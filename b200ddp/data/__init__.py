from .datasets import FooDataset, SyntheticDenoising, SyntheticImageNet, SyntheticSpanCorruption, SyntheticImageText, SyntheticTokens
from .loader import BatchLoader, DevicePrefetcher

__all__ = ["FooDataset", "SyntheticDenoising", "SyntheticImageNet", "SyntheticSpanCorruption", "SyntheticImageText", "SyntheticTokens", "BatchLoader", "DevicePrefetcher"]
