from .datasets import FooDataset, SyntheticDenoising, SyntheticImageNet, SyntheticImageText, SyntheticTokens
from .loader import BatchLoader, DevicePrefetcher

__all__ = ["FooDataset", "SyntheticDenoising", "SyntheticImageNet", "SyntheticImageText", "SyntheticTokens", "BatchLoader", "DevicePrefetcher"]
