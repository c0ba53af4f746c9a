from .datasets import FooDataset, SyntheticImageNet, SyntheticImageText, SyntheticTokens
from .loader import BatchLoader, DevicePrefetcher

__all__ = ["FooDataset", "SyntheticImageNet", "SyntheticImageText", "SyntheticTokens", "BatchLoader", "DevicePrefetcher"]
