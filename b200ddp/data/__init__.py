from .datasets import FooDataset, SyntheticDenoising, SyntheticImageNet, SyntheticSpanCorruption, SyntheticImageText, SyntheticSpeech, SyntheticTokens
from .loader import BatchLoader, DevicePrefetcher

__all__ = ["FooDataset", "SyntheticDenoising", "SyntheticImageNet", "SyntheticSpanCorruption", "SyntheticImageText", "SyntheticSpeech", "SyntheticTokens", "BatchLoader", "DevicePrefetcher"]
