"""Synthetic datasets.  ``FooDataset`` mirrors the reference (``dataset.py:6-17``: X ~ N(0,1)^(n,10),
Y ~ N(0,1)^(n,5), held in host memory, drawn from the global torch RNG *after* seeding so every rank
holds the same data).  The ImageNet- and token-shaped variants feed the benchmark configurations
(there is no network for real data)."""
from __future__ import annotations

from typing import Tuple

import torch
from torch.utils.data import Dataset


class FooDataset(Dataset):
    def __init__(self, samples: int, in_features: int = 10, out_features: int = 5) -> None:
        self.samples = int(samples)
        self.X = torch.randn(self.samples, in_features)
        self.Y = torch.randn(self.samples, out_features)

    def __len__(self) -> int:
        return self.samples

    def __getitem__(self, index) -> Tuple[torch.Tensor, torch.Tensor]:
        return self.X[index], self.Y[index]

    def batch(self, indices: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """Whole-batch gather (one index_select instead of B ``__getitem__`` calls + collate)."""
        return self.X.index_select(0, indices), self.Y.index_select(0, indices)

    def batch_into(self, indices: torch.Tensor, outs) -> None:
        """Gather straight into caller-owned (pinned) buffers: one pass over the data."""
        torch.index_select(self.X, 0, indices, out=outs[0])
        torch.index_select(self.Y, 0, indices, out=outs[1])


class SyntheticImageNet(Dataset):
    """ImageNet-shaped samples: image fp32 (or uint8) [3,224,224]; target either a dense fp32
    [classes] vector (what the reference's hard-coded MSELoss needs) or an int64 class id."""

    def __init__(self, samples: int = 1024, classes: int = 1000, size: int = 224, image_dtype=torch.float32,
                 dense_target: bool = True, seed: int = 1234):
        g = torch.Generator().manual_seed(seed)
        self.samples = int(samples)
        if image_dtype == torch.uint8:
            self.X = torch.randint(0, 256, (self.samples, 3, size, size), dtype=torch.uint8, generator=g)
        else:
            self.X = torch.randn(self.samples, 3, size, size, generator=g).to(image_dtype)
        labels = torch.randint(0, classes, (self.samples,), generator=g)
        self.labels = labels
        self.dense_target = dense_target
        if dense_target:
            self.Y = torch.zeros(self.samples, classes)
            self.Y[torch.arange(self.samples), labels] = 1.0
        else:
            self.Y = labels

    def __len__(self) -> int:
        return self.samples

    def __getitem__(self, index):
        return self.X[index], self.Y[index]

    def batch(self, indices: torch.Tensor):
        return self.X.index_select(0, indices), self.Y.index_select(0, indices)

    def batch_into(self, indices: torch.Tensor, outs) -> None:
        """Gather straight into caller-owned (pinned) buffers: one pass over the data."""
        torch.index_select(self.X, 0, indices, out=outs[0])
        torch.index_select(self.Y, 0, indices, out=outs[1])


class SyntheticTokens(Dataset):
    """Token ids [seq] + MLM labels [seq] (-100 = not predicted) for the BERT config."""

    def __init__(self, samples: int = 512, seq_len: int = 512, vocab: int = 30522, mask_prob: float = 0.15, seed: int = 1234):
        g = torch.Generator().manual_seed(seed)
        self.samples = int(samples)
        self.X = torch.randint(0, vocab, (self.samples, seq_len), generator=g)
        labels = torch.randint(0, vocab, (self.samples, seq_len), generator=g)
        masked = torch.rand(self.samples, seq_len, generator=g) < mask_prob
        self.Y = torch.where(masked, labels, torch.full_like(labels, -100))

    def __len__(self) -> int:
        return self.samples

    def __getitem__(self, index):
        return self.X[index], self.Y[index]

    def batch(self, indices: torch.Tensor):
        return self.X.index_select(0, indices), self.Y.index_select(0, indices)

    def batch_into(self, indices: torch.Tensor, outs) -> None:
        """Gather straight into caller-owned (pinned) buffers: one pass over the data."""
        torch.index_select(self.X, 0, indices, out=outs[0])
        torch.index_select(self.Y, 0, indices, out=outs[1])
