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
    """Token ids [seq] + MLM labels [seq] (-100 = not predicted) for the BERT config.

    ``min_len < seq_len`` gives right-padded rows: each row's length is uniform in [min_len, seq_len] (seeded), its
    prefix holds tokens from [1, vocab) and the tail is ``PAD_ID`` labelled -100.  ``lengths`` then holds the lengths and
    ``pad_token_id`` is ``PAD_ID``; without padding both are None and the tensors are those of fixed-length rows.

    ``pack=True`` packs documents instead: ``samples`` documents with lengths uniform in [min_len, seq_len] (``min_len``
    defaults to ``seq_len``), each starting with ``CLS_ID`` and holding tokens from [1, vocab) other than ``CLS_ID``,
    are placed into rows of ``seq_len`` by first-fit decreasing (longest first, ties in document order).  Row tails are
    ``PAD_ID`` labelled -100, the ``CLS_ID`` tokens are labelled -100 too.  ``lengths`` then holds each row's filled
    length, ``cls_token_id`` is ``CLS_ID``, and ``doc_ids`` / ``doc_lengths`` list each row's documents (in row order).

    ``causal=True`` gives causal-LM rows (GPT) in the same three layouts: within a document ``labels[t] = ids[t + 1]``,
    and each document's last token and the padding are labelled -100.  Tokens come from [1, vocab); packed documents
    start with ``BOS_ID`` instead of ``CLS_ID`` (and hold no other ``BOS_ID``), and ``bos_token_id`` is set instead of
    ``cls_token_id``.  ``bos_token_id`` picks another start id for causal packed documents (1, Llama's ``<s>``, for
    SmolLM; 151643, ``<|endoftext|>``, for Qwen2.5); GPT-2's 50256 stays the default."""

    PAD_ID = 0
    CLS_ID = 101                   # [CLS] in the BERT vocabulary
    BOS_ID = 50256                 # <|endoftext|> in the GPT-2 vocabulary, which starts each GPT-2 document
    LLAMA_BOS_ID = 1               # <s> in the Llama / SmolLM vocabularies
    QWEN_BOS_ID = 151643           # <|endoftext|> in the Qwen2.5 vocabulary, which starts each Qwen2.5 document

    def __init__(self, samples: int = 512, seq_len: int = 512, vocab: int = 30522, mask_prob: float = 0.15, seed: int = 1234,
                 min_len: int | None = None, pack: bool = False, causal: bool = False, bos_token_id: int | None = None):
        if min_len is not None and not 1 <= min_len <= seq_len:
            raise ValueError(f"SyntheticTokens: min_len must lie in [1, seq_len = {seq_len}], got {min_len}")
        g = torch.Generator().manual_seed(seed)
        self.samples = int(samples)
        self.lengths = None
        self.pad_token_id = None
        self.cls_token_id = None
        self.bos_token_id = None
        self.doc_ids = self.doc_lengths = None
        if pack:
            self._pack(g, seq_len, vocab, mask_prob, seq_len if min_len is None else min_len, causal, bos_token_id)
            return
        if causal:
            self._causal_rows(g, seq_len, vocab, min_len)
            return
        if min_len is None or min_len == seq_len:
            self.X = torch.randint(0, vocab, (self.samples, seq_len), generator=g)
        else:
            self.lengths = torch.randint(min_len, seq_len + 1, (self.samples,), generator=g)
            self.pad_token_id = self.PAD_ID
            self.X = torch.randint(1, vocab, (self.samples, seq_len), generator=g)
        labels = torch.randint(0, vocab, (self.samples, seq_len), generator=g)
        masked = torch.rand(self.samples, seq_len, generator=g) < mask_prob
        self.Y = torch.where(masked, labels, torch.full_like(labels, -100))
        if self.lengths is not None:
            pad = torch.arange(seq_len)[None, :] >= self.lengths[:, None]
            self.X.masked_fill_(pad, self.PAD_ID)
            self.Y.masked_fill_(pad, -100)

    def _causal_rows(self, g: torch.Generator, seq_len: int, vocab: int, min_len: int | None) -> None:
        """Fixed-length or right-padded causal-LM rows: next-token labels, -100 at each row's last token and padding."""
        self.X = torch.randint(1, vocab, (self.samples, seq_len), generator=g)
        length = torch.full((self.samples,), seq_len)
        if min_len is not None and min_len < seq_len:
            self.lengths = length = torch.randint(min_len, seq_len + 1, (self.samples,), generator=g)
            self.pad_token_id = self.PAD_ID
            self.X.masked_fill_(torch.arange(seq_len)[None, :] >= length[:, None], self.PAD_ID)
        self.Y = torch.cat([self.X[:, 1:], torch.full((self.samples, 1), -100)], 1)
        self.Y.masked_fill_(torch.arange(seq_len)[None, :] >= (length - 1)[:, None], -100)

    def _pack(self, g: torch.Generator, seq_len: int, vocab: int, mask_prob: float, min_len: int, causal: bool = False,
              bos_token_id: int | None = None) -> None:
        start_id = (self.BOS_ID if bos_token_id is None else bos_token_id) if causal else self.CLS_ID
        if causal and (start_id == self.PAD_ID or not 0 < start_id < vocab):
            raise ValueError(f"SyntheticTokens: the start id must lie in [1, vocab = {vocab}) and differ from PAD_ID, got {start_id}")
        need = start_id if causal else start_id + 1
        if vocab <= need:
            raise ValueError(f"SyntheticTokens: packing needs vocab > {need} (token {start_id} starts a document)")
        lens = torch.randint(min_len, seq_len + 1, (self.samples,), generator=g)
        total = int(lens.sum())
        tokens = torch.randint(1, vocab - 1, (total,), generator=g)
        tokens += tokens >= start_id                               # [1, vocab) without start_id
        offsets = torch.cumsum(lens, 0) - lens
        if causal:                                                 # next token inside the document, -100 at its last
            tokens[offsets] = start_id
            labels = torch.cat([tokens[1:], torch.full((1,), -100)])
            labels[offsets + lens - 1] = -100
        else:
            labels = torch.randint(0, vocab, (total,), generator=g)
            masked = torch.rand(total, generator=g) < mask_prob
            labels = torch.where(masked, labels, torch.full_like(labels, -100))
            tokens[offsets] = start_id
            labels[offsets] = -100
        lens_l, offsets_l = lens.tolist(), offsets.tolist()
        rows, free = [], []
        for i in sorted(range(self.samples), key=lambda i: (-lens_l[i], i)):   # first-fit decreasing
            r = next((r for r, f in enumerate(free) if f >= lens_l[i]), len(rows))
            if r == len(rows):
                rows.append([])
                free.append(seq_len)
            rows[r].append(i)
            free[r] -= lens_l[i]
        self.X = torch.full((len(rows), seq_len), self.PAD_ID, dtype=torch.long)
        self.Y = torch.full((len(rows), seq_len), -100, dtype=torch.long)
        for r, docs in enumerate(rows):
            at = 0
            for i in docs:
                n, o = lens_l[i], offsets_l[i]
                self.X[r, at:at + n] = tokens[o:o + n]
                self.Y[r, at:at + n] = labels[o:o + n]
                at += n
        self.samples = len(rows)
        self.doc_ids = rows
        self.doc_lengths = [[lens_l[i] for i in docs] for docs in rows]
        self.lengths = torch.tensor([seq_len - f for f in free])
        self.pad_token_id = self.PAD_ID
        if causal:
            self.bos_token_id = start_id
        else:
            self.cls_token_id = start_id

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
