"""Synthetic datasets.  ``FooDataset`` mirrors the reference (``dataset.py:6-17``: X ~ N(0,1)^(n,10),
Y ~ N(0,1)^(n,5), held in host memory, drawn from the global torch RNG *after* seeding so every rank
holds the same data).  The ImageNet- and token-shaped variants feed the benchmark configurations
(there is no network for real data)."""
from __future__ import annotations

import math
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


class SyntheticImageText(Dataset):
    """Image-caption pairs for CLIP: ``X`` images fp32 [3, size, size] as in ``SyntheticImageNet`` and ``Y`` caption ids
    int64 [context] (seeded).  A caption is ``SOT_ID``, tokens from [1, SOT_ID), ``EOT_ID``, then pad 0, with total lengths
    (SOT and EOT included) uniform in [8, context].  ``samples`` is rounded down to a multiple of ``batch`` (at least one
    batch): with ``batch`` the global batch, every batch holds whole pairs and no partial batch reaches the loss."""

    SOT_ID = 49406                 # <|startoftext|> in CLIP's vocabulary
    EOT_ID = 49407                 # <|endoftext|>
    PAD_ID = 0

    def __init__(self, samples: int = 1024, batch: int = 1, size: int = 224, context: int = 77, min_len: int = 8, seed: int = 1234):
        if not 2 <= min_len <= context:
            raise ValueError(f"SyntheticImageText: min_len must lie in [2, context = {context}], got {min_len}")
        g = torch.Generator().manual_seed(seed)
        batch = max(1, int(batch))
        self.samples = max(batch, int(samples) // batch * batch)
        self.X = torch.randn(self.samples, 3, size, size, generator=g)
        lens = torch.randint(min_len, context + 1, (self.samples,), generator=g)
        pos = torch.arange(context)[None, :]
        ids = torch.randint(1, self.SOT_ID, (self.samples, context), generator=g)
        ids[:, 0] = self.SOT_ID
        ids = torch.where(pos == (lens - 1)[:, None], torch.full_like(ids, self.EOT_ID), ids)
        self.Y = torch.where(pos >= lens[:, None], torch.full_like(ids, self.PAD_ID), ids)
        self.caption_lengths = lens

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


class SyntheticSpeech(Dataset):
    """Waveform / transcript pairs for Whisper (seeded): ``X`` int16 PCM [samples, 480000] (30 seconds at 16 kHz) and ``Y``
    labels int64 [seq_len].  A transcript holds n tokens from [0, ``EOT_ID``) followed by ``EOT_ID``, then -100; n + 1 is
    ``seq_len`` or, with ``min_len``, uniform in [min_len, seq_len].  The clip carries one segment per token, a tone whose
    pitch follows the token plus noise, over the first n / seq_len of the clip, and silence after it.  There is no pad id:
    the labels' -100 padding gives the transcript lengths.  128 clips take 123 MB."""

    EOT_ID = 50256                 # <|endoftext|>
    SAMPLES = 480000
    RATE = 16000

    def __init__(self, samples: int = 128, seq_len: int = 448, min_len: int | None = None, seed: int = 1234):
        if min_len is not None and not 1 <= min_len <= seq_len:
            raise ValueError(f"SyntheticSpeech: min_len must lie in [1, seq_len = {seq_len}], got {min_len}")
        g = torch.Generator().manual_seed(seed)
        self.samples = int(samples)
        lens = torch.full((self.samples,), seq_len) if min_len is None else torch.randint(min_len, seq_len + 1, (self.samples,), generator=g)
        pos = torch.arange(seq_len)[None, :]
        ids = torch.randint(0, self.EOT_ID, (self.samples, seq_len), generator=g)
        ids = torch.where(pos == (lens - 1)[:, None], torch.full_like(ids, self.EOT_ID), ids)
        self.Y = torch.where(pos >= lens[:, None], torch.full_like(ids, -100), ids)
        self.X = torch.zeros(self.samples, self.SAMPLES, dtype=torch.int16)
        seg = self.SAMPLES // seq_len
        for i in range(self.samples):
            n = int(lens[i]) - 1
            if n == 0:
                continue
            freq = (100.0 + 60.0 * (ids[i, :n] % 64).double()).repeat_interleave(seg)
            amp = (2000.0 + 6000.0 * torch.rand(n, generator=g, dtype=torch.float64)).repeat_interleave(seg)
            t = torch.arange(n * seg, dtype=torch.float64) / self.RATE
            wave = amp * torch.sin(2 * math.pi * freq * t) + 300.0 * torch.randn(n * seg, generator=g, dtype=torch.float64)
            self.X[i, :n * seg] = wave.round().clamp(-32768, 32767).to(torch.int16)

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
    ``cls_token_id``.  ``bos_token_id`` picks another start id for causal packed documents (a model's own, from its
    entry in ``b200ddp.models.MODEL_REGISTRY``); ``BOS_ID`` is the default.  ``cls_token_id`` does the same for MLM packed
    documents (ModernBERT's [CLS] is 50281); ``CLS_ID`` is the default."""

    PAD_ID = 0
    CLS_ID = 101                   # [CLS] in the BERT vocabulary
    BOS_ID = 50256                 # <|endoftext|> in the GPT-2 vocabulary, which starts each GPT-2 document

    def __init__(self, samples: int = 512, seq_len: int = 512, vocab: int = 30522, mask_prob: float = 0.15, seed: int = 1234,
                 min_len: int | None = None, pack: bool = False, causal: bool = False, bos_token_id: int | None = None,
                 cls_token_id: int = CLS_ID):
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
            self._pack(g, seq_len, vocab, mask_prob, seq_len if min_len is None else min_len, causal, bos_token_id, cls_token_id)
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
              bos_token_id: int | None = None, cls_token_id: int = CLS_ID) -> None:
        start_id = (self.BOS_ID if bos_token_id is None else bos_token_id) if causal else cls_token_id
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


class SyntheticSpanCorruption(Dataset):
    """Source / target pairs for T5's span-corruption objective (seeded): ``X`` source ids [seq_len], right-padded with
    ``PAD_ID``; ``Y`` labels [target_width], the target ids, -100 at padding.

    A document is n text tokens from [3, 32000) (T5's special ids are 0 to 2; its sentinels 32099, 32098, ... sit above
    the text vocabulary).  ``round(0.15 n)`` of them (at least 1, at most n - 1) are noise, in ``max(round(noise / 3),
    1)`` spans; noise and kept tokens are each split into that many non-empty runs by a random segmentation, and the
    runs alternate kept, noise, kept, noise ... as in T5's ``random_spans_noise_mask``.  The source is ``start_id`` +
    the kept runs with each noise span replaced by the next sentinel + ``EOS_ID``; the target is ``start_id`` + (sentinel,
    its span's tokens) for every span + the next sentinel + ``EOS_ID``.  ``start_id`` (2, <unk>) never occurs in the text,
    so packed documents can be found on both sides.

    Sources are ``seq_len`` tokens long (the longest n whose source fits), or uniform in [``min_len``, ``seq_len``].
    Targets are right-padded to ``target_width(seq_len)``: the longest target a source of ``seq_len`` tokens can have,
    rounded up to 128 (128 at 512, 256 at 1024).  ``pack=True`` places the pairs first-fit decreasing by source length
    (ties in pair order) into the first row where both the source and the target still fit: short documents have a
    larger target-to-source ratio, so the source alone does not bound the target row.  ``bos_token_id`` is then
    ``start_id``, and ``doc_ids`` / ``doc_lengths`` list each row's pairs and source lengths.  ``lengths`` holds each
    row's filled source length."""

    PAD_ID = 0
    EOS_ID = 1
    TEXT_END = 32000
    FIRST_SENTINEL = 32099

    def __init__(self, samples: int = 512, seq_len: int = 512, vocab: int = 32128, start_id: int = 2, min_len: int | None = None,
                 pack: bool = False, noise_density: float = 0.15, mean_span: float = 3.0, seed: int = 1234):
        if min_len is not None and not 4 <= min_len <= seq_len:
            raise ValueError(f"SyntheticSpanCorruption: min_len must lie in [4, seq_len = {seq_len}], got {min_len}")
        if vocab <= self.FIRST_SENTINEL or not 1 < start_id < 3:
            raise ValueError(f"SyntheticSpanCorruption: needs T5's vocabulary (> {self.FIRST_SENTINEL} ids) and start_id 2, "
                             f"got vocab {vocab} and start_id {start_id}")
        self.noise_density, self.mean_span = noise_density, mean_span
        g = torch.Generator().manual_seed(seed)
        n = int(samples)
        src_lens = torch.full((n,), seq_len) if min_len is None else torch.randint(min_len, seq_len + 1, (n,), generator=g)
        self.target_width = self.target_width_for(seq_len, noise_density, mean_span)
        sources, targets = [], []
        for L in src_lens.tolist():
            text = torch.randint(3, self.TEXT_END, (self._text_len(L),), generator=g)
            s, t = self._corrupt(text, g)
            sources.append(torch.cat([torch.tensor([start_id]), s, torch.tensor([self.EOS_ID])]))
            targets.append(torch.cat([torch.tensor([start_id]), t, torch.tensor([self.EOS_ID])]))
        self.pad_token_id = self.PAD_ID
        self.bos_token_id = None
        self.doc_ids = self.doc_lengths = None
        slen = [len(x) for x in sources]
        tlen = [len(y) for y in targets]
        if pack:
            rows, free_s, free_t = [], [], []
            for i in sorted(range(n), key=lambda i: (-slen[i], i)):    # first-fit decreasing by source length
                r = next((r for r in range(len(rows)) if free_s[r] >= slen[i] and free_t[r] >= tlen[i]), len(rows))
                if r == len(rows):
                    rows.append([])
                    free_s.append(seq_len)
                    free_t.append(self.target_width)
                rows[r].append(i)
                free_s[r] -= slen[i]
                free_t[r] -= tlen[i]
            self.doc_ids = rows
            self.doc_lengths = [[slen[i] for i in docs] for docs in rows]
            self.bos_token_id = start_id
        else:
            rows = [[i] for i in range(n)]
        self.samples = len(rows)
        self.X = torch.full((self.samples, seq_len), self.PAD_ID, dtype=torch.long)
        self.Y = torch.full((self.samples, self.target_width), -100, dtype=torch.long)
        for r, docs in enumerate(rows):
            a = b = 0
            for i in docs:
                self.X[r, a:a + slen[i]] = sources[i]
                self.Y[r, b:b + tlen[i]] = targets[i]
                a, b = a + slen[i], b + tlen[i]
        self.lengths = (self.X != self.PAD_ID).sum(1)

    @staticmethod
    def _spans(n: int, density: float, mean_span: float):
        noise = min(max(int(round(n * density)), 1), n - 1)
        return noise, max(int(round(noise / mean_span)), 1)

    @classmethod
    def _lens(cls, n: int, density: float = 0.15, mean_span: float = 3.0):
        """(source, target) lengths of a document of n text tokens, start and end ids included."""
        noise, spans = cls._spans(n, density, mean_span)
        return (n - noise) + spans + 2, noise + spans + 3

    def _text_len(self, src_len: int) -> int:
        """The longest text whose source fits in src_len tokens."""
        n = 2
        while self._lens(n + 1, self.noise_density, self.mean_span)[0] <= src_len:
            n += 1
        return n

    @classmethod
    def target_width_for(cls, seq_len: int, density: float = 0.15, mean_span: float = 3.0) -> int:
        """Label columns for sources of up to seq_len tokens: the longest target, rounded up to 128."""
        longest, n = 0, 2
        while cls._lens(n, density, mean_span)[0] <= seq_len:
            longest = max(longest, cls._lens(n, density, mean_span)[1])
            n += 1
        return (longest + 127) // 128 * 128

    @staticmethod
    def _segment(items: int, segments: int, g: torch.Generator) -> list:
        """items split into `segments` non-empty runs at random (T5's random_segmentation)."""
        cuts = (torch.randperm(items - 1, generator=g)[:segments - 1] + 1).sort().values.tolist()
        edges = [0] + cuts + [items]
        return [b - a for a, b in zip(edges[:-1], edges[1:])]

    def _corrupt(self, text: torch.Tensor, g: torch.Generator):
        """(source body, target body) of one document: kept runs and sentinels; sentinels and noise runs, then the next
        sentinel."""
        n = text.numel()
        noise, spans = self._spans(n, self.noise_density, self.mean_span)
        kept_runs = self._segment(n - noise, spans, g)
        noise_runs = self._segment(noise, spans, g)
        src, tgt, at = [], [], 0
        for k in range(spans):
            sentinel = torch.tensor([self.FIRST_SENTINEL - k])
            src += [text[at:at + kept_runs[k]], sentinel]
            at += kept_runs[k]
            tgt += [sentinel, text[at:at + noise_runs[k]]]
            at += noise_runs[k]
        tgt.append(torch.tensor([self.FIRST_SENTINEL - spans]))
        return torch.cat(src), torch.cat(tgt)

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


class SyntheticDenoising(Dataset):
    """Source / target pairs for BART's text-infilling objective (seeded): ``X`` source ids [seq_len], right-padded with
    ``PAD_ID``; ``Y`` labels [seq_len], the target ids, -100 at padding.

    A target document is ``start_id`` followed by tokens from [4, vocab) other than ``start_id`` and ``mask_id`` (BART's
    special ids are 0 to 3 and its <mask>); ``start_id`` is neither ``PAD_ID`` nor BART's decoder start id 2.  Its source is the same document with spans of the tokens after the start
    replaced, each span by one ``mask_id``: span lengths are Poisson(3) clipped to at least 1 (the last one cut to the
    budget), covering ``round(0.3 n)`` of the document's n tokens, so a source is never longer than its target.

    Targets are ``seq_len`` tokens long, or uniform in [``min_len``, ``seq_len``] with ``min_len``.  ``pack=True`` places
    the pairs into rows by first-fit decreasing target length (longest first, ties in pair order); the k-th source and
    the k-th target of a row are one pair, and since no source is longer than its target every source fits.
    ``bos_token_id`` is then ``start_id`` and ``doc_ids`` / ``doc_lengths`` list each row's pairs and target lengths.
    ``pad_token_id`` is always ``PAD_ID`` (sources are shorter than their targets) and ``lengths`` holds each row's
    filled target length."""

    PAD_ID = 0

    def __init__(self, samples: int = 512, seq_len: int = 512, vocab: int = 50265, start_id: int = 3, mask_id: int = 50264,
                 min_len: int | None = None, pack: bool = False, mask_ratio: float = 0.3, mean_span: float = 3.0, seed: int = 1234):
        if min_len is not None and not 1 <= min_len <= seq_len:
            raise ValueError(f"SyntheticDenoising: min_len must lie in [1, seq_len = {seq_len}], got {min_len}")
        if not (0 < start_id < vocab and start_id != 2 and 4 <= mask_id < vocab and start_id != mask_id):
            raise ValueError(f"SyntheticDenoising: start_id must lie in [1, vocab = {vocab}) other than the pad id 0 and the decoder "
                             f"start id 2, mask_id in [4, vocab), and the two must differ; got {start_id} and {mask_id}")
        g = torch.Generator().manual_seed(seed)
        n = int(samples)
        lens = torch.full((n,), seq_len) if min_len is None else torch.randint(min_len, seq_len + 1, (n,), generator=g)
        lens_l = lens.tolist()
        excluded = sorted(i for i in (start_id, mask_id) if i >= 4)
        targets, sources = [], []
        for L in lens_l:
            body = torch.randint(4, vocab - len(excluded), (L - 1,), generator=g)
            for e in excluded:                                      # [4, vocab) without start_id and mask_id
                body += body >= e
            targets.append(torch.cat([torch.tensor([start_id]), body]))
            sources.append(torch.cat([torch.tensor([start_id]), self._infill(body, g, mask_id, mask_ratio, mean_span)]))
        self.pad_token_id = self.PAD_ID
        self.bos_token_id = None
        self.doc_ids = self.doc_lengths = None
        if pack:
            rows, free = [], []
            for i in sorted(range(n), key=lambda i: (-lens_l[i], i)):   # first-fit decreasing by target length
                r = next((r for r, f in enumerate(free) if f >= lens_l[i]), len(rows))
                if r == len(rows):
                    rows.append([])
                    free.append(seq_len)
                rows[r].append(i)
                free[r] -= lens_l[i]
            self.doc_ids = rows
            self.doc_lengths = [[lens_l[i] for i in docs] for docs in rows]
            self.bos_token_id = start_id
        else:
            rows = [[i] for i in range(n)]
        self.samples = len(rows)
        self.X = torch.full((self.samples, seq_len), self.PAD_ID, dtype=torch.long)
        self.Y = torch.full((self.samples, seq_len), -100, dtype=torch.long)
        for r, docs in enumerate(rows):
            a = b = 0
            for i in docs:
                s, t = sources[i], targets[i]
                self.X[r, a:a + len(s)] = s
                self.Y[r, b:b + len(t)] = t
                a, b = a + len(s), b + len(t)
        self.lengths = (self.Y != -100).sum(1)

    @staticmethod
    def _infill(body: torch.Tensor, g: torch.Generator, mask_id: int, ratio: float, mean_span: float) -> torch.Tensor:
        """body with spans covering round(ratio * len) of its tokens replaced by one mask_id each."""
        n = body.numel()
        budget = int(round(ratio * n))
        spans = []
        while sum(spans) < budget:
            spans += torch.poisson(torch.full((16,), mean_span), generator=g).clamp(min=1).long().tolist()
        out, total = [], 0
        for s in spans:
            if total >= budget:
                break
            out.append(min(s, budget - total))
            total += out[-1]
        spans = out
        # the n - budget kept tokens and the spans in a random interleaving (stars and bars)
        slots = len(spans) + n - budget
        is_span = torch.zeros(slots, dtype=torch.bool)
        is_span[torch.randperm(slots, generator=g)[:len(spans)]] = True
        width = torch.ones(slots, dtype=torch.long)
        width[is_span] = torch.tensor(spans, dtype=torch.long)
        first = torch.cumsum(width, 0) - width                    # each slot's first token in body
        return torch.where(is_span, torch.full_like(first, mask_id), body[first.clamp(max=max(n - 1, 0))] if n else first)

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
