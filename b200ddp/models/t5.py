"""T5 encoder-decoder (t5-small, t5-base) for sequence-to-sequence training, as ``transformers``'
``T5ForConditionalGeneration`` defines it: pre-RMSNorm blocks (eps 1e-6), no biases anywhere, no position embeddings but
one learned relative position bias per stack (bidirectional in the encoder, unidirectional in the decoder's
self-attention; cross-attention has none), unscaled attention scores, ReLU feed-forward ``wi`` / ``wo``, a
``final_layer_norm`` per stack, and the LM head tied to ``shared`` with the decoder output scaled by ``d_model ** -0.5``.
No dropout.

Self-attention runs on ``ops.relative_attention`` (the bias inside the attention kernels on CUDA in bf16, the dense
reference on the CPU and in fp32), its table built once per stack and forward by ``ops.relative_position_table``.
Cross-attention is ``ops.cross_attention(8 q, ...)``: the kernel's 1/sqrt(64) = 1/8 undoes the exact x8, so the scores
are T5's unscaled ones.  Fixed-length, right-padded and packed rows take one path, as in ``models/bart.py``, whose
``shift_documents_right`` derives the decoder input (decoder start id 0, -100 -> pad 0)."""
from __future__ import annotations

from dataclasses import dataclass, replace

import torch
import torch.nn as nn

from ..ops import (Linear, LinearCrossEntropyLoss, RMSNorm, cross_attention, cross_bounds, document_bounds, linear,
                   relative_attention, relative_position_table)
from ..ops.functional import relative_position_buckets
from .bart import shift_documents_right

CROSS_SCALE = 8.0                  # 1 / the cross-attention kernel's 1/sqrt(64): exact in bf16


@dataclass
class T5Config:
    vocab_size: int = 32128
    d_model: int = 512
    num_layers: int = 6
    num_decoder_layers: int = 6
    num_heads: int = 8
    d_kv: int = 64
    d_ff: int = 2048
    num_buckets: int = 32
    eps: float = 1e-6
    max_position: int = 1024       # the longest sequence trained: T5 has no position table, and 1024 source tokens carry
                                   # about 57 of its 100 sentinels
    decoder_start_token_id: int = 0
    pad_token_id: int | None = None  # right-padded rows: length = non-pad count (sources) or non -100 count (labels)
    bos_token_id: int | None = None  # packed rows: a document starts at each such id (and at 0) on both sides
    fused_lm_loss: bool = False    # forward returns the scaled decoder output; ``lm_head_loss`` applies the head


class T5SelfAttention(nn.Module):
    """layer.0 of a block: RMSNorm, fused q | k | v, the biased attention, o."""

    def __init__(self, c: T5Config, causal: bool):
        super().__init__()
        self.heads, self.causal = c.num_heads, causal
        inner = c.num_heads * c.d_kv
        self.layer_norm = RMSNorm(c.d_model, eps=c.eps)
        self.qkv = Linear(c.d_model, 3 * inner, bias=False)
        self.o = Linear(inner, c.d_model, bias=False)

    def forward(self, x, bounds, table):
        return x + self.o(relative_attention(self.qkv(self.layer_norm(x)), bounds, table, self.heads, self.causal))


class T5CrossAttention(nn.Module):
    """layer.1 of a decoder block (``EncDecAttention``): RMSNorm, q, fused k | v of the encoder output, o."""

    def __init__(self, c: T5Config):
        super().__init__()
        self.heads = c.num_heads
        inner = c.num_heads * c.d_kv
        self.layer_norm = RMSNorm(c.d_model, eps=c.eps)
        self.q = Linear(c.d_model, inner, bias=False)
        self.cross_kv = Linear(c.d_model, 2 * inner, bias=False)
        self.o = Linear(inner, c.d_model, bias=False)

    def forward(self, x, enc, q_bounds, kv_bounds):
        q = self.q(self.layer_norm(x)) * CROSS_SCALE
        return x + self.o(cross_attention(q, self.cross_kv(enc), q_bounds, kv_bounds, self.heads))


class T5FeedForward(nn.Module):
    def __init__(self, c: T5Config):
        super().__init__()
        self.layer_norm = RMSNorm(c.d_model, eps=c.eps)
        self.wi = Linear(c.d_model, c.d_ff, bias=False, activation="relu")
        self.wo = Linear(c.d_ff, c.d_model, bias=False)

    def forward(self, x):
        return x + self.wo(self.wi(self.layer_norm(x)))


class T5Block(nn.Module):
    def __init__(self, c: T5Config, decoder: bool):
        super().__init__()
        self.self_attn = T5SelfAttention(c, causal=decoder)
        self.cross_attn = T5CrossAttention(c) if decoder else None
        self.ff = T5FeedForward(c)

    def forward(self, x, bounds, table, enc=None, q_bounds=None, kv_bounds=None):
        x = self.self_attn(x, bounds, table)
        if self.cross_attn is not None:
            x = self.cross_attn(x, enc, q_bounds, kv_bounds)
        return self.ff(x)


class T5Stack(nn.Module):
    """One side's relative bias embedding (block 0's in transformers), blocks and ``final_layer_norm``."""

    def __init__(self, c: T5Config, n: int, decoder: bool):
        super().__init__()
        self.decoder = decoder
        self.relative_attention_bias = nn.Embedding(c.num_buckets, c.num_heads)
        # the bucket of each clamped distance: moves with the module, so a forward never copies it to the device
        self.register_buffer("buckets", relative_position_buckets(not decoder, c.num_buckets), persistent=False)
        self.block = nn.ModuleList([T5Block(c, decoder) for _ in range(n)])
        self.final_layer_norm = RMSNorm(c.d_model, eps=c.eps)

    def forward(self, x, bounds, enc=None, q_bounds=None, kv_bounds=None):
        table = relative_position_table(self.relative_attention_bias.weight, not self.decoder, self.buckets)
        for blk in self.block:
            x = blk(x, bounds, table, enc, q_bounds, kv_bounds)
        return self.final_layer_norm(x)


class T5ForConditionalGeneration(nn.Module):
    """Encoder-decoder + LM head tied to ``shared``; ``forward(input_ids, labels)`` returns logits [B, Sq, vocab] (or, with
    ``T5Config.fused_lm_loss``, the scaled decoder output for ``lm_head_loss()``)."""

    def __init__(self, config: T5Config | None = None):
        super().__init__()
        c = self.config = config or T5Config()
        self.shared = nn.Embedding(c.vocab_size, c.d_model)
        self.encoder = T5Stack(c, c.num_layers, decoder=False)
        self.decoder = T5Stack(c, c.num_decoder_layers, decoder=True)
        self._init()

    @torch.no_grad()
    def _init(self):
        """transformers' ``T5PreTrainedModel._init_weights`` at ``initializer_factor`` 1."""
        c = self.config
        d, inner = c.d_model, c.num_heads * c.d_kv
        nn.init.normal_(self.shared.weight, std=1.0)
        for stack in (self.encoder, self.decoder):
            nn.init.normal_(stack.relative_attention_bias.weight, std=d ** -0.5)
            for blk in stack.block:
                nn.init.normal_(blk.self_attn.qkv.weight[:inner], std=(d * c.d_kv) ** -0.5)      # q
                nn.init.normal_(blk.self_attn.qkv.weight[inner:], std=d ** -0.5)                 # k, v
                nn.init.normal_(blk.self_attn.o.weight, std=inner ** -0.5)
                if blk.cross_attn is not None:
                    nn.init.normal_(blk.cross_attn.q.weight, std=(d * c.d_kv) ** -0.5)
                    nn.init.normal_(blk.cross_attn.cross_kv.weight, std=d ** -0.5)
                    nn.init.normal_(blk.cross_attn.o.weight, std=inner ** -0.5)
                nn.init.normal_(blk.ff.wi.weight, std=d ** -0.5)
                nn.init.normal_(blk.ff.wo.weight, std=c.d_ff ** -0.5)

    def forward(self, input_ids, labels):
        c = self.config
        enc_bounds, _ = document_bounds(input_ids, c.bos_token_id, c.pad_token_id)
        dec_ids, dec_bounds, _ = shift_documents_right(labels, c.decoder_start_token_id, c.pad_token_id, c.bos_token_id, 0)
        q_bounds, kv_bounds = cross_bounds(enc_bounds, dec_bounds)
        x = self.encoder(self.shared(input_ids), enc_bounds)
        y = self.decoder(self.shared(dec_ids), dec_bounds, x, q_bounds, kv_bounds)
        y = y * c.d_model ** -0.5                                 # transformers' scale_decoder_outputs (tied head)
        if c.fused_lm_loss:
            return y
        return linear(y, self.shared.weight)

    def lm_head_loss(self, ignore_index: int = -100) -> LinearCrossEntropyLoss:
        """Criterion over ``forward``'s scaled decoder output with ``fused_lm_loss``: the tied head, no bias."""
        return LinearCrossEntropyLoss(lambda: (self.shared.weight, None), ignore_index)

    def load_hf_state_dict(self, hf: dict) -> None:
        """Load a ``transformers.T5ForConditionalGeneration`` state dict strictly: self-attention q / k / v fused into
        ``qkv``, cross-attention k / v into ``cross_kv``, each stack's ``relative_attention_bias`` from its block 0;
        ``encoder.embed_tokens`` / ``decoder.embed_tokens`` / ``lm_head`` are tied to ``shared``.  Missing and unexpected
        keys raise ``KeyError``."""
        c = self.config
        out = {}
        used = set()

        def get(k):
            if k not in hf:
                raise KeyError(f"load_hf_state_dict: missing key {k}")
            used.add(k)
            return hf[k]

        out["shared.weight"] = get("shared.weight")
        for k in ("encoder.embed_tokens.weight", "decoder.embed_tokens.weight", "lm_head.weight"):   # tied to shared
            if k in hf:
                used.add(k)
        for side, n in (("encoder", c.num_layers), ("decoder", c.num_decoder_layers)):
            out[f"{side}.relative_attention_bias.weight"] = get(f"{side}.block.0.layer.0.SelfAttention.relative_attention_bias.weight")
            out[f"{side}.final_layer_norm.weight"] = get(f"{side}.final_layer_norm.weight")
            for i in range(n):
                s, d = f"{side}.block.{i}.layer", f"{side}.block.{i}"
                out[f"{d}.self_attn.layer_norm.weight"] = get(f"{s}.0.layer_norm.weight")
                out[f"{d}.self_attn.qkv.weight"] = torch.cat([get(f"{s}.0.SelfAttention.{x}.weight") for x in "qkv"])
                out[f"{d}.self_attn.o.weight"] = get(f"{s}.0.SelfAttention.o.weight")
                ff = 2 if side == "decoder" else 1
                if side == "decoder":
                    out[f"{d}.cross_attn.layer_norm.weight"] = get(f"{s}.1.layer_norm.weight")
                    out[f"{d}.cross_attn.q.weight"] = get(f"{s}.1.EncDecAttention.q.weight")
                    out[f"{d}.cross_attn.cross_kv.weight"] = torch.cat([get(f"{s}.1.EncDecAttention.{x}.weight") for x in "kv"])
                    out[f"{d}.cross_attn.o.weight"] = get(f"{s}.1.EncDecAttention.o.weight")
                out[f"{d}.ff.layer_norm.weight"] = get(f"{s}.{ff}.layer_norm.weight")
                out[f"{d}.ff.wi.weight"] = get(f"{s}.{ff}.DenseReluDense.wi.weight")
                out[f"{d}.ff.wo.weight"] = get(f"{s}.{ff}.DenseReluDense.wo.weight")
        unknown = set(hf) - used
        if unknown:
            raise KeyError(f"load_hf_state_dict: unexpected keys {sorted(unknown)[:8]}")
        own = self.state_dict()
        self.load_state_dict({k: v.to(own[k].dtype).contiguous() for k, v in out.items()}, strict=True)


T5_SMALL = T5Config()
T5_BASE = T5Config(d_model=768, num_layers=12, num_decoder_layers=12, num_heads=12, d_ff=3072)


def _build(preset: T5Config, pad_token_id, bos_token_id, fused_lm_loss) -> T5ForConditionalGeneration:
    return T5ForConditionalGeneration(replace(preset, pad_token_id=pad_token_id, bos_token_id=bos_token_id, fused_lm_loss=fused_lm_loss))


def t5_small(pad_token_id: int | None = None, bos_token_id: int | None = None, fused_lm_loss: bool = False) -> nn.Module:
    """t5-small (6 + 6 layers, d 512, 8 heads, d_ff 2048).  ``pad_token_id`` takes right-padded rows (sources padded with
    it, labels with -100); ``bos_token_id`` packed rows whose documents start with that id on both sides."""
    return _build(T5_SMALL, pad_token_id, bos_token_id, fused_lm_loss)


def t5_base(pad_token_id: int | None = None, bos_token_id: int | None = None, fused_lm_loss: bool = False) -> nn.Module:
    """t5-base (12 + 12 layers, d 768, 12 heads, d_ff 3072); the arguments as ``t5_small``'s."""
    return _build(T5_BASE, pad_token_id, bos_token_id, fused_lm_loss)
