"""GPT-2 (124 M) causal language model for the "GPT-2 DDP bf16, seq 1024" config.
Pre-LN decoder blocks: every linear is a ``b200ddp.ops.Linear`` (wgmma GEMM, the MLP's with the tanh GELU), every
LayerNorm the hand-written kernel, the loss the fused cross-entropy, and the LM head is tied to the token embedding.
Attention on fixed-length rows uses torch's SDPA with ``is_causal=True`` (library flash attention); with
``GPTConfig.pad_token_id`` set, right-padded rows run on the native causal kernel (``ops.causal_attention``) with one
document ``(0, length)`` per row, so tiles of padding are skipped; with ``GPTConfig.bos_token_id`` set, rows hold
packed documents (each starting with that id), attention is causal inside each document and position ids restart in
each.  The state dict is the same in every mode; ``load_hf_state_dict`` reads ``transformers.GPT2LMHeadModel``'s."""
from __future__ import annotations

from dataclasses import dataclass, replace

import torch
import torch.nn as nn
import torch.nn.functional as F

from ..ops import LayerNorm, Linear, LinearCrossEntropyLoss, causal_attention, document_bounds, linear


@dataclass
class GPTConfig:
    vocab_size: int = 50257
    max_position: int = 1024
    hidden: int = 768
    layers: int = 12
    heads: int = 12
    intermediate: int = 3072
    eps: float = 1e-5
    pad_vocab_to: int = 64         # LM head rows padded so logits rows keep the 16-byte pitch TMA needs (50257 -> 50304)
    fp8: bool = False              # block linears (qkv, attn_out, ffn_in, ffn_out) on FP8 tensor cores; same parameters
    pad_token_id: int | None = None  # right-padded input: length = non-pad count per row, attention on the native kernel
    bos_token_id: int | None = None  # packed input: a document starts at each such id (and at 0), attention stays inside it
    fused_lm_loss: bool = False    # forward returns the final hidden states; ``lm_head_loss`` applies the head inside the loss

    @property
    def padded_vocab(self) -> int:
        m = max(1, self.pad_vocab_to)
        return (self.vocab_size + m - 1) // m * m


class GPTBlock(nn.Module):
    def __init__(self, c: GPTConfig):
        super().__init__()
        self.heads = c.heads
        self.ln_1 = LayerNorm(c.hidden, eps=c.eps)
        # Q, K and V are one stored [3*hidden, hidden] projection (rows: query, key, value), as GPT-2's own c_attn
        self.qkv = Linear(c.hidden, 3 * c.hidden, fp8=c.fp8)
        self.attn_out = Linear(c.hidden, c.hidden, fp8=c.fp8)
        self.ln_2 = LayerNorm(c.hidden, eps=c.eps)
        self.ffn_in = Linear(c.hidden, c.intermediate, activation="gelu_tanh", fp8=c.fp8)
        self.ffn_out = Linear(c.intermediate, c.hidden, fp8=c.fp8)

    def forward(self, x, bounds=None):
        B, S, H = x.shape
        qkv = self.qkv(self.ln_1(x))
        if bounds is not None:
            a = causal_attention(qkv, bounds, self.heads)  # [B, S, H], the layout attn_out reads
        else:
            q, k, v = (t.view(B, S, self.heads, H // self.heads).transpose(1, 2) for t in qkv.split(H, dim=-1))
            a = F.scaled_dot_product_attention(q, k, v, is_causal=True).transpose(1, 2).reshape(B, S, H)
        x = x + self.attn_out(a)
        return x + self.ffn_out(self.ffn_in(self.ln_2(x)))


class GPTModel(nn.Module):
    def __init__(self, config: GPTConfig | None = None):
        super().__init__()
        c = self.config = config or GPTConfig()
        self.wte = nn.Embedding(c.padded_vocab, c.hidden)
        self.wpe = nn.Embedding(c.max_position, c.hidden)
        self.h = nn.ModuleList([GPTBlock(c) for _ in range(c.layers)])
        self.ln_f = LayerNorm(c.hidden, eps=c.eps)
        self.apply(self._init)

    @staticmethod
    def _init(m):
        if isinstance(m, (Linear, nn.Embedding)):
            nn.init.normal_(m.weight, std=0.02)
            if getattr(m, "bias", None) is not None:
                nn.init.zeros_(m.bias)

    def forward(self, input_ids):
        B, S = input_ids.shape
        c = self.config
        if S > c.max_position:
            raise ValueError(f"GPTModel: sequence length {S} exceeds max_position {c.max_position}")
        bounds = position_ids = None
        if c.bos_token_id is not None or c.pad_token_id is not None:
            # documents (one per row without a BOS id) and per-document positions, on the device (no host synchronisation)
            bounds, position_ids = document_bounds(input_ids, c.bos_token_id, c.pad_token_id)
            if c.bos_token_id is None:
                position_ids = None
        pos = self.wpe(torch.arange(S, device=input_ids.device))[None] if position_ids is None else self.wpe(position_ids)
        x = self.wte(input_ids) + pos
        for block in self.h:
            x = block(x, bounds)
        return self.ln_f(x)


class GPTLMHeadModel(nn.Module):
    """Decoder + LM head tied to the token embedding (no bias); forward returns logits [B, S, padded vocab].  The padded
    vocabulary rows get a large negative logit bias (a non-persistent buffer, through the GEMM epilogue), so they take
    no probability and leave the loss unchanged.  With ``GPTConfig.fused_lm_loss`` forward returns the final hidden states
    [B, S, hidden] instead and ``lm_head_loss()`` is the criterion that applies the head (``ops.linear_cross_entropy``)."""

    def __init__(self, config: GPTConfig | None = None):
        super().__init__()
        self.transformer = GPTModel(config)
        c = self.transformer.config
        bias = torch.zeros(c.padded_vocab)
        bias[c.vocab_size:] = -1e4
        self.register_buffer("vocab_bias", bias, persistent=False)

    @property
    def config(self) -> GPTConfig:
        return self.transformer.config

    def forward(self, input_ids):
        h = self.transformer(input_ids)
        if self.config.fused_lm_loss:
            return h
        return linear(h, self.transformer.wte.weight, self.vocab_bias.to(h.dtype))

    def lm_head_loss(self, ignore_index: int = -100) -> LinearCrossEntropyLoss:
        """Criterion over ``forward``'s hidden states with ``fused_lm_loss``: the tied head and the padded-vocabulary bias,
        read from this model at every call."""
        return LinearCrossEntropyLoss(lambda: (self.transformer.wte.weight, self.vocab_bias), ignore_index)

    def load_hf_state_dict(self, hf: dict) -> None:
        """Load a ``transformers.GPT2LMHeadModel`` state dict.  Its ``Conv1D`` weights are stored [in, out] and are
        transposed here; ``c_attn`` is already the fused query | key | value projection.  Vocabulary rows beyond the
        checkpoint's are zero."""
        c = self.config
        own = self.state_dict()
        out = {}

        def put(dst, src, transpose=False):
            t = hf[src].t() if transpose else hf[src]
            if own[dst].shape != t.shape:                         # padded vocabulary
                full = torch.zeros_like(own[dst])
                full[:t.shape[0]] = t
                t = full
            out[dst] = t.to(own[dst].dtype).contiguous()

        put("transformer.wte.weight", "transformer.wte.weight")
        put("transformer.wpe.weight", "transformer.wpe.weight")
        for wb in ("weight", "bias"):
            put(f"transformer.ln_f.{wb}", f"transformer.ln_f.{wb}")
            for i in range(c.layers):
                for src, dst in (("ln_1", "ln_1"), ("ln_2", "ln_2")):
                    put(f"transformer.h.{i}.{dst}.{wb}", f"transformer.h.{i}.{src}.{wb}")
                for src, dst in (("attn.c_attn", "qkv"), ("attn.c_proj", "attn_out"), ("mlp.c_fc", "ffn_in"),
                                 ("mlp.c_proj", "ffn_out")):
                    put(f"transformer.h.{i}.{dst}.{wb}", f"transformer.h.{i}.{src}.{wb}", transpose=wb == "weight")
        self.load_state_dict(out, strict=True)


GPT2 = GPTConfig()


def gpt2(fp8: bool = False, pad_token_id: int | None = None, bos_token_id: int | None = None,
         fused_lm_loss: bool = False) -> nn.Module:
    """GPT-2 small (124 M) with its LM head; ``fp8=True`` puts the 48 block linears on FP8 tensor cores (embeddings and
    the tied LM head stay bf16).  ``pad_token_id`` takes right-padded input; ``bos_token_id`` takes packed documents,
    each starting with that id (causal attention stays inside a document and position ids restart in each).
    ``fused_lm_loss=True``: forward returns hidden states and ``lm_head_loss()`` computes the loss without the logits."""
    return GPTLMHeadModel(replace(GPT2, fp8=fp8, pad_token_id=pad_token_id, bos_token_id=bos_token_id, fused_lm_loss=fused_lm_loss))
