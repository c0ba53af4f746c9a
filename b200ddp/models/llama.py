"""Llama-architecture causal language model; the defaults are SmolLM-135M (hidden 576, 30 layers, 9 query heads over 3
K/V heads, SwiGLU intermediate 1536, vocabulary 49152, tied embeddings, 134,515,008 parameters).
Pre-norm decoder blocks: RMSNorm -> fused q | k | v projection (bias-free unless ``attention_bias``) -> rotary
embedding -> grouped-query causal attention -> o_proj -> RMSNorm -> fused gate | up projection -> SwiGLU -> down_proj.
Every linear is a ``b200ddp.ops.Linear`` (wgmma GEMM, or FP8 with ``fp8=True``), every norm, the rotary embedding, SwiGLU and attention
are the hand-written kernels, and the LM head is tied to the token embedding.  Attention always runs on the native
causal kernel with documents from ``document_bounds``: one full-length document per row for fixed-length rows, one per
row up to its length with ``LlamaConfig.pad_token_id``, and packed documents (each starting with ``bos_token_id``, with
position ids restarting in each) with ``LlamaConfig.bos_token_id``.  ``load_hf_state_dict`` reads
``transformers.LlamaForCausalLM``'s and ``transformers.Qwen2ForCausalLM``'s state dicts.

``qwen2_5_1_5b`` is Qwen2.5-1.5B: the same blocks with a bias on the q | k | v projection (``attention_bias``), head dim
128 (12 query heads over 2 K/V heads at hidden 1536), SwiGLU intermediate 8960, vocabulary 151936, rope theta 1e6, RMSNorm
eps 1e-6 and tied embeddings: 1,543,714,304 parameters."""
from __future__ import annotations

from dataclasses import dataclass

import torch
import torch.nn as nn

from ..ops import Linear, LinearCrossEntropyLoss, RMSNorm, causal_attention, document_bounds, linear, rotary, rotary_cos_sin, swiglu


@dataclass
class LlamaConfig:
    vocab_size: int = 49152
    max_position: int = 2048
    hidden: int = 576
    layers: int = 30
    heads: int = 9
    kv_heads: int = 3
    intermediate: int = 1536
    eps: float = 1e-5
    rope_theta: float = 10000.0
    attention_bias: bool = False   # a bias on the fused q | k | v projection only, laid out [q_bias | k_bias | v_bias]
    fp8: bool = False              # block linears (qkv, o_proj, gate_up, down_proj) on FP8 tensor cores; same parameters
    pad_token_id: int | None = None  # right-padded input: length = non-pad count per row
    bos_token_id: int | None = None  # packed input: a document starts at each such id (and at 0), attention stays inside it
    fused_lm_loss: bool = False    # forward returns the final hidden states; ``lm_head_loss`` applies the head inside the loss

    @property
    def head_dim(self) -> int:
        return self.hidden // self.heads


class LlamaBlock(nn.Module):
    def __init__(self, c: LlamaConfig):
        super().__init__()
        self.heads, self.kv_heads = c.heads, c.kv_heads
        d = c.head_dim
        self.input_layernorm = RMSNorm(c.hidden, eps=c.eps)
        # q | k | v in one stored [(heads + 2 * kv_heads) * d, hidden] projection, so attention reads it without a copy
        self.qkv = Linear(c.hidden, (c.heads + 2 * c.kv_heads) * d, bias=c.attention_bias, fp8=c.fp8)
        self.o_proj = Linear(c.heads * d, c.hidden, bias=False, fp8=c.fp8)
        self.post_attention_layernorm = RMSNorm(c.hidden, eps=c.eps)
        self.gate_up = Linear(c.hidden, 2 * c.intermediate, bias=False, fp8=c.fp8)   # gate | up
        self.down_proj = Linear(c.intermediate, c.hidden, bias=False, fp8=c.fp8)

    def forward(self, x, bounds, position_ids, cos_sin):
        qkv = rotary(self.qkv(self.input_layernorm(x)), position_ids, cos_sin, self.heads, self.kv_heads)
        x = x + self.o_proj(causal_attention(qkv, bounds, self.heads, self.kv_heads))
        return x + self.down_proj(swiglu(self.gate_up(self.post_attention_layernorm(x))))


class LlamaModel(nn.Module):
    def __init__(self, config: LlamaConfig | None = None):
        super().__init__()
        c = self.config = config or LlamaConfig()
        if c.hidden % c.heads or c.heads % c.kv_heads:
            raise ValueError(f"LlamaConfig: heads must divide hidden and kv_heads must divide heads, got hidden={c.hidden}, "
                             f"heads={c.heads}, kv_heads={c.kv_heads}")
        self.embed_tokens = nn.Embedding(c.vocab_size, c.hidden)
        self.layers = nn.ModuleList([LlamaBlock(c) for _ in range(c.layers)])
        self.norm = RMSNorm(c.hidden, eps=c.eps)
        self.register_buffer("cos_sin", rotary_cos_sin(c.max_position, c.head_dim, c.rope_theta), persistent=False)
        self.apply(self._init)

    @staticmethod
    def _init(m):
        if isinstance(m, (Linear, nn.Embedding)):
            nn.init.normal_(m.weight, std=0.02)
        if isinstance(m, Linear) and m.bias is not None:
            nn.init.zeros_(m.bias)

    def _apply(self, fn, recurse=True):
        # the rotary table stays fp32 whatever dtype the parameters are cast to
        table = self.cos_sin
        out = super()._apply(fn, recurse)
        self.cos_sin = table.to(device=self.cos_sin.device, dtype=torch.float32)
        return out

    def forward(self, input_ids):
        B, S = input_ids.shape
        c = self.config
        if S > c.max_position:
            raise ValueError(f"LlamaModel: sequence length {S} exceeds max_position {c.max_position}")
        # documents and per-document positions, on the device (no host synchronisation); the positions are converted
        # once here to the int32 ids the rotary kernel reads, rather than once per layer
        bounds, position_ids = document_bounds(input_ids, c.bos_token_id, c.pad_token_id)
        position_ids = position_ids.to(torch.int32)
        x = self.embed_tokens(input_ids)
        for layer in self.layers:
            x = layer(x, bounds, position_ids, self.cos_sin)
        return self.norm(x)


class LlamaForCausalLM(nn.Module):
    """Decoder + LM head tied to the token embedding (no bias); forward returns logits [B, S, vocab], or with
    ``LlamaConfig.fused_lm_loss`` the final hidden states [B, S, hidden], to be scored by ``lm_head_loss()``."""

    def __init__(self, config: LlamaConfig | None = None):
        super().__init__()
        self.model = LlamaModel(config)

    @property
    def config(self) -> LlamaConfig:
        return self.model.config

    def forward(self, input_ids):
        h = self.model(input_ids)
        return h if self.config.fused_lm_loss else linear(h, self.model.embed_tokens.weight)

    def lm_head_loss(self, ignore_index: int = -100) -> LinearCrossEntropyLoss:
        """Criterion over ``forward``'s hidden states with ``fused_lm_loss``: the tied head, read from this model at every call."""
        return LinearCrossEntropyLoss(lambda: (self.model.embed_tokens.weight, None), ignore_index)

    def load_hf_state_dict(self, hf: dict) -> None:
        """Load a ``transformers.LlamaForCausalLM`` or ``transformers.Qwen2ForCausalLM`` state dict: q / k / v (weights, and
        biases when the config has ``attention_bias``) and gate / up are concatenated into the fused projections, a tied
        ``lm_head.weight`` is ignored."""
        own = self.state_dict()
        out = {"model.embed_tokens.weight": hf["model.embed_tokens.weight"], "model.norm.weight": hf["model.norm.weight"]}
        for i in range(self.config.layers):
            src, dst = f"model.layers.{i}.", f"model.layers.{i}."
            out[dst + "qkv.weight"] = torch.cat([hf[src + f"self_attn.{n}_proj.weight"] for n in "qkv"], 0)
            if self.config.attention_bias:
                out[dst + "qkv.bias"] = torch.cat([hf[src + f"self_attn.{n}_proj.bias"] for n in "qkv"], 0)
            out[dst + "o_proj.weight"] = hf[src + "self_attn.o_proj.weight"]
            out[dst + "gate_up.weight"] = torch.cat([hf[src + "mlp.gate_proj.weight"], hf[src + "mlp.up_proj.weight"]], 0)
            out[dst + "down_proj.weight"] = hf[src + "mlp.down_proj.weight"]
            for n in ("input_layernorm", "post_attention_layernorm"):
                out[dst + f"{n}.weight"] = hf[src + f"{n}.weight"]
        self.load_state_dict({k: v.to(own[k].dtype).contiguous() for k, v in out.items()}, strict=True)


def smollm_135m(fp8: bool = False, pad_token_id: int | None = None, bos_token_id: int | None = None,
                fused_lm_loss: bool = False) -> nn.Module:
    """SmolLM-135M with its tied LM head; ``fp8=True`` puts the 120 block linears on FP8 tensor cores (embedding and LM
    head stay bf16).  ``pad_token_id`` takes right-padded input; ``bos_token_id`` takes packed documents, each starting
    with that id (attention stays inside a document and position ids restart in each).  ``fused_lm_loss=True``: forward
    returns hidden states and ``lm_head_loss()`` computes the loss without the logits."""
    return LlamaForCausalLM(LlamaConfig(fp8=fp8, pad_token_id=pad_token_id, bos_token_id=bos_token_id, fused_lm_loss=fused_lm_loss))


def qwen2_5_1_5b(fp8: bool = False, pad_token_id: int | None = None, bos_token_id: int | None = None,
                 fused_lm_loss: bool = False) -> nn.Module:
    """Qwen2.5-1.5B with its tied LM head (32768 positions); ``fp8=True`` puts the 112 block linears on FP8 tensor cores.
    ``pad_token_id``, ``bos_token_id`` and ``fused_lm_loss`` as for ``smollm_135m``."""
    return LlamaForCausalLM(LlamaConfig(vocab_size=151936, max_position=32768, hidden=1536, layers=28, heads=12, kv_heads=2,
                                        intermediate=8960, eps=1e-6, rope_theta=1e6, attention_bias=True, fp8=fp8,
                                        pad_token_id=pad_token_id, bos_token_id=bos_token_id, fused_lm_loss=fused_lm_loss))
