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
eps 1e-6 and tied embeddings: 1,543,714,304 parameters.

``granite_3_0_1b_a400m`` is Granite-3.0-1B-A400M, a sparse mixture of experts: every block's SwiGLU is 32 experts of
width 512 of which each token uses 8 (``ops.MoE``: native routing, expert sort and grouped wgmma GEMMs), 16 query heads
over 8 K/V heads at hidden 1024, 24 layers, Granite's four multipliers and a vocabulary of 49155 padded to 49216:
1,334,690,816 parameters.  ``load_hf_state_dict`` also reads ``transformers.GraniteMoeForCausalLM``'s state dicts.

``qwen3_0_6b`` is Qwen3-0.6B: 16 query heads over 8 K/V heads of dim 128 at hidden 1024 (``explicit_head_dim``: the
heads are 2048 wide together), each query and key head RMS-normalised over its 128 elements with a learned weight
before rotary (``qk_norm``: ``ops.qk_norm_rotary``, one fused kernel per direction), 28 layers, SwiGLU intermediate 3072,
vocabulary 151936, rope theta 1e6, RMSNorm eps 1e-6 and tied embeddings: 596,049,920 parameters.
``load_hf_state_dict`` also reads ``transformers.Qwen3ForCausalLM``'s state dicts."""
from __future__ import annotations

import math
from dataclasses import dataclass, replace

import torch
import torch.nn as nn

from ..ops import (Linear, LinearCrossEntropyLoss, MoE, RMSNorm, causal_attention, document_bounds, linear, qk_norm_rotary, rotary,
                   rotary_cos_sin, swiglu)


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
    # sparse mixture of experts: with num_experts > 0 every block's SwiGLU is num_experts experts of width `intermediate`,
    # experts_per_token of them per token; router_aux_loss_coef > 0 keeps the load-balancing statistics (router_aux_loss)
    num_experts: int = 0
    experts_per_token: int = 0
    router_aux_loss_coef: float = 0.0
    # Granite's multipliers (the defaults leave the model as it is, with no extra op): embedding output, attention scores
    # (None = 1 / sqrt(head_dim)), both residual branches, and 1 / logits_scaling on the final hidden states
    embedding_multiplier: float = 1.0
    attention_multiplier: float | None = None
    residual_multiplier: float = 1.0
    logits_scaling: float = 1.0
    pad_vocab_to: int = 1          # embedding / LM-head rows padded to a multiple of this (GPT-2's mechanism)
    # attention head width when it is not hidden // heads (Qwen3: 16 heads of 128 at hidden 1024); None = hidden // heads
    explicit_head_dim: int | None = None
    qk_norm: bool = False          # per-head RMSNorm of q and k (weights q_norm / k_norm [head_dim]) before rotary (Qwen3)

    @property
    def head_dim(self) -> int:
        return self.hidden // self.heads if self.explicit_head_dim is None else self.explicit_head_dim

    @property
    def padded_vocab(self) -> int:
        m = max(1, self.pad_vocab_to)
        return (self.vocab_size + m - 1) // m * m

    @property
    def q_scale(self) -> float:
        """Factor on q that turns the attention kernels' 1 / sqrt(head_dim) into ``attention_multiplier``."""
        return 1.0 if self.attention_multiplier is None else self.attention_multiplier * math.sqrt(self.head_dim)


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
        if c.num_experts > 0:
            self.moe = MoE(c.hidden, c.intermediate, c.num_experts, c.experts_per_token, aux=c.router_aux_loss_coef > 0)
        else:
            self.gate_up = Linear(c.hidden, 2 * c.intermediate, bias=False, fp8=c.fp8)   # gate | up
            self.down_proj = Linear(c.intermediate, c.hidden, bias=False, fp8=c.fp8)
        if c.qk_norm:
            self.q_norm = RMSNorm(d, eps=c.eps)
            self.k_norm = RMSNorm(d, eps=c.eps)
        self.q_scale, self.residual = c.q_scale, c.residual_multiplier

    def _add(self, x, y):
        return x + y if self.residual == 1.0 else torch.add(x, y, alpha=self.residual)

    def forward(self, x, bounds, position_ids, cos_sin):
        qkv = self.qkv(self.input_layernorm(x))
        if hasattr(self, "q_norm"):
            qkv = qk_norm_rotary(qkv, self.q_norm.weight, self.k_norm.weight, position_ids, cos_sin, self.heads, self.kv_heads,
                                 self.q_norm.eps)
        else:
            qkv = rotary(qkv, position_ids, cos_sin, self.heads, self.kv_heads, self.q_scale)
        x = self._add(x, self.o_proj(causal_attention(qkv, bounds, self.heads, self.kv_heads)))
        h = self.post_attention_layernorm(x)
        return self._add(x, self.moe(h) if hasattr(self, "moe") else self.down_proj(swiglu(self.gate_up(h))))


class LlamaModel(nn.Module):
    def __init__(self, config: LlamaConfig | None = None):
        super().__init__()
        c = self.config = config or LlamaConfig()
        if (c.explicit_head_dim is None and c.hidden % c.heads) or c.heads % c.kv_heads:
            raise ValueError(f"LlamaConfig: heads must divide hidden (unless explicit_head_dim is set) and kv_heads must divide "
                             f"heads, got hidden={c.hidden}, heads={c.heads}, kv_heads={c.kv_heads}")
        if c.explicit_head_dim is not None and (c.explicit_head_dim < 2 or c.explicit_head_dim % 2):
            raise ValueError(f"LlamaConfig: explicit_head_dim must be a positive even number, got {c.explicit_head_dim}")
        if c.qk_norm and c.q_scale != 1.0:
            raise ValueError("LlamaConfig: qk_norm has no query-scale variant; leave attention_multiplier at None")
        if not (c.q_scale > 0 and math.frexp(c.q_scale)[0] == 0.5):
            raise ValueError(f"LlamaConfig: attention_multiplier * sqrt(head_dim) must be a power of two (it scales q exactly in "
                             f"bf16), got {c.attention_multiplier} * sqrt({c.head_dim})")
        if c.num_experts > 0 and not 1 <= c.experts_per_token <= c.num_experts:
            raise ValueError(f"LlamaConfig: experts_per_token must lie in [1, num_experts = {c.num_experts}], got {c.experts_per_token}")
        if c.num_experts > 0 and c.fp8:
            raise ValueError("LlamaConfig: fp8 covers dense block linears; the mixture-of-experts layers have no FP8 path")
        self.embed_tokens = nn.Embedding(c.padded_vocab, c.hidden)
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
        if c.embedding_multiplier != 1.0:
            x = x * c.embedding_multiplier
        for layer in self.layers:
            x = layer(x, bounds, position_ids, self.cos_sin)
        return self.norm(x)


class LlamaForCausalLM(nn.Module):
    """Decoder + LM head tied to the token embedding (no bias); forward returns logits [B, S, vocab], or with
    ``LlamaConfig.fused_lm_loss`` the final hidden states [B, S, hidden], to be scored by ``lm_head_loss()``.

    With ``pad_vocab_to`` padding the vocabulary, the logits are [B, S, padded vocab] and the padded rows get a -1e4 logit
    bias (a non-persistent buffer, as GPT-2's), so they take no probability.  ``logits_scaling`` multiplies the final
    hidden states by 1 / logits_scaling before the head, in both paths; Hugging Face divides the logits instead, so the
    two differ by bf16 rounding only."""

    def __init__(self, config: LlamaConfig | None = None):
        super().__init__()
        self.model = LlamaModel(config)
        c = self.model.config
        bias = None
        if c.padded_vocab != c.vocab_size:
            bias = torch.zeros(c.padded_vocab)
            bias[c.vocab_size:] = -1e4
        self.register_buffer("vocab_bias", bias, persistent=False)

    @property
    def config(self) -> LlamaConfig:
        return self.model.config

    def forward(self, input_ids):
        h = self.model(input_ids)
        if self.config.logits_scaling != 1.0:
            h = h * (1.0 / self.config.logits_scaling)
        if self.config.fused_lm_loss:
            return h
        bias = None if self.vocab_bias is None else self.vocab_bias.to(h.dtype)
        return linear(h, self.model.embed_tokens.weight, bias)

    def lm_head_loss(self, ignore_index: int = -100) -> LinearCrossEntropyLoss:
        """Criterion over ``forward``'s hidden states with ``fused_lm_loss``: the tied head (and the padded-vocabulary bias),
        read from this model at every call."""
        return LinearCrossEntropyLoss(lambda: (self.model.embed_tokens.weight, self.vocab_bias), ignore_index)

    def router_aux_loss(self) -> torch.Tensor:
        """Hugging Face's ``load_balancing_loss_func`` over every layer of the last forward (``attention_mask=None``): E times
        the sum over experts of (fraction of token slots routed to the expert) x (mean router probability), both averaged over
        all layers' tokens together.  Needs ``router_aux_loss_coef > 0``.  Takes the statistics out of the layers, so one
        forward gives one aux loss: left behind, they would keep that forward's autograd graph (and its parameters' gradient
        accumulators) alive into the next step, which a CUDA-graph capture cannot take."""
        states = [layer.moe.aux_state for layer in self.model.layers]
        if any(s is None for s in states):
            raise RuntimeError("router_aux_loss needs a forward of a model built with num_experts > 0 and router_aux_loss_coef > 0, "
                               "and takes that forward's statistics once")
        for layer in self.model.layers:
            layer.moe.aux_state = None
        n = float(sum(s[2] for s in states))
        probs = torch.stack([s[0] for s in states]).sum(0)
        counts = torch.stack([s[1] for s in states]).sum(0).float()
        return (counts * probs).sum() * (self.config.num_experts / (n * n))

    def load_hf_state_dict(self, hf: dict) -> None:
        """Load a ``transformers.LlamaForCausalLM``, ``transformers.Qwen2ForCausalLM``, ``transformers.Qwen3ForCausalLM`` or
        ``transformers.GraniteMoeForCausalLM`` state dict: q / k / v (weights, and biases when the config has
        ``attention_bias``) and gate / up are concatenated into the fused projections, Qwen3's ``self_attn.q_norm`` /
        ``k_norm`` weights (with ``qk_norm``) and GraniteMoe's ``block_sparse_moe`` router and expert weights are taken as
        they are, embedding rows beyond the checkpoint's vocabulary are zero, and a tied ``lm_head.weight`` is ignored."""
        own = self.state_dict()
        emb = hf["model.embed_tokens.weight"]
        if emb.shape[0] != own["model.embed_tokens.weight"].shape[0]:       # padded vocabulary: zero rows beyond the checkpoint's
            emb = torch.cat([emb, emb.new_zeros(own["model.embed_tokens.weight"].shape[0] - emb.shape[0], emb.shape[1])])
        out = {"model.embed_tokens.weight": emb, "model.norm.weight": hf["model.norm.weight"]}
        for i in range(self.config.layers):
            src, dst = f"model.layers.{i}.", f"model.layers.{i}."
            out[dst + "qkv.weight"] = torch.cat([hf[src + f"self_attn.{n}_proj.weight"] for n in "qkv"], 0)
            if self.config.attention_bias:
                out[dst + "qkv.bias"] = torch.cat([hf[src + f"self_attn.{n}_proj.bias"] for n in "qkv"], 0)
            out[dst + "o_proj.weight"] = hf[src + "self_attn.o_proj.weight"]
            if self.config.num_experts > 0:
                moe = src + "block_sparse_moe."
                out[dst + "moe.router.weight"] = hf[moe + "router.layer.weight"]
                out[dst + "moe.w_gate_up"] = hf[moe + "input_linear.weight"]
                out[dst + "moe.w_down"] = hf[moe + "output_linear.weight"]
            else:
                out[dst + "gate_up.weight"] = torch.cat([hf[src + "mlp.gate_proj.weight"], hf[src + "mlp.up_proj.weight"]], 0)
                out[dst + "down_proj.weight"] = hf[src + "mlp.down_proj.weight"]
            for n in ("input_layernorm", "post_attention_layernorm"):
                out[dst + f"{n}.weight"] = hf[src + f"{n}.weight"]
            if self.config.qk_norm:
                for n in ("q_norm", "k_norm"):
                    out[dst + f"{n}.weight"] = hf[src + f"self_attn.{n}.weight"]
        self.load_state_dict({k: v.to(own[k].dtype).contiguous() for k, v in out.items()}, strict=True)


SMOLLM_135M = LlamaConfig()
QWEN2_5_1_5B = LlamaConfig(vocab_size=151936, max_position=32768, hidden=1536, layers=28, heads=12, kv_heads=2,
                           intermediate=8960, eps=1e-6, rope_theta=1e6, attention_bias=True)
QWEN3_0_6B = LlamaConfig(vocab_size=151936, max_position=40960, hidden=1024, layers=28, heads=16, kv_heads=8,
                         intermediate=3072, eps=1e-6, rope_theta=1e6, explicit_head_dim=128, qk_norm=True)
GRANITE_3_0_1B_A400M = LlamaConfig(vocab_size=49155, max_position=4096, hidden=1024, layers=24, heads=16, kv_heads=8,
                                   intermediate=512, eps=1e-6, rope_theta=10000.0, num_experts=32, experts_per_token=8,
                                   router_aux_loss_coef=0.001, embedding_multiplier=12.0, attention_multiplier=0.015625,
                                   residual_multiplier=0.22, logits_scaling=6.0, pad_vocab_to=64)


def smollm_135m(fp8: bool = False, pad_token_id: int | None = None, bos_token_id: int | None = None,
                fused_lm_loss: bool = False) -> nn.Module:
    """SmolLM-135M with its tied LM head; ``fp8=True`` puts the 120 block linears on FP8 tensor cores (embedding and LM
    head stay bf16).  ``pad_token_id`` takes right-padded input; ``bos_token_id`` takes packed documents, each starting
    with that id (attention stays inside a document and position ids restart in each).  ``fused_lm_loss=True``: forward
    returns hidden states and ``lm_head_loss()`` computes the loss without the logits."""
    return LlamaForCausalLM(replace(SMOLLM_135M, fp8=fp8, pad_token_id=pad_token_id, bos_token_id=bos_token_id,
                                    fused_lm_loss=fused_lm_loss))


def qwen2_5_1_5b(fp8: bool = False, pad_token_id: int | None = None, bos_token_id: int | None = None,
                 fused_lm_loss: bool = False) -> nn.Module:
    """Qwen2.5-1.5B with its tied LM head (32768 positions); ``fp8=True`` puts the 112 block linears on FP8 tensor cores.
    ``pad_token_id``, ``bos_token_id`` and ``fused_lm_loss`` as for ``smollm_135m``."""
    return LlamaForCausalLM(replace(QWEN2_5_1_5B, fp8=fp8, pad_token_id=pad_token_id, bos_token_id=bos_token_id,
                                    fused_lm_loss=fused_lm_loss))


def qwen3_0_6b(fp8: bool = False, pad_token_id: int | None = None, bos_token_id: int | None = None,
               fused_lm_loss: bool = False) -> nn.Module:
    """Qwen3-0.6B with its tied LM head (40960 positions): 28 blocks of grouped-query attention (16 query heads over 8 K/V
    heads of dim 128 at hidden 1024, so heads * head_dim = 2048 is not the hidden size) with per-head q / k RMSNorm before
    rotary, SwiGLU intermediate 3072, vocabulary 151936; ``fp8=True`` puts the 112 block linears on FP8 tensor cores.
    ``pad_token_id``, ``bos_token_id`` and ``fused_lm_loss`` as for ``smollm_135m``."""
    return LlamaForCausalLM(replace(QWEN3_0_6B, fp8=fp8, pad_token_id=pad_token_id, bos_token_id=bos_token_id,
                                    fused_lm_loss=fused_lm_loss))


def granite_3_0_1b_a400m(pad_token_id: int | None = None, bos_token_id: int | None = None, fused_lm_loss: bool = False,
                         router_aux_loss_coef: float = GRANITE_3_0_1B_A400M.router_aux_loss_coef) -> nn.Module:
    """Granite-3.0-1B-A400M with its tied LM head (4096 positions): 24 blocks of grouped-query attention (16 query heads
    over 8 K/V heads, head dim 64) and a mixture of 32 SwiGLU experts of width 512, 8 per token; embedding multiplier 12,
    attention multiplier 1/64, residual multiplier 0.22, logits scaling 6; vocabulary 49155 padded to 49216.
    ``router_aux_loss_coef`` (transformers' default 0.001; 0 turns it off) weights ``router_aux_loss`` in the training
    loss.  ``pad_token_id``, ``bos_token_id`` and ``fused_lm_loss`` as for ``smollm_135m``."""
    return LlamaForCausalLM(replace(GRANITE_3_0_1B_A400M, router_aux_loss_coef=router_aux_loss_coef, pad_token_id=pad_token_id,
                                    bos_token_id=bos_token_id, fused_lm_loss=fused_lm_loss))
