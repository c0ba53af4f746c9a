"""Mamba-2 state-space causal language model (transformers' ``Mamba2ForCausalLM``); the presets are mamba2-130m (hidden 768,
24 layers, 24 heads, 128,989,632 parameters) and mamba2-370m (hidden 1024, 48 layers, 32 heads, 368,346,624 parameters),
with one group, head dim 64, state 128, expand 2, conv width 4, no linear biases, a conv bias, vocabulary 50288 (the
released checkpoints' padded GPT-NeoX vocabulary), RMSNorm eps 1e-5 and the LM head tied to the embedding.

Each block: fp32 residual stream -> RMSNorm (its input cast to the weight's dtype first) -> bias-free ``in_proj`` to
zxbcdt [T, W] = z [0, E) | xBC [E, 2E + 2N) | dt [2E + 2N, W), W = 2E + 2N + H -> ``ops.causal_conv1d_window`` over the xBC
columns (x | B | C = silu(conv(xBC) + bias)) -> ``ops.ssd_scan`` (dt = softplus(dt + dt_bias), A = -exp(A_log), D skip)
-> ``ops.gated_rms_norm`` (weight * rmsnorm(y silu(z)), z read in place) -> bias-free ``out_proj`` -> fp32 residual add.
The three backwards fill disjoint columns of one in_proj gradient through ``ops.Mamba2GradLink``.  The state resets at each
document start of ``document_bounds``: one document per row for fixed rows, one per row up to its length with
``Mamba2Config.pad_token_id``, and packed documents (each starting with ``bos_token_id``) with ``Mamba2Config.bos_token_id``.

In bf16 on the GPU the linears are the wgmma kernels and the conv, scan and gated norm are native kernels
(``csrc/mamba.cu``, ``csrc/mamba2.cu``, ``csrc/layernorm.cu``); on the CPU, and in fp32 anywhere, the ops run torch
references with the arithmetic of transformers' ``torch_forward``.  ``A_log``, ``D`` and ``dt_bias`` (all [H]) stay fp32
under ``to_mixed_bf16``; the AdamW rule of this project (decay iff ``ndim >= 2``) decays none of the three.
``load_hf_state_dict`` reads transformers' state dict."""
from __future__ import annotations

import math
from dataclasses import dataclass, replace

import torch
import torch.nn as nn

from ..ops import (Linear, LinearCrossEntropyLoss, Mamba2GradLink, RMSNorm, causal_conv1d_window, document_bounds, gated_rms_norm, linear,
                   ssd_scan)


@dataclass
class Mamba2Config:
    vocab_size: int = 50288
    max_position: int = 2048       # no positions: a training cap on the sequence length (the released checkpoints' context)
    hidden: int = 768
    layers: int = 24
    heads: int = 24
    head_dim: int = 64
    state: int = 128
    n_groups: int = 1
    conv_kernel: int = 4
    expand: int = 2
    eps: float = 1e-5
    initializer_range: float = 0.1
    time_step_min: float = 0.001
    time_step_max: float = 0.1
    time_step_floor: float = 1e-4
    pad_token_id: int | None = None  # right-padded input: length = non-pad count per row
    bos_token_id: int | None = None  # packed input: a document starts at each such id (and at 0), the state resets there
    fused_lm_loss: bool = False    # forward returns the final hidden states; ``lm_head_loss`` applies the head inside the loss

    @property
    def intermediate(self) -> int:
        return self.expand * self.hidden

    @property
    def conv_dim(self) -> int:
        return self.intermediate + 2 * self.n_groups * self.state


class Mamba2Mixer(nn.Module):
    """transformers' ``Mamba2Mixer`` parameters (``in_proj``, ``conv1d`` [conv_dim, 1, 4] with bias, ``dt_bias``, ``A_log``,
    ``D``, ``norm.weight``, ``out_proj``) on the native conv, SSD scan and gated norm."""

    keep_fp32_params = ("A_log", "D", "dt_bias")      # the scan reads them in fp32

    def __init__(self, c: Mamba2Config):
        super().__init__()
        E, H = c.intermediate, c.heads
        if c.head_dim != 64 or c.state != 128 or c.n_groups != 1 or c.conv_kernel != 4 or H * c.head_dim != E:
            raise ValueError(f"Mamba2Config: the kernels take head dim 64, state 128, one group, conv width 4 and heads * head_dim = "
                             f"expand * hidden, got {c.head_dim}, {c.state}, {c.n_groups}, {c.conv_kernel} and {H} * {c.head_dim} vs {E}")
        self.E, self.H, self.eps = E, H, c.eps
        self.in_proj = Linear(c.hidden, 2 * E + 2 * c.state + H, bias=False)
        self.conv1d = nn.Conv1d(c.conv_dim, c.conv_dim, c.conv_kernel, groups=c.conv_dim, padding=c.conv_kernel - 1, bias=True)
        self.dt_bias = nn.Parameter(torch.empty(H))
        self.A_log = nn.Parameter(torch.log(torch.arange(1, H + 1, dtype=torch.float32)))
        self.norm = nn.Module()
        self.norm.weight = nn.Parameter(torch.ones(E))
        self.D = nn.Parameter(torch.ones(H))
        self.out_proj = Linear(E, c.hidden, bias=False)
        with torch.no_grad():
            std = c.initializer_range
            nn.init.normal_(self.in_proj.weight, std=std)
            dt = torch.exp(torch.rand(H) * (math.log(c.time_step_max) - math.log(c.time_step_min)) + math.log(c.time_step_min))
            dt = dt.clamp(min=c.time_step_floor)
            self.dt_bias.copy_(dt + torch.log(-torch.expm1(-dt)))      # inverse softplus
            nn.init.kaiming_uniform_(self.conv1d.weight, a=math.sqrt(5))
            nn.init.zeros_(self.conv1d.bias)
            nn.init.kaiming_uniform_(self.out_proj.weight, a=math.sqrt(5))

    def forward(self, x, bounds):
        E, H = self.E, self.H
        zxbcdt = self.in_proj(x)
        link = Mamba2GradLink(zxbcdt)
        xbc = causal_conv1d_window(zxbcdt, self.conv1d.weight, self.conv1d.bias, bounds, col=E, link=link)
        y = ssd_scan(xbc, zxbcdt[..., zxbcdt.shape[-1] - H:], self.A_log, self.D, self.dt_bias, bounds, link=link)
        y = gated_rms_norm(y, zxbcdt[..., :E], self.norm.weight, self.eps, link=link)
        return self.out_proj(y)


class Mamba2Block(nn.Module):
    def __init__(self, c: Mamba2Config):
        super().__init__()
        self.norm = RMSNorm(c.hidden, eps=c.eps)
        self.mixer = Mamba2Mixer(c)

    def forward(self, residual, bounds):
        return residual + self.mixer(self.norm(residual.to(self.norm.weight.dtype)), bounds)


class Mamba2Model(nn.Module):
    def __init__(self, config: Mamba2Config | None = None):
        super().__init__()
        c = self.config = config or Mamba2Config()
        self.embeddings = nn.Embedding(c.vocab_size, c.hidden)
        nn.init.normal_(self.embeddings.weight, std=c.initializer_range)
        self.layers = nn.ModuleList([Mamba2Block(c) for _ in range(c.layers)])
        self.norm_f = RMSNorm(c.hidden, eps=c.eps)

    def forward(self, input_ids):
        c = self.config
        if input_ids.shape[1] > c.max_position:
            raise ValueError(f"Mamba2Model: sequence length {input_ids.shape[1]} exceeds max_position {c.max_position}")
        bounds, _ = document_bounds(input_ids, c.bos_token_id, c.pad_token_id)
        bounds = bounds.to(torch.int32)
        x = self.embeddings(input_ids).float()        # residual_in_fp32
        for layer in self.layers:
            x = layer(x, bounds)
        return self.norm_f(x.to(self.norm_f.weight.dtype))


class Mamba2ForCausalLM(nn.Module):
    """Backbone + LM head tied to the embedding (no bias); forward returns logits [B, S, vocab], or with
    ``Mamba2Config.fused_lm_loss`` the final hidden states [B, S, hidden], to be scored by ``lm_head_loss()``."""

    def __init__(self, config: Mamba2Config | None = None):
        super().__init__()
        self.backbone = Mamba2Model(config)

    @property
    def config(self) -> Mamba2Config:
        return self.backbone.config

    def forward(self, input_ids):
        h = self.backbone(input_ids)
        if self.config.fused_lm_loss:
            return h
        return linear(h, self.backbone.embeddings.weight)

    def lm_head_loss(self, ignore_index: int = -100) -> LinearCrossEntropyLoss:
        """Criterion over ``forward``'s hidden states with ``fused_lm_loss``: the tied head, read from this model at every call."""
        return LinearCrossEntropyLoss(lambda: (self.backbone.embeddings.weight, None), ignore_index)

    def load_hf_state_dict(self, hf: dict) -> None:
        """Load a ``transformers.Mamba2ForCausalLM`` state dict: the names are the same, and the tied ``lm_head.weight`` must
        equal the embedding."""
        hf = dict(hf)
        head = hf.pop("lm_head.weight", None)
        if head is not None and not torch.equal(head, hf["backbone.embeddings.weight"]):
            raise ValueError("load_hf_state_dict: lm_head.weight differs from backbone.embeddings.weight; this model ties them")
        own = self.state_dict()
        self.load_state_dict({k: v.to(own[k].dtype) if k in own else v for k, v in hf.items()}, strict=True)


MAMBA2_130M = Mamba2Config()
MAMBA2_370M = Mamba2Config(hidden=1024, layers=48, heads=32)


def _build(preset: Mamba2Config, pad_token_id, bos_token_id, fused_lm_loss) -> Mamba2ForCausalLM:
    return Mamba2ForCausalLM(replace(preset, pad_token_id=pad_token_id, bos_token_id=bos_token_id, fused_lm_loss=fused_lm_loss))


def mamba2_130m(pad_token_id: int | None = None, bos_token_id: int | None = None, fused_lm_loss: bool = False) -> nn.Module:
    """mamba2-130m with its tied LM head.  ``pad_token_id`` takes right-padded input; ``bos_token_id`` takes packed
    documents, each starting with that id (the state resets there).  ``fused_lm_loss=True``: forward returns hidden states
    and ``lm_head_loss()`` computes the loss without the logits."""
    return _build(MAMBA2_130M, pad_token_id, bos_token_id, fused_lm_loss)


def mamba2_370m(pad_token_id: int | None = None, bos_token_id: int | None = None, fused_lm_loss: bool = False) -> nn.Module:
    """mamba2-370m (hidden 1024, 48 layers, 32 heads); arguments as for ``mamba2_130m``."""
    return _build(MAMBA2_370M, pad_token_id, bos_token_id, fused_lm_loss)
