"""Mamba-1 state-space causal language model (transformers' ``MambaForCausalLM``); the presets are mamba-130m (hidden 768,
24 layers, 129,135,360 parameters) and mamba-370m (hidden 1024, 48 layers, 371,516,416 parameters), with intermediate
E = 2 hidden, state N = 16, conv width 4, ``time_step_rank`` = ceil(hidden / 16), vocabulary 50280, RMSNorm eps 1e-5 and
the LM head tied to the embedding.

Each block: fp32 residual stream -> RMSNorm (its input cast to the weight's dtype first) -> bias-free ``in_proj`` to
x | z [T, 2E] -> ``ops.causal_conv1d`` (u = silu(conv(x) + bias)) -> bias-free ``x_proj`` to dt | B | C -> bias-free
``dt_proj`` on dt (its bias is added inside the scan in fp32, then softplus, as transformers' CUDA path does) ->
``ops.selective_scan`` (y gated by silu(z)) -> bias-free ``out_proj`` -> fp32 residual add.  The state resets at each
document start of ``document_bounds``: one document per row for fixed rows, one per row up to its length with
``MambaConfig.pad_token_id``, and packed documents (each starting with ``bos_token_id``) with ``MambaConfig.bos_token_id``.

In bf16 on the GPU the linears are the wgmma kernels and the conv and scan are the native kernels in ``csrc/mamba.cu``;
on the CPU, and in fp32 anywhere, the ops run torch references with the arithmetic of transformers' ``slow_forward``.
``A_log``, ``D`` and ``dt_proj.bias`` stay fp32 under ``to_mixed_bf16``.  Under the AdamW rule of this project (decay iff
``ndim >= 2``) ``A_log`` [E, 16] is decayed and ``D`` [E] is not.  ``load_hf_state_dict`` reads transformers' state dict."""
from __future__ import annotations

import math
from dataclasses import dataclass, replace

import torch
import torch.nn as nn

from ..ops import Linear, LinearCrossEntropyLoss, MambaGradLink, RMSNorm, causal_conv1d, document_bounds, linear, selective_scan


@dataclass
class MambaConfig:
    vocab_size: int = 50280
    max_position: int = 2048       # no positions: a training cap on the sequence length (the released checkpoints' context)
    hidden: int = 768
    layers: int = 24
    state: int = 16
    conv_kernel: int = 4
    expand: int = 2
    time_step_rank: int | None = None   # None = ceil(hidden / 16)
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
    def rank(self) -> int:
        return math.ceil(self.hidden / 16) if self.time_step_rank is None else self.time_step_rank


class MambaMixer(nn.Module):
    """transformers' ``MambaMixer`` parameters (``in_proj``, ``conv1d`` [E, 1, 4] with bias, ``x_proj``, ``dt_proj``,
    ``A_log``, ``D``, ``out_proj``) on the native conv and scan."""

    keep_fp32_params = ("A_log", "D", "dt_proj.bias")      # the scan reads them in fp32

    def __init__(self, c: MambaConfig):
        super().__init__()
        E, N, R = c.intermediate, c.state, c.rank
        if N != 16 or c.conv_kernel != 4:
            raise ValueError(f"MambaConfig: the kernels take state 16 and conv width 4, got {N} and {c.conv_kernel}")
        self.in_proj = Linear(c.hidden, 2 * E, bias=False)
        self.conv1d = nn.Conv1d(E, E, c.conv_kernel, groups=E, padding=c.conv_kernel - 1, bias=True)
        self.x_proj = Linear(E, R + 2 * N, bias=False)
        self.dt_proj = Linear(R, E, bias=True)
        self.A_log = nn.Parameter(torch.log(torch.arange(1, N + 1, dtype=torch.float32)).repeat(E, 1))
        self.D = nn.Parameter(torch.ones(E))
        self.out_proj = Linear(E, c.hidden, bias=False)
        self.rank = R
        with torch.no_grad():
            std = c.initializer_range
            nn.init.normal_(self.in_proj.weight, std=std)
            nn.init.normal_(self.x_proj.weight, std=std)
            nn.init.uniform_(self.dt_proj.weight, -R ** -0.5, R ** -0.5)
            dt = torch.exp(torch.rand(E) * (math.log(c.time_step_max) - math.log(c.time_step_min)) + math.log(c.time_step_min))
            dt = dt.clamp(min=c.time_step_floor)
            self.dt_proj.bias.copy_(dt + torch.log(-torch.expm1(-dt)))      # inverse softplus
            nn.init.kaiming_uniform_(self.conv1d.weight, a=math.sqrt(5))
            nn.init.zeros_(self.conv1d.bias)
            nn.init.kaiming_uniform_(self.out_proj.weight, a=math.sqrt(5))

    def forward(self, x, bounds):
        link = MambaGradLink()
        xz = self.in_proj(x)
        u = causal_conv1d(xz, self.conv1d.weight, self.conv1d.bias, bounds, link)
        xbc = self.x_proj(u)
        delta_raw = linear(xbc[..., :self.rank], self.dt_proj.weight)
        y = selective_scan(u, delta_raw, xbc, xz, self.A_log, self.D, self.dt_proj.bias, bounds, link)
        return self.out_proj(y)


class MambaBlock(nn.Module):
    def __init__(self, c: MambaConfig):
        super().__init__()
        self.norm = RMSNorm(c.hidden, eps=c.eps)
        self.mixer = MambaMixer(c)

    def forward(self, residual, bounds):
        return residual + self.mixer(self.norm(residual.to(self.norm.weight.dtype)), bounds)


class MambaModel(nn.Module):
    def __init__(self, config: MambaConfig | None = None):
        super().__init__()
        c = self.config = config or MambaConfig()
        self.embeddings = nn.Embedding(c.vocab_size, c.hidden)
        nn.init.normal_(self.embeddings.weight, std=c.initializer_range)
        self.layers = nn.ModuleList([MambaBlock(c) for _ in range(c.layers)])
        self.norm_f = RMSNorm(c.hidden, eps=c.eps)

    def forward(self, input_ids):
        c = self.config
        if input_ids.shape[1] > c.max_position:
            raise ValueError(f"MambaModel: sequence length {input_ids.shape[1]} exceeds max_position {c.max_position}")
        bounds, _ = document_bounds(input_ids, c.bos_token_id, c.pad_token_id)
        bounds = bounds.to(torch.int32)
        x = self.embeddings(input_ids).float()        # residual_in_fp32
        for layer in self.layers:
            x = layer(x, bounds)
        return self.norm_f(x.to(self.norm_f.weight.dtype))


class MambaForCausalLM(nn.Module):
    """Backbone + LM head tied to the embedding (no bias); forward returns logits [B, S, vocab], or with
    ``MambaConfig.fused_lm_loss`` the final hidden states [B, S, hidden], to be scored by ``lm_head_loss()``."""

    def __init__(self, config: MambaConfig | None = None):
        super().__init__()
        self.backbone = MambaModel(config)

    @property
    def config(self) -> MambaConfig:
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
        """Load a ``transformers.MambaForCausalLM`` state dict: the names are the same, and the tied ``lm_head.weight`` must
        equal the embedding."""
        hf = dict(hf)
        head = hf.pop("lm_head.weight", None)
        if head is not None and not torch.equal(head, hf["backbone.embeddings.weight"]):
            raise ValueError("load_hf_state_dict: lm_head.weight differs from backbone.embeddings.weight; this model ties them")
        own = self.state_dict()
        self.load_state_dict({k: v.to(own[k].dtype) if k in own else v for k, v in hf.items()}, strict=True)


MAMBA_130M = MambaConfig()
MAMBA_370M = MambaConfig(hidden=1024, layers=48)


def _build(preset: MambaConfig, pad_token_id, bos_token_id, fused_lm_loss) -> MambaForCausalLM:
    return MambaForCausalLM(replace(preset, pad_token_id=pad_token_id, bos_token_id=bos_token_id, fused_lm_loss=fused_lm_loss))


def mamba_130m(pad_token_id: int | None = None, bos_token_id: int | None = None, fused_lm_loss: bool = False) -> nn.Module:
    """mamba-130m with its tied LM head.  ``pad_token_id`` takes right-padded input; ``bos_token_id`` takes packed
    documents, each starting with that id (the state resets there).  ``fused_lm_loss=True``: forward returns hidden states
    and ``lm_head_loss()`` computes the loss without the logits."""
    return _build(MAMBA_130M, pad_token_id, bos_token_id, fused_lm_loss)


def mamba_370m(pad_token_id: int | None = None, bos_token_id: int | None = None, fused_lm_loss: bool = False) -> nn.Module:
    """mamba-370m (hidden 1024, 48 layers); arguments as for ``mamba_130m``."""
    return _build(MAMBA_370M, pad_token_id, bos_token_id, fused_lm_loss)
