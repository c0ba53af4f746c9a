"""``nn.Module`` wrappers over ``ops.functional`` (drop-in for nn.Linear / nn.LayerNorm / loss modules).
Reference call sites: ``nn.Linear`` x2 + ``nn.ReLU`` in ``model.py:11-16``, ``nn.MSELoss`` in ``ddp.py:164``."""
from __future__ import annotations

import math
import os
from typing import Optional

import torch
import torch.nn as nn

from . import functional as Fn


class Linear(nn.Module):
    """``nn.Linear`` replacement with an optional fused activation epilogue.  ``fp8=True`` runs forward, data gradient and
    weight gradient on FP8 tensor cores (E4M3 activations / weights, E5M2 gradients, per-tensor power-of-two scales); the
    parameters, their names and shapes are the same either way."""

    def __init__(self, in_features: int, out_features: int, bias: bool = True, activation: Optional[str] = None,
                 device=None, dtype=None, fp8: bool = False):
        super().__init__()
        if fp8 and (in_features % 16 or out_features % 16):
            raise ValueError(f"fp8 Linear needs in_features and out_features divisible by 16, got {in_features} -> {out_features}")
        self.in_features, self.out_features, self.activation = in_features, out_features, activation
        self.fp8 = bool(fp8)
        self.weight = nn.Parameter(torch.empty(out_features, in_features, device=device, dtype=dtype))
        self.bias = nn.Parameter(torch.empty(out_features, device=device, dtype=dtype)) if bias else None
        self.reset_parameters()

    def reset_parameters(self) -> None:
        # same init law as nn.Linear so seeds give the same starting point as the reference model
        nn.init.kaiming_uniform_(self.weight, a=math.sqrt(5))
        if self.bias is not None:
            bound = 1 / math.sqrt(self.in_features) if self.in_features > 0 else 0
            nn.init.uniform_(self.bias, -bound, bound)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return Fn.linear(x, self.weight, self.bias, self.activation, fp8=self.fp8)

    def extra_repr(self) -> str:
        return (f"in={self.in_features}, out={self.out_features}, bias={self.bias is not None}, act={self.activation}"
                + (", fp8=True" if self.fp8 else ""))


class Conv2dTC(nn.Conv2d):
    """Bias-free ``nn.Conv2d`` (same parameter name, shape and init, so checkpoints and DDP bucket layouts are unchanged)
    whose stride-1 1x1 / 3x3 instances run forward, data gradient and (where it wins) weight gradient on the hand-written
    wgmma kernels for channels_last bf16 CUDA tensors; everything else (CPU, fp32, stride 2, odd channel counts) takes
    the stock path.  ``forward_with_stats`` additionally hands the following BatchNorm its statistics from the epilogue."""

    def __init__(self, in_channels: int, out_channels: int, kernel_size: int = 1, stride: int = 1, **kw):
        super().__init__(in_channels, out_channels, kernel_size, stride=stride, padding=(kernel_size - 1) // 2, bias=False, **kw)

    def _native(self, x: torch.Tensor) -> bool:
        return self.stride[0] == self.stride[1] and Fn.conv_tc_wanted(x, self.weight, self.stride[0], self.padding[0])

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if self._native(x):
            return Fn.conv2d_tc(x, self.weight, False)[0]
        return super().forward(x)

    def forward_with_stats(self, x: torch.Tensor):
        """(y, partial BatchNorm statistics [2, G, C_out] from the convolution's epilogue, or None on the stock path)."""
        if self._native(x):
            return Fn.conv2d_tc(x, self.weight, True)
        return super().forward(x), None


class PointwiseConv2d(Conv2dTC):
    def __init__(self, in_channels: int, out_channels: int, stride: int = 1, **kw):
        super().__init__(in_channels, out_channels, 1, stride=stride, **kw)


class Conv3x3(Conv2dTC):
    def __init__(self, in_channels: int, out_channels: int, stride: int = 1, **kw):
        super().__init__(in_channels, out_channels, 3, stride=stride, **kw)


class StemConv7x7(nn.Conv2d):
    """The ResNet stem: bias-free ``nn.Conv2d(3, 64, 7, stride=2, padding=3)`` (same parameter name / shape / init) that runs
    forward and weight gradient on the wgmma kernels for channels_last bf16 CUDA input, and hands the following BatchNorm
    its statistics from the epilogue; anything else takes the stock path."""

    def __init__(self, in_channels: int = 3, out_channels: int = 64, **kw):
        super().__init__(in_channels, out_channels, 7, stride=2, padding=3, bias=False, **kw)

    def _native(self, x: torch.Tensor) -> bool:
        return Fn.stem_conv_supported(x, self.weight, self.stride, self.padding)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if self._native(x):
            return Fn.stem_conv(x, self.weight, False)[0]
        return super().forward(x)

    def forward_with_stats(self, x: torch.Tensor):
        if self._native(x):
            return Fn.stem_conv(x, self.weight, True)
        return super().forward(x), None


class LayerNorm(nn.Module):
    def __init__(self, hidden: int, eps: float = 1e-5, device=None, dtype=None):
        super().__init__()
        self.eps = eps
        self.weight = nn.Parameter(torch.ones(hidden, device=device, dtype=dtype))
        self.bias = nn.Parameter(torch.zeros(hidden, device=device, dtype=dtype))

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return Fn.layer_norm(x, self.weight, self.bias, self.eps)


class RMSNorm(nn.Module):
    """Llama's RMSNorm: y = x * rsqrt(mean(x^2) + eps) * weight (no mean, no bias)."""

    def __init__(self, hidden: int, eps: float = 1e-5, device=None, dtype=None):
        super().__init__()
        self.eps = eps
        self.weight = nn.Parameter(torch.ones(hidden, device=device, dtype=dtype))

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return Fn.rms_norm(x, self.weight, self.eps)


class MSELoss(nn.Module):
    def forward(self, out: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
        return Fn.mse_loss(out, target)


class CrossEntropyLoss(nn.Module):
    def __init__(self, ignore_index: int = -100):
        super().__init__()
        self.ignore_index = ignore_index

    def forward(self, logits: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
        return Fn.cross_entropy(logits, target, self.ignore_index)
