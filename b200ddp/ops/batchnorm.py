"""Fused training BatchNorm2d (+ residual add) (+ ReLU) for channels_last activations (``csrc/batchnorm.cu``).

Drop-in for ``nn.BatchNorm2d`` (same parameter / buffer names, so checkpoints and bucket layouts are unchanged) with two
extra knobs: ``relu=True`` fuses the activation, and ``forward(x, residual=...)`` fuses the Bottleneck shortcut add.  On
CPU, in eval mode, or for layouts the kernel does not cover, it computes the same thing with stock torch ops.

The reference's own model has no normalisation (``model.py:8-16``); this op exists for the ResNet-50 / ResNet-152 configs
the benchmark runs, where the stock ATen BatchNorm + add + ReLU kernels are a large share of the step."""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import _ext


class _FusedBN(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, residual, weight, bias, module, relu, partials=None):
        C = _ext.get()
        ws = module._workspace(x)
        momentum = module.momentum if module.momentum is not None else 0.1
        if partials is not None:
            # statistics already reduced per 32-row group by the producing GEMM: finish + apply, x is read once
            y, stats, mask = C.bn_forward_partials(x, residual, weight, bias, module.running_mean, module.running_var,
                                                   module.num_batches_tracked, module.eps, momentum, relu, partials)
        else:
            y, stats, mask = C.bn_forward(x, residual, weight, bias, module.running_mean, module.running_var,
                                          module.num_batches_tracked, module.eps, momentum, relu, ws[0], ws[1])
        ctx.save_for_backward(x, mask if relu else None, weight, stats)    # 1 bit / element instead of keeping y for the mask
        ctx.relu = relu
        ctx.has_residual = residual is not None
        ctx.module = module
        return y

    @staticmethod
    def backward(ctx, dy):
        C = _ext.get()
        x, y, weight, stats = ctx.saved_tensors
        ws = ctx.module._workspace(x)
        need_dres = ctx.has_residual and ctx.relu
        dx, dres, dparams = C.bn_backward(dy, x, y, weight, stats, ctx.relu, need_dres, ws[2], ws[3])
        if ctx.has_residual and not ctx.relu:
            dres = dy                                  # plain add: the shortcut receives dy unchanged
        return dx, (dres if ctx.has_residual else None), dparams[0], dparams[1], None, None, None


class FusedBatchNormAct2d(nn.BatchNorm2d):
    def __init__(self, num_features: int, eps: float = 1e-5, momentum: float = 0.1, relu: bool = False, **kwargs):
        super().__init__(num_features, eps=eps, momentum=momentum, **kwargs)
        self.relu = relu
        self._ws = {}

    def _workspace(self, x: torch.Tensor):
        """Persistent per-shape scratch (partials + self-resetting block counters): allocated once, outside any graph."""
        key = (tuple(x.shape), x.device)
        ws = self._ws.get(key)
        if ws is None:
            C = _ext.get()
            R = x.numel() // x.shape[1]
            pf, cn = C.bn_workspace(R, x.shape[1])
            mk = lambda n, dt: torch.zeros(max(int(n), 1), dtype=dt, device=x.device)   # noqa: E731
            ws = (mk(pf, torch.float32), mk(cn, torch.int32), mk(pf, torch.float32), mk(cn, torch.int32))
            self._ws[key] = ws
        return ws

    def _fusable(self, x: torch.Tensor) -> bool:
        return (x.is_cuda and self.training and self.track_running_stats and x.dim() == 4 and x.shape[1] % 8 == 0
                and x.dtype in (torch.bfloat16, torch.float32) and self.weight is not None and self.weight.dtype == torch.float32
                and x.is_contiguous(memory_format=torch.channels_last))

    def forward(self, x: torch.Tensor, residual: Optional[torch.Tensor] = None,
                partials: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``partials``: optional [2, groups, C] partial statistics of ``x`` from the kernel that produced it
        (``functional.conv2d_tc``); ignored on the stock fallback path, which recomputes them."""
        if self._fusable(x) and (residual is None or (residual.dtype == x.dtype and residual.shape == x.shape)):
            if residual is not None and not residual.is_contiguous(memory_format=torch.channels_last):
                residual = residual.contiguous(memory_format=torch.channels_last)
            return _FusedBN.apply(x, residual, self.weight, self.bias, self, self.relu, partials)
        y = super().forward(x)
        if residual is not None:
            y = y + residual
        return F.relu(y) if self.relu else y

    def extra_repr(self) -> str:
        return super().extra_repr() + f", relu={self.relu}"


class _MaxPool3x3s2(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        y, idx = _ext.get().maxpool3x3s2_fwd(x)
        ctx.save_for_backward(idx)
        ctx.hw = (x.shape[2], x.shape[3])
        return y

    @staticmethod
    def backward(ctx, dy):
        (idx,) = ctx.saved_tensors
        return _ext.get().maxpool3x3s2_bwd(dy, idx, ctx.hw[0], ctx.hw[1])


class MaxPool3x3s2(nn.Module):
    """``nn.MaxPool2d(3, stride=2, padding=1)`` (the ResNet stem pool) with native channels_last kernels on CUDA."""

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if (x.is_cuda and x.dim() == 4 and x.shape[1] % 8 == 0 and x.dtype in (torch.bfloat16, torch.float32)
                and x.is_contiguous(memory_format=torch.channels_last)):
            return _MaxPool3x3s2.apply(x)
        return F.max_pool2d(x, 3, stride=2, padding=1)
