"""Mixed-precision placement: bf16 weights/activations with BatchNorm kept in fp32 (cuDNN's fast NHWC
batch-norm kernels want bf16 activations with fp32 scale/bias/statistics).  This is the working version of
what the reference's ``--fp16`` asks apex for (O2: half model + fp32 master weights, ``ddp.py:174-180``); the
fp32 masters live in the fused optimizers (``b200ddp.optim.FusedSGD``, ``b200ddp.optim.FusedAdamW``)."""
from __future__ import annotations

import torch
import torch.nn as nn

_KEEP_FP32 = (nn.modules.batchnorm._BatchNorm,)


def to_mixed_bf16(model: nn.Module, keep_norm_fp32: bool = True) -> nn.Module:
    """bf16 weights, with BatchNorm (``keep_norm_fp32``) and the parameters a module names in ``keep_fp32_params`` (CLIP's
    ``logit_scale``, whose exponential bf16 would round) left in fp32."""
    model.to(torch.bfloat16)
    if keep_norm_fp32:
        for m in model.modules():
            if isinstance(m, _KEEP_FP32):
                m.float()
    for m in model.modules():
        for name in getattr(m, "keep_fp32_params", ()):
            p = m.get_parameter(name)                 # a dotted name reaches into a child (Mamba's "dt_proj.bias")
            p.data = p.data.float()
    return model


def is_dense(t: torch.Tensor) -> bool:
    """True when the tensor's elements occupy one gap-free block of storage (any permutation of strides)."""
    if t.is_contiguous():
        return True
    if t.numel() == 0:
        return True
    # sort dims by stride; a dense layout has stride[i] == product of the sizes of all faster dims
    dims = sorted(((st, sz) for st, sz in zip(t.stride(), t.shape) if sz != 1), key=lambda p: p[0])
    expect = 1
    for st, sz in dims:
        if st != expect:
            return False
        expect *= sz
    return True
