"""Autograd bindings for the hand-written sm_90a kernels.

Every op has two bodies: CUDA tensors go to the native extension (and raise if it is missing - no
silent fallback on a GPU box); CPU tensors use plain PyTorch math so the CPU test-suite and the gloo
plumbing config run without a GPU.  This is a device split inside one framework, not a multi-backend
kernel dispatch.

Reference call sites being replaced: ``nn.Linear``/``nn.ReLU`` in ``model.py:11-16`` (cuBLASLt +
clamp kernels), ``nn.MSELoss`` in ``ddp.py:164,222``; LayerNorm / cross-entropy / GELU are needed by the
BERT config.
"""
from __future__ import annotations

import math
import os
from typing import Optional

import torch
import torch.nn.functional as F

from .. import _ext

EPI_NONE, EPI_BIAS, EPI_BIAS_RELU, EPI_BIAS_GELU = 0, 1, 2, 3
_ACT_TO_EPI = {None: EPI_BIAS, "relu": EPI_BIAS_RELU, "gelu": EPI_BIAS_GELU}


def _C():
    return _ext.get()


# ------------------------------------------------------------------------------------------------
# Linear
# ------------------------------------------------------------------------------------------------
def _tc_ok(M: int, N: int, K: int) -> bool:
    """wgmma path needs 16-byte row pitches for TMA for all three GEMMs (fwd, dgrad, wgrad)."""
    return K % 8 == 0 and N % 8 == 0 and M % 8 == 0


class _LinearTC(torch.autograd.Function):
    """bf16 linear on wgmma: fwd y = act(x W^T + b); bwd dgrad/wgrad without transposes (MN-major
    operand descriptors), ReLU/GELU backward applied to dy before the two GEMMs."""

    @staticmethod
    def forward(ctx, x, weight, bias, activation):
        C = _C()
        x2 = x.reshape(-1, x.shape[-1])
        if not x2.is_contiguous():
            x2 = x2.contiguous()
        epi = _ACT_TO_EPI[activation] if bias is not None else EPI_NONE
        if bias is None and activation is not None:
            raise ValueError("fused activation needs a bias (use bias=True)")
        if activation == "gelu":
            # keep the pre-activation for the backward (GELU' needs it): two launches, one extra tensor
            pre = C.gemm_nt(x2, weight, bias, EPI_BIAS, None)
            y = C.gelu_fwd(pre)
            ctx.save_for_backward(x2, weight, pre)
        else:
            y = C.gemm_nt(x2, weight, bias, epi, None)
            ctx.save_for_backward(x2, weight, y if activation == "relu" else None)
        ctx.activation = activation
        ctx.has_bias = bias is not None
        ctx.x_shape = x.shape
        return y.view(*x.shape[:-1], weight.shape[0])

    @staticmethod
    def backward(ctx, dy):
        C = _C()
        x2, weight, aux = ctx.saved_tensors
        dy2 = dy.reshape(-1, dy.shape[-1])
        if ctx.activation == "relu":
            dy2 = dy2 * (aux > 0).to(dy2.dtype)
        elif ctx.activation == "gelu":
            dy2 = C.gelu_bwd(dy2.contiguous(), aux)          # dy * gelu'(pre) in one pass
        if not dy2.is_contiguous():
            dy2 = dy2.contiguous()
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            # dx[M,K] = dy[M,N] @ W[N,K]   : A = dy (K-major over N), B = W stored [N,K] = "[K_red, N_out]" MN-major
            dx = C.gemm(dy2, weight, None, False, True, EPI_NONE, False, None).view(ctx.x_shape)
        if ctx.needs_input_grad[1]:
            # dW[N,K] = dy^T[N,M] @ x[M,K] : A = dy stored [M,N] (MN-major), B = x stored [M,K] (MN-major)
            dw = C.gemm(dy2, x2, None, True, True, EPI_NONE, False, None)
        if ctx.has_bias and ctx.needs_input_grad[2]:
            db = dy2.sum(0)
        return dx, dw, db, None


class _LinearSmall(torch.autograd.Function):
    """fp32 linear for shapes below one tensor-core tile (FooModel): CUDA-core kernels, fused
    bias+ReLU forward, single-launch dx/dw/db backward."""

    @staticmethod
    def forward(ctx, x, weight, bias, relu):
        C = _C()
        xc = x.contiguous()
        y = C.small_linear_fwd(xc, weight.contiguous(), bias, bool(relu))
        ctx.save_for_backward(xc, weight, y)
        ctx.relu = bool(relu)
        ctx.has_bias = bias is not None
        return y

    @staticmethod
    def backward(ctx, dy):
        C = _C()
        x, weight, y = ctx.saved_tensors
        dx, dw, db = C.small_linear_bwd(dy, x, weight.contiguous(), y, ctx.relu, ctx.needs_input_grad[0], ctx.has_bias)
        return (dx if ctx.needs_input_grad[0] else None), dw, (db if ctx.has_bias else None), None


def linear(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor] = None,
           activation: Optional[str] = None) -> torch.Tensor:
    """y = act(x @ weight.T + bias), activation in {None, "relu", "gelu"}."""
    if x.is_cuda:
        N, K = weight.shape
        M = x.numel() // K
        if x.dtype == torch.bfloat16 and weight.dtype == torch.bfloat16 and _tc_ok(M, N, K) \
                and (bias is not None or activation is None) and os.environ.get("B200DDP_DISABLE_TC", "0") != "1":
            return _LinearTC.apply(x, weight, bias, activation)
        if x.dtype == torch.float32 and weight.dtype == torch.float32 and N * (K + 1) * 4 <= 48 * 1024 and M * N * 4 <= 48 * 1024 \
                and activation in (None, "relu"):
            return _LinearSmall.apply(x, weight, bias, activation == "relu")
        _C()  # loud failure if the extension is missing; otherwise this shape has no native kernel yet
        y = F.linear(x, weight, bias)
    else:
        y = F.linear(x, weight, bias)
    if activation == "relu":
        y = F.relu(y)
    elif activation == "gelu":
        y = F.gelu(y)
    return y


# ------------------------------------------------------------------------------------------------
# Convolutions on wgmma (csrc/conv_wgmma.cu, csrc/conv_wgrad_wgmma.cu)
# ------------------------------------------------------------------------------------------------
def _conv_policy() -> str:
    """B200DDP_CONV: ``auto`` (default) = the hand-written wgmma kernels for the layer shapes where they beat the library
    per layer, the library elsewhere; ``native`` = the wgmma kernels wherever they apply
    (every stride-1 1x1 / 3x3 convolution: forward, data gradient, BatchNorm-statistics epilogue); ``lib`` = library only."""
    return os.environ.get("B200DDP_CONV", "auto")


def _fprop_native(cin: int, cout: int, k: int, pixels: int) -> bool:
    mode = _conv_policy()
    if mode == "native":
        return True
    if mode == "lib":
        return False
    # No layer shape is selected inside the training step: `auto` == library.
    return False


def _dgrad_native(cin: int, cout: int, k: int, pixels: int) -> bool:
    """Data gradient: the wgmma kernel under ``native``; under ``auto`` no layer shape beats the library yet."""
    return _conv_policy() == "native"


def _wgrad_native(cin: int, cout: int, k: int, pixels: int) -> bool:
    """Which weight-gradient kernel runs (B200DDP_CONV_WGRAD=native|lib|auto overrides; default follows B200DDP_CONV)."""
    mode = os.environ.get("B200DDP_CONV_WGRAD", "auto")
    if mode == "native":
        return True
    if mode == "lib" or _conv_policy() == "lib":
        return False
    if _conv_policy() == "native":
        return k == 1 and pixels >= 25088 and not (cin == 64 and cout == 64)
    return False


def conv_tc_supported(x: torch.Tensor, weight: torch.Tensor, stride: int, padding: int) -> bool:
    """stride-1 'same' 1x1 / 3x3 convolutions of channels_last bf16 CUDA tensors with channel counts that are multiples of 64."""
    k = weight.shape[2]
    return (x.is_cuda and x.dtype == torch.bfloat16 and weight.dtype == torch.bfloat16 and x.dim() == 4 and stride == 1
            and weight.shape[2] == weight.shape[3] and k in (1, 3) and padding == (k - 1) // 2
            and x.shape[1] % 64 == 0 and weight.shape[0] % 64 == 0 and x.shape[3] + 2 <= 256 and _conv_policy() != "lib")


def conv_tc_wanted(x: torch.Tensor, weight: torch.Tensor, stride: int, padding: int) -> bool:
    """Supported AND selected by the policy for this layer shape."""
    if not conv_tc_supported(x, weight, stride, padding):
        return False
    n, cin, h, w = x.shape
    return _fprop_native(cin, weight.shape[0], weight.shape[2], n * h * w)


def _cl(t: torch.Tensor) -> torch.Tensor:
    return t if t.is_contiguous(memory_format=torch.channels_last) else t.contiguous(memory_format=torch.channels_last)


class _ConvTC(torch.autograd.Function):
    """y = conv(x, w) (stride 1, 'same' padding) as a wgmma implicit GEMM; optionally also returns the per-CTA partial
    column sums / sums of squares of y from the epilogue, so the BatchNorm that follows never re-reads y for its statistics.
    Backward: data gradient on the same kernel (mirrored taps, filter read MN-major - no transposed weights), weight
    gradient on the split-pixel wgmma kernel or the library (``_wgrad_native``)."""

    @staticmethod
    def forward(ctx, x, w, want_stats):
        C = _C()
        xc, wc = _cl(x), _cl(w)
        k = w.shape[2]
        y, st = C.conv_fprop(xc, wc, 1, (k - 1) // 2, -1, 0, 0, bool(want_stats))
        ctx.save_for_backward(xc, wc)
        ctx.k = k
        ctx.w_strides = w.stride()
        if want_stats:
            ctx.mark_non_differentiable(st)
            return y, st
        return y, None

    @staticmethod
    def backward(ctx, dy, _dstats):
        C = _C()
        x, w = ctx.saved_tensors
        k = ctx.k
        pad = (k - 1) // 2
        dyc = _cl(dy)
        dx = dw = None
        n, cin, h, wd = x.shape
        if ctx.needs_input_grad[0]:
            if _dgrad_native(cin, w.shape[0], k, n * h * wd):
                dx = C.conv_dgrad(dyc, w, 1, pad, -1, 0, 0)[0]
            else:
                dx = torch.ops.aten.convolution_backward(dyc, x, w, None, [1, 1], [pad, pad], [1, 1], False, [0, 0], 1,
                                                         [True, False, False])[0]
        if ctx.needs_input_grad[1]:
            if _wgrad_native(cin, w.shape[0], k, n * h * wd):
                dw = C.conv_wgrad(dyc, x, k, 1, pad, 0, 0, 0)
            else:
                dw = torch.ops.aten.convolution_backward(dyc, x, w, None, [1, 1], [pad, pad], [1, 1], False, [0, 0], 1,
                                                         [False, True, False])[1]
            if k == 1 and tuple(dw.stride()) != tuple(ctx.w_strides):
                dw = dw.as_strided(dw.shape, ctx.w_strides)      # same memory order; match the parameter's strides so autograd steals it
        return dx, dw, None


def conv2d_tc(x: torch.Tensor, weight: torch.Tensor, want_stats: bool = False):
    """(y, partial BatchNorm statistics or None).  Caller checks ``conv_tc_supported`` first."""
    return _ConvTC.apply(x, weight, want_stats)


# ------------------------------------------------------------------------------------------------
# The strided 7x7 stem (reference hot path: the model's first convolution, the reference ddp.py:221,231)
# ------------------------------------------------------------------------------------------------
def _stem_policy() -> str:
    """B200DDP_STEM: ``native`` (default) = the wgmma stem kernels where they apply, ``lib`` = library."""
    return os.environ.get("B200DDP_STEM", "native")


def stem_conv_supported(x: torch.Tensor, weight: torch.Tensor, stride, padding) -> bool:
    """[N,3,H,W] channels_last bf16 CUDA input that needs no gradient, [64,3,7,7] channels_last bf16 filter, stride 2,
    padding 3, even H / W with W / 2 a multiple of 16 and <= 128 (one output row per accumulator tile)."""
    if _stem_policy() == "lib" or not (x.is_cuda and x.dim() == 4 and x.dtype == torch.bfloat16 and weight.dtype == torch.bfloat16):
        return False
    if tuple(weight.shape) != (64, 3, 7, 7) or tuple(stride) != (2, 2) or tuple(padding) != (3, 3) or x.shape[1] != 3:
        return False
    if x.requires_grad and torch.is_grad_enabled():
        return False                                     # no data-gradient kernel: the first layer's input is data
    if not (x.is_contiguous(memory_format=torch.channels_last) and weight.is_contiguous(memory_format=torch.channels_last)):
        return False
    return bool(_C().stem_conv_supported(int(x.shape[2]), int(x.shape[3])))


class _StemConv(torch.autograd.Function):
    """y = conv7x7/s2(x, w) on the wgmma tap-GEMM: the input is repacked into a zero-bordered image of row pairs whose
    overlapping 128-byte windows ARE the im2col rows (one TMA tensor map, nothing materialised; csrc/conv.h); optional
    BatchNorm-statistics epilogue.  Backward: weight gradient over the same windows on the dedicated split-pixel wgmma
    kernel (``B200DDP_STEM_WGRAD=generic`` selects the general kernel); the input gets no gradient."""

    @staticmethod
    def forward(ctx, x, w, want_stats):
        resident = os.environ.get("B200DDP_STEM_RESIDENT", "1") != "0"
        y, st, xp = _C().stem_conv_fprop(x, w, bool(want_stats), resident)
        ctx.save_for_backward(xp)
        ctx.hw = (int(x.shape[2]), int(x.shape[3]))
        ctx.w_strides = w.stride()
        if want_stats:
            ctx.mark_non_differentiable(st)
            return y, st
        return y, None

    @staticmethod
    def backward(ctx, dy, _dstats):
        (xp,) = ctx.saved_tensors
        dw = None
        if ctx.needs_input_grad[1]:
            variant = 1 if os.environ.get("B200DDP_STEM_WGRAD", "dedicated") == "generic" else 0
            dw = _C().stem_conv_wgrad(_cl(dy), xp, ctx.hw[0], ctx.hw[1], variant)
            if tuple(dw.stride()) != tuple(ctx.w_strides):
                dw = dw.as_strided(dw.shape, ctx.w_strides)
        return None, dw, None


def stem_conv(x: torch.Tensor, weight: torch.Tensor, want_stats: bool = False):
    """(y, partial BatchNorm statistics or None).  Caller checks ``stem_conv_supported`` first."""
    return _StemConv.apply(x, weight, want_stats)


# ------------------------------------------------------------------------------------------------
# Losses: forward computes loss AND input gradient in one launch
# ------------------------------------------------------------------------------------------------
class _MSEFused(torch.autograd.Function):
    @staticmethod
    def forward(ctx, out, target):
        loss, dout = _C().mse_fwd_bwd(out.contiguous(), target.contiguous(), 1.0)
        ctx.save_for_backward(dout)
        return loss.to(out.dtype) if out.dtype != torch.float32 else loss

    @staticmethod
    def backward(ctx, g):
        (dout,) = ctx.saved_tensors
        return dout * g.to(dout.dtype), None


def mse_loss(out: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
    """mean((out-target)^2) - reference criterion ``nn.MSELoss`` (``ddp.py:164``)."""
    if out.is_cuda and out.dtype in (torch.float32, torch.bfloat16) and out.dtype == target.dtype and out.shape == target.shape:
        return _MSEFused.apply(out, target)
    return F.mse_loss(out.float(), target.float())


class _XentFused(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, targets, ignore_index):
        loss, dlogits = _C().xent_fwd_bwd(logits.contiguous(), targets.contiguous(), int(ignore_index), 1.0)
        ctx.save_for_backward(dlogits)
        return loss

    @staticmethod
    def backward(ctx, g):
        (dlogits,) = ctx.saved_tensors
        return dlogits * g.to(dlogits.dtype), None, None


def cross_entropy(logits: torch.Tensor, targets: torch.Tensor, ignore_index: int = -100) -> torch.Tensor:
    """Softmax cross-entropy, mean over non-ignored rows; logits [..., C], targets [...]."""
    if logits.is_cuda and logits.dtype in (torch.float32, torch.bfloat16):
        flat = logits.reshape(-1, logits.shape[-1])
        return _XentFused.apply(flat, targets.reshape(-1), ignore_index)
    return F.cross_entropy(logits.reshape(-1, logits.shape[-1]).float(), targets.reshape(-1), ignore_index=ignore_index)


# ------------------------------------------------------------------------------------------------
# LayerNorm
# ------------------------------------------------------------------------------------------------
class _LayerNormFused(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, gamma, beta, eps):
        xc = x.contiguous()
        y, mean, rstd = _C().layernorm_fwd(xc, gamma.contiguous(), beta.contiguous(), float(eps))
        ctx.save_for_backward(xc, gamma, mean, rstd)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, gamma, mean, rstd = ctx.saved_tensors
        dx, dgamma, dbeta = _C().layernorm_bwd(dy.contiguous(), x, gamma.contiguous(), mean, rstd)
        return dx, dgamma, dbeta, None


def layer_norm(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float = 1e-5) -> torch.Tensor:
    if x.is_cuda and x.dtype in (torch.float32, torch.bfloat16) and gamma.dtype == x.dtype and x.shape[-1] * 8 <= 96 * 1024:
        return _LayerNormFused.apply(x, gamma, beta, eps)
    return F.layer_norm(x, (x.shape[-1],), gamma, beta, eps)
