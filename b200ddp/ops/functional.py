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
# GELU variants: the erf form ("gelu", BERT) and the tanh approximation ("gelu_tanh", GPT-2's ``gelu_new``).  Both run as
# a bias epilogue plus one elementwise pass (csrc/loss.cu) that keeps the pre-activation for the backward.
_GELU_TANH = {"gelu": False, "gelu_tanh": True}


def _gelu_tanh_grad(p: torch.Tensor) -> torch.Tensor:
    """d/dp of 0.5 p (1 + tanh(sqrt(2 / pi) (p + 0.044715 p^3))), in p's dtype."""
    k = math.sqrt(2.0 / math.pi)
    t = torch.tanh(k * (p + 0.044715 * p * p * p))
    return 0.5 * (1.0 + t) + 0.5 * p * (1.0 - t * t) * k * (1.0 + 3.0 * 0.044715 * p * p)


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
        if bias is None and activation is not None:
            raise ValueError("fused activation needs a bias (use bias=True)")
        if activation in _GELU_TANH:
            # keep the pre-activation for the backward (GELU' needs it): two launches, one extra tensor
            pre = C.gemm_nt(x2, weight, bias, EPI_BIAS, None)
            y = C.gelu_fwd(pre, _GELU_TANH[activation])
            ctx.save_for_backward(x2, weight, pre)
        else:
            y = C.gemm_nt(x2, weight, bias, _ACT_TO_EPI[activation] if bias is not None else EPI_NONE, None)
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
        elif ctx.activation in _GELU_TANH:
            dy2 = C.gelu_bwd(dy2.contiguous(), aux, _GELU_TANH[ctx.activation])   # dy * gelu'(pre) in one pass
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


# ------------------------------------------------------------------------------------------------
# FP8 linear (csrc/fp8.cu, csrc/gemm_wgmma.cu): E4M3 x / W, E5M2 dy, current per-tensor power-of-two scales
# ------------------------------------------------------------------------------------------------
FP8_FORMATS = {"e4m3": (torch.float8_e4m3fn, 448.0), "e5m2": (torch.float8_e5m2, 57344.0)}


def fp8_scale(amax: float, fmt: str) -> float:
    """s = 2^e with e the largest integer such that amax * 2^e <= fmax, e clamped to [-126, 127]; amax = 0 gives 1.
    The same rule as ``fp8_scale_exponent`` in csrc/fp8.cu, evaluated exactly on the mantissas."""
    fmax = FP8_FORMATS[fmt][1]
    if not (amax > 0.0) or not math.isfinite(amax):
        return 1.0
    ma, ea = math.frexp(amax)
    mf, ef = math.frexp(fmax)
    e = ef - ea - (1 if ma > mf else 0)
    return math.ldexp(1.0, min(max(e, -126), 127))


def fp8_quantize_reference(t: torch.Tensor, fmt: str):
    """(q, s) on the CPU: q = (t.float() * s).to(float8) - bitwise what the CUDA quantiser writes."""
    s = fp8_scale(float(t.detach().abs().max().float()) if t.numel() else 0.0, fmt)
    return (t.detach().float() * s).to(FP8_FORMATS[fmt][0]), s


def _fp8_round_trip(t: torch.Tensor, fmt: str) -> torch.Tensor:
    """fp32 values of t after quantisation and exact dequantisation."""
    q, s = fp8_quantize_reference(t, fmt)
    return q.float() / s


def _fp8_check(x2: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor], need_transpose_x: bool) -> None:
    M, K = x2.shape
    N = weight.shape[0]
    if x2.dtype != torch.bfloat16 or weight.dtype != torch.bfloat16 or (bias is not None and bias.dtype != torch.bfloat16):
        raise ValueError(f"fp8 linear on CUDA needs bf16 input, weight and bias, got {x2.dtype} x {weight.dtype} "
                         f"(input {tuple(x2.shape)}, weight {tuple(weight.shape)})")
    if K % 16 or N % 16:
        raise ValueError(f"fp8 linear needs in_features and out_features divisible by 16, got weight {tuple(weight.shape)}")
    if need_transpose_x and M % 16:
        raise ValueError(f"fp8 linear backward needs the row count divisible by 16 (the weight gradient reduces over rows "
                         f"of a transposed FP8 copy), got input {tuple(x2.shape)}")


class _LinearFP8(torch.autograd.Function):
    """FP8 linear: y = act(x W^T + b) with x, W quantised to E4M3 and dy to E5M2 (per-tensor power-of-two scales).
    FP8 wgmma takes K-major operands only, so every quantisation writes the transposed copy the backward needs:
    forward x8 [M,K] . W8 [N,K], dgrad dy8 [M,N] . W8^T [K,N], wgrad dy8^T [N,M] . x8^T [K,M].  The bias gradient comes
    from the column sums of the dy quantisation pass.  Parameters and gradients stay bf16.
    CPU body: the same recipe emulated exactly (same scales, a torch.float8 round trip, fp32 matmuls)."""

    @staticmethod
    def forward(ctx, x, weight, bias, activation, grad_enabled):
        x2 = x.reshape(-1, x.shape[-1])
        if not x2.is_contiguous():
            x2 = x2.contiguous()
        if bias is None and activation is not None:
            raise ValueError("fused activation needs a bias (use bias=True)")
        # transposed copies only where a backward will read them (no_grad inference needs none)
        need_dx, need_dw = grad_enabled and ctx.needs_input_grad[0], grad_enabled and ctx.needs_input_grad[1]
        ctx.activation = activation
        ctx.has_bias = bias is not None
        ctx.x_shape = x.shape
        if x.is_cuda:
            C = _C()
            _fp8_check(x2, weight, bias, need_dw)
            xq, xqt, xs, _ = C.fp8_quantize(x2, "e4m3", need_dw, False)
            wq, wqt, ws, _ = C.fp8_quantize(weight.contiguous(), "e4m3", need_dx, False)
            if activation in _GELU_TANH:
                pre = C.gemm_fp8(xq, wq, xs, ws, bias, EPI_BIAS)
                y = C.gelu_fwd(pre, _GELU_TANH[activation])
            else:
                pre = None
                y = C.gemm_fp8(xq, wq, xs, ws, bias, _ACT_TO_EPI[activation] if bias is not None else EPI_NONE)
                if activation == "relu":
                    pre = y
            ctx.save_for_backward(xqt, xs, wqt, ws, pre)
        else:
            xd = _fp8_round_trip(x2, "e4m3")
            wd = _fp8_round_trip(weight, "e4m3")
            acc = xd @ wd.t()
            if bias is not None:
                acc = acc + bias.float()
            pre = acc.to(x.dtype)
            if activation == "gelu":
                y = F.gelu(pre.float()).to(x.dtype)
            elif activation == "gelu_tanh":
                y = F.gelu(pre.float(), approximate="tanh").to(x.dtype)
            elif activation == "relu":
                y = F.relu(pre)
            else:
                y = pre
            ctx.save_for_backward(xd, wd, pre if activation is not None else None)
            ctx.dtypes = (x.dtype, weight.dtype, bias.dtype if bias is not None else None)
        return y.view(*x.shape[:-1], weight.shape[0])

    @staticmethod
    def backward(ctx, dy):
        dy2 = dy.reshape(-1, dy.shape[-1])
        dx = dw = db = None
        if dy.is_cuda:
            C = _C()
            xqt, xs, wqt, ws, aux = ctx.saved_tensors
            if ctx.activation == "relu":
                dy2 = dy2 * (aux > 0).to(dy2.dtype)
            elif ctx.activation in _GELU_TANH:
                dy2 = C.gelu_bwd(dy2.contiguous(), aux, _GELU_TANH[ctx.activation])
            if not dy2.is_contiguous():
                dy2 = dy2.contiguous()
            if dy2.shape[0] % 16:
                raise ValueError(f"fp8 linear backward needs the row count divisible by 16, got gradient {tuple(dy2.shape)}")
            need_db = ctx.has_bias and ctx.needs_input_grad[2]
            dyq, dyqt, dys, colsum = C.fp8_quantize(dy2, "e5m2", ctx.needs_input_grad[1], need_db)
            if ctx.needs_input_grad[0]:
                dx = C.gemm_fp8(dyq, wqt, dys, ws, None, EPI_NONE).view(ctx.x_shape)       # [M,K], reduction over N
            if ctx.needs_input_grad[1]:
                dw = C.gemm_fp8(dyqt, xqt, dys, xs, None, EPI_NONE)                        # [N,K], reduction over M
            if need_db:
                db = colsum.to(dy.dtype)
        else:
            xd, wd, aux = ctx.saved_tensors
            x_dtype, w_dtype, b_dtype = ctx.dtypes
            if ctx.activation == "relu":
                dy2 = dy2 * (aux > 0).to(dy2.dtype)
            elif ctx.activation == "gelu":
                p = aux.float()                                    # gelu'(p) = Phi(p) + p phi(p)
                dgelu = 0.5 * (1.0 + torch.erf(p * math.sqrt(0.5))) + p * torch.exp(-0.5 * p * p) / math.sqrt(2.0 * math.pi)
                dy2 = (dy2.float() * dgelu).to(dy.dtype)
            elif ctx.activation == "gelu_tanh":
                dy2 = (dy2.float() * _gelu_tanh_grad(aux.float())).to(dy.dtype)
            dyd = _fp8_round_trip(dy2, "e5m2")
            if ctx.needs_input_grad[0]:
                dx = (dyd @ wd).to(x_dtype).view(ctx.x_shape)
            if ctx.needs_input_grad[1]:
                dw = (dyd.t() @ xd).to(w_dtype)
            if ctx.has_bias and ctx.needs_input_grad[2]:
                db = dy2.float().sum(0).to(b_dtype)
        return dx, dw, db, None, None


def linear(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor] = None,
           activation: Optional[str] = None, fp8: bool = False) -> torch.Tensor:
    """y = act(x @ weight.T + bias), activation in {None, "relu", "gelu", "gelu_tanh"} ("gelu" is the erf form,
    "gelu_tanh" the tanh approximation).  ``fp8=True`` runs the three GEMMs on FP8 tensor cores (``_LinearFP8``); on CUDA
    it needs bf16 tensors and raises ``ValueError`` for anything else."""
    if fp8:
        return _LinearFP8.apply(x, weight, bias, activation, torch.is_grad_enabled())
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
    elif activation == "gelu_tanh":
        y = F.gelu(y, approximate="tanh")
    return y


# ------------------------------------------------------------------------------------------------
# Key-padding attention (csrc/attention.cu): Q / K / V read straight out of the fused projection
# ------------------------------------------------------------------------------------------------
ATTENTION_HEAD_DIM = 64
ATTENTION_SEQ_MULTIPLE = 128
CAUSAL_WIDE_HEAD_DIM = 128      # the causal kernels also run at this head dim (grouped-query or multi-head)


def _key_mask(seq_lens: torch.Tensor, S: int, device) -> torch.Tensor:
    """[B, S] bool: key j of sequence b is visible iff j < seq_lens[b] (lengths clamped to [0, S], like the kernel)."""
    lens = seq_lens.to(device=device, dtype=torch.long).clamp(0, S)
    return torch.arange(S, device=device)[None, :] < lens[:, None]


def attention_reference(qkv: torch.Tensor, seq_lens: torch.Tensor, heads: int) -> torch.Tensor:
    """softmax(Q K^T / sqrt(d)) V with the key-padding mask, in fp32 (fp64 stays fp64); a sequence of length 0 gives zeros.
    qkv [B, S, 3 * hidden] (query | key | value column blocks), returns [B, S, hidden] in qkv's dtype.  Differentiable."""
    return _masked_attention_reference(qkv, _key_mask(seq_lens, qkv.shape[1], qkv.device)[:, None, None, :], heads)


def _masked_attention_reference(qkv: torch.Tensor, keep: torch.Tensor, heads: int) -> torch.Tensor:
    """Body of the references: ``keep`` is a bool mask broadcastable to [B, heads, S (query), S (key)]."""
    B, S, W = qkv.shape
    hidden = W // 3
    hd = hidden // heads
    ct = torch.promote_types(qkv.dtype, torch.float32)
    q, k, v = (t.to(ct).reshape(B, S, heads, hd).transpose(1, 2) for t in qkv.split(hidden, dim=-1))
    scores = (q @ k.transpose(-1, -2)) * (1.0 / math.sqrt(hd))
    # a finite fill keeps an all-hidden row free of NaN; multiplying by the mask then zeroes it (and its gradients)
    p = torch.softmax(scores.masked_fill(~keep, torch.finfo(ct).min), dim=-1) * keep
    return (p @ v).transpose(1, 2).reshape(B, S, hidden).to(qkv.dtype)


def _attention_check(qkv: torch.Tensor, seq_lens: torch.Tensor, heads: int) -> None:
    _qkv_check(qkv, heads)
    B = qkv.shape[0]
    if seq_lens.dim() != 1 or seq_lens.shape[0] != B or seq_lens.is_floating_point() or seq_lens.is_complex():
        raise ValueError(f"attention needs integer seq_lens [B] = [{B}], got {seq_lens.dtype} {tuple(seq_lens.shape)}")


def _qkv_check(qkv: torch.Tensor, heads: int) -> None:
    if qkv.dim() != 3 or qkv.shape[-1] % 3:
        raise ValueError(f"attention needs qkv [B, S, 3 * hidden], got {tuple(qkv.shape)}")
    B, S, W = qkv.shape
    if heads < 1 or (W // 3) % heads or (W // 3) // heads != ATTENTION_HEAD_DIM:
        raise ValueError(f"attention on CUDA supports head dim {ATTENTION_HEAD_DIM} only, got hidden {W // 3} over {heads} heads")
    if qkv.dtype != torch.bfloat16:
        raise ValueError(f"attention on CUDA needs bf16 qkv, got {qkv.dtype}")
    if S % ATTENTION_SEQ_MULTIPLE or S == 0:
        raise ValueError(f"attention on CUDA needs the sequence length to be a multiple of {ATTENTION_SEQ_MULTIPLE}, got {S}")
    if not qkv.is_contiguous():
        raise ValueError("attention on CUDA needs a contiguous qkv (the fused projection's output)")


# mask modes of _Attention: name -> (native forward, native backward, CPU reference)
_ATTENTION_MODES = {
    "key_padding": ("attention_fwd", "attention_bwd", lambda: attention_reference),
    "packed": ("packed_attention_fwd", "packed_attention_bwd", lambda: packed_attention_reference),
    "causal": ("causal_attention_fwd", "causal_attention_bwd", lambda: causal_attention_reference),
}


class _Attention(torch.autograd.Function):
    """Key-padding (``mode="key_padding"``, mask = seq_lens [B]), packed-document (``"packed"``, mask = bounds [B, S, 2])
    or causal-document (``"causal"``, the same bounds) attention.  CUDA body: the sm_90a kernels (forward keeps the row
    log-sum-exp; backward is three deterministic launches writing one dqkv tensor, the exact gradient the qkv linear
    consumes).  CPU body: the matching reference (backward by recomputation through autograd)."""

    @staticmethod
    def forward(ctx, qkv, mask, heads, mode):
        ctx.heads, ctx.mode = heads, mode
        if qkv.is_cuda:
            B, S, W = qkv.shape
            m = mask.to(device=qkv.device, dtype=torch.int32).contiguous()
            o, lse = getattr(_C(), _ATTENTION_MODES[mode][0])(qkv.view(B * S, W), m, heads)
            ctx.save_for_backward(qkv, o, lse, m)
            return o.view(B, S, W // 3)
        ctx.save_for_backward(qkv, mask)
        return _ATTENTION_MODES[mode][2]()(qkv, mask, heads)

    @staticmethod
    def backward(ctx, dy):
        if dy.is_cuda:
            qkv, o, lse, m = ctx.saved_tensors
            B, S, W = qkv.shape
            do = dy.reshape(B * S, W // 3).to(torch.bfloat16).contiguous()
            if do.data_ptr() % 16:                                # the kernels read dO in 16-byte vectors / TMA boxes
                do = do.clone()
            dqkv = getattr(_C(), _ATTENTION_MODES[ctx.mode][1])(do, qkv.view(B * S, W), o, lse, m, ctx.heads)
            return dqkv.view(B, S, W), None, None, None
        qkv, mask = ctx.saved_tensors
        ref = _ATTENTION_MODES[ctx.mode][2]()
        with torch.enable_grad():
            x = qkv.detach().requires_grad_(True)
            (g,) = torch.autograd.grad(ref(x, mask, ctx.heads), x, dy)
        return g, None, None, None


def attention(qkv: torch.Tensor, seq_lens: torch.Tensor, heads: int) -> torch.Tensor:
    """Multi-head attention over right-padded sequences: qkv [B, S, 3 * hidden] (the fused projection's output, column
    blocks query | key | value), seq_lens [B] integer lengths (key j of sequence b is visible iff j < seq_lens[b]; every
    query row is computed).  Returns [B, S, hidden].  On CUDA: bf16, head dim 64, S % 128 == 0 and contiguous qkv, else
    ``ValueError``; lengths stay on the device (no host synchronisation, CUDA-graph safe)."""
    if qkv.is_cuda:
        _attention_check(qkv, seq_lens, heads)
    return _Attention.apply(qkv, seq_lens, heads, "key_padding")


# ------------------------------------------------------------------------------------------------
# Packed-document attention (csrc/attention.cu, segment mode): several documents per row, block-diagonal mask
# ------------------------------------------------------------------------------------------------
def document_bounds(input_ids: torch.Tensor, cls_token_id: Optional[int], pad_token_id: Optional[int]):
    """Documents of packed rows, on the device with no host synchronisation (CUDA-graph safe).

    input_ids [B, S].  A row's length is its non-pad count (S when ``pad_token_id`` is None); positions at or beyond it
    are padding, whatever their id.  A document starts at position 0 and at every ``cls_token_id`` below the length, and
    runs to the next start or the length; with ``cls_token_id=None`` each row is one document ``(0, length)``.  Returns ``(bounds, position_ids)``: bounds int32 [B, S, 2] holds each
    position's document as (start, end), (0, 0) for padding; position_ids long [B, S] restart at 0 in each document and
    are 0 for padding."""
    B, S = input_ids.shape
    pos = torch.arange(S, device=input_ids.device).expand(B, S)
    if pad_token_id is None:
        lens = torch.full((B, 1), S, device=input_ids.device, dtype=torch.long)
    else:
        lens = (input_ids != pad_token_id).sum(1, keepdim=True)
    valid = pos < lens
    is_start = (pos == 0) if cls_token_id is None else (input_ids == cls_token_id) | (pos == 0)
    is_start = is_start & valid
    start = torch.where(is_start, pos, 0).cummax(1).values                   # the last start at or before each position
    nxt = torch.where(is_start, pos, S)[:, 1:]                                  # the first start after each position
    nxt = torch.cat([nxt, torch.full((B, 1), S, device=pos.device, dtype=pos.dtype)], 1).flip(1).cummin(1).values.flip(1)
    end = torch.minimum(nxt, lens)
    bounds = torch.stack([torch.where(valid, start, 0), torch.where(valid, end, 0)], -1).to(torch.int32)
    return bounds, torch.where(valid, pos - start, 0)


def _bounds_mask(bounds: torch.Tensor, S: int, device) -> torch.Tensor:
    """[B, S, S] bool: query i sees key j iff start[i] <= j < end[i] (start clamped to [0, S], end to [start, S], like
    the kernel)."""
    b = bounds.to(device=device, dtype=torch.long).reshape(-1, S, 2)
    start = b[..., 0].clamp(0, S)
    end = torch.maximum(b[..., 1].clamp(max=S), start)
    j = torch.arange(S, device=device)
    return (j >= start[..., None]) & (j < end[..., None])


def packed_attention_reference(qkv: torch.Tensor, bounds: torch.Tensor, heads: int) -> torch.Tensor:
    """softmax(Q K^T / sqrt(d)) V where query i sees key j of its row iff bounds[b, i, 0] <= j < bounds[b, i, 1], in
    fp32 (fp64 stays fp64); a row that sees no key gives zeros.  qkv [B, S, 3 * hidden], bounds integer [B, S, 2];
    returns [B, S, hidden] in qkv's dtype.  Differentiable."""
    return _masked_attention_reference(qkv, _bounds_mask(bounds, qkv.shape[1], qkv.device)[:, None], heads)


def packed_attention(qkv: torch.Tensor, bounds: torch.Tensor, heads: int) -> torch.Tensor:
    """Multi-head attention over packed documents: qkv [B, S, 3 * hidden] (the fused projection's output), bounds
    integer [B, S, 2] (``document_bounds``): query i of a row sees key j of the same row iff start[i] <= j < end[i].
    Rows with start == end (padding) give zeros and get zero gradients.  Returns [B, S, hidden].  On CUDA: bf16, head
    dim 64, S % 128 == 0 and contiguous qkv, else ``ValueError``; bounds stay on the device (CUDA-graph safe)."""
    if qkv.is_cuda:
        _qkv_check(qkv, heads)
        _bounds_check(qkv, bounds, "packed attention")
    return _Attention.apply(qkv, bounds, heads, "packed")


def _bounds_check(qkv: torch.Tensor, bounds: torch.Tensor, who: str) -> None:
    B, S = qkv.shape[:2]
    if tuple(bounds.shape) != (B, S, 2) or bounds.is_floating_point() or bounds.is_complex():
        raise ValueError(f"{who} needs integer bounds [B, S, 2] = [{B}, {S}, 2], got {bounds.dtype} {tuple(bounds.shape)}")


# ------------------------------------------------------------------------------------------------
# Causal document attention (csrc/attention.cu, causal mode): packed documents, each causal (decoder LMs)
# ------------------------------------------------------------------------------------------------
def _causal_mask(bounds: torch.Tensor, S: int, device) -> torch.Tensor:
    """[B, S, S] bool: query i sees key j iff start[i] <= j <= i and j < end[i] (bounds clamped like the kernel)."""
    i = torch.arange(S, device=device)
    return _bounds_mask(bounds, S, device) & (i[None, :] <= i[:, None])


def causal_attention_reference(qkv: torch.Tensor, bounds: torch.Tensor, heads: int, kv_heads: Optional[int] = None) -> torch.Tensor:
    """softmax(Q K^T / sqrt(d)) V where query i sees key j of its row iff bounds[b, i, 0] <= j <= i and
    j < bounds[b, i, 1], in fp32 (fp64 stays fp64), as a dense mask; a row that sees no key gives zeros.  qkv
    [B, S, 3 * hidden], bounds integer [B, S, 2]; returns [B, S, hidden] in qkv's dtype.  Differentiable.
    ``kv_heads`` (grouped-query attention): qkv is [B, S, (heads + 2 * kv_heads) * d], query head h reads K/V head
    h // (heads // kv_heads); K and V are repeated per group (Hugging Face's ``repeat_kv``)."""
    if kv_heads is not None and kv_heads != heads:
        qkv = _repeat_kv(qkv, heads, kv_heads)
    return _masked_attention_reference(qkv, _causal_mask(bounds, qkv.shape[1], qkv.device)[:, None], heads)


def _repeat_kv(qkv: torch.Tensor, heads: int, kv_heads: int) -> torch.Tensor:
    """[B, S, (heads + 2 * kv_heads) * d] -> [B, S, 3 * heads * d]: each K/V head repeated heads // kv_heads times."""
    B, S, Wd = qkv.shape
    d = Wd // (heads + 2 * kv_heads)
    q, k, v = qkv.split([heads * d, kv_heads * d, kv_heads * d], dim=-1)
    rep = heads // kv_heads
    k, v = (t.reshape(B, S, kv_heads, 1, d).expand(B, S, kv_heads, rep, d).reshape(B, S, heads * d) for t in (k, v))
    return torch.cat([q, k, v], -1)


def _gqa_check(qkv: torch.Tensor, heads: int, kv_heads: int, head_dim: int = ATTENTION_HEAD_DIM) -> None:
    if heads < 1 or kv_heads < 1 or heads % kv_heads:
        raise ValueError(f"grouped-query attention needs kv_heads dividing heads, got heads={heads}, kv_heads={kv_heads}")
    if qkv.dim() != 3 or qkv.shape[-1] != (heads + 2 * kv_heads) * head_dim:
        raise ValueError(f"grouped-query attention on CUDA needs qkv [B, S, (heads + 2 * kv_heads) * {head_dim}] = "
                         f"[B, S, {(heads + 2 * kv_heads) * head_dim}], got {tuple(qkv.shape)}")
    if qkv.dtype != torch.bfloat16:
        raise ValueError(f"attention on CUDA needs bf16 qkv, got {qkv.dtype}")
    S = qkv.shape[1]
    if S % ATTENTION_SEQ_MULTIPLE or S == 0:
        raise ValueError(f"attention on CUDA needs the sequence length to be a multiple of {ATTENTION_SEQ_MULTIPLE}, got {S}")
    if not qkv.is_contiguous():
        raise ValueError("attention on CUDA needs a contiguous qkv (the fused projection's output)")


class _GqaAttention(torch.autograd.Function):
    """Grouped-query causal-document attention.  CUDA body: the sm_90a GQA kernels of the head dim, 64 or 128 (dK / dV
    accumulate across each group in registers: one writer per element, deterministic).  CPU body:
    ``causal_attention_reference`` with K / V repeated."""

    @staticmethod
    def forward(ctx, qkv, bounds, heads, kv_heads):
        ctx.heads, ctx.kv_heads = heads, kv_heads
        if qkv.is_cuda:
            B, S, Wd = qkv.shape
            d = Wd // (heads + 2 * kv_heads)
            m = bounds.to(device=qkv.device, dtype=torch.int32).contiguous()
            fwd = _C().causal_attention_d128_fwd if d == CAUSAL_WIDE_HEAD_DIM else _C().causal_gqa_attention_fwd
            o, lse = fwd(qkv.view(B * S, Wd), m, heads, kv_heads)
            ctx.save_for_backward(qkv, o, lse, m)
            return o.view(B, S, heads * d)
        ctx.save_for_backward(qkv, bounds)
        return causal_attention_reference(qkv, bounds, heads, kv_heads)

    @staticmethod
    def backward(ctx, dy):
        if dy.is_cuda:
            qkv, o, lse, m = ctx.saved_tensors
            B, S, Wd = qkv.shape
            do = dy.reshape(B * S, -1).to(torch.bfloat16).contiguous()
            if do.data_ptr() % 16:
                do = do.clone()
            wide = o.shape[-1] == ctx.heads * CAUSAL_WIDE_HEAD_DIM
            bwd = _C().causal_attention_d128_bwd if wide else _C().causal_gqa_attention_bwd
            dqkv = bwd(do, qkv.view(B * S, Wd), o, lse, m, ctx.heads, ctx.kv_heads)
            return dqkv.view(B, S, Wd), None, None, None
        qkv, bounds = ctx.saved_tensors
        with torch.enable_grad():
            x = qkv.detach().requires_grad_(True)
            (g,) = torch.autograd.grad(causal_attention_reference(x, bounds, ctx.heads, ctx.kv_heads), x, dy)
        return g, None, None, None


def causal_attention(qkv: torch.Tensor, bounds: torch.Tensor, heads: int, kv_heads: Optional[int] = None) -> torch.Tensor:
    """Causal multi-head attention inside documents: qkv [B, S, 3 * hidden] (the fused projection's output), bounds
    integer [B, S, 2] (``document_bounds``; with ``cls_token_id=None`` it gives right-padded rows one document each):
    query i of a row sees key j iff start[i] <= j <= i and j < end[i].  Rows with start == end (padding) give zeros and
    get zero gradients.  Returns [B, S, hidden].  On CUDA: bf16, head dim 64, S % 128 == 0 and contiguous qkv, else
    ``ValueError``; bounds stay on the device (CUDA-graph safe).  Tiles above the diagonal are never visited.

    ``kv_heads`` other than None or ``heads`` selects grouped-query attention: qkv is [B, S, (heads + 2 * kv_heads) * 64]
    (query | key | value column blocks) and query head h reads K/V head h // (heads // kv_heads); the output stays
    [B, S, heads * 64].

    Head dim 128 (qkv [B, S, (heads + 2 * kv_heads) * 128], kv_heads None meaning ``heads``) runs on CUDA on the head-dim-128
    kernels, with the same layouts, masks and checks; the output is [B, S, heads * 128]."""
    kv = heads if kv_heads is None else kv_heads
    if qkv.is_cuda and heads >= 1 and kv >= 1 and qkv.dim() == 3 and qkv.shape[-1] == (heads + 2 * kv) * CAUSAL_WIDE_HEAD_DIM:
        _gqa_check(qkv, heads, kv, CAUSAL_WIDE_HEAD_DIM)
        _bounds_check(qkv, bounds, "causal attention")
        return _GqaAttention.apply(qkv, bounds, heads, kv)
    if kv_heads is not None and kv_heads != heads:
        if qkv.is_cuda:
            _gqa_check(qkv, heads, kv_heads)
            _bounds_check(qkv, bounds, "causal attention")
        elif heads < 1 or kv_heads < 1 or heads % kv_heads or qkv.dim() != 3 or qkv.shape[-1] % (heads + 2 * kv_heads):
            raise ValueError(f"grouped-query attention needs kv_heads dividing heads and qkv [B, S, (heads + 2 * kv_heads) * d], "
                             f"got heads={heads}, kv_heads={kv_heads}, qkv {tuple(qkv.shape)}")
        return _GqaAttention.apply(qkv, bounds, heads, kv_heads)
    if qkv.is_cuda:
        _qkv_check(qkv, heads)
        _bounds_check(qkv, bounds, "causal attention")
    return _Attention.apply(qkv, bounds, heads, "causal")


# ------------------------------------------------------------------------------------------------
# Llama building blocks: rotary position embedding (csrc/rotary.cu), RMSNorm (csrc/layernorm.cu), SwiGLU (csrc/loss.cu)
# ------------------------------------------------------------------------------------------------
def rotary_cos_sin(max_position: int, head_dim: int = ATTENTION_HEAD_DIM, theta: float = 10000.0) -> torch.Tensor:
    """fp32 [max_position, 2, head_dim // 2]: cos and sin of p * theta^(-2i / head_dim), computed in fp64 on the host."""
    inv = theta ** (-torch.arange(0, head_dim, 2, dtype=torch.float64) / head_dim)
    ang = torch.arange(max_position, dtype=torch.float64)[:, None] * inv[None, :]
    return torch.stack([ang.cos(), ang.sin()], 1).float()


def _rotary_reference(qkv: torch.Tensor, position_ids: torch.Tensor, cos_sin: torch.Tensor, heads: int, kv_heads: int,
                      inverse: bool = False) -> torch.Tensor:
    B, S, Wd = qkv.shape
    d = Wd // (heads + 2 * kv_heads)
    half = d // 2
    ct = torch.promote_types(qkv.dtype, torch.float32)
    pos = position_ids.to(device=qkv.device, dtype=torch.long).reshape(B, S).clamp(0, cos_sin.shape[0] - 1)
    cs = cos_sin.to(device=qkv.device, dtype=ct)[pos]                        # [B, S, 2, half]
    cos, sin = cs[:, :, None, 0], cs[:, :, None, 1]
    if inverse:
        sin = -sin
    qk, v = qkv.to(ct).split([(heads + kv_heads) * d, kv_heads * d], dim=-1)
    x = qk.reshape(B, S, heads + kv_heads, d)
    lo, hi = x[..., :half], x[..., half:]
    out = torch.cat([lo * cos - hi * sin, hi * cos + lo * sin], -1).reshape(B, S, -1)
    return torch.cat([out, v], -1).to(qkv.dtype)


class _Rotary(torch.autograd.Function):
    @staticmethod
    def forward(ctx, qkv, position_ids, cos_sin, heads, kv_heads):
        ctx.heads, ctx.kv_heads = heads, kv_heads
        if qkv.is_cuda:
            B, S, Wd = qkv.shape
            pos = position_ids.to(device=qkv.device, dtype=torch.int32).reshape(-1).contiguous()
            table = cos_sin.to(device=qkv.device, dtype=torch.float32).contiguous()
            ctx.save_for_backward(pos, table)
            return _C().rotary(qkv.reshape(B * S, Wd).contiguous(), pos, table, heads, kv_heads, False).view(B, S, Wd)
        ctx.save_for_backward(position_ids, cos_sin)
        return _rotary_reference(qkv, position_ids, cos_sin, heads, kv_heads)

    @staticmethod
    def backward(ctx, dy):
        pos, table = ctx.saved_tensors
        if dy.is_cuda:
            B, S, Wd = dy.shape
            dx = _C().rotary(dy.reshape(B * S, Wd).to(torch.bfloat16).contiguous(), pos, table, ctx.heads, ctx.kv_heads, True)
            return dx.view(B, S, Wd), None, None, None, None
        return _rotary_reference(dy, pos, table, ctx.heads, ctx.kv_heads, inverse=True), None, None, None, None


def rotary(qkv: torch.Tensor, position_ids: torch.Tensor, cos_sin: torch.Tensor, heads: int, kv_heads: int) -> torch.Tensor:
    """Rotary position embedding (Hugging Face's ``rotate_half`` convention: element i of a head pairs with i + d/2) of
    the query and key heads of qkv [B, S, (heads + 2 * kv_heads) * d]; the value heads pass through.  position_ids
    integer [B, S] (clamped to the table), cos_sin fp32 [max_position, 2, d / 2] (``rotary_cos_sin``).  Out of place.  On
    CUDA: bf16 and d = 64 or 128, else ``ValueError``; positions stay on the device (CUDA-graph safe)."""
    if qkv.dim() != 3 or heads < 1 or kv_heads < 1 or qkv.shape[-1] % (heads + 2 * kv_heads) or \
            (qkv.shape[-1] // (heads + 2 * kv_heads)) % 2:
        raise ValueError(f"rotary needs qkv [B, S, (heads + 2 * kv_heads) * d] with an even d, got {tuple(qkv.shape)} for "
                         f"heads={heads}, kv_heads={kv_heads}")
    d = qkv.shape[-1] // (heads + 2 * kv_heads)
    if tuple(position_ids.shape) != tuple(qkv.shape[:2]) or position_ids.is_floating_point() or position_ids.is_complex():
        raise ValueError(f"rotary needs integer position_ids {tuple(qkv.shape[:2])}, got {position_ids.dtype} {tuple(position_ids.shape)}")
    if cos_sin.dim() != 3 or tuple(cos_sin.shape[1:]) != (2, d // 2) or cos_sin.shape[0] < 1:
        raise ValueError(f"rotary needs cos_sin [max_position, 2, {d // 2}], got {tuple(cos_sin.shape)}")
    if qkv.is_cuda and (qkv.dtype != torch.bfloat16 or d not in (ATTENTION_HEAD_DIM, CAUSAL_WIDE_HEAD_DIM)):
        raise ValueError(f"rotary on CUDA needs bf16 qkv and head dim {ATTENTION_HEAD_DIM} or {CAUSAL_WIDE_HEAD_DIM}, got {qkv.dtype}, "
                         f"head dim {d}")
    return _Rotary.apply(qkv, position_ids, cos_sin, heads, kv_heads)


def _rms_norm_reference(x: torch.Tensor, weight: torch.Tensor, eps: float) -> torch.Tensor:
    xf = x.float()
    return (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps) * weight.float()).to(x.dtype)


class _RMSNormFused(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, eps):
        xc = x.contiguous()
        y, rstd = _C().rmsnorm_fwd(xc, weight.contiguous(), float(eps))
        ctx.save_for_backward(xc, weight, rstd)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, weight, rstd = ctx.saved_tensors
        dx, dw = _C().rmsnorm_bwd(dy.contiguous().to(x.dtype), x, weight.contiguous(), rstd)
        return dx, dw, None


def rms_norm(x: torch.Tensor, weight: torch.Tensor, eps: float = 1e-5) -> torch.Tensor:
    """y = x * rsqrt(mean(x^2) + eps) * weight over the last dimension (statistics in fp32).  On CUDA: the LayerNorm
    fast-path kernels up to hidden 1024 and the wide RMSNorm kernels up to 4096 (hidden % 8 == 0, bf16 or fp32 with weight
    of the same dtype), else ``ValueError``; the weight gradient is a deterministic column reduction."""
    if x.dim() < 1 or weight.dim() != 1 or weight.shape[0] != x.shape[-1]:
        raise ValueError(f"rms_norm needs x [..., hidden] and weight [hidden], got {tuple(x.shape)} and {tuple(weight.shape)}")
    if x.is_cuda:
        n = x.shape[-1]
        if x.dtype not in (torch.float32, torch.bfloat16) or weight.dtype != x.dtype or n % 8 or n > 4096:
            raise ValueError(f"rms_norm on CUDA needs bf16 or fp32 x and weight of one dtype and hidden % 8 == 0, <= 4096; got "
                             f"{x.dtype} x {weight.dtype}, hidden {n}")
        if weight.device != x.device:
            raise ValueError(f"rms_norm needs the weight on x's device ({x.device}), got {weight.device}")
        return _RMSNormFused.apply(x, weight, eps)
    return _rms_norm_reference(x, weight, eps)


class _SwiGLU(torch.autograd.Function):
    @staticmethod
    def forward(ctx, gate_up):
        gu = gate_up.contiguous()
        ctx.save_for_backward(gu)
        return _C().swiglu_fwd(gu)

    @staticmethod
    def backward(ctx, dy):
        (gu,) = ctx.saved_tensors
        return _C().swiglu_bwd(dy.to(gu.dtype).contiguous(), gu)


def _swiglu_reference(gate_up: torch.Tensor) -> torch.Tensor:
    g, u = gate_up.float().chunk(2, dim=-1)
    return (F.silu(g) * u).to(gate_up.dtype)


def swiglu(gate_up: torch.Tensor) -> torch.Tensor:
    """silu(gate) * up from one projection [..., 2 * I] with column blocks gate | up; returns [..., I].  On CUDA: one
    vectorised pass each way (the backward writes d[gate | up] together); bf16 and I % 8 == 0, else ``ValueError``."""
    if gate_up.dim() < 1 or gate_up.shape[-1] % 2:
        raise ValueError(f"swiglu needs [..., 2 * I] (gate | up), got {tuple(gate_up.shape)}")
    if gate_up.is_cuda:
        if gate_up.dtype != torch.bfloat16 or (gate_up.shape[-1] // 2) % 8:
            raise ValueError(f"swiglu on CUDA needs bf16 and I % 8 == 0, got {gate_up.dtype} {tuple(gate_up.shape)}")
        return _SwiGLU.apply(gate_up)
    return _swiglu_reference(gate_up)


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
