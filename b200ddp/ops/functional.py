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
# GELU variants: the erf form ("gelu", BERT), the tanh approximation ("gelu_tanh", GPT-2's ``gelu_new``) and QuickGELU
# ("quick_gelu", x sigmoid(1.702 x), CLIP's).  All run as a bias epilogue plus one elementwise pass (csrc/loss.cu) that keeps
# the pre-activation for the backward.
_GELU_TANH = {"gelu": False, "gelu_tanh": True}
_GELUS = (*_GELU_TANH, "quick_gelu")
QUICK_GELU_C = 1.702


def _gelu_fwd(C, pre: torch.Tensor, activation: str) -> torch.Tensor:
    return C.clip.quick_gelu_fwd(pre) if activation == "quick_gelu" else C.gelu_fwd(pre, _GELU_TANH[activation])


def _gelu_bwd(C, dy: torch.Tensor, pre: torch.Tensor, activation: str) -> torch.Tensor:
    return C.clip.quick_gelu_bwd(dy, pre) if activation == "quick_gelu" else C.gelu_bwd(dy, pre, _GELU_TANH[activation])


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


_ZERO_BIAS = {}                  # (features, dtype, device) -> zeros, never written


def _zero_bias(n: int, dtype, device) -> torch.Tensor:
    key = (n, dtype, str(device))
    if key not in _ZERO_BIAS:
        _ZERO_BIAS[key] = torch.zeros(n, dtype=dtype, device=device)
    return _ZERO_BIAS[key]


class _LinearTC(torch.autograd.Function):
    """bf16 linear on wgmma: fwd y = act(x W^T + b); bwd dgrad/wgrad without transposes (MN-major
    operand descriptors), ReLU/GELU backward applied to dy before the two GEMMs."""

    @staticmethod
    def forward(ctx, x, weight, bias, activation):
        C = _C()
        x2 = x.reshape(-1, x.shape[-1])
        if not x2.is_contiguous():
            x2 = x2.contiguous()
        if bias is None and activation not in (None, "relu", *_GELUS):
            raise ValueError("fused activation needs a bias (use bias=True)")
        if activation in _GELUS:
            # keep the pre-activation for the backward (GELU' needs it): two launches, one extra tensor
            pre = C.gemm_nt(x2, weight, bias, EPI_BIAS if bias is not None else EPI_NONE, None)
            y = _gelu_fwd(C, pre, activation)
            ctx.save_for_backward(x2, weight, pre)
        else:
            epi_bias = bias
            if bias is None and activation == "relu":            # bias-free ReLU (T5's wi): a zero bias feeds the ReLU epilogue
                epi_bias = _zero_bias(weight.shape[0], weight.dtype, weight.device)
            y = C.gemm_nt(x2, weight, epi_bias, _ACT_TO_EPI[activation] if epi_bias is not None else EPI_NONE, None)
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
        elif ctx.activation in _GELUS:
            dy2 = _gelu_bwd(C, dy2.contiguous(), aux, ctx.activation)          # dy * gelu'(pre) in one pass
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
    """y = act(x @ weight.T + bias), activation in {None, "relu", "gelu", "gelu_tanh", "quick_gelu"} ("gelu" is the erf
    form, "gelu_tanh" the tanh approximation, "quick_gelu" x sigmoid(1.702 x)).  ``fp8=True`` runs the three GEMMs on FP8
    tensor cores (``_LinearFP8``); on CUDA it needs bf16 tensors and raises ``ValueError`` for anything else, and it has no
    QuickGELU."""
    if fp8:
        if activation == "quick_gelu":
            raise ValueError("fp8 linear has no quick_gelu activation")
        return _LinearFP8.apply(x, weight, bias, activation, torch.is_grad_enabled())
    if x.is_cuda:
        N, K = weight.shape
        M = x.numel() // K
        if x.dtype == torch.bfloat16 and weight.dtype == torch.bfloat16 and _tc_ok(M, N, K) \
                and (bias is not None or activation in (None, "relu", *_GELUS)) and os.environ.get("B200DDP_DISABLE_TC", "0") != "1":
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
    elif activation == "quick_gelu":
        y = y * torch.sigmoid(QUICK_GELU_C * y)                       # transformers' QuickGELUActivation
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


def window_bounds(bounds: torch.Tensor, window: int) -> torch.Tensor:
    """Bidirectional sliding-window bounds inside documents: int32 [B, S, 2] where position i's interval (start, end)
    becomes (max(start, i - window), min(end, i + window + 1)), so query i sees key j iff both lie in one document and
    |i - j| <= window (ModernBERT's local attention with ``window = local_attention // 2``).  The mask stays symmetric,
    which is what ``packed_attention``'s key-side gradient needs, and its kernels skip every tile outside the window.
    Padding rows (start == end) stay empty; ``window >= S - 1`` returns ``bounds`` itself.  Torch ops on bounds' device,
    no host synchronisation (CUDA-graph safe).  A negative or non-integer window raises ``ValueError``."""
    if isinstance(window, bool) or not isinstance(window, int) or window < 0:
        raise ValueError(f"window_bounds needs a non-negative integer window, got {window!r}")
    if bounds.dim() != 3 or bounds.shape[-1] != 2 or bounds.is_floating_point() or bounds.is_complex():
        raise ValueError(f"window_bounds needs integer bounds [B, S, 2], got {bounds.dtype} {tuple(bounds.shape)}")
    S = bounds.shape[1]
    if window >= S - 1:
        return bounds
    b = bounds.to(torch.int32)
    i = torch.arange(S, device=b.device, dtype=torch.int32)[None, :]
    start, end = b[..., 0], b[..., 1]
    win = torch.stack([torch.maximum(start, i - window), torch.minimum(end, i + window + 1)], -1)
    return torch.where((start == end)[..., None], b, win)


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
# Cross-attention (csrc/cross_attention.cu): queries of one sequence attend to the keys / values of another
# ------------------------------------------------------------------------------------------------
def _interval_mask(bounds: torch.Tensor, n: int, device) -> torch.Tensor:
    """[B, R, n] bool: row r sees column j iff start[r] <= j < end[r] (start clamped to [0, n], end to [start, n], like
    the kernels)."""
    b = bounds.to(device=device, dtype=torch.long)
    start = b[..., 0].clamp(0, n)
    end = torch.maximum(b[..., 1].clamp(max=n), start)
    j = torch.arange(n, device=device)
    return (j >= start[..., None]) & (j < end[..., None])


def cross_attention_reference(q: torch.Tensor, kv: torch.Tensor, q_bounds: torch.Tensor, heads: int) -> torch.Tensor:
    """softmax(Q K^T / sqrt(d)) V where query i of row b sees key j of row b iff q_bounds[b, i, 0] <= j < q_bounds[b, i, 1],
    as a dense mask in fp32 (fp64 stays fp64); a query that sees no key gives zeros.  q [B, Sq, hidden], kv
    [B, Sk, 2 * hidden] (key | value column blocks), q_bounds integer [B, Sq, 2]; returns [B, Sq, hidden] in q's dtype.
    Differentiable."""
    B, Sq, hidden = q.shape
    Sk = kv.shape[1]
    hd = hidden // heads
    ct = torch.promote_types(q.dtype, torch.float32)
    qh = q.to(ct).reshape(B, Sq, heads, hd).transpose(1, 2)
    k, v = (t.to(ct).reshape(B, Sk, heads, hd).transpose(1, 2) for t in kv.split(hidden, dim=-1))
    keep = _interval_mask(q_bounds, Sk, q.device)[:, None]
    scores = (qh @ k.transpose(-1, -2)) * (1.0 / math.sqrt(hd))
    p = torch.softmax(scores.masked_fill(~keep, torch.finfo(ct).min), dim=-1) * keep
    return (p @ v).transpose(1, 2).reshape(B, Sq, hidden).to(q.dtype)


def _cross_check(q: torch.Tensor, kv: torch.Tensor, q_bounds: torch.Tensor, kv_bounds: torch.Tensor, heads: int) -> None:
    if q.dim() != 3 or kv.dim() != 3 or q.shape[0] != kv.shape[0] or kv.shape[-1] != 2 * q.shape[-1]:
        raise ValueError(f"cross attention needs q [B, Sq, hidden] and kv [B, Sk, 2 * hidden], got {tuple(q.shape)} and {tuple(kv.shape)}")
    B, Sq, hidden = q.shape
    Sk = kv.shape[1]
    if heads < 1 or hidden % heads or hidden // heads != ATTENTION_HEAD_DIM:
        raise ValueError(f"cross attention on CUDA supports head dim {ATTENTION_HEAD_DIM} only, got hidden {hidden} over {heads} heads")
    if q.dtype != torch.bfloat16 or kv.dtype != torch.bfloat16:
        raise ValueError(f"cross attention on CUDA needs bf16 q and kv, got {q.dtype} and {kv.dtype}")
    if Sq == 0 or Sk == 0 or Sq % ATTENTION_SEQ_MULTIPLE or Sk % ATTENTION_SEQ_MULTIPLE:
        raise ValueError(f"cross attention on CUDA needs both lengths to be multiples of {ATTENTION_SEQ_MULTIPLE}, got Sq={Sq}, Sk={Sk}")
    if not q.is_contiguous() or not kv.is_contiguous():
        raise ValueError("cross attention on CUDA needs contiguous q and kv (the projections' outputs)")
    for name, t, S in (("q_bounds", q_bounds, Sq), ("kv_bounds", kv_bounds, Sk)):
        if tuple(t.shape) != (B, S, 2) or t.is_floating_point() or t.is_complex():
            raise ValueError(f"cross attention needs integer {name} [B, {'Sq' if S == Sq else 'Sk'}, 2] = [{B}, {S}, 2], "
                             f"got {t.dtype} {tuple(t.shape)}")


class _CrossAttention(torch.autograd.Function):
    """CUDA body: the sm_90a cross-attention kernels (forward keeps the row log-sum-exp; backward is four deterministic
    launches writing dq and dkv, the gradients the two projections consume).  CPU body: ``cross_attention_reference``
    (backward by recomputation through autograd)."""

    @staticmethod
    def forward(ctx, q, kv, q_bounds, kv_bounds, heads):
        ctx.heads = heads
        if q.is_cuda:
            B, Sq, hidden = q.shape
            Sk = kv.shape[1]
            qb = q_bounds.to(device=q.device, dtype=torch.int32).contiguous()
            kb = kv_bounds.to(device=q.device, dtype=torch.int32).contiguous()
            o, lse = _C().cross.cross_attention_fwd(q.view(B * Sq, hidden), kv.view(B * Sk, 2 * hidden), qb, heads)
            ctx.save_for_backward(q, kv, o, lse, qb, kb)
            return o.view(B, Sq, hidden)
        ctx.save_for_backward(q, kv, q_bounds)
        return cross_attention_reference(q, kv, q_bounds, heads)

    @staticmethod
    def backward(ctx, dy):
        if dy.is_cuda:
            q, kv, o, lse, qb, kb = ctx.saved_tensors
            B, Sq, hidden = q.shape
            Sk = kv.shape[1]
            do = dy.reshape(B * Sq, hidden).to(torch.bfloat16).contiguous()
            if do.data_ptr() % 16:                                # the kernels read dO in 16-byte vectors / TMA boxes
                do = do.clone()
            dq, dkv = _C().cross.cross_attention_bwd(do, q.view(B * Sq, hidden), kv.view(B * Sk, 2 * hidden), o, lse, qb, kb, ctx.heads)
            return dq.view(B, Sq, hidden), dkv.view(B, Sk, 2 * hidden), None, None, None
        q, kv, q_bounds = ctx.saved_tensors
        with torch.enable_grad():
            x, y = q.detach().requires_grad_(True), kv.detach().requires_grad_(True)
            dq, dkv = torch.autograd.grad(cross_attention_reference(x, y, q_bounds, ctx.heads), (x, y), dy)
        return dq, dkv, None, None, None


def cross_attention(q: torch.Tensor, kv: torch.Tensor, q_bounds: torch.Tensor, kv_bounds: torch.Tensor, heads: int) -> torch.Tensor:
    """Multi-head cross-attention: q [B, Sq, hidden] (the query projection's output), kv [B, Sk, 2 * hidden] (the fused
    key | value projection of the other sequence), q_bounds integer [B, Sq, 2]: query i of row b sees key j of row b iff
    q_bounds[b, i, 0] <= j < q_bounds[b, i, 1]; kv_bounds integer [B, Sk, 2]: for key j, the interval of queries that see
    it.  The two must describe the same mask (``cross_bounds`` builds such a pair); the kernels trust it rather than
    check it, which would need a host synchronisation.  A query that sees no key gives zeros; a key no query sees gets
    zero gradients.  Returns [B, Sq, hidden].  On CUDA: bf16, head dim 64, Sq and Sk multiples of 128, contiguous q and
    kv, else ``ValueError``; bounds stay on the device (CUDA-graph safe)."""
    if q.is_cuda:
        _cross_check(q, kv, q_bounds, kv_bounds, heads)
    return _CrossAttention.apply(q, kv, q_bounds, kv_bounds, heads)


# ------------------------------------------------------------------------------------------------
# T5's relative position bias (csrc/attention.cu, kBias): a learned, bucketed bias added to the unscaled scores
# ------------------------------------------------------------------------------------------------
RELATIVE_MAX_DISTANCE = 128
RELATIVE_TABLE_COLS = 2 * RELATIVE_MAX_DISTANCE + 1    # the distances k - i clamped to [-128, 128]
_RELATIVE_BUCKETS = {}                                  # (bidirectional, num_buckets, device) -> int32 [257]


def relative_position_bucket(rel: torch.Tensor, bidirectional: bool, num_buckets: int = 32, max_distance: int = 128) -> torch.Tensor:
    """T5's bucket of each relative position ``rel = key - query`` (long), with transformers' float32 expression
    (``T5Attention._relative_position_bucket``), so the bucket edges fall where transformers puts them.  Bidirectional
    (encoder): half the buckets for positive distances; unidirectional (decoder): only ``rel <= 0`` is told apart."""
    rel = torch.as_tensor(rel).long()
    buckets = torch.zeros_like(rel)
    if bidirectional:
        num_buckets //= 2
        buckets = buckets + (rel > 0).long() * num_buckets
        rel = rel.abs()
    else:
        rel = -torch.min(rel, torch.zeros_like(rel))
    max_exact = num_buckets // 2
    large = max_exact + (torch.log(rel.float() / max_exact) / math.log(max_distance / max_exact) * (num_buckets - max_exact)).long()
    large = torch.min(large, torch.full_like(large, num_buckets - 1))
    return buckets + torch.where(rel < max_exact, rel, large)


def _relative_buckets(bidirectional: bool, num_buckets: int, device) -> torch.Tensor:
    """int32 [257]: the bucket of each clamped distance c - 128, computed on the host once per configuration and device."""
    key = (bool(bidirectional), int(num_buckets), str(device))
    if key not in _RELATIVE_BUCKETS:
        _RELATIVE_BUCKETS[key] = relative_position_buckets(bidirectional, num_buckets).to(device)
    return _RELATIVE_BUCKETS[key]


class _RelativeTable(torch.autograd.Function):
    """CUDA body: one gather kernel forward; backward one kernel that folds dtable into d weight bucket by bucket in a
    fixed order (no atomics).  CPU body: indexing, in fp32 (fp64 stays fp64)."""

    @staticmethod
    def forward(ctx, weight, bidirectional, buckets):
        idx = _relative_buckets(bidirectional, weight.shape[0], weight.device) if buckets is None else buckets
        ctx.save_for_backward(weight, idx)
        if weight.is_cuda:
            return _C().t5.relative_table_fwd(weight.contiguous(), idx)
        return weight.to(torch.promote_types(weight.dtype, torch.float32))[idx.long()].t().contiguous()

    @staticmethod
    def backward(ctx, dtable):
        weight, idx = ctx.saved_tensors
        if dtable.is_cuda:
            return _C().t5.relative_table_bwd(dtable.float().contiguous(), idx, weight.contiguous()), None, None
        dw = torch.zeros(weight.shape, dtype=dtable.dtype)
        dw.index_add_(0, idx.long(), dtable.t())
        return dw.to(weight.dtype), None, None


def relative_position_buckets(bidirectional: bool, num_buckets: int = 32) -> torch.Tensor:
    """int32 [257] on the CPU: the bucket of each clamped distance c - 128 (``relative_position_bucket``).  A module that
    keeps it as a buffer hands ``relative_position_table`` a device copy made when the module moved, so no forward (and no
    CUDA-graph capture) copies it to the device."""
    rel = torch.arange(-RELATIVE_MAX_DISTANCE, RELATIVE_MAX_DISTANCE + 1)
    return relative_position_bucket(rel, bidirectional, num_buckets, RELATIVE_MAX_DISTANCE).to(torch.int32)


def relative_position_table(weight: torch.Tensor, bidirectional: bool, buckets: Optional[torch.Tensor] = None) -> torch.Tensor:
    """T5's bias per head and clamped distance: weight [num_buckets, heads] (the ``relative_attention_bias`` embedding)
    -> fp32 [heads, 257], column c holding the bias of distance ``key - query = c - 128`` (exact at any length: every
    distance beyond +-128 falls in the bucket of +-128).  Differentiable.  A stack builds it once per forward and hands it
    to all its layers, so autograd sums their fp32 gradients before the one fold into the weight.  ``buckets``:
    ``relative_position_buckets(bidirectional, num_buckets)`` on weight's device; without it a copy cached per device is
    used, made on the first call."""
    if weight.dim() != 2 or not weight.is_floating_point():
        raise ValueError(f"relative_position_table needs a floating weight [num_buckets, heads], got {weight.dtype} {tuple(weight.shape)}")
    if buckets is not None and (tuple(buckets.shape) != (RELATIVE_TABLE_COLS,) or buckets.dtype != torch.int32 or buckets.device != weight.device):
        raise ValueError(f"relative_position_table needs int32 buckets [{RELATIVE_TABLE_COLS}] on weight's device, got "
                         f"{buckets.dtype} {tuple(buckets.shape)} on {buckets.device}")
    return _RelativeTable.apply(weight, bidirectional, buckets)


def relative_attention_reference(qkv: torch.Tensor, bounds: torch.Tensor, table: torch.Tensor, heads: int, causal: bool) -> torch.Tensor:
    """softmax(Q K^T + bias) V with T5's unscaled scores, bias[h, i, j] = table[h, clamp(j - i, -128, 128) + 128], under the
    mask of ``packed_attention`` (causal=False) or ``causal_attention`` (causal=True), as a dense mask in fp32 (fp64 stays
    fp64); a row that sees no key gives zeros.  qkv [B, S, 3 * hidden], bounds integer [B, S, 2], table [heads, 257];
    returns [B, S, hidden] in qkv's dtype.  Differentiable in qkv and table."""
    B, S, W = qkv.shape
    hidden = W // 3
    hd = hidden // heads
    ct = torch.promote_types(qkv.dtype, torch.float32)
    q, k, v = (t.to(ct).reshape(B, S, heads, hd).transpose(1, 2) for t in qkv.split(hidden, dim=-1))
    pos = torch.arange(S, device=qkv.device)
    col = (pos[None, :] - pos[:, None]).clamp(-RELATIVE_MAX_DISTANCE, RELATIVE_MAX_DISTANCE) + RELATIVE_MAX_DISTANCE
    keep = (_causal_mask if causal else _bounds_mask)(bounds, S, qkv.device)[:, None]
    scores = q @ k.transpose(-1, -2) + table.to(ct)[:, col]
    p = torch.softmax(scores.masked_fill(~keep, torch.finfo(ct).min), dim=-1) * keep
    return (p @ v).transpose(1, 2).reshape(B, S, hidden).to(qkv.dtype)


class _RelativeAttention(torch.autograd.Function):
    """CUDA body: the kBias instantiations of the segment / causal kernels (backward: dqkv, and dtable through per-CTA
    partials and a fixed-order finish, no atomics).  CPU body: ``relative_attention_reference``."""

    @staticmethod
    def forward(ctx, qkv, bounds, table, heads, causal):
        ctx.heads, ctx.causal = heads, causal
        if qkv.is_cuda:
            B, S, W = qkv.shape
            m = bounds.to(device=qkv.device, dtype=torch.int32).contiguous()
            t = table.float().contiguous()
            o, lse = _C().t5.relative_attention_fwd(qkv.view(B * S, W), m, t, heads, causal)
            ctx.save_for_backward(qkv, o, lse, m, t)
            return o.view(B, S, W // 3)
        ctx.save_for_backward(qkv, bounds, table)
        return relative_attention_reference(qkv, bounds, table, heads, causal)

    @staticmethod
    def backward(ctx, dy):
        if dy.is_cuda:
            qkv, o, lse, m, t = ctx.saved_tensors
            B, S, W = qkv.shape
            do = dy.reshape(B * S, W // 3).to(torch.bfloat16).contiguous()
            if do.data_ptr() % 16:                                # the kernels read dO in TMA boxes
                do = do.clone()
            dqkv, dtable = _C().t5.relative_attention_bwd(do, qkv.view(B * S, W), o, lse, m, t, ctx.heads, ctx.causal)
            return dqkv.view(B, S, W), None, dtable, None, None
        qkv, bounds, table = ctx.saved_tensors
        with torch.enable_grad():
            x, tb = qkv.detach().requires_grad_(True), table.detach().requires_grad_(True)
            dx, dt = torch.autograd.grad(relative_attention_reference(x, bounds, tb, ctx.heads, ctx.causal), (x, tb), dy)
        return dx, None, dt, None, None


def relative_attention(qkv: torch.Tensor, bounds: torch.Tensor, table: torch.Tensor, heads: int, causal: bool) -> torch.Tensor:
    """T5's self-attention: ``packed_attention`` (causal=False) or ``causal_attention`` (causal=True) over the documents of
    bounds [B, S, 2], with the scores unscaled and T5's relative bias added, table [heads, 257]
    (``relative_position_table``).  The distance is ``key - query`` inside a row, which inside a packed document is the
    in-document distance.  Returns [B, S, hidden], with gradients for qkv and table.  On CUDA: bf16 qkv, head dim 64,
    S % 128 == 0, contiguous qkv and a [heads, 257] table, else ``ValueError``; no host synchronisation (CUDA-graph
    safe)."""
    if qkv.is_cuda:
        _qkv_check(qkv, heads)
        _bounds_check(qkv, bounds, "relative attention")
        if tuple(table.shape) != (heads, RELATIVE_TABLE_COLS) or not table.is_floating_point():
            raise ValueError(f"relative attention needs a table [heads, {RELATIVE_TABLE_COLS}] = [{heads}, {RELATIVE_TABLE_COLS}], "
                             f"got {table.dtype} {tuple(table.shape)}")
    return _RelativeAttention.apply(qkv, bounds, table, heads, causal)


def _document_table(bounds: torch.Tensor, slots: int):
    """Per position, the index of its document in its row (counting from 0, -1 for padding), and a table
    [B, slots + 1, 2] (slots >= S) of each row's k-th document's (start, end), (0, 0) where the row has no k-th document."""
    B, S, _ = bounds.shape
    b = bounds.to(torch.long)
    start, end = b[..., 0], b[..., 1]
    pos = torch.arange(S, device=b.device)
    is_start = (start == pos) & (end > start)
    index = torch.where(end > start, is_start.long().cumsum(1) - 1, -1)
    slot = torch.where(is_start, index, slots)
    table = torch.zeros(B, slots + 1, 2, dtype=torch.long, device=b.device)
    table.scatter_(1, slot[..., None].expand(B, S, 2), torch.where(is_start[..., None], b, 0))
    table[:, slots] = 0
    return index, table


def cross_bounds(enc_bounds: torch.Tensor, dec_bounds: torch.Tensor):
    """Cross-attention bounds of paired documents: the k-th decoder document of a row sees the k-th encoder document of
    the same row.  enc_bounds [B, Sk, 2] and dec_bounds [B, Sq, 2] are the two sides' ``document_bounds``.  Returns
    ``(q_bounds, kv_bounds)`` int32 [B, Sq, 2] and [B, Sk, 2]: each decoder position gets its partner document's (start,
    end), each encoder position its partner's; padding positions and documents without a partner get (0, 0).  Both
    describe the same mask, as ``cross_attention`` requires.  Torch ops on the bounds' device, no host synchronisation."""
    if enc_bounds.dim() != 3 or dec_bounds.dim() != 3 or enc_bounds.shape[0] != dec_bounds.shape[0] or enc_bounds.shape[-1] != 2 \
            or dec_bounds.shape[-1] != 2:
        raise ValueError(f"cross_bounds needs enc_bounds [B, Sk, 2] and dec_bounds [B, Sq, 2], got {tuple(enc_bounds.shape)} "
                         f"and {tuple(dec_bounds.shape)}")
    slots = max(enc_bounds.shape[1], dec_bounds.shape[1])
    enc_index, enc_table = _document_table(enc_bounds, slots)
    dec_index, dec_table = _document_table(dec_bounds, slots)

    def partner(index, table):
        got = torch.gather(table, 1, torch.where(index >= 0, index, slots)[..., None].expand(*index.shape, 2))
        return got.to(torch.int32)

    return partner(dec_index, enc_table), partner(enc_index, dec_table)


# ------------------------------------------------------------------------------------------------
# Llama building blocks: rotary position embedding (csrc/rotary.cu), RMSNorm (csrc/layernorm.cu), SwiGLU (csrc/loss.cu)
# ------------------------------------------------------------------------------------------------
def rotary_cos_sin(max_position: int, head_dim: int = ATTENTION_HEAD_DIM, theta: float = 10000.0) -> torch.Tensor:
    """fp32 [max_position, 2, head_dim // 2]: cos and sin of p * theta^(-2i / head_dim), computed in fp64 on the host."""
    inv = theta ** (-torch.arange(0, head_dim, 2, dtype=torch.float64) / head_dim)
    ang = torch.arange(max_position, dtype=torch.float64)[:, None] * inv[None, :]
    return torch.stack([ang.cos(), ang.sin()], 1).float()


def _rotary_reference(qkv: torch.Tensor, position_ids: torch.Tensor, cos_sin: torch.Tensor, heads: int, kv_heads: int,
                      inverse: bool = False, q_scale: float = 1.0) -> torch.Tensor:
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
    out = torch.cat([lo * cos - hi * sin, hi * cos + lo * sin], -1)
    if q_scale != 1.0:
        out = torch.cat([out[:, :, :heads] * q_scale, out[:, :, heads:]], 2)
    return torch.cat([out.reshape(B, S, -1), v], -1).to(qkv.dtype)


class _Rotary(torch.autograd.Function):
    @staticmethod
    def forward(ctx, qkv, position_ids, cos_sin, heads, kv_heads, q_scale):
        ctx.heads, ctx.kv_heads, ctx.q_scale = heads, kv_heads, q_scale
        if qkv.is_cuda:
            B, S, Wd = qkv.shape
            pos = position_ids.to(device=qkv.device, dtype=torch.int32).reshape(-1).contiguous()
            table = cos_sin.to(device=qkv.device, dtype=torch.float32).contiguous()
            ctx.save_for_backward(pos, table)
            return _C().rotary(qkv.reshape(B * S, Wd).contiguous(), pos, table, heads, kv_heads, False, q_scale).view(B, S, Wd)
        ctx.save_for_backward(position_ids, cos_sin)
        return _rotary_reference(qkv, position_ids, cos_sin, heads, kv_heads, q_scale=q_scale)

    @staticmethod
    def backward(ctx, dy):
        pos, table = ctx.saved_tensors
        if dy.is_cuda:
            B, S, Wd = dy.shape
            dx = _C().rotary(dy.reshape(B * S, Wd).to(torch.bfloat16).contiguous(), pos, table, ctx.heads, ctx.kv_heads, True, ctx.q_scale)
            return dx.view(B, S, Wd), None, None, None, None, None
        return (_rotary_reference(dy, pos, table, ctx.heads, ctx.kv_heads, inverse=True, q_scale=ctx.q_scale),
                None, None, None, None, None)


def rotary(qkv: torch.Tensor, position_ids: torch.Tensor, cos_sin: torch.Tensor, heads: int, kv_heads: int,
           q_scale: float = 1.0) -> torch.Tensor:
    """Rotary position embedding (Hugging Face's ``rotate_half`` convention: element i of a head pairs with i + d/2) of
    the query and key heads of qkv [B, S, (heads + 2 * kv_heads) * d]; the value heads pass through.  position_ids
    integer [B, S] (clamped to the table), cos_sin fp32 [max_position, 2, d / 2] (``rotary_cos_sin``).  Out of place.  On
    CUDA: bf16 and d = 64 or 128, else ``ValueError``; positions stay on the device (CUDA-graph safe).

    ``q_scale``, a positive power of two (exact in bf16, else ``ValueError``), also multiplies the query heads: it folds
    an attention score scale other than 1 / sqrt(d) (Granite's ``attention_multiplier``) into q."""
    if not (q_scale > 0 and math.frexp(q_scale)[0] == 0.5):
        raise ValueError(f"rotary: q_scale must be a positive power of two (exact in bf16), got {q_scale}")
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
    return _Rotary.apply(qkv, position_ids, cos_sin, heads, kv_heads, float(q_scale))


def _qk_norm_rotary_reference(qkv: torch.Tensor, q_weight: torch.Tensor, k_weight: torch.Tensor, position_ids: torch.Tensor,
                              cos_sin: torch.Tensor, heads: int, kv_heads: int, eps: float) -> torch.Tensor:
    B, S, Wd = qkv.shape
    d = Wd // (heads + 2 * kv_heads)
    ct = torch.promote_types(qkv.dtype, torch.float32)
    x = qkv.to(ct)
    qk, v = x.split([(heads + kv_heads) * d, kv_heads * d], dim=-1)
    qk = qk.reshape(B, S, heads + kv_heads, d)
    w = torch.cat([q_weight.to(ct).expand(heads, d), k_weight.to(ct).expand(kv_heads, d)])
    qk = qk * torch.rsqrt(qk.pow(2).mean(-1, keepdim=True) + eps) * w
    normed = torch.cat([qk.reshape(B, S, -1), v], -1)
    return _rotary_reference(normed, position_ids, cos_sin, heads, kv_heads).to(qkv.dtype)


class _QkNormRotary(torch.autograd.Function):
    @staticmethod
    def forward(ctx, qkv, q_weight, k_weight, position_ids, cos_sin, heads, kv_heads, eps):
        ctx.heads, ctx.kv_heads, ctx.eps = heads, kv_heads, eps
        if qkv.is_cuda:
            B, S, Wd = qkv.shape
            x = qkv.reshape(B * S, Wd).contiguous()
            pos = position_ids.to(device=qkv.device, dtype=torch.int32).reshape(-1).contiguous()
            table = cos_sin.to(device=qkv.device, dtype=torch.float32).contiguous()
            wq, wk = q_weight.contiguous(), k_weight.contiguous()
            y, rstd = _C().qk_norm_rotary_fwd(x, wq, wk, pos, table, heads, kv_heads, eps)
            ctx.save_for_backward(x, rstd, wq, wk, pos, table)
            return y.view(B, S, Wd)
        ctx.save_for_backward(qkv, q_weight, k_weight, position_ids, cos_sin)
        return _qk_norm_rotary_reference(qkv, q_weight, k_weight, position_ids, cos_sin, heads, kv_heads, eps)

    @staticmethod
    def backward(ctx, dy):
        if dy.is_cuda:
            x, rstd, wq, wk, pos, table = ctx.saved_tensors
            B, S, Wd = dy.shape
            dx, dwq, dwk = _C().qk_norm_rotary_bwd(dy.reshape(B * S, Wd).to(torch.bfloat16).contiguous(), x, rstd, wq, wk, pos, table,
                                                   ctx.heads, ctx.kv_heads)
            return dx.view(B, S, Wd), dwq, dwk, None, None, None, None, None
        qkv, q_weight, k_weight, position_ids, cos_sin = ctx.saved_tensors
        with torch.enable_grad():                    # the CPU body's gradient is autograd through the reference
            ins = [t.detach().requires_grad_(True) for t in (qkv, q_weight, k_weight)]
            y = _qk_norm_rotary_reference(*ins, position_ids, cos_sin, ctx.heads, ctx.kv_heads, ctx.eps)
            grads = torch.autograd.grad(y, ins, dy)
        return (*grads, None, None, None, None, None)


def qk_norm_rotary(qkv: torch.Tensor, q_weight: torch.Tensor, k_weight: torch.Tensor, position_ids: torch.Tensor,
                   cos_sin: torch.Tensor, heads: int, kv_heads: int, eps: float = 1e-6) -> torch.Tensor:
    """Qwen3's per-head q / k RMSNorm followed by rotary, in Hugging Face's ``Qwen3Attention`` order (norm, then rope):
    every query head h of qkv [B, S, (heads + 2 * kv_heads) * d] becomes rope(x * rsqrt(mean(x^2) + eps) * q_weight) over
    its d elements, every key head the same with k_weight ([d] each); value heads pass through.  position_ids and cos_sin
    as for ``rotary``.  Out of place.

    On CUDA one kernel per direction (statistics and rotation in fp32, one bf16 rounding), with bf16 qkv, d = 128,
    16-byte aligned qkv and bf16 weights on qkv's device, else ``ValueError``; positions stay on the device (CUDA-graph
    safe).  The weight gradients are deterministic (per-CTA partials summed in a fixed order).  The backward keeps the
    pre-norm qkv and fp32 rstd [B * S, heads + kv_heads]: at 16,384 tokens and Qwen3-0.6B's 4096-wide qkv, about 134 MB
    per layer (plus 1.6 MB of rstd)."""
    if qkv.dim() != 3 or heads < 1 or kv_heads < 1 or qkv.shape[-1] % (heads + 2 * kv_heads) or \
            (qkv.shape[-1] // (heads + 2 * kv_heads)) % 2:
        raise ValueError(f"qk_norm_rotary needs qkv [B, S, (heads + 2 * kv_heads) * d] with an even d, got {tuple(qkv.shape)} for "
                         f"heads={heads}, kv_heads={kv_heads}")
    d = qkv.shape[-1] // (heads + 2 * kv_heads)
    if q_weight.shape != (d,) or k_weight.shape != (d,):
        raise ValueError(f"qk_norm_rotary needs q_weight and k_weight [{d}], got {tuple(q_weight.shape)} and {tuple(k_weight.shape)}")
    if tuple(position_ids.shape) != tuple(qkv.shape[:2]) or position_ids.is_floating_point() or position_ids.is_complex():
        raise ValueError(f"qk_norm_rotary needs integer position_ids {tuple(qkv.shape[:2])}, got {position_ids.dtype} "
                         f"{tuple(position_ids.shape)}")
    if cos_sin.dim() != 3 or tuple(cos_sin.shape[1:]) != (2, d // 2) or cos_sin.shape[0] < 1:
        raise ValueError(f"qk_norm_rotary needs cos_sin [max_position, 2, {d // 2}], got {tuple(cos_sin.shape)}")
    if not eps > 0:
        raise ValueError(f"qk_norm_rotary needs eps > 0, got {eps}")
    if qkv.is_cuda:
        if qkv.dtype != torch.bfloat16 or d != CAUSAL_WIDE_HEAD_DIM:
            raise ValueError(f"qk_norm_rotary on CUDA needs bf16 qkv and head dim {CAUSAL_WIDE_HEAD_DIM}, got {qkv.dtype}, head dim {d}")
        if any(w.dtype != torch.bfloat16 or w.device != qkv.device for w in (q_weight, k_weight)):
            raise ValueError(f"qk_norm_rotary on CUDA needs bf16 weights on qkv's device ({qkv.device}), got "
                             f"{q_weight.dtype} on {q_weight.device} and {k_weight.dtype} on {k_weight.device}")
        if qkv.is_contiguous() and qkv.data_ptr() % 16:
            raise ValueError("qk_norm_rotary on CUDA needs 16-byte aligned qkv")
    return _QkNormRotary.apply(qkv, q_weight, k_weight, position_ids, cos_sin, heads, kv_heads, float(eps))


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


class _GeGLU(torch.autograd.Function):
    @staticmethod
    def forward(ctx, input_gate):
        ctx.save_for_backward(input_gate)
        return _C().geglu_fwd(input_gate)

    @staticmethod
    def backward(ctx, dy):
        (ig,) = ctx.saved_tensors
        return _C().geglu_bwd(dy.to(ig.dtype).contiguous(), ig)


def _geglu_reference(input_gate: torch.Tensor) -> torch.Tensor:
    a, g = input_gate.to(torch.promote_types(input_gate.dtype, torch.float32)).chunk(2, dim=-1)
    return (F.gelu(a) * g).to(input_gate.dtype)


def geglu(input_gate: torch.Tensor) -> torch.Tensor:
    """gelu(input) * gate (the erf form of GELU) from one projection [..., 2 * I] with column blocks input | gate; returns
    [..., I] (ModernBERT's MLP).  CPU: the fp32 reference, differentiated by autograd.  On CUDA: one vectorised pass each
    way (the backward writes d[input | gate] together); bf16, I % 8 == 0 and a contiguous 16-byte aligned input, else
    ``ValueError``."""
    if input_gate.dim() < 1 or input_gate.shape[-1] % 2:
        raise ValueError(f"geglu needs [..., 2 * I] (input | gate), got {tuple(input_gate.shape)}")
    if input_gate.is_cuda:
        if input_gate.dtype != torch.bfloat16 or (input_gate.shape[-1] // 2) % 8:
            raise ValueError(f"geglu on CUDA needs bf16 and I % 8 == 0, got {input_gate.dtype} {tuple(input_gate.shape)}")
        if not input_gate.is_contiguous() or input_gate.data_ptr() % 16:
            raise ValueError("geglu on CUDA needs a contiguous, 16-byte aligned input")
        return _GeGLU.apply(input_gate)
    return _geglu_reference(input_gate)


# ------------------------------------------------------------------------------------------------
# Mixture of experts (csrc/moe.cu routing / permutation / combine, csrc/gemm_wgmma.cu grouped GEMMs)
# ------------------------------------------------------------------------------------------------
MOE_MAX_EXPERTS = 64
MOE_MAX_TOP_K = 8
MOE_ALIGN = 128            # each expert's segment of the permuted rows starts at a multiple of this


def moe_capacity(tokens: int, experts: int, top_k: int) -> int:
    """Rows of the permuted buffers: every expert's segment padded to a multiple of 128, for any routing."""
    return (tokens * top_k + experts * (MOE_ALIGN - 1) + MOE_ALIGN - 1) // MOE_ALIGN * MOE_ALIGN


def moe_route_reference(logits: torch.Tensor, top_k: int):
    """(ids [T, k] long, gates [T, k] fp32): the top-k logits of each row, ties to the lower expert (a stable sort), and
    the softmax over them in fp32.  Differentiable in the gates."""
    ids = torch.sort(logits.float(), dim=-1, descending=True, stable=True).indices[:, :top_k]
    return ids, torch.softmax(logits.float().gather(1, ids), dim=-1)


def moe_permute_reference(ids: torch.Tensor, experts: int):
    """The expert-sorted layout the native permutation writes, from ids [T, k]: (counts [E], offsets [E + 1] (segment
    starts, multiples of 128), fwd_map [capacity] (row -> t * k + j, -1 in padding), inv_map [T, k] (t * k + j -> row),
    tile_expert [capacity / 128] (-1 for unused tiles)), all int32.  Within an expert, rows keep the order of t * k + j."""
    T, k = ids.shape
    flat = ids.reshape(-1).long()
    counts = torch.bincount(flat, minlength=experts)
    padded = (counts + MOE_ALIGN - 1) // MOE_ALIGN * MOE_ALIGN
    offsets = torch.cat([padded.new_zeros(1), padded.cumsum(0)])
    cap = moe_capacity(T, experts, k)
    order = torch.sort(flat, stable=True).indices                     # assignments grouped by expert, in order
    starts = torch.cat([counts.new_zeros(1), counts.cumsum(0)])[:-1]
    sorted_e = flat[order]
    rows = offsets[sorted_e] + torch.arange(T * k) - starts[sorted_e]
    fwd = torch.full((cap,), -1, dtype=torch.long)
    fwd[rows] = order
    inv = torch.empty(T * k, dtype=torch.long)
    inv[order] = rows
    tile0 = torch.arange(cap // MOE_ALIGN) * MOE_ALIGN
    owner = ((tile0[:, None] >= offsets[None, :-1]) & (tile0[:, None] < offsets[None, 1:])).int()
    tiles = torch.where(owner.any(1), owner.argmax(1), -1)
    return tuple(t.to(torch.int32) for t in (counts, offsets, fwd, inv.view(T, k), tiles))


def _moe_reference(x, router_weight, w_gate_up, w_down, top_k, aux=False, routing_logits=None):
    """Hugging Face's ``GraniteMoeMoE`` with the stable tie rule: the router logits in x's dtype, then in fp32; top-k and
    a softmax over the chosen logits in fp32, rounded to x's dtype; each expert a SwiGLU over its rows (w_gate_up [E, 2I,
    H], gate | up, and w_down [E, H, I]); the k gated outputs of a token summed in fp32 in slot order.  With ``aux`` also
    returns each expert's sum of full-softmax probabilities (fp32, differentiable) and its token count (int32).
    ``routing_logits`` [T, E], if given, decides which experts each token takes (the gates still come from this call's
    logits): an fp32 reference then routes exactly like the bf16 run it checks."""
    H = x.shape[-1]
    E = router_weight.shape[0]
    x2 = x.reshape(-1, H)
    T = x2.shape[0]
    logits = F.linear(x2, router_weight).float()
    ids = moe_route_reference(logits if routing_logits is None else routing_logits, top_k)[0]
    gates = torch.softmax(logits.gather(1, ids), dim=-1).to(x.dtype)
    slots = x2.new_zeros(T, top_k, H)
    for e in range(E):
        tok, slot = (ids == e).nonzero(as_tuple=True)
        if tok.numel() == 0:
            continue
        g, u = F.linear(x2[tok], w_gate_up[e]).chunk(2, dim=-1)
        y = F.linear(F.silu(g) * u, w_down[e])
        slots = slots.index_put((tok, slot), y * gates[tok, slot, None])
    out = slots.float().sum(1).to(x.dtype).view(x.shape)
    if not aux:
        return out
    return out, torch.softmax(logits, dim=-1).sum(0), torch.bincount(ids.reshape(-1), minlength=E).to(torch.int32)


class _MoE(torch.autograd.Function):
    """CUDA body of ``moe``: route, permute, gather, grouped gate|up GEMM, SwiGLU, grouped down GEMM, combine.  The backward
    gathers the permuted input again from x rather than keeping it (one more memory-bound pass instead of [capacity, H]
    per layer alive until the backward).  No host synchronisation: every shape follows from (T, E, k)."""

    @staticmethod
    def forward(ctx, x2, logits, w_gate_up, w_down, top_k, aux):
        C = _C()
        ctx.set_materialize_grads(False)
        E = w_gate_up.shape[0]
        ids, gates, probsum = C.moe_route(logits, top_k, aux)
        counts, offsets, fwd, inv, tiles = C.moe_permute(ids, E)
        gu = C.moe_gemm(C.moe_gather(x2, fwd, top_k), w_gate_up, tiles, False)
        h = C.swiglu_fwd(gu)
        y = C.moe_gemm(h, w_down, tiles, False)
        out = C.moe_combine(y, inv, gates)
        ctx.save_for_backward(x2, logits, w_gate_up, w_down, ids, gates, offsets, fwd, inv, tiles, gu, h, y)
        ctx.top_k, ctx.aux = top_k, aux
        if not aux:
            return out
        ctx.mark_non_differentiable(counts)
        return out, probsum, counts

    @staticmethod
    def backward(ctx, dout, dprobsum=None, _dcounts=None):
        C = _C()
        x2, logits, w_gate_up, w_down, ids, gates, offsets, fwd, inv, tiles, gu, h, y = ctx.saved_tensors
        if dout is None:
            dout = torch.zeros_like(x2)
        dy, dgates = C.moe_combine_bwd(dout.to(torch.bfloat16).contiguous(), y, fwd, gates)
        dw_down = C.moe_gemm_wgrad(dy, h, offsets) if ctx.needs_input_grad[3] else None
        dgu = C.swiglu_bwd(C.moe_gemm(dy, w_down, tiles, True), gu)
        dx = dw_gu = None
        if ctx.needs_input_grad[0]:
            dx = C.moe_combine(C.moe_gemm(dgu, w_gate_up, tiles, True), inv, None)
        if ctx.needs_input_grad[2]:
            dw_gu = C.moe_gemm_wgrad(dgu, C.moe_gather(x2, fwd, ctx.top_k), offsets)
        dp = dprobsum.float().contiguous() if ctx.aux and dprobsum is not None else None
        dlogits = C.moe_router_bwd(logits, ids, dgates, dp) if ctx.needs_input_grad[1] else None
        return dx, dlogits, dw_gu, dw_down, None, None


def moe(x: torch.Tensor, router_weight: torch.Tensor, w_gate_up: torch.Tensor, w_down: torch.Tensor, top_k: int,
        aux: bool = False):
    """Sparse mixture-of-experts SwiGLU layer (Hugging Face's ``GraniteMoeMoE``), dropless: x [..., H], router_weight
    [E, H], w_gate_up [E, 2I, H] (rows gate | up), w_down [E, H, I].  Each token goes to its top_k experts by router logit
    (ties to the lower expert), weighted by the softmax over those k logits in fp32 rounded to x's dtype; the k outputs
    are summed in fp32 in slot order.  Returns the output [..., H]; with ``aux=True`` also each expert's sum over tokens
    of the full router softmax (fp32 [E], differentiable: the load-balancing loss) and its token count (int32 [E]).

    On CUDA (bf16; E <= 64 and a multiple of 8, 1 <= top_k <= min(E, 8), H and I multiples of 64, tokens a multiple of
    8, else ``ValueError``): native routing, a stable expert sort into 128-aligned segments, grouped wgmma GEMMs and a
    gather-based combine; deterministic, no atomics and no host synchronisation (CUDA-graph safe).  CPU: ``_moe_reference``."""
    H = x.shape[-1] if x.dim() >= 1 else -1
    E = router_weight.shape[0] if router_weight.dim() == 2 else -1
    if router_weight.dim() != 2 or router_weight.shape[1] != H or w_gate_up.dim() != 3 or w_down.dim() != 3 or \
            w_gate_up.shape[0] != E or w_down.shape[0] != E or w_gate_up.shape[2] != H or w_gate_up.shape[1] % 2 or \
            tuple(w_down.shape[1:]) != (H, w_gate_up.shape[1] // 2):
        raise ValueError(f"moe needs x [..., H], router_weight [E, H], w_gate_up [E, 2I, H] and w_down [E, H, I], got x "
                         f"{tuple(x.shape)}, router {tuple(router_weight.shape)}, gate_up {tuple(w_gate_up.shape)}, down "
                         f"{tuple(w_down.shape)}")
    if not 1 <= top_k <= min(E, MOE_MAX_TOP_K):
        raise ValueError(f"moe needs 1 <= top_k <= min(experts, {MOE_MAX_TOP_K}), got top_k={top_k} with {E} experts")
    if not x.is_cuda:
        return _moe_reference(x, router_weight, w_gate_up, w_down, top_k, aux)
    I = w_down.shape[2]
    T = x.numel() // H
    if any(t.dtype != torch.bfloat16 for t in (x, router_weight, w_gate_up, w_down)):
        raise ValueError(f"moe on CUDA needs bf16 x and weights, got {x.dtype}, {router_weight.dtype}, {w_gate_up.dtype}, {w_down.dtype}")
    if E > MOE_MAX_EXPERTS or E % 8 or H % 64 or I % 64 or T == 0 or T % 8:
        raise ValueError(f"moe on CUDA needs E <= {MOE_MAX_EXPERTS} and a multiple of 8, H and I multiples of 64 and a positive "
                         f"token count that is a multiple of 8, got E={E}, H={H}, I={I}, tokens={T}")
    x2 = x.reshape(T, H).contiguous()
    logits = linear(x2, router_weight)                               # bf16 [T, E] on the wgmma GEMM, as Hugging Face's router
    outs = _MoE.apply(x2, logits, w_gate_up.contiguous(), w_down.contiguous(), int(top_k), bool(aux))
    if not aux:
        return outs.view(x.shape)
    out, probsum, counts = outs
    return out.view(x.shape), probsum, counts


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
# LM head + cross-entropy without the logits (csrc/gemm_wgmma.cu LM epilogues, csrc/loss.cu combine)
# ------------------------------------------------------------------------------------------------
# Vocabulary columns per backward slice: the bf16 logit gradient of one slice, [tokens, LM_LOSS_SLICE], is the largest
# buffer the backward allocates (67 MB at 8192 tokens).  On an H100 (700 W) the Qwen2.5 head backward (8192 x 151936 x 1536)
# took 27.0 - 28.3 ms at 4096, 8192, 16384 and 32768 columns in two runs of `bench/kernel_bench.py --only lmloss`, with no
# width fastest in both, so the narrowest, with the smallest buffer, is used.
LM_LOSS_SLICE = 4096


class _LinearCrossEntropy(torch.autograd.Function):
    """Forward: one GEMM whose epilogue reduces each row's logits per 128-column tile to (max, sum exp), then a fixed-order
    merge to the row log-sum-exp and the mean loss.  Backward, per vocabulary slice: the GEMM again, its epilogue writing
    the bf16 logit gradient, then dh += dlogits . weight[slice] (fp32), dweight[slice] = dlogits^T . hidden and, for a
    trained bias, dbias[slice] = the column sums of dlogits.  The upstream gradient and the valid-row count stay on the
    device (CUDA-graph safe).  Nothing of size [tokens, vocab] is allocated.  ``rows`` (int32 [1] on the device, or None):
    only the leading rows below it carry labels, and every GEMM visits only the 128-row tiles below it."""

    @staticmethod
    def forward(ctx, hidden, weight, targets, bias, ignore_index, rows):
        h2 = hidden.reshape(-1, hidden.shape[-1]).contiguous()
        t = targets.reshape(-1).to(torch.long).contiguous()
        w = weight.contiguous()
        b = bias.detach().contiguous() if bias is not None else None
        loss, lse, row_loss = _C().lm_loss_fwd(h2, w, t, b, int(ignore_index), rows=rows)
        ctx.save_for_backward(h2, w, t, b, lse, row_loss, rows)
        ctx.ignore_index = int(ignore_index)
        ctx.h_shape = hidden.shape
        return loss

    @staticmethod
    def backward(ctx, g):
        h2, w, t, b, lse, row_loss, rows = ctx.saved_tensors
        gs = g.detach().float().reshape(1).contiguous()
        dh, dw, db = _C().lm_loss_bwd(h2, w, t, b, lse, row_loss, gs, ctx.ignore_index, LM_LOSS_SLICE,
                                      ctx.needs_input_grad[0], ctx.needs_input_grad[1], rows=rows,
                                      need_dbias=ctx.needs_input_grad[3])
        return (dh.view(ctx.h_shape) if dh is not None else None), dw, None, db, None, None


class _GatherRows(torch.autograd.Function):
    """out[r] = x[index[r]] for r < count, zero rows after (``compact_rows``' order); the backward scatters the gradient
    back, exactly zero on the other rows of x."""

    @staticmethod
    def forward(ctx, x, index, count):
        ctx.save_for_backward(index, count)
        return _C().gather_rows(x, index, count)

    @staticmethod
    def backward(ctx, g):
        index, count = ctx.saved_tensors
        return _C().scatter_rows(g.contiguous(), index, count), None, None


def compact_rows(targets: torch.Tensor, ignore_index: int = -100, num_classes: Optional[int] = None):
    """The rows that carry a label, first and in their original order: ``(index int32 [T], count int32 [1], compacted
    targets int64 [T])`` for targets [T].  A row is labelled by ``cross_entropy``'s rule: its target is not
    ``ignore_index``, not negative and below ``num_classes`` (no upper bound when None).  ``index`` is a permutation of the
    rows (the unlabelled ones follow, also in order) and the compacted targets hold ``ignore_index`` from ``count`` on.
    On CUDA it runs on the device with no host synchronisation, so ``count`` stays there; the CPU body uses
    ``torch.nonzero``."""
    if targets.dim() != 1 or targets.is_floating_point() or targets.is_complex() or targets.numel() == 0:
        raise ValueError(f"compact_rows needs integer targets [T] with T >= 1, got {targets.dtype} {tuple(targets.shape)}")
    vocab = num_classes if num_classes is not None else torch.iinfo(torch.int64).max
    t = targets.to(torch.long).contiguous()
    if t.is_cuda:
        return _C().compact_rows(t, int(ignore_index), int(vocab))
    valid = (t != ignore_index) & (t >= 0) & (t < vocab)
    index = torch.cat([torch.nonzero(valid)[:, 0], torch.nonzero(~valid)[:, 0]]).to(torch.int32)
    count = valid.sum(dtype=torch.int32).reshape(1)
    out = torch.where(torch.arange(t.numel()) < count, t[index.long()], torch.full_like(t, ignore_index))
    return index, count, out


def _linear_cross_entropy_reference(hidden, weight, targets, bias, ignore_index):
    """CPU body: ``cross_entropy(linear(hidden, weight, bias), targets)`` with the same ignore rule (targets equal to
    ``ignore_index``, negative or >= V are ignored; all ignored gives 0).  Differentiable through autograd."""
    logits = F.linear(hidden.reshape(-1, hidden.shape[-1]), weight, bias).float()
    t = targets.reshape(-1)
    valid = (t != ignore_index) & (t >= 0) & (t < logits.shape[-1])
    picked = logits.gather(1, torch.where(valid, t, 0)[:, None])[:, 0]
    rows = torch.where(valid, torch.logsumexp(logits, -1) - picked, 0.0)
    return rows.sum() / valid.sum().clamp(min=1)


def linear_cross_entropy(hidden: torch.Tensor, weight: torch.Tensor, targets: torch.Tensor, bias: Optional[torch.Tensor] = None,
                         ignore_index: int = -100, sparse: bool = False) -> torch.Tensor:
    """Mean over non-ignored rows of ``cross_entropy(linear(hidden, weight, bias), targets)``: hidden [..., H], weight [V, H],
    bias [V] or None, targets [...] integer.  Targets equal to ``ignore_index``, negative or >= V are ignored; when every row
    is ignored the loss and the gradients are 0.  On CUDA the [tokens, V] logits are never allocated (``_LinearCrossEntropy``):
    bf16 hidden / weight / bias, H and V multiples of 8, else ``ValueError``.  The bias gets a gradient when it requires one
    (a trained decoder bias); a bias without one (GPT-2's padded-vocabulary mask) is a constant.

    ``sparse=True`` scores the labelled rows alone (masked-LM prediction, where most rows are ignored): they are compacted
    to the front (``compact_rows``), the head runs on the tiles that hold them, and the hidden-state gradient is scattered
    back, exactly zero on the other rows.  Same loss and gradients as ``sparse=False``; on CUDA the number of labelled rows
    stays on the device, so the call captures into a CUDA graph that replays on batches with other counts."""
    if hidden.dim() < 1 or weight.dim() != 2 or weight.shape[1] != hidden.shape[-1] or \
            tuple(targets.shape) != tuple(hidden.shape[:-1]) or (bias is not None and tuple(bias.shape) != (weight.shape[0],)):
        raise ValueError(f"linear_cross_entropy needs hidden [..., H], weight [V, H], targets [...] and bias [V], got hidden "
                         f"{tuple(hidden.shape)}, weight {tuple(weight.shape)}, targets {tuple(targets.shape)}, bias "
                         f"{None if bias is None else tuple(bias.shape)}")
    if targets.is_floating_point() or targets.is_complex():
        raise ValueError(f"linear_cross_entropy needs integer targets, got {targets.dtype}")
    V, H = weight.shape
    if sparse and hidden.numel() > 0:
        index, count, targets = compact_rows(targets.reshape(-1), ignore_index, V)
        h2 = hidden.reshape(-1, H)
        if not hidden.is_cuda:
            return _linear_cross_entropy_reference(h2[index.long()], weight, targets, bias, ignore_index)
        hidden, rows = _GatherRows.apply(h2.contiguous(), index, count), count
    else:
        rows = None
    if not hidden.is_cuda:
        return _linear_cross_entropy_reference(hidden, weight, targets, bias, ignore_index)
    if hidden.dtype != torch.bfloat16 or weight.dtype != torch.bfloat16 or (bias is not None and bias.dtype != torch.bfloat16):
        raise ValueError(f"linear_cross_entropy on CUDA needs bf16 hidden, weight and bias, got {hidden.dtype}, {weight.dtype}, "
                         f"{None if bias is None else bias.dtype}")
    if H % 8 or V % 8 or hidden.numel() == 0:
        raise ValueError(f"linear_cross_entropy on CUDA needs H and V multiples of 8 and at least one row, got weight "
                         f"{tuple(weight.shape)}, hidden {tuple(hidden.shape)}")
    return _LinearCrossEntropy.apply(hidden, weight, targets, bias, ignore_index, rows)


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


def layer_norm(x: torch.Tensor, gamma: torch.Tensor, beta: Optional[torch.Tensor], eps: float = 1e-5) -> torch.Tensor:
    """LayerNorm over the last dimension; ``beta=None`` is the bias-free form (ModernBERT's), which on CUDA runs the same
    fused kernel with a zero beta whose gradient is dropped."""
    if x.is_cuda and x.dtype in (torch.float32, torch.bfloat16) and gamma.dtype == x.dtype and x.shape[-1] * 8 <= 96 * 1024:
        return _LayerNormFused.apply(x, gamma, gamma.new_zeros(gamma.shape) if beta is None else beta, eps)
    return F.layer_norm(x, (x.shape[-1],), gamma, beta, eps)


# ------------------------------------------------------------------------------------------------
# Vision Transformer patch embedding (csrc/vit.cu): the images of a batch as documents of one token stream
# ------------------------------------------------------------------------------------------------
def image_token_rows(batch: int, tokens_per_image: int) -> int:
    """Rows of the token stream of `batch` images of `tokens_per_image` tokens each: their count rounded up to a multiple
    of 128, the row multiple of the attention kernels."""
    return -(-batch * tokens_per_image // ATTENTION_SEQ_MULTIPLE) * ATTENTION_SEQ_MULTIPLE


def image_token_bounds(batch: int, tokens_per_image: int, device=None) -> torch.Tensor:
    """Document bounds int32 [1, T, 2] (T = ``image_token_rows``) of `batch` images laid out one after another in one token
    stream: the rows of image b, [b n, (b + 1) n) with n = tokens_per_image, hold (b n, (b + 1) n); the padding rows past
    batch n hold (0, 0).  ``packed_attention(qkv.view(1, T, 3 * hidden), bounds, heads)`` then attends within each image.
    Torch ops on static shapes: no host synchronisation (CUDA-graph safe)."""
    if batch < 1 or tokens_per_image < 1:
        raise ValueError(f"image_token_bounds needs batch >= 1 and tokens_per_image >= 1, got {batch}, {tokens_per_image}")
    T = image_token_rows(batch, tokens_per_image)
    t = torch.arange(T, device=device, dtype=torch.int32)
    start = t - t % tokens_per_image
    real = t < batch * tokens_per_image
    zero = torch.zeros((), device=device, dtype=torch.int32)
    return torch.stack([torch.where(real, start, zero), torch.where(real, start + tokens_per_image, zero)], -1).view(1, T, 2)


def patch_embed_reference(images: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor], class_token: torch.Tensor,
                          pos_embedding: torch.Tensor) -> torch.Tensor:
    """torchvision's ViT input stage (``conv_proj``, flatten, class token, position embedding) laid out as ``patch_embed``'s
    token stream [T, D]: image b's class token at row b (N + 1), its N patches after it, zero rows past B (N + 1).
    Differentiable."""
    B = images.shape[0]
    D, p = weight.shape[0], weight.shape[-1]
    x = F.conv2d(images, weight, bias, stride=p).flatten(2).transpose(1, 2)
    x = torch.cat([class_token.expand(B, -1, -1), x], 1) + pos_embedding
    per = x.shape[1]
    return F.pad(x.reshape(B * per, D), (0, 0, 0, image_token_rows(B, per) - B * per))


def _patch_embed_check(images, weight, bias, class_token, pos_embedding) -> None:
    if images.dim() != 4 or weight.dim() != 4 or weight.shape[1] != images.shape[1] or weight.shape[2] != weight.shape[3]:
        raise ValueError(f"patch_embed needs images [B, C, H, W] and a square weight [D, C, p, p], got {tuple(images.shape)} "
                         f"and {tuple(weight.shape)}")
    B, C, H, W = images.shape
    D, p = weight.shape[0], weight.shape[-1]
    if p % 8 or H % p or W % p or D % 8:
        raise ValueError(f"patch_embed on CUDA needs a patch size p % 8 == 0 that divides H and W, and D % 8 == 0, got p = {p}, "
                         f"image {H}x{W}, D = {D}")
    per = (H // p) * (W // p) + 1
    if class_token.numel() != D or pos_embedding.numel() != per * D or (bias is not None and bias.numel() != D):
        raise ValueError(f"patch_embed needs class_token of {D} elements, pos_embedding [1, {per}, {D}] and bias [{D}], got "
                         f"{tuple(class_token.shape)}, {tuple(pos_embedding.shape)}, {None if bias is None else tuple(bias.shape)}")
    ts = [images, weight, class_token, pos_embedding] + ([bias] if bias is not None else [])
    if any(t.dtype != torch.bfloat16 for t in ts):
        raise ValueError(f"patch_embed on CUDA needs bf16 tensors, got {[t.dtype for t in ts]}")
    if not (images.is_contiguous() or images.is_contiguous(memory_format=torch.channels_last)):
        raise ValueError("patch_embed on CUDA needs contiguous or channels_last images")
    if images.requires_grad and torch.is_grad_enabled():
        raise ValueError("patch_embed gives the images no gradient; pass images that do not require one")


class _PatchAssemble(torch.autograd.Function):
    """GEMM output [T, D] -> tokens: class token + pos[0], patch + pos[1 + i], zero padding rows (csrc/vit.cu).  Backward is
    one launch: the patch rows' gradient (zero at class and padding rows, so the linear's weight and bias gradients sum
    patch rows only) and d pos / d class_token as fixed-order fp32 sums over the images."""

    @staticmethod
    def forward(ctx, y, class_token, pos_embedding, batch):
        ctx.batch, ctx.per = batch, pos_embedding.numel() // y.shape[1]
        ctx.shapes = class_token.shape, pos_embedding.shape
        return _C().vit.patch_assemble(y, class_token.contiguous(), pos_embedding.contiguous(), batch)

    @staticmethod
    def backward(ctx, dy):
        dy = dy.contiguous()
        if dy.data_ptr() % 16:                                    # the kernel reads dy in 16-byte vectors
            dy = dy.clone()
        dpatch, dpos, dcls = _C().vit.patch_embed_bwd(dy, ctx.batch, ctx.per)
        return dpatch, dcls.view(ctx.shapes[0]), dpos.view(ctx.shapes[1]), None


def patch_embed(images: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor], class_token: torch.Tensor,
                pos_embedding: torch.Tensor) -> torch.Tensor:
    """A Vision Transformer's input stage as one token stream: images [B, C, H, W], the patch convolution's weight
    [D, C, p, p] (stride p) and bias [D], class_token [1, 1, D] and pos_embedding [1, N + 1, D] (N = H W / p²; torchvision's
    ``conv_proj``, ``class_token`` and ``encoder.pos_embedding``).  Returns tokens [T, D], T = ``image_token_rows(B, N + 1)``:
    image b's class token (class_token + pos[0]) at row b (N + 1), its patches (patch + pos[1 + i], raster order) after it,
    exact zeros in the padding rows past B (N + 1); ``image_token_bounds(B, N + 1)`` are its attention bounds.

    On CUDA (bf16, contiguous or channels_last images, p % 8 == 0, D % 8 == 0, else ``ValueError``): one kernel writes the
    patch matrix [T, C p²] in token order (zero class and padding rows) in the flattened weight's K order, the wgmma
    ``linear`` runs on all T rows, and one kernel adds the class token and the position embedding.  The gradients of the
    weight, bias, class token and position embedding do not depend on the output gradient at padding rows; the images get
    none.  On CPU: ``patch_embed_reference``."""
    if not images.is_cuda:
        return patch_embed_reference(images, weight, bias, class_token, pos_embedding)
    _patch_embed_check(images, weight, bias, class_token, pos_embedding)
    B, _, H, W = images.shape
    D, p = weight.shape[0], weight.shape[-1]
    per = (H // p) * (W // p) + 1
    patches = _C().vit.patchify(images, p, image_token_rows(B, per))
    y = linear(patches, weight.reshape(D, -1), bias)               # a channels_last weight is copied into (c, ky, kx) order
    return _PatchAssemble.apply(y, class_token, pos_embedding, B)


# ------------------------------------------------------------------------------------------------
# ConvNeXt (csrc/convnext.cu): the depthwise 7x7 convolution on NHWC activations, and the patchify convolutions as gathers
# ------------------------------------------------------------------------------------------------
DWCONV_KERNEL = 7
DWCONV_MAX_CHANNELS = 1024


def depthwise_conv2d_reference(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor]) -> torch.Tensor:
    """``depthwise_conv2d`` through ``F.conv2d(groups=C)`` on the NCHW view of x [B, H, W, C]; returns [B, H, W, C]."""
    return F.conv2d(x.permute(0, 3, 1, 2), weight, bias, padding=DWCONV_KERNEL // 2, groups=x.shape[-1]).permute(0, 2, 3, 1)


def _depthwise_check(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor]) -> None:
    C = x.shape[-1] if x.dim() == 4 else -1
    if x.dim() != 4 or tuple(weight.shape) != (C, 1, DWCONV_KERNEL, DWCONV_KERNEL) or bias is None or tuple(bias.shape) != (C,):
        raise ValueError(f"depthwise_conv2d needs x [B, H, W, C], weight [C, 1, 7, 7] and bias [C], got {tuple(x.shape)}, "
                         f"{tuple(weight.shape)} and {None if bias is None else tuple(bias.shape)}")
    if C < 8 or C > DWCONV_MAX_CHANNELS or C % 8 or x.numel() == 0:
        raise ValueError(f"depthwise_conv2d on CUDA needs 8 <= C <= {DWCONV_MAX_CHANNELS}, C % 8 == 0 and a non-empty x, got "
                         f"{tuple(x.shape)}")
    if weight.dtype != torch.bfloat16 or bias.dtype != torch.bfloat16:
        raise ValueError(f"depthwise_conv2d on CUDA needs bf16 x, weight and bias, got {x.dtype}, {weight.dtype}, {bias.dtype}")


def _aligned16(t: torch.Tensor) -> torch.Tensor:
    t = t.contiguous()
    return t.clone() if t.data_ptr() % 16 else t                     # the kernels move 16-byte vectors


class _DepthwiseConv2d(torch.autograd.Function):
    """x [B, H, W, C] bf16 -> y (csrc/convnext.cu).  Backward: the data gradient is the forward kernel flipped, and one
    pass plus an in-order finish gives the weight and bias gradients."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        C = x.shape[-1]
        w = weight.reshape(C, DWCONV_KERNEL * DWCONV_KERNEL).contiguous()     # free for a contiguous or channels_last weight
        ctx.save_for_backward(x, w)
        ctx.weight_shape = weight.shape
        return _C().convnext.dwconv_fwd(x, w, bias.contiguous())

    @staticmethod
    def backward(ctx, dy):
        x, w = ctx.saved_tensors
        dy = _aligned16(dy)
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = _C().convnext.dwconv_dgrad(dy, w)
        if ctx.needs_input_grad[1] or ctx.needs_input_grad[2]:
            dw, db = _C().convnext.dwconv_wgrad(dy, x)
            dw = dw.view(ctx.weight_shape)
        return dx, dw, db


def depthwise_conv2d(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor]) -> torch.Tensor:
    """ConvNeXt's depthwise convolution (kernel 7, stride 1, padding 3, one filter per channel) on NHWC activations:
    x [B, H, W, C], weight [C, 1, 7, 7] (contiguous or channels_last), bias [C] -> y [B, H, W, C].

    CUDA with bf16 tensors runs the native kernels: fp32 sums in a fixed order and one bf16 rounding, bitwise repeatable,
    no host synchronisation; it needs 8 <= C <= 1024 with C % 8 == 0 and a bias, else ``ValueError``.  The weight and bias
    gradients do not depend on the output gradient anywhere but at real pixels.  Everything else runs
    ``depthwise_conv2d_reference``."""
    if not (x.is_cuda and x.dtype == torch.bfloat16):
        return depthwise_conv2d_reference(x, weight, bias)
    _depthwise_check(x, weight, bias)
    return _DepthwiseConv2d.apply(_aligned16(x), weight, bias)


def patchify_nhwc(x: torch.Tensor, patch: int) -> torch.Tensor:
    """The rows of a patch convolution (kernel = stride = ``patch``, no padding) over x [B, H, W, C] (any strides): one
    row per output pixel in raster order, its p² C inputs in (ky, kx, c) order, [B (H / p) (W / p), p² C].  Times
    ``weight.permute(0, 2, 3, 1).reshape(D, -1)`` this is the convolution.  A torch permutation copy; its backward is the
    inverse permutation."""
    B, H, W, C = x.shape
    if H % patch or W % patch:
        raise ValueError(f"patchify_nhwc needs H and W divisible by {patch}, got {tuple(x.shape)}")
    return x.reshape(B, H // patch, patch, W // patch, patch, C).permute(0, 1, 3, 2, 4, 5).reshape(-1, patch * patch * C)


# ------------------------------------------------------------------------------------------------
# Swin Transformer (csrc/swin.cu): shifted-window attention on raster token rows
# ------------------------------------------------------------------------------------------------
SWIN_WINDOW = 7
SWIN_HEAD_DIM = 32
SWIN_MASK = -100.0                   # torchvision's value between shift regions, not -inf
SWIN_V2_WINDOW = 8


def swin_relative_position_index(device=None, window: int = SWIN_WINDOW) -> torch.Tensor:
    """int64 [w^4] for window w (7 by default): entry w^2 i + j is (yi - yj + w - 1) (2w - 1) + (xi - xj + w - 1) for the
    window's tokens i = w yi + xi and j = w yj + xj, the table row of their relative position (torchvision's
    ``relative_position_index``)."""
    t = torch.arange(window * window, device=device)
    y, x = t // window, t % window
    return ((y[:, None] - y[None, :] + window - 1) * (2 * window - 1) + (x[:, None] - x[None, :] + window - 1)).flatten()


def swin_v2_relative_coords_table(window: int = SWIN_V2_WINDOW, device=None) -> torch.Tensor:
    """fp32 [1, 2w - 1, 2w - 1, 2]: entry (dy + w - 1, dx + w - 1) is f(8 dy / (w - 1)), f(8 dx / (w - 1)) with
    f(t) = sign(t) log2(|t| + 1) / 3, the input of Swin V2's continuous position bias MLP (torchvision's
    ``relative_coords_table``)."""
    r = torch.arange(-(window - 1), window, dtype=torch.float32, device=device)
    t = torch.stack(torch.meshgrid([r, r], indexing="ij")).permute(1, 2, 0).contiguous().unsqueeze(0)
    t = t / (window - 1) * 8
    return torch.sign(t) * torch.log2(torch.abs(t) + 1.0) / 3.0


def _shift_pair(shift, window: int = SWIN_WINDOW) -> tuple[int, int]:
    sy, sx = (shift, shift) if isinstance(shift, int) else tuple(shift)
    if not (0 <= sy < window and 0 <= sx < window):
        raise ValueError(f"window_attention needs 0 <= shift < {window}, got {shift}")
    return int(sy), int(sx)


def _shift_regions(n: int, shift: int, device, window: int = SWIN_WINDOW) -> torch.Tensor:
    """The shift region of each shifted coordinate 0 .. n-1: [0, n-w), [n-w, n-shift), [n-shift, n); one region at shift 0."""
    c = torch.arange(n, device=device)
    if shift == 0:
        return torch.zeros_like(c)
    return (c >= n - window).long() + (c >= n - shift).long()


def _window_attention_torch(qkv, table, scale, batch, height, width, heads, shift, window, who):
    """Both references: V1's scaled dot product when ``scale`` is None, else V2's cosine scores times scale [heads]."""
    sy, sx = _shift_pair(shift, window)
    B, H, W, w = batch, height, width, window
    if H % w or W % w or qkv.dim() != 2 or qkv.shape[0] != B * H * W or qkv.shape[1] % (3 * heads):
        raise ValueError(f"{who} needs qkv [B H W, 3C] with H and W multiples of {w}, got {tuple(qkv.shape)} "
                         f"for {B} x {H} x {W} and {heads} heads")
    dtype = qkv.dtype if qkv.dtype in (torch.float32, torch.float64) else torch.float32
    C = qkv.shape[1] // 3
    d = C // heads
    x = qkv.to(dtype).view(B, H, W, 3 * C)
    if sy or sx:
        x = torch.roll(x, shifts=(-sy, -sx), dims=(1, 2))
    n = (H // w) * (W // w)
    x = x.view(B, H // w, w, W // w, w, 3 * C).permute(0, 1, 3, 2, 4, 5).reshape(B * n, w * w, 3, heads, d).permute(2, 0, 3, 1, 4)
    q, k, v = x[0], x[1], x[2]
    bias = table.to(dtype)[swin_relative_position_index(table.device, w)].view(w * w, w * w, heads).permute(2, 0, 1)
    if scale is None:
        attn = (q * d ** -0.5) @ k.transpose(-2, -1) + bias
    else:
        attn = (F.normalize(q, dim=-1) @ F.normalize(k, dim=-1).transpose(-2, -1)) * scale.to(dtype).view(heads, 1, 1) + bias
    if sy or sx:
        region = _shift_regions(H, sy, qkv.device, w)[:, None] * 3 + _shift_regions(W, sx, qkv.device, w)[None, :]
        region = region.view(H // w, w, W // w, w).permute(0, 2, 1, 3).reshape(n, w * w)
        mask = torch.where(region[:, :, None] != region[:, None, :], SWIN_MASK, 0.0).to(dtype)
        attn = (attn.view(B, n, heads, w * w, w * w) + mask[None, :, None]).view(B * n, heads, w * w, w * w)
    o = (attn.softmax(-1) @ v).transpose(1, 2).reshape(B, H // w, W // w, w, w, C).permute(0, 1, 3, 2, 4, 5).reshape(B, H, W, C)
    if sy or sx:
        o = torch.roll(o, shifts=(sy, sx), dims=(1, 2))
    return o.reshape(B * H * W, C).to(qkv.dtype)


def window_attention_reference(qkv: torch.Tensor, table: torch.Tensor, batch: int, height: int, width: int, heads: int,
                               shift) -> torch.Tensor:
    """``window_attention`` in torch, fp32 for bf16 input: roll the map by -shift, partition it into 7 x 7 windows, dense
    scores with the relative position bias and the -100 region mask, softmax, and the reverse partition and roll.  Needs
    height and width multiples of 7; any head dim."""
    return _window_attention_torch(qkv, table, None, batch, height, width, heads, shift, SWIN_WINDOW, "window_attention_reference")


class _WindowAttention(torch.autograd.Function):
    """qkv [B H W, 3C] bf16, table fp32 [169, heads] -> o [B H W, C] (csrc/swin.cu).  Backward: one kernel per window for
    dqkv and the window's table partials, and an in-order finish for dtable."""

    @staticmethod
    def forward(ctx, qkv, table, batch, height, width, sy, sx):
        o, lse = _C().swin.attention_fwd(qkv, table, batch, height, width, sy, sx)
        ctx.save_for_backward(qkv, table, o, lse)
        ctx.geometry = (batch, height, width, sy, sx)
        return o

    @staticmethod
    def backward(ctx, dout):
        qkv, table, o, lse = ctx.saved_tensors
        dqkv, dtable = _C().swin.attention_bwd(_aligned16(dout), qkv, o, lse, table, *ctx.geometry)
        return dqkv, dtable, None, None, None, None, None


def window_attention(qkv: torch.Tensor, table: torch.Tensor, batch: int, height: int, width: int, heads: int, shift) -> torch.Tensor:
    """Swin's (shifted) window attention on raster token rows: qkv [B H W, 3C] with rows in (b, y, x) order and columns
    [q heads | k heads | v heads] (torchvision's reshape order), table [169, heads] -> [B H W, C].  Window 7; ``shift`` is
    an int or a (y, x) pair in [0, 7).

    The token at (y, x) sits at shifted coordinates y' = (y - sy) mod H, x' = (x - sx) mod W, in window (y' / 7, x' / 7)
    at local index i = 7 (y' % 7) + x' % 7, and scores its window's tokens j with
    d^-0.5 q_i . k_j + table[(yi - yj + 6) 13 + (xi - xj + 6), h] - 100 [i and j lie in different shift regions]; the
    regions are [0, H-7), [H-7, H-sy), [H-sy, H) along y' (one region when sy = 0) and the same along x'.  Each token's
    output lands on its own row, so no roll, partition or permute is materialised.

    CUDA bf16 input runs the native kernels (head dim 32; H and W multiples of 7; else ``ValueError``): fp32 softmax and
    sums, bitwise repeatable, no host synchronisation, the table gradient summed in a fixed order and rounded once to the
    table's dtype.  Everything else runs ``window_attention_reference``."""
    sy, sx = _shift_pair(shift)
    if not (qkv.is_cuda and qkv.dtype == torch.bfloat16):
        return window_attention_reference(qkv, table, batch, height, width, heads, (sy, sx))
    rows = batch * height * width
    if qkv.dim() != 2 or qkv.shape[0] != rows or qkv.shape[1] != 3 * SWIN_HEAD_DIM * heads or tuple(table.shape) != (169, heads):
        raise ValueError(f"window_attention on CUDA needs qkv [B H W, 96 heads] (head dim {SWIN_HEAD_DIM}) and table [169, heads], "
                         f"got {tuple(qkv.shape)} and {tuple(table.shape)} for {batch} x {height} x {width} and {heads} heads")
    if height % SWIN_WINDOW or width % SWIN_WINDOW or min(batch, height, width) < 1:
        raise ValueError(f"window_attention on CUDA needs H and W positive multiples of {SWIN_WINDOW}, got {height} x {width}")
    return _WindowAttention.apply(_aligned16(qkv), table.float().contiguous(), batch, height, width, sy, sx)


def window_attention_v2_reference(qkv: torch.Tensor, table: torch.Tensor, scale: torch.Tensor, batch: int, height: int, width: int,
                                  heads: int, shift) -> torch.Tensor:
    """``window_attention_v2`` in torch, fp32 for bf16 input: as ``window_attention_reference`` at window 8, with the
    scores scale_h cos(q_i, k_j) (``F.normalize``, eps 1e-12) in place of d^-0.5 q_i . k_j.  Needs height and width
    multiples of 8; any head dim."""
    return _window_attention_torch(qkv, table, scale, batch, height, width, heads, shift, SWIN_V2_WINDOW, "window_attention_v2_reference")


class _WindowAttentionV2(torch.autograd.Function):
    """qkv [B H W, 3C] bf16, table fp32 [225, heads], scale fp32 [heads] -> o [B H W, C] (csrc/swin.cu).  Backward: one
    kernel per window for dqkv and the window's table and scale partials, and an in-order finish for dtable and dscale."""

    @staticmethod
    def forward(ctx, qkv, table, scale, batch, height, width, sy, sx):
        o, lse = _C().swin_v2.attention_fwd(qkv, table, scale, batch, height, width, sy, sx)
        ctx.save_for_backward(qkv, table, scale, o, lse)
        ctx.geometry = (batch, height, width, sy, sx)
        return o

    @staticmethod
    def backward(ctx, dout):
        qkv, table, scale, o, lse = ctx.saved_tensors
        dqkv, dtable, dscale = _C().swin_v2.attention_bwd(_aligned16(dout), qkv, o, lse, table, scale, *ctx.geometry)
        return dqkv, dtable, dscale, None, None, None, None, None


def window_attention_v2(qkv: torch.Tensor, table: torch.Tensor, scale: torch.Tensor, batch: int, height: int, width: int, heads: int,
                        shift) -> torch.Tensor:
    """Swin V2's (shifted) cosine window attention on raster token rows: qkv [B H W, 3C] as in ``window_attention``,
    table [225, heads] (torchvision's ``16 sigmoid(cpb_mlp(relative_coords_table))``), scale [heads]
    (``exp(min(logit_scale, log 100))``) -> [B H W, C].  Window 8; ``shift`` is an int or a (y, x) pair in [0, 8).

    Token i scores its window's tokens j with scale_h cos(q_i, k_j) + table[(yi - yj + 7) 15 + (xi - xj + 7), h] - 100
    [i and j lie in different shift regions], cos the dot product of the rows divided by max(norm, 1e-12); windows and
    regions are ``window_attention``'s with 8 in place of 7.

    CUDA bf16 input runs the native kernels (head dim 32; H and W multiples of 8; else ``ValueError``): the normalised
    q and k rounded once to bf16, fp32 softmax and sums, bitwise repeatable, no host synchronisation, the table and scale
    gradients summed in a fixed order and rounded once to their dtype.  Everything else runs
    ``window_attention_v2_reference``."""
    sy, sx = _shift_pair(shift, SWIN_V2_WINDOW)
    if not (qkv.is_cuda and qkv.dtype == torch.bfloat16):
        return window_attention_v2_reference(qkv, table, scale, batch, height, width, heads, (sy, sx))
    rows = batch * height * width
    if (qkv.dim() != 2 or qkv.shape[0] != rows or qkv.shape[1] != 3 * SWIN_HEAD_DIM * heads or tuple(table.shape) != (225, heads)
            or tuple(scale.shape) != (heads,)):
        raise ValueError(f"window_attention_v2 on CUDA needs qkv [B H W, 96 heads] (head dim {SWIN_HEAD_DIM}), table [225, heads] "
                         f"and scale [heads], got {tuple(qkv.shape)}, {tuple(table.shape)} and {tuple(scale.shape)} for "
                         f"{batch} x {height} x {width} and {heads} heads")
    if height % SWIN_V2_WINDOW or width % SWIN_V2_WINDOW or min(batch, height, width) < 1:
        raise ValueError(f"window_attention_v2 on CUDA needs H and W positive multiples of {SWIN_V2_WINDOW}, got {height} x {width}")
    return _WindowAttentionV2.apply(_aligned16(qkv), table.float().contiguous(), scale.float().contiguous(), batch, height, width, sy, sx)


# ------------------------------------------------------------------------------------------------
# Mamba (csrc/mamba.cu): causal depthwise conv1d + SiLU and the selective scan on token rows, reset at document starts
# ------------------------------------------------------------------------------------------------
MAMBA_CONV_WIDTH = 4
MAMBA_STATE = 16
MAMBA_SOFTPLUS_THRESHOLD = 20.0      # torch's softplus threshold


def _ref_dtype(t: torch.Tensor):
    return torch.float64 if t.dtype == torch.float64 else torch.float32


def _mamba_positions(bounds: torch.Tensor, device):
    """(real [B, S], start [B, S] long, reset [B, S]) from document bounds: a position is real when start < end, and the
    state resets at a document's first position."""
    b = bounds.to(device=device, dtype=torch.long)
    S = b.shape[1]
    pos = torch.arange(S, device=device)
    real = b[..., 0] < b[..., 1]
    start = b[..., 0].clamp(min=0)
    return real, start, real & ((start >= pos) | (pos == 0))


def causal_conv1d_reference(xz: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor, bounds: torch.Tensor) -> torch.Tensor:
    """``causal_conv1d`` in torch, fp32 (fp64 for fp64 input): u[t] = silu(bias + sum_j w[:, j] x[t - 3 + j]) with x the first
    half of xz [B, S, 2E], taps before the document start reading zero and padding positions giving zero.  Differentiable."""
    dtype = _ref_dtype(xz)
    B, S, E2 = xz.shape
    E = E2 // 2
    x = xz[..., :E].to(dtype)
    w = weight.reshape(E, MAMBA_CONV_WIDTH).to(dtype)
    real, start, _ = _mamba_positions(bounds, xz.device)
    pos = torch.arange(S, device=xz.device)
    pre = bias.to(dtype).expand(B, S, E)
    for j in range(MAMBA_CONV_WIDTH):
        shift = MAMBA_CONV_WIDTH - 1 - j
        xs = F.pad(x, (0, 0, shift, 0))[:, :S]
        keep = (pos - shift >= start) & real
        pre = pre + w[:, j] * torch.where(keep[..., None], xs, torch.zeros_like(xs))
    return torch.where(real[..., None], F.silu(pre), torch.zeros_like(pre)).to(xz.dtype)


def selective_scan_reference(u: torch.Tensor, delta_raw: torch.Tensor, xbc: torch.Tensor, xz: torch.Tensor, A_log: torch.Tensor,
                             D: torch.Tensor, dt_bias: torch.Tensor, bounds: torch.Tensor) -> torch.Tensor:
    """``selective_scan`` in torch, fp32 (fp64 for fp64 input), a loop over the sequence as in transformers'
    ``MambaMixer.slow_forward`` with the state reset at each document start and zero output at padding.  Differentiable."""
    dtype = _ref_dtype(u)
    B, S, E = u.shape
    N = MAMBA_STATE
    R = xbc.shape[-1] - 2 * N
    uu, z = u.to(dtype), xz[..., E:].to(dtype)
    Bm, Cm = xbc[..., R:R + N].to(dtype), xbc[..., R + N:].to(dtype)
    delta = F.softplus(delta_raw.to(dtype) + dt_bias.to(dtype), threshold=MAMBA_SOFTPLUS_THRESHOLD)
    A = -torch.exp(A_log.to(dtype))
    real, _, reset = _mamba_positions(bounds, u.device)
    h = torch.zeros(B, E, N, dtype=dtype, device=u.device)
    ys = []
    for t in range(S):
        dA = torch.exp(delta[:, t, :, None] * A)
        h = torch.where(reset[:, t, None, None], torch.zeros_like(h), dA * h) + delta[:, t, :, None] * Bm[:, t, None, :] * uu[:, t, :, None]
        h = torch.where(real[:, t, None, None], h, torch.zeros_like(h))
        ys.append((h * Cm[:, t, None, :]).sum(-1))
    y = (torch.stack(ys, 1) + uu * D.to(dtype)) * F.silu(z)
    return torch.where(real[..., None], y, torch.zeros_like(y)).to(u.dtype)


class MambaGradLink:
    """Hands the [T, 2E] gradient buffer of in_proj's output from ``selective_scan``'s backward, which writes its z half,
    to ``causal_conv1d``'s backward, which writes its x half and returns it whole: no zero fill, no add, no concatenation.
    Pass one fresh link to both ops of a mixer; the scan's backward always runs first (its input u is the conv's output)."""

    def __init__(self):
        self.dxz = None


def _mamba_check(who: str, xz: torch.Tensor, bounds: torch.Tensor) -> None:
    if xz.dim() != 3 or tuple(bounds.shape) != (xz.shape[0], xz.shape[1], 2) or bounds.is_floating_point() or bounds.is_complex():
        raise ValueError(f"{who} needs xz [B, S, 2E] and integer bounds [B, S, 2], got {tuple(xz.shape)} and {bounds.dtype} "
                         f"{tuple(bounds.shape)}")
    if xz.shape[-1] % 16 or xz.shape[-1] == 0:
        raise ValueError(f"{who} needs E = xz.shape[-1] / 2 a positive multiple of 8, got xz {tuple(xz.shape)}")


def _mamba_native(who: str, *ts: torch.Tensor) -> bool:
    """True for CUDA bf16 activations (the native kernels), False for CPU ones or CUDA fp32 / fp64 ones (the reference);
    any other CUDA dtype, or a mix, raises ``ValueError`` rather than falling back to the reference's loop."""
    if not any(t.is_cuda for t in ts):
        return False
    dtypes = {t.dtype for t in ts}
    if all(t.is_cuda for t in ts) and dtypes == {torch.bfloat16}:
        return True
    if all(t.is_cuda for t in ts) and dtypes <= {torch.float32, torch.float64}:
        return False
    raise ValueError(f"{who} on CUDA needs bf16 activations (the native kernels) or fp32 / fp64 ones (the reference), got "
                     f"{[str(t.dtype) for t in ts]} on {[str(t.device) for t in ts]}")


def _rows(t: torch.Tensor) -> torch.Tensor:
    return _aligned16(t.reshape(-1, t.shape[-1]))


class _CausalConv1d(torch.autograd.Function):
    """xz [B, S, 2E] bf16 -> u [B, S, E] (csrc/mamba.cu).  Backward: dx into the x half of the link's buffer (or a new one
    with a zero z half), fp32 weight and bias gradients summed in a fixed order."""

    @staticmethod
    def forward(ctx, xz, weight, bias, bounds, link):
        B, S, E2 = xz.shape
        x2, w, b = _rows(xz), weight.reshape(E2 // 2, MAMBA_CONV_WIDTH).float().contiguous(), bias.float().contiguous()
        bd = _aligned16(bounds.to(torch.int32))                      # the kernels read (start, end) as int2
        ctx.save_for_backward(x2, w, b, bd)
        ctx.link, ctx.dtypes, ctx.weight_shape = link, (weight.dtype, bias.dtype), weight.shape
        return _C().mamba.conv_fwd(x2, w, b, bd).view(B, S, E2 // 2)

    @staticmethod
    def backward(ctx, du):
        x2, w, b, bd = ctx.saved_tensors
        link = ctx.link
        given = link.dxz if link is not None else None
        dxz, dw, db = _C().mamba.conv_bwd(_rows(du), x2, w, b, bd, given)
        if given is None:
            dxz[:, dxz.shape[1] // 2:].zero_()
        else:
            link.dxz = None
        return (dxz.view(*du.shape[:2], -1), dw.view(ctx.weight_shape).to(ctx.dtypes[0]), db.to(ctx.dtypes[1]), None, None)


def causal_conv1d(xz: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor, bounds: torch.Tensor,
                  link: Optional[MambaGradLink] = None) -> torch.Tensor:
    """Mamba's causal depthwise convolution of width 4 with SiLU over the x half of in_proj's output xz [B, S, 2E]:
    u[t] = silu(bias + sum_j weight[:, 0, j] x[t - 3 + j]), weight [E, 1, 4], bias [E].  Taps before the document start
    of ``bounds`` (int32 [B, S, 2], ``document_bounds``) read zero, and padding positions (start == end) give zero.

    CUDA bf16 xz runs the native kernels (E % 8 == 0, else ``ValueError``): fp32 sums with one bf16 rounding, bitwise
    repeatable, no host synchronisation; its data gradient lands in the x half of the [B, S, 2E] gradient, whose z half
    ``selective_scan`` fills when both get the same ``link``.  CPU input, and CUDA fp32 or fp64 input, run
    ``causal_conv1d_reference``; CUDA input of any other dtype raises ``ValueError``."""
    _mamba_check("causal_conv1d", xz, bounds)
    E = xz.shape[-1] // 2
    if tuple(weight.shape) != (E, 1, MAMBA_CONV_WIDTH) or tuple(bias.shape) != (E,):
        raise ValueError(f"causal_conv1d needs weight [E, 1, 4] and bias [E] for E = {E}, got {tuple(weight.shape)} and {tuple(bias.shape)}")
    if not _mamba_native("causal_conv1d", xz):
        return causal_conv1d_reference(xz, weight, bias, bounds)
    return _CausalConv1d.apply(xz, weight, bias, bounds, link)


class _SelectiveScan(torch.autograd.Function):
    """(u, delta_raw [B, S, E], xbc [B, S, R + 32], xz [B, S, 2E]) bf16 -> y [B, S, E] (csrc/mamba.cu); each chunk's fp32
    start state is kept for the backward."""

    @staticmethod
    def forward(ctx, u, delta_raw, xbc, xz, A_log, D, dt_bias, bounds, link):
        B, S, E = u.shape
        ins = [_rows(u), _rows(delta_raw), _rows(xbc), _rows(xz), A_log.float().contiguous(), D.float().contiguous(),
               dt_bias.float().contiguous(), _aligned16(bounds.to(torch.int32))]
        y, hst, sumd = _C().mamba.scan_fwd(*ins)
        ctx.save_for_backward(*ins, hst, sumd)
        ctx.link, ctx.dtypes, ctx.shapes = link, (A_log.dtype, D.dtype, dt_bias.dtype), (u.shape, xbc.shape, xz.shape)
        return y.view(B, S, E)

    @staticmethod
    def backward(ctx, dy):
        du, ddraw, dxbc, dxz, dA_log, dD, dbias = _C().mamba.scan_bwd(_rows(dy), *ctx.saved_tensors)
        ushape, xbcshape, xzshape = ctx.shapes
        if ctx.link is not None:
            ctx.link.dxz, dxz = dxz, None
        else:
            dxz[:, :xzshape[-1] // 2].zero_()
            dxz = dxz.view(xzshape)
        tA, tD, tb = ctx.dtypes
        return (du.view(ushape), ddraw.view(ushape), dxbc.view(xbcshape), dxz, dA_log.to(tA), dD.to(tD), dbias.to(tb), None, None)


def selective_scan(u: torch.Tensor, delta_raw: torch.Tensor, xbc: torch.Tensor, xz: torch.Tensor, A_log: torch.Tensor, D: torch.Tensor,
                   dt_bias: torch.Tensor, bounds: torch.Tensor, link: Optional[MambaGradLink] = None) -> torch.Tensor:
    """Mamba-1's selective scan with the state reset at every document start: per row, channel e and state n,
    delta = softplus(delta_raw + dt_bias) (threshold 20), A = -exp(A_log),
    h_t = exp(delta_t A) h_{t-1} + delta_t B_t u_t with h = 0 before each document, y_t = (C_t . h_t + D u_t) silu(z_t).
    u and delta_raw [B, S, E]; xbc [B, S, R + 32] is x_proj's output dt | B | C (B and C read in place); z is the second
    half of xz [B, S, 2E]; A_log [E, 16]; D and dt_bias [E]; bounds int32 [B, S, 2] (``document_bounds``).  Padding
    positions give y = 0 and zero gradients.

    CUDA bf16 activations run the native chunked scan (E % 8 == 0 and N = 16, else ``ValueError``): the state is fp32
    throughout, gradients are summed in a fixed order (bitwise repeatable), nothing is read back to the host.  The
    gradient of xz has its z half only; with a ``link`` shared with ``causal_conv1d`` the conv's backward completes and
    returns it.  CPU activations, and CUDA fp32 or fp64 ones, run ``selective_scan_reference``; CUDA activations of
    any other dtype, or of mixed dtypes, raise ``ValueError``."""
    _mamba_check("selective_scan", xz, bounds)
    B, S, E2 = xz.shape
    E = E2 // 2
    if tuple(u.shape) != (B, S, E) or tuple(delta_raw.shape) != (B, S, E) or xbc.dim() != 3 or tuple(xbc.shape[:2]) != (B, S) \
            or xbc.shape[-1] < 2 * MAMBA_STATE:
        raise ValueError(f"selective_scan needs u and delta_raw [B, S, E] = [{B}, {S}, {E}] and xbc [B, S, R + 32], got "
                         f"{tuple(u.shape)}, {tuple(delta_raw.shape)} and {tuple(xbc.shape)}")
    if tuple(A_log.shape) != (E, MAMBA_STATE) or tuple(D.shape) != (E,) or tuple(dt_bias.shape) != (E,):
        raise ValueError(f"selective_scan needs A_log [E, 16] and D, dt_bias [E] for E = {E}, got {tuple(A_log.shape)}, "
                         f"{tuple(D.shape)} and {tuple(dt_bias.shape)}")
    if not _mamba_native("selective_scan", u, delta_raw, xbc, xz):
        return selective_scan_reference(u, delta_raw, xbc, xz, A_log, D, dt_bias, bounds)
    return _SelectiveScan.apply(u, delta_raw, xbc, xz, A_log, D, dt_bias, bounds, link)


# ------------------------------------------------------------------------------------------------
# Mamba-2 (csrc/mamba2.cu, the conv in csrc/mamba.cu, the gated norm in csrc/layernorm.cu): the causal conv over the xBC
# column window of in_proj's output, the chunked SSD scan and the gated RMSNorm on token rows, reset at document starts
# ------------------------------------------------------------------------------------------------
MAMBA2_HEAD_DIM = 64
MAMBA2_STATE = 128
MAMBA2_CHUNK = 64        # rows per chunk of the SSD (the result does not depend on it in exact arithmetic)


class Mamba2GradLink:
    """Hands one [B, S, W] gradient buffer of in_proj's output zxbcdt between the backwards of a Mamba-2 mixer: the gated
    norm writes its z columns, ``ssd_scan`` its dt columns, and ``causal_conv1d_window`` its xBC columns and returns it
    whole: no zero fill, no add, no concatenation.  Build one per mixer call from zxbcdt and pass it to all three ops; the
    conv's backward runs last (its output feeds the scan, whose output feeds the norm)."""

    def __init__(self, zxbcdt: torch.Tensor):
        self.shape, self.like = tuple(zxbcdt.shape), zxbcdt
        self.base = zxbcdt.data_ptr()
        self.buffer = None

    def window(self, view: torch.Tensor) -> torch.Tensor:
        """The columns of the gradient buffer under ``view`` (a column window of zxbcdt), allocating the buffer first."""
        col = (view.data_ptr() - self.base) // view.element_size()
        if self.buffer is None:
            self.buffer = torch.empty(self.shape, dtype=self.like.dtype, device=self.like.device)
            self.like = None
        return self.buffer[..., col:col + view.shape[-1]]


def _row_view(t: torch.Tensor) -> torch.Tensor:
    """[..., C] -> [T, C] read in place when its rows have unit column stride, a pitch that is a multiple of 8 and a 16-byte
    aligned start (a column window of a contiguous tensor), else a contiguous copy."""
    r = t.reshape(-1, t.shape[-1])
    if r.stride(-1) != 1 or r.stride(0) % 8 or r.stride(0) < r.shape[1] or r.data_ptr() % 16:
        r = r.contiguous()
        if r.data_ptr() % 16:
            r = r.clone()
    return r


def _mamba2_check_rows(who: str, x: torch.Tensor, bounds: torch.Tensor) -> None:
    if x.dim() != 3 or tuple(bounds.shape) != (x.shape[0], x.shape[1], 2) or bounds.is_floating_point() or bounds.is_complex():
        raise ValueError(f"{who} needs activations [B, S, *] and integer bounds [B, S, 2], got {tuple(x.shape)} and {bounds.dtype} "
                         f"{tuple(bounds.shape)}")


def causal_conv1d_window_reference(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor, bounds: torch.Tensor,
                                   col: int = 0) -> torch.Tensor:
    """``causal_conv1d_window`` in torch, fp32 (fp64 for fp64 input): u[t] = silu(bias + sum_j w[:, j] x[t - 3 + j]) over the
    columns [col, col + C) of x [B, S, W], taps before the document start reading zero and padding positions giving zero.
    Differentiable."""
    dtype = _ref_dtype(x)
    B, S, _ = x.shape
    C = weight.shape[0]
    xs0 = x[..., col:col + C].to(dtype)
    w = weight.reshape(C, MAMBA_CONV_WIDTH).to(dtype)
    real, start, _ = _mamba_positions(bounds, x.device)
    pos = torch.arange(S, device=x.device)
    pre = bias.to(dtype).expand(B, S, C)
    for j in range(MAMBA_CONV_WIDTH):
        shift = MAMBA_CONV_WIDTH - 1 - j
        xs = F.pad(xs0, (0, 0, shift, 0))[:, :S]
        keep = (pos - shift >= start) & real
        pre = pre + w[:, j] * torch.where(keep[..., None], xs, torch.zeros_like(xs))
    return torch.where(real[..., None], F.silu(pre), torch.zeros_like(pre)).to(x.dtype)


class _CausalConv1dWindow(torch.autograd.Function):
    """zxbcdt [B, S, W] bf16 -> u [B, S, C] from the columns [col, col + C) (csrc/mamba.cu).  Backward: dx into those
    columns of the link's buffer, which it returns whole (or of a new buffer with zeros elsewhere); fp32 weight and bias
    gradients summed in a fixed order."""

    @staticmethod
    def forward(ctx, x, weight, bias, bounds, col, link):
        B, S, W = x.shape
        C = weight.shape[0]
        xw = _row_view(x[..., col:col + C])
        w, b = weight.reshape(C, MAMBA_CONV_WIDTH).float().contiguous(), bias.float().contiguous()
        bd = _aligned16(bounds.to(torch.int32))                      # the kernels read (start, end) as int2
        ctx.save_for_backward(x, xw, w, b, bd)
        ctx.link, ctx.col, ctx.dtypes, ctx.weight_shape = link, col, (weight.dtype, bias.dtype), weight.shape
        return _C().mamba2.conv_fwd(xw, w, b, bd).view(B, S, C)

    @staticmethod
    def backward(ctx, du):
        x, xw, w, b, bd = ctx.saved_tensors
        C = w.shape[0]
        if ctx.link is not None:
            dx = ctx.link.window(x[..., ctx.col:ctx.col + C])
            full, ctx.link.buffer = ctx.link.buffer, None
        else:
            full = torch.zeros_like(x)
            dx = full[..., ctx.col:ctx.col + C]
        _, dw, db = _C().mamba2.conv_bwd(_rows(du), xw, w, b, bd, dx.reshape(-1, C))
        return full, dw.view(ctx.weight_shape).to(ctx.dtypes[0]), db.to(ctx.dtypes[1]), None, None, None


def causal_conv1d_window(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor, bounds: torch.Tensor, col: int = 0,
                         link: Optional[Mamba2GradLink] = None) -> torch.Tensor:
    """Mamba-2's causal depthwise convolution of width 4 with SiLU over the columns [col, col + C) of x [B, S, W] (in_proj's
    output, read in place), weight [C, 1, 4], bias [C]: u[t] = silu(bias + sum_j weight[:, 0, j] x[t - 3 + j]) -> [B, S, C].
    Taps before the document start of ``bounds`` (int32 [B, S, 2], ``document_bounds``) read zero; padding positions give zero.

    CUDA bf16 x runs the native kernels (C and col multiples of 8, else ``ValueError``): fp32 sums with one bf16 rounding,
    bitwise repeatable, no host synchronisation.  The gradient of x is [B, S, W]: with a ``link`` shared with ``ssd_scan``
    and ``gated_rms_norm`` it is their common buffer, complete; without one its other columns are zero.  CPU x, and CUDA
    fp32 or fp64 x, run ``causal_conv1d_window_reference``; CUDA x of any other dtype raises ``ValueError``."""
    _mamba2_check_rows("causal_conv1d_window", x, bounds)
    C = weight.shape[0]
    if tuple(weight.shape) != (C, 1, MAMBA_CONV_WIDTH) or tuple(bias.shape) != (C,) or col < 0 or col + C > x.shape[-1]:
        raise ValueError(f"causal_conv1d_window needs weight [C, 1, 4], bias [C] and columns [col, col + C) inside x, got "
                         f"{tuple(weight.shape)}, {tuple(bias.shape)}, col {col} and x {tuple(x.shape)}")
    if not _mamba_native("causal_conv1d_window", x):
        return causal_conv1d_window_reference(x, weight, bias, bounds, col)
    if C % 8 or col % 8 or x.shape[-1] % 8:
        raise ValueError(f"causal_conv1d_window's kernels need C, col and W multiples of 8, got C {C}, col {col}, W {x.shape[-1]}")
    return _CausalConv1dWindow.apply(x, weight, bias, bounds, col, link)


def _ssd_shapes(who: str, xbc: torch.Tensor, dt: torch.Tensor, A_log, D, dt_bias, bounds, head_dim: int, state_size: int,
                n_groups: int):
    _mamba2_check_rows(who, xbc, bounds)
    if head_dim != MAMBA2_HEAD_DIM or state_size != MAMBA2_STATE or n_groups != 1:
        raise ValueError(f"{who} takes head dim 64, state 128 and one group, got head dim {head_dim}, state {state_size}, "
                         f"{n_groups} groups")
    B, S, _ = xbc.shape
    H = dt.shape[-1] if dt.dim() == 3 else -1
    if dt.dim() != 3 or tuple(dt.shape[:2]) != (B, S) or xbc.shape[-1] != H * head_dim + 2 * state_size:
        raise ValueError(f"{who} needs dt [B, S, H] and xbc [B, S, 64 H + 256] (x | B | C), got {tuple(dt.shape)} and {tuple(xbc.shape)}")
    if any(tuple(t.shape) != (H,) for t in (A_log, D, dt_bias)):
        raise ValueError(f"{who} needs A_log, D and dt_bias [H] for H = {H}, got {tuple(A_log.shape)}, {tuple(D.shape)} and "
                         f"{tuple(dt_bias.shape)}")
    return B, S, H


def ssd_scan_reference(xbc: torch.Tensor, dt: torch.Tensor, A_log: torch.Tensor, D: torch.Tensor, dt_bias: torch.Tensor,
                       bounds: torch.Tensor, head_dim: int = MAMBA2_HEAD_DIM, state_size: int = MAMBA2_STATE,
                       n_groups: int = 1) -> torch.Tensor:
    """``ssd_scan`` in torch, fp32 (fp64 for fp64 input): the chunked SSD of transformers' ``Mamba2Mixer.torch_forward``
    (intra-chunk C B^T o L, chunk states, their recurrence, state -> output) with the state reset at each document start:
    L and the chunk states only join rows of one document, and a chunk's incoming state reaches only rows whose document
    began before the chunk.  Padding positions give y = 0.  Differentiable."""
    B, S, H = _ssd_shapes("ssd_scan_reference", xbc, dt, A_log, D, dt_bias, bounds, head_dim, state_size, n_groups)
    dtype = _ref_dtype(xbc)
    P, N, L = head_dim, state_size, MAMBA2_CHUNK
    E = H * P
    dev = xbc.device
    real, start, _ = _mamba_positions(bounds, dev)
    pad = (L - S % L) % L
    nc = (S + pad) // L
    pos = torch.arange(S + pad, device=dev)
    real = F.pad(real, (0, pad))
    start = F.pad(start, (0, pad), value=0)
    v = dt.to(dtype) + dt_bias.to(dtype)
    dts = F.softplus(v, threshold=MAMBA_SOFTPLUS_THRESHOLD) * real[:, :S, None]
    xs = F.pad(xbc.to(dtype), (0, 0, 0, pad))
    x = xs[..., :E].reshape(B, nc, L, H, P)
    Bm, Cm = xs[..., E:E + N].reshape(B, nc, L, N), xs[..., E + N:].reshape(B, nc, L, N)
    dts = F.pad(dts, (0, 0, 0, pad)).reshape(B, nc, L, H)
    A = -torch.exp(A_log.to(dtype))
    cum = torch.cumsum(A * dts, dim=2)                                    # [B, nc, L, H]
    real_c, start_c, pos_c = real.reshape(B, nc, L), start.reshape(B, nc, L), pos.reshape(nc, L)
    # same document, j <= i, both real
    tri = torch.tril(torch.ones(L, L, dtype=torch.bool, device=dev))
    same = (pos_c[None, :, None, :] >= start_c[..., :, None]) & tri & real_c[..., :, None] & real_c[..., None, :]   # [B, nc, i, j]
    diff = cum[:, :, :, None, :] - cum[:, :, None, :, :]                  # [B, nc, i, j, H]
    Lm = torch.exp(torch.where(same[..., None], diff, torch.full_like(diff, -math.inf))) * dts[:, :, None, :, :]
    CB = torch.einsum("bcin,bcjn->bcij", Cm, Bm)
    y = torch.einsum("bcijh,bcjhp->bcihp", Lm * CB[..., None], x)
    # each chunk's outgoing state: the rows of its last document
    last = start_c[..., -1]
    for_state = real_c & real_c[..., -1:] & (start_c == last[..., None])                 # [B, nc, L]
    wdecay = torch.exp(torch.where(for_state[..., None], cum[:, :, -1:, :] - cum, torch.full_like(cum, -math.inf))) * dts
    states = torch.einsum("bcjh,bcjn,bcjhp->bchnp", wdecay, Bm, x)
    carry = real_c[..., -1] & (last < pos_c[None, :, 0])                                 # [B, nc]
    dec = torch.where(carry[..., None], torch.exp(cum[:, :, -1, :]), torch.zeros_like(cum[:, :, -1, :]))   # [B, nc, H]
    h = torch.zeros(B, H, N, P, dtype=dtype, device=dev)
    hin = []
    for c in range(nc):
        hin.append(h)
        h = dec[:, c, :, None, None] * h + states[:, c]
    hin = torch.stack(hin, 1)                                                            # [B, nc, H, N, P]
    off = real_c & (start_c < pos_c[None, :, :1])                                        # [B, nc, L]
    ecum = torch.exp(torch.where(off[..., None], cum, torch.full_like(cum, -math.inf)))
    y = y + torch.einsum("bcin,bchnp->bcihp", Cm, hin) * ecum[..., None]
    y = y + D.to(dtype)[:, None] * x
    y = y.reshape(B, S + pad, E)[:, :S]
    return torch.where(real[:, :S, None], y, torch.zeros_like(y)).to(xbc.dtype)


class _SsdScan(torch.autograd.Function):
    """(xbc [B, S, 64 H + 256], dt [B, S, H] view) bf16 -> y [B, S, 64 H] (csrc/mamba2.cu); nothing but the inputs is kept
    for the backward, which recomputes the chunk states."""

    @staticmethod
    def forward(ctx, xbc, dt, A_log, D, dt_bias, bounds, link):
        B, S, _ = xbc.shape
        ins = [_rows(xbc), _row_view(dt), A_log.float().contiguous(), D.float().contiguous(), dt_bias.float().contiguous(),
               _aligned16(bounds.to(torch.int32))]
        y = _C().mamba2.ssd_fwd(*ins)
        ctx.save_for_backward(dt, *ins)
        ctx.link, ctx.dtypes, ctx.xshape = link, (A_log.dtype, D.dtype, dt_bias.dtype), xbc.shape
        return y.view(B, S, -1)

    @staticmethod
    def backward(ctx, dy):
        dt, *ins = ctx.saved_tensors
        given = ctx.link.window(dt) if ctx.link is not None else None
        dxbc, ddt, dA_log, dD, dbias = _C().mamba2.ssd_bwd(_rows(dy), *ins, None if given is None else given.reshape(-1, dt.shape[-1]))
        tA, tD, tb = ctx.dtypes
        return (dxbc.view(ctx.xshape), None if given is not None else ddt.view(dt.shape), dA_log.to(tA), dD.to(tD), dbias.to(tb),
                None, None)


def ssd_scan(xbc: torch.Tensor, dt: torch.Tensor, A_log: torch.Tensor, D: torch.Tensor, dt_bias: torch.Tensor, bounds: torch.Tensor,
             head_dim: int = MAMBA2_HEAD_DIM, state_size: int = MAMBA2_STATE, n_groups: int = 1,
             link: Optional[Mamba2GradLink] = None) -> torch.Tensor:
    """Mamba-2's SSD scan with the state reset at every document start: per row, head h (head dim 64) and state n (128),
    dt = softplus(dt + dt_bias) (threshold 20), A = -exp(A_log), h_t = exp(dt_t A) h_{t-1} + dt_t B_t x_t^T with h = 0 before
    each document, y_t = C_t h_t + D x_t.  xbc [B, S, 64 H + 256] is the conv's output x | B | C (one group: B and C shared by
    all heads); dt [B, S, H] may be a column view of in_proj's output; A_log, D, dt_bias [H]; bounds int32 [B, S, 2]
    (``document_bounds``).  Padding positions give y = 0 and zero gradients.  Head dims other than 64, states other than
    128 and more than one group raise ``ValueError``.

    CUDA bf16 activations run the native chunked scan on tensor cores (H a multiple of 8, else ``ValueError``): bf16
    operands with fp32 sums and fp32 chunk states, gradients summed in a fixed order (bitwise repeatable), nothing read back
    to the host.  With a ``link`` the gradient of dt goes into the link's buffer instead of being returned.  CPU activations,
    and CUDA fp32 or fp64 ones, run ``ssd_scan_reference``; CUDA activations of any other dtype, or of mixed dtypes, raise
    ``ValueError``."""
    _ssd_shapes("ssd_scan", xbc, dt, A_log, D, dt_bias, bounds, head_dim, state_size, n_groups)
    if not _mamba_native("ssd_scan", xbc, dt):
        return ssd_scan_reference(xbc, dt, A_log, D, dt_bias, bounds)
    if dt.shape[-1] % 8:
        raise ValueError(f"ssd_scan's kernels need the head count a multiple of 8, got {dt.shape[-1]}")
    return _SsdScan.apply(xbc, dt, A_log, D, dt_bias, bounds, link)


def gated_rms_norm_reference(y: torch.Tensor, z: torch.Tensor, weight: torch.Tensor, eps: float) -> torch.Tensor:
    """``gated_rms_norm`` in torch as transformers' ``MambaRMSNormGated``: g = y silu(z) in fp32 (fp64 for fp64 input),
    weight * g * rsqrt(mean(g^2) + eps).  Differentiable."""
    dtype = _ref_dtype(y)
    g = y.to(dtype) * F.silu(z.to(dtype))
    g = g * torch.rsqrt(g.pow(2).mean(-1, keepdim=True) + eps)
    return (weight.to(dtype) * g).to(y.dtype)


class _GatedRmsNorm(torch.autograd.Function):
    """(y [B, S, E], z [B, S, E] view) bf16 -> weight * rmsnorm(y silu(z)) (csrc/layernorm.cu)."""

    @staticmethod
    def forward(ctx, y, z, weight, eps, link):
        y2, z2, w = _rows(y), _row_view(z), weight.to(torch.bfloat16).contiguous()
        out, rstd = _C().mamba2.gated_norm_fwd(y2, z2, w, eps)
        ctx.save_for_backward(z, y2, z2, w, rstd)
        ctx.link, ctx.wdtype = link, weight.dtype
        return out.view(y.shape)

    @staticmethod
    def backward(ctx, dout):
        z, y2, z2, w, rstd = ctx.saved_tensors
        given = ctx.link.window(z) if ctx.link is not None else None
        dy, dz, dw = _C().mamba2.gated_norm_bwd(_rows(dout), y2, z2, w, rstd, None if given is None else given.reshape(-1, z.shape[-1]))
        return dy.view(dout.shape), None if given is not None else dz.view(z.shape), dw.to(ctx.wdtype), None, None


def gated_rms_norm(y: torch.Tensor, z: torch.Tensor, weight: torch.Tensor, eps: float,
                   link: Optional[Mamba2GradLink] = None) -> torch.Tensor:
    """Mamba-2's gated RMSNorm over the last dim: weight * g / sqrt(mean(g^2) + eps) with g = y silu(z); y [..., E], z [..., E]
    (it may be a column view of in_proj's output, read in place), weight [E].

    CUDA bf16 y and z run the native wide RMSNorm kernels' gated variant (1024 < E <= 4096, E % 8 == 0, else ``ValueError``):
    fp32 statistics, one bf16 rounding, dweight summed in a fixed order.  With a ``link`` the gradient of z goes into the
    link's buffer instead of being returned.  CPU input, and CUDA fp32 or fp64 input, run ``gated_rms_norm_reference``;
    CUDA input of any other dtype, or of mixed dtypes, raises ``ValueError``."""
    if y.shape != z.shape or y.dim() < 1 or tuple(weight.shape) != (y.shape[-1],):
        raise ValueError(f"gated_rms_norm needs y and z of one shape [..., E] and weight [E], got {tuple(y.shape)}, {tuple(z.shape)} "
                         f"and {tuple(weight.shape)}")
    if not _mamba_native("gated_rms_norm", y, z):
        return gated_rms_norm_reference(y, z, weight, eps)
    E = y.shape[-1]
    if E % 8 or not 1024 < E <= 4096 or y.numel() == 0:
        raise ValueError(f"gated_rms_norm's kernels need 1024 < E <= 4096 with E % 8 == 0 and at least one row, got {tuple(y.shape)}")
    return _GatedRmsNorm.apply(y, z, weight, float(eps), link)


# ------------------------------------------------------------------------------------------------
# CLIP (csrc/clip.cu): captions as causal documents of one token stream, the contrastive loss over the global batch
# ------------------------------------------------------------------------------------------------
def caption_token_bounds(input_ids: torch.Tensor, eos_token_id: int):
    """Causal-document bounds of B captions laid out one after another in one token stream: ``(bounds int32 [1, T, 2],
    pooled long [B])`` for input_ids [B, L], T = ``image_token_rows(B, L)``.  Caption b owns rows [L b, L (b + 1)); with e_b
    its first ``eos_token_id`` (transformers' ``(ids == eos).int().argmax(-1)``, so 0 for a caption without one), rows
    L b + j with j <= e_b hold (L b, L b + e_b + 1) and every later row, and the padding past L B, holds (0, 0).
    ``causal_attention(qkv.view(1, T, 3 * hidden), bounds, heads)`` then gives the pooled row L b + e_b (``pooled[b]``) the
    same keys as the dense L x L causal mask, and never visits a row past an EOT.  Torch ops on input_ids' device: no host
    synchronisation (CUDA-graph safe)."""
    if input_ids.dim() != 2 or input_ids.is_floating_point() or input_ids.is_complex() or input_ids.numel() == 0:
        raise ValueError(f"caption_token_bounds needs integer input_ids [B, L], got {input_ids.dtype} {tuple(input_ids.shape)}")
    B, L = input_ids.shape
    dev = input_ids.device
    eot = (input_ids == eos_token_id).int().argmax(-1)
    T = image_token_rows(B, L)
    t = torch.arange(T, device=dev)
    b = torch.clamp(t // L, max=B - 1)
    first = b * L
    e = eot[b]
    keep = (t < B * L) & (t - first <= e)
    zero = torch.zeros((), device=dev, dtype=torch.long)
    bounds = torch.stack([torch.where(keep, first, zero), torch.where(keep, first + e + 1, zero)], -1).to(torch.int32)
    return bounds.view(1, T, 2), torch.arange(B, device=dev) * L + eot


def _vector_norm(x: torch.Tensor) -> torch.Tensor:
    """transformers' ``_get_vector_norm``: sqrt(sum(x^2)) over the last dimension, kept."""
    return torch.pow(torch.sum(torch.pow(x, 2), dim=-1, keepdim=True), 0.5)


class _L2Normalize(torch.autograd.Function):
    """u = x / ||x|| per row (csrc/clip.cu); the backward rnorm (du - u <u, du>) recomputes u from x in fp32."""

    @staticmethod
    def forward(ctx, x):
        u, rnorm = _C().clip.l2norm_fwd(x)
        ctx.save_for_backward(x, rnorm)
        return u

    @staticmethod
    def backward(ctx, du):
        x, rnorm = ctx.saved_tensors
        return _C().clip.l2norm_bwd(du.to(torch.bfloat16).contiguous(), x, rnorm)


class _ContrastiveLoss(torch.autograd.Function):
    """Forward: z_img = u_img U_txt^T and z_txt = u_txt U_img^T on the wgmma GEMM (fp32 out), then one fused cross-entropy
    (csrc/clip.cu) that writes the loss, both bf16 logit gradients and d logit_scale.  Backward: the four products
    du_img = dz_img U_txt, dU_txt = dz_img^T u_img, du_txt = dz_txt U_img and dU_img = dz_txt^T u_txt on the same GEMM
    (MN-major operands, no transposed copies), each dz first scaled by the upstream gradient on the device."""

    @staticmethod
    def forward(ctx, u_img, u_txt, U_img, U_txt, logit_scale, offset):
        C = _C()
        z_img = C.gemm(u_img, U_txt, None, False, False, EPI_NONE, True, None)
        z_txt = C.gemm(u_txt, U_img, None, False, False, EPI_NONE, True, None)
        loss, dscale, dz_img, dz_txt = C.clip.contrastive_xent(z_img, z_txt, logit_scale.reshape(1), int(offset))
        ctx.save_for_backward(u_img, u_txt, U_img, U_txt, dz_img, dz_txt, dscale)
        ctx.scale_shape = logit_scale.shape
        return loss

    @staticmethod
    def backward(ctx, g):
        C = _C()
        u_img, u_txt, U_img, U_txt, dz_img, dz_txt, dscale = ctx.saved_tensors
        g = g.detach().float()
        dz_img, dz_txt = dz_img * g, dz_txt * g                   # bf16 out, one rounding of the fp32 product
        du_img = C.gemm(dz_img, U_txt, None, False, True, EPI_NONE, False, None)
        du_txt = C.gemm(dz_txt, U_img, None, False, True, EPI_NONE, False, None)
        dU_txt = C.gemm(dz_img, u_img, None, True, True, EPI_NONE, False, None)
        dU_img = C.gemm(dz_txt, u_txt, None, True, True, EPI_NONE, False, None)
        return du_img, du_txt, dU_img, dU_txt, (dscale * g).view(ctx.scale_shape), None


def _gather_features(x: torch.Tensor, group) -> torch.Tensor:
    """The rows of every rank of ``group``, in rank order, with autograd: the backward sums the gradient of the gathered
    rows across ranks and returns this rank's slice (``torch.distributed.nn.functional.all_gather``)."""
    from torch.distributed.nn.functional import all_gather
    return torch.cat(all_gather(x.contiguous(), group=group), 0)


def clip_loss(image_embeds: torch.Tensor, text_embeds: torch.Tensor, logit_scale: torch.Tensor, group=None) -> torch.Tensor:
    """CLIP's contrastive loss over the global batch: with u = x / ||x|| per row, s = exp(logit_scale) (no clamp), and the
    N = world B normalised features of every rank gathered in rank order (U_img, U_txt),
    (CE(s u_img U_txt^T, rank B + r) + CE(s u_txt U_img^T, rank B + r)) / 2 averaged over the B local rows -
    transformers' ``clip_loss`` on the global batch's similarity rows this rank owns.  image_embeds, text_embeds [B, D]
    (unnormalised), logit_scale a one-element tensor.

    Ranks: ``group``, or the default process group when one is initialised.  Above one rank the gather is
    ``torch.distributed.nn.functional.all_gather``, whose backward sums the features' gradients over the ranks, so that
    averaging the parameter gradients across ranks (DDP) gives the gradient of the global-batch mean loss.  One rank runs
    no collective.

    On CUDA: bf16 embeds with B % 8 == 0 and D % 8 == 0, else ``ValueError``.  The normalisation, the cross-entropy with its
    gradients (``_ContrastiveLoss``) and the GEMMs are native and read nothing back to the host.  On CPU: torch ops."""
    if image_embeds.dim() != 2 or tuple(text_embeds.shape) != tuple(image_embeds.shape) or image_embeds.shape[0] < 1:
        raise ValueError(f"clip_loss needs image_embeds and text_embeds [B, D] of one shape with B >= 1, got "
                         f"{tuple(image_embeds.shape)} and {tuple(text_embeds.shape)}")
    if logit_scale.numel() != 1:
        raise ValueError(f"clip_loss needs a one-element logit_scale, got {tuple(logit_scale.shape)}")
    world, rank = 1, 0
    if torch.distributed.is_available() and torch.distributed.is_initialized():
        group = torch.distributed.group.WORLD if group is None else group
        world, rank = torch.distributed.get_world_size(group), torch.distributed.get_rank(group)
    B, D = image_embeds.shape
    if image_embeds.is_cuda:
        if image_embeds.dtype != torch.bfloat16 or text_embeds.dtype != torch.bfloat16 or B % 8 or D % 8:
            raise ValueError(f"clip_loss on CUDA needs bf16 embeds with B % 8 == 0 and D % 8 == 0, got {image_embeds.dtype} and "
                             f"{text_embeds.dtype} [{B}, {D}]")
        if logit_scale.device != image_embeds.device:
            raise ValueError(f"clip_loss needs logit_scale on the embeds' device ({image_embeds.device}), got {logit_scale.device}")
        u_img, u_txt = _L2Normalize.apply(image_embeds.contiguous()), _L2Normalize.apply(text_embeds.contiguous())
    else:
        u_img, u_txt = image_embeds / _vector_norm(image_embeds), text_embeds / _vector_norm(text_embeds)
    if world > 1:
        U_img, U_txt = _gather_features(u_img, group), _gather_features(u_txt, group)
    else:
        U_img, U_txt = u_img, u_txt
    if image_embeds.is_cuda:
        return _ContrastiveLoss.apply(u_img, u_txt, U_img, U_txt, logit_scale.float(), rank * B)
    s = logit_scale.exp()
    labels = torch.arange(B, device=image_embeds.device) + rank * B
    return (F.cross_entropy((u_img @ U_txt.t()) * s, labels) + F.cross_entropy((u_txt @ U_img.t()) * s, labels)) / 2.0


# ------------------------------------------------------------------------------------------------
# Whisper's audio side (csrc/whisper.cu): the log-mel front end and the gathers of the two-convolution stem
# ------------------------------------------------------------------------------------------------
WHISPER_SAMPLES = 480000         # a 30-second clip at 16 kHz
WHISPER_N_FFT, WHISPER_HOP = 400, 160


def whisper_mel_filters(num_mel_bins: int = 80, n_fft: int = WHISPER_N_FFT, sampling_rate: int = 16000) -> torch.Tensor:
    """Whisper's mel filterbank, fp64 [n_fft // 2 + 1, num_mel_bins]: triangular filters on the Slaney mel scale between 0 Hz
    and sampling_rate / 2, each scaled to unit area (Slaney normalisation), as ``WhisperFeatureExtractor.mel_filters``."""
    f_sp, min_log_hz, min_log_mel, logstep = 200.0 / 3, 1000.0, 15.0, math.log(6.4) / 27.0

    def hz_to_mel(f):
        return torch.where(f >= min_log_hz, min_log_mel + torch.log(f.clamp(min=min_log_hz) / min_log_hz) / logstep, f / f_sp)

    def mel_to_hz(m):
        return torch.where(m >= min_log_mel, min_log_hz * torch.exp(logstep * (m - min_log_mel)), f_sp * m)

    edges = torch.tensor([0.0, sampling_rate / 2], dtype=torch.float64)
    mels = hz_to_mel(edges)
    freqs = mel_to_hz(torch.linspace(float(mels[0]), float(mels[1]), num_mel_bins + 2, dtype=torch.float64))
    fft_freqs = torch.linspace(0, sampling_rate // 2, n_fft // 2 + 1, dtype=torch.float64)
    diff = freqs[1:] - freqs[:-1]
    slopes = freqs[None, :] - fft_freqs[:, None]
    down, up = -slopes[:, :-2] / diff[:-1], slopes[:, 2:] / diff[1:]
    filters = torch.clamp(torch.minimum(down, up), min=0.0)
    return filters * (2.0 / (freqs[2:] - freqs[:-2]))[None, :]


def log_mel_spectrogram_reference(waveform: torch.Tensor, mel_filters: torch.Tensor, dtype=torch.float64) -> torch.Tensor:
    """Whisper's log-mel features of int16 waveforms [B, N] in ``dtype``: [B, mels, N / 160], as transformers'
    ``WhisperFeatureExtractor`` (its ``_torch_extract_fbank_features``) computes them from waveform / 32768."""
    x = waveform.to(dtype) / 32768.0
    window = torch.hann_window(WHISPER_N_FFT, periodic=True, dtype=dtype, device=x.device)
    stft = torch.stft(x, WHISPER_N_FFT, WHISPER_HOP, window=window, center=True, pad_mode="reflect", return_complex=True)
    power = stft[..., :-1].abs() ** 2
    L = (mel_filters.to(dtype=dtype, device=x.device).T @ power).clamp(min=1e-10).log10()
    M = L.amax(dim=(1, 2), keepdim=True)
    return (torch.maximum(L, M - 8.0) + 4.0) / 4.0


def log_mel_spectrogram(waveform: torch.Tensor, mel_filters: torch.Tensor, out_dtype=torch.bfloat16,
                        out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Whisper's log-mel features [B, 80, 3000] in ``out_dtype`` (bf16 or fp32) of 30-second int16 PCM clips
    ``waveform`` [B, 480000] (shorter clips zero-padded by the caller, as the feature extractor pads them), through
    ``mel_filters`` [201, 80] (``whisper_mel_filters()``).  Written into ``out`` when given.  Anything else raises
    ``ValueError``.  On CUDA the native kernels compute it in fp32 in a fixed order without host synchronisation (CUDA-graph
    safe, bitwise repeatable); on CPU ``log_mel_spectrogram_reference`` in fp32."""
    if waveform.dtype != torch.int16 or waveform.dim() != 2 or waveform.shape[0] < 1 or waveform.shape[1] != WHISPER_SAMPLES \
            or not waveform.is_contiguous():
        raise ValueError(f"log_mel_spectrogram needs contiguous int16 waveforms [B, {WHISPER_SAMPLES}] with B >= 1, got "
                         f"{waveform.dtype} {tuple(waveform.shape)}{'' if waveform.is_contiguous() else ' strided'}")
    if tuple(mel_filters.shape) != (WHISPER_N_FFT // 2 + 1, 80) or not mel_filters.is_floating_point():
        raise ValueError(f"log_mel_spectrogram needs floating mel_filters [201, 80], got {mel_filters.dtype} {tuple(mel_filters.shape)}")
    if out_dtype not in (torch.bfloat16, torch.float32):
        raise ValueError(f"log_mel_spectrogram writes bf16 or fp32, got {out_dtype}")
    B = waveform.shape[0]
    if out is not None and (out.dtype != out_dtype or tuple(out.shape) != (B, 80, 3000) or not out.is_contiguous()
                            or out.device != waveform.device):
        raise ValueError(f"log_mel_spectrogram needs out to be a contiguous {out_dtype} [{B}, 80, 3000] on {waveform.device}, got "
                         f"{out.dtype} {tuple(out.shape)} on {out.device}")
    if waveform.is_cuda:
        filters = mel_filters.to(device=waveform.device, dtype=torch.float32).contiguous()
        return _C().whisper.log_mel(waveform, filters, out_dtype == torch.bfloat16, out)
    y = log_mel_spectrogram_reference(waveform, mel_filters, torch.float32).to(out_dtype)
    return out.copy_(y) if out is not None else y


def encoder_rows(frames: int) -> int:
    """Rows per clip of Whisper's encoder for ``frames`` mel frames: the stride-2 convolution's frames / 2 outputs, rounded
    up to a multiple of 128 so the attention kernels take them (1536 for 3000 frames: 1500 real rows and 36 padding rows)."""
    n = frames // 2
    return (n + ATTENTION_SEQ_MULTIPLE - 1) // ATTENTION_SEQ_MULTIPLE * ATTENTION_SEQ_MULTIPLE


def mel_patches_reference(features: torch.Tensor) -> torch.Tensor:
    """P1 [B F, 3 C] of features [B, C, F]: P1[b F + t, j C + c] = features[b, c, t + j - 1], zero outside [0, F)."""
    B, C, T = features.shape
    p = F.pad(features, (1, 1))
    return torch.stack([p[..., j:j + T] for j in range(3)], 1).permute(0, 3, 1, 2).reshape(B * T, 3 * C)


def mel_patches(features: torch.Tensor) -> torch.Tensor:
    """The im2col rows of Whisper's first convolution (width 3, padding 1) over mel features [B, 80, F]: [B F, 240] with
    column j 80 + c holding channel c at frame t + j - 1 (``mel_patches_reference``), so that
    ``linear(P1, conv1.weight.permute(0, 2, 1).reshape(d, 240))`` is the convolution.  Forward only: the features take no
    gradient.  On CUDA: bf16 features, else ``ValueError``; a native gather."""
    if features.dim() != 3 or features.shape[1] != 80:
        raise ValueError(f"mel_patches needs features [B, 80, F], got {tuple(features.shape)}")
    if features.is_cuda:
        if features.dtype != torch.bfloat16:
            raise ValueError(f"mel_patches on CUDA needs bf16 features, got {features.dtype}")
        return _C().whisper.mel_patches(features.contiguous())
    return mel_patches_reference(features)


def frame_patches_reference(h1: torch.Tensor, frames: int, rows: int) -> torch.Tensor:
    """P2 [B rows, 3 d] of h1 [B frames, d]: row (b, l) for l < frames / 2 holds h1[b, 2l - 1] | h1[b, 2l] | h1[b, 2l + 1]
    (h1[b, -1] = 0), rows l >= frames / 2 are zero.  Differentiable."""
    d = h1.shape[1]
    B, L = h1.shape[0] // frames, frames // 2
    hp = F.pad(h1.view(B, frames, d), (0, 0, 1, 1))
    idx = 2 * torch.arange(L, device=h1.device)
    p = torch.cat([hp[:, idx + j] for j in range(3)], -1)
    return F.pad(p, (0, 0, 0, rows - L)).reshape(B * rows, 3 * d)


class _FramePatches(torch.autograd.Function):
    """The stride-2 gather forward; its backward is a col2im gather (each dh1 row sums its at most two taps in order)."""

    @staticmethod
    def forward(ctx, h1, frames, rows):
        ctx.geometry = (frames, rows)
        return _C().whisper.frame_patches(h1, frames, rows)

    @staticmethod
    def backward(ctx, dp2):
        frames, rows = ctx.geometry
        return _C().whisper.frame_patches_bwd(dp2.contiguous(), frames, rows), None, None


def frame_patches(h1: torch.Tensor, frames: int, rows: int) -> torch.Tensor:
    """The im2col rows of Whisper's second convolution (width 3, stride 2, padding 1) over h1 [B frames, d]: [B rows, 3 d]
    (``frame_patches_reference``), rows >= frames / 2 zero, so that ``linear(P2, conv2.weight.permute(0, 2, 1).reshape(d,
    3 d))`` gives the encoder's rows.  frames even, rows >= frames / 2.  On CUDA: bf16 h1 with d % 8 == 0, else
    ``ValueError``; native gathers both ways, the backward summing each h1 row's taps in fp32 with one bf16 rounding."""
    if h1.dim() != 2 or frames < 2 or frames % 2 or h1.shape[0] % frames or rows < frames // 2:
        raise ValueError(f"frame_patches needs h1 [B frames, d] with even frames >= 2 and rows >= frames / 2, got "
                         f"{tuple(h1.shape)}, frames {frames}, rows {rows}")
    if h1.is_cuda:
        if h1.dtype != torch.bfloat16 or h1.shape[1] % 8:
            raise ValueError(f"frame_patches on CUDA needs bf16 h1 with d % 8 == 0, got {h1.dtype} {tuple(h1.shape)}")
        return _FramePatches.apply(h1.contiguous(), frames, rows)
    return frame_patches_reference(h1, frames, rows)


# ------------------------------------------------------------------------------------------------
# Masked-autoencoder pretraining (csrc/mae.cu): per-image shuffling, the masked patch embedding, the decoder's unshuffle,
# per-image attention at head dim 32 and the pixel reconstruction loss, on ``patch_embed``'s token streams
# ------------------------------------------------------------------------------------------------
MAE_HEAD_DIM = 32
MAE_MAX_TOKENS = 256
MAE_NORM_PIX_EPS = 1e-6


def mae_shuffle_reference(noise: torch.Tensor, keep: int):
    """transformers' ``random_masking`` indices with a stable sort: (ids_keep [B, keep], ids_restore [B, N]), int64.  Patch i
    of image b has rank ids_restore[b, i] in its image's ascending noise (ties by index) and is kept iff that is below keep."""
    ids_shuffle = torch.argsort(noise, dim=1, stable=True)
    return ids_shuffle[:, :keep], torch.argsort(ids_shuffle, dim=1)


def mae_shuffle(noise: torch.Tensor, keep: int):
    """(ids_keep [B, keep], ids_restore [B, N]) of noise [B, N]: the patches ranked by ascending noise, ties in index order,
    the first `keep` kept.  CUDA: one kernel, int32 results, no host synchronisation (N <= 1024); the ranks of noise without
    NaNs equal a stable ``argsort``'s.  CPU: ``mae_shuffle_reference``."""
    if not noise.is_cuda:
        return mae_shuffle_reference(noise, keep)
    return _C().mae.shuffle(noise.float().contiguous(), int(keep))


def mae_patch_embed_reference(images: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor], class_token: torch.Tensor,
                              pos_embedding: torch.Tensor, ids_keep: torch.Tensor) -> torch.Tensor:
    """transformers' ViTMAE embeddings (the patch convolution, + pos[1:], the kept patches gathered, the class token + pos[0]
    in front) as ``mae_patch_embed``'s token stream [image_token_rows(B, keep + 1), D].  Differentiable."""
    B, keep = ids_keep.shape
    D, p = weight.shape[0], weight.shape[-1]
    x = F.conv2d(images, weight, bias, stride=p).flatten(2).transpose(1, 2) + pos_embedding[:, 1:]
    x = torch.gather(x, 1, ids_keep.long().unsqueeze(-1).expand(-1, -1, D))
    x = torch.cat([(class_token + pos_embedding[:, :1]).expand(B, -1, -1), x], 1)
    return F.pad(x.reshape(B * (keep + 1), D), (0, 0, 0, image_token_rows(B, keep + 1) - B * (keep + 1)))


class _MaeAssemble(torch.autograd.Function):
    """GEMM output [T, D] -> encoder tokens (csrc/mae.cu).  Backward: dy at patch rows for the weight-gradient GEMM and
    d class_token as a fixed-order sum over the images; the frozen position table gets none."""

    @staticmethod
    def forward(ctx, y, class_token, pos_embedding, ids_keep):
        ctx.batch, ctx.per, ctx.cls_shape = ids_keep.shape[0], ids_keep.shape[1] + 1, class_token.shape
        return _C().mae.patch_assemble(y, class_token.contiguous(), pos_embedding.contiguous(), ids_keep)

    @staticmethod
    def backward(ctx, dy):
        dpatch, dcls = _C().mae.patch_embed_bwd(_aligned16(dy), ctx.batch, ctx.per)
        return dpatch, dcls.view(ctx.cls_shape), None, None


def mae_patch_embed(images: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor], class_token: torch.Tensor,
                    pos_embedding: torch.Tensor, ids_keep: torch.Tensor) -> torch.Tensor:
    """The masked autoencoder's encoder input as one token stream: images [B, C, H, W], the patch convolution's weight
    [D, C, p, p] and bias [D], class_token [1, 1, D], a frozen pos_embedding [1, N + 1, D] and ids_keep [B, keep].  Returns
    [T, D], T = ``image_token_rows(B, keep + 1)``: image b's class token + pos[0] at row b (keep + 1), then its kept patch
    ids_keep[b, j] + pos[1 + ids_keep[b, j]] for j = 0 .. keep - 1, zero padding rows; ``image_token_bounds(B, keep + 1)``
    are its attention bounds.

    On CUDA (the requirements of ``patch_embed``, a pos_embedding that needs no gradient, else ``ValueError``): one kernel
    writes the kept patches' rows of the patch matrix, the wgmma ``linear`` runs on all T rows and one kernel adds the class
    token and positions (fp32, one rounding).  On CPU: ``mae_patch_embed_reference``."""
    if not images.is_cuda:
        return mae_patch_embed_reference(images, weight, bias, class_token, pos_embedding, ids_keep)
    _patch_embed_check(images, weight, bias, class_token, pos_embedding)
    if pos_embedding.requires_grad:
        raise ValueError("mae_patch_embed treats pos_embedding as a frozen table; pass one with requires_grad=False")
    B, keep = ids_keep.shape
    D, p = weight.shape[0], weight.shape[-1]
    ids_keep = ids_keep.to(torch.int32).contiguous()
    patches = _C().mae.patchify(images, ids_keep, p, image_token_rows(B, keep + 1))
    y = linear(patches, weight.reshape(D, -1), bias)
    return _MaeAssemble.apply(y, class_token, pos_embedding, ids_keep)


def mae_unshuffle_reference(y: torch.Tensor, mask_token: torch.Tensor, pos_embedding: torch.Tensor, ids_restore: torch.Tensor,
                            keep: int) -> torch.Tensor:
    """transformers' ViTMAE decoder input on token streams: the encoder stream y [Te, E] (B images of keep + 1 rows) ->
    [image_token_rows(B, N + 1), E] by its ``cat``, ``gather``, ``cat`` and the position add.  Differentiable."""
    B, N = ids_restore.shape
    E = y.shape[1]
    x = y[:B * (keep + 1)].view(B, keep + 1, E)
    x_ = torch.cat([x[:, 1:], mask_token.view(1, 1, E).expand(B, N - keep, E)], 1)
    x_ = torch.gather(x_, 1, ids_restore.long().unsqueeze(-1).expand(-1, -1, E))
    z = torch.cat([x[:, :1], x_], 1) + pos_embedding.view(1, N + 1, E)
    return F.pad(z.reshape(B * (N + 1), E), (0, 0, 0, image_token_rows(B, N + 1) - B * (N + 1)))


class _MaeUnshuffle(torch.autograd.Function):
    """Encoder stream -> decoder stream (csrc/mae.cu).  Backward: a gather of each encoder row's one decoder row, and
    d mask_token as a fixed-order fp32 sum over the masked rows."""

    @staticmethod
    def forward(ctx, y, mask_token, pos_embedding, ids_keep, ids_restore):
        ctx.save_for_backward(ids_keep, ids_restore)
        ctx.rows, ctx.mask_shape = y.shape[0], mask_token.shape
        B, N = ids_restore.shape
        return _C().mae.unshuffle(y, mask_token.contiguous(), pos_embedding.contiguous(), ids_restore, ids_keep.shape[1],
                                  image_token_rows(B, N + 1))

    @staticmethod
    def backward(ctx, dz):
        ids_keep, ids_restore = ctx.saved_tensors
        dy, dmask = _C().mae.unshuffle_bwd(_aligned16(dz), ids_keep, ids_restore, ctx.rows)
        return dy, dmask.view(ctx.mask_shape), None, None, None


def mae_unshuffle(y: torch.Tensor, mask_token: torch.Tensor, pos_embedding: torch.Tensor, ids_keep: torch.Tensor,
                  ids_restore: torch.Tensor) -> torch.Tensor:
    """The masked autoencoder's decoder input: the encoder stream y [Te, E] (B images of keep + 1 rows, keep =
    ``ids_keep.shape[1]``), mask_token [1, 1, E], a frozen pos_embedding [1, N + 1, E], ids_keep [B, keep] and ids_restore
    [B, N] from ``mae_shuffle``.  Returns [image_token_rows(B, N + 1), E]: row b (N + 1) is image b's class row, row
    b (N + 1) + 1 + i its encoder row of rank ids_restore[b, i] if that is below keep, else mask_token, each plus its
    position; zero padding rows.

    CUDA (bf16): one kernel, fp32 add and one rounding; backward one gather kernel with per-CTA partials for d mask_token and
    an in-order finish.  CPU: ``mae_unshuffle_reference``."""
    if not y.is_cuda:
        return mae_unshuffle_reference(y, mask_token, pos_embedding, ids_restore, ids_keep.shape[1])
    if pos_embedding.requires_grad:
        raise ValueError("mae_unshuffle treats pos_embedding as a frozen table; pass one with requires_grad=False")
    if y.dtype != torch.bfloat16 or mask_token.dtype != torch.bfloat16 or pos_embedding.dtype != torch.bfloat16:
        raise ValueError(f"mae_unshuffle on CUDA needs bf16 tensors, got {y.dtype}, {mask_token.dtype}, {pos_embedding.dtype}")
    return _MaeUnshuffle.apply(_aligned16(y), mask_token, pos_embedding, ids_keep.to(torch.int32).contiguous(),
                               ids_restore.to(torch.int32).contiguous())


def image_attention_reference(qkv: torch.Tensor, batch: int, tokens: int, heads: int) -> torch.Tensor:
    """``image_attention`` in torch (fp32 for bf16 input): dense softmax attention within each image's `tokens` rows, zero
    padding rows.  Any head dim."""
    T, W = qkv.shape
    dtype = qkv.dtype if qkv.dtype in (torch.float32, torch.float64) else torch.float32
    x = qkv[:batch * tokens].to(dtype).view(batch, tokens, 3, heads, W // (3 * heads)).permute(2, 0, 3, 1, 4)
    q, k, v = x[0], x[1], x[2]
    a = ((q * q.shape[-1] ** -0.5) @ k.transpose(-2, -1)).softmax(-1)
    o = (a @ v).transpose(1, 2).reshape(batch * tokens, W // 3)
    return F.pad(o, (0, 0, 0, T - batch * tokens)).to(qkv.dtype)


class _ImageAttention(torch.autograd.Function):
    """qkv [T, 3C] bf16 -> o [T, C] (csrc/mae.cu).  Backward: one kernel per (image, head)."""

    @staticmethod
    def forward(ctx, qkv, batch, tokens):
        o, lse = _C().mae.attention_fwd(qkv, batch, tokens)
        ctx.save_for_backward(qkv, o, lse)
        ctx.geometry = (batch, tokens)
        return o

    @staticmethod
    def backward(ctx, dout):
        qkv, o, lse = ctx.saved_tensors
        return _C().mae.attention_bwd(_aligned16(dout), qkv, o, lse, *ctx.geometry), None, None


def image_attention(qkv: torch.Tensor, batch: int, tokens: int, heads: int) -> torch.Tensor:
    """Per-image self-attention on a token stream: qkv [T, 3C] (columns q heads | k heads | v heads), image b's rows
    [b tokens, (b + 1) tokens), rows past batch tokens padding.  Returns [T, C]; padding rows are zero and get zero gradient.

    CUDA bf16 input runs the native kernels (head dim 32, tokens <= 256, else ``ValueError``): fp32 online softmax and sums,
    bitwise repeatable, no host synchronisation.  Everything else runs ``image_attention_reference``."""
    if not (qkv.is_cuda and qkv.dtype == torch.bfloat16):
        return image_attention_reference(qkv, batch, tokens, heads)
    if qkv.dim() != 2 or qkv.shape[1] != 3 * MAE_HEAD_DIM * heads:
        raise ValueError(f"image_attention on CUDA needs qkv [T, {3 * MAE_HEAD_DIM} heads] (head dim {MAE_HEAD_DIM}), got "
                         f"{tuple(qkv.shape)} for {heads} heads")
    if not (1 <= tokens <= MAE_MAX_TOKENS) or batch < 1 or batch * tokens > qkv.shape[0]:
        raise ValueError(f"image_attention on CUDA needs 1 <= tokens <= {MAE_MAX_TOKENS} and batch * tokens <= T, got {batch} x "
                         f"{tokens} for T = {qkv.shape[0]}")
    return _ImageAttention.apply(_aligned16(qkv), batch, tokens)


def mae_patchify(images: torch.Tensor, patch: int) -> torch.Tensor:
    """transformers' ``ViTMAEForPreTraining.patchify``: [B, C, H, W] -> [B, N, p p C] in (ky, kx, c) order."""
    B, C, H, W = images.shape
    x = images.reshape(B, C, H // patch, patch, W // patch, patch)
    return torch.einsum("nchpwq->nhwpqc", x).reshape(B, (H // patch) * (W // patch), patch * patch * C)


def mae_loss_reference(pred: torch.Tensor, images: torch.Tensor, ids_restore: torch.Tensor, keep: int, norm_pix: bool) -> torch.Tensor:
    """transformers' ``forward_loss`` on the decoder stream pred [Td, C p p] (image b's patch i at row b (N + 1) + 1 + i),
    in pred's dtype (fp32 for bf16)."""
    B, N = ids_restore.shape
    dtype = pred.dtype if pred.dtype in (torch.float32, torch.float64) else torch.float32
    p = int(round(math.sqrt(pred.shape[1] // images.shape[1])))
    x = pred[:B * (N + 1)].to(dtype).view(B, N + 1, -1)[:, 1:]
    target = mae_patchify(images.to(dtype), p)
    if norm_pix:
        mean = target.mean(dim=-1, keepdim=True)
        var = target.var(dim=-1, keepdim=True)
        target = (target - mean) / (var + MAE_NORM_PIX_EPS) ** 0.5
    mask = (ids_restore >= keep).to(dtype)
    return (((x - target) ** 2).mean(dim=-1) * mask).sum() / mask.sum()


class _MaeLoss(torch.autograd.Function):
    """pred [Td, C p p] bf16 -> loss fp32 [] (csrc/mae.cu).  Backward: the target recomputed from the image, the incoming
    gradient read on the device."""

    @staticmethod
    def forward(ctx, pred, images, ids_restore, keep, norm_pix):
        ctx.save_for_backward(pred, images, ids_restore)
        ctx.keep, ctx.norm_pix = keep, norm_pix
        return _C().mae.loss(pred, images, ids_restore, keep, norm_pix)

    @staticmethod
    def backward(ctx, dloss):
        pred, images, ids_restore = ctx.saved_tensors
        dpred = _C().mae.loss_bwd(dloss.float().reshape(1).contiguous(), pred, images, ids_restore, ctx.keep, ctx.norm_pix)
        return dpred, None, None, None, None


def mae_loss(pred: torch.Tensor, images: torch.Tensor, ids_restore: torch.Tensor, keep: int, norm_pix: bool) -> torch.Tensor:
    """The masked autoencoder's pixel reconstruction loss: pred [Td, C p p] on the decoder stream (image b's patch i at row
    b (N + 1) + 1 + i), images [B, C, H, W] and ids_restore [B, N].  The target is image b's patch i in (ky, kx, c) order,
    with ``norm_pix`` normalised by its mean and unbiased variance (+ 1e-6); the loss is the mean over the B (N - keep) masked
    patches of the per-patch mean of (pred - target)^2.

    CUDA bf16 runs the native kernels (C p^2 <= 768, p % 8 == 0, contiguous or channels_last images, else ``ValueError``):
    fixed-order fp32 sums, a backward that writes zeros at class, visible and padding rows and keeps nothing [Td, C p p]-sized
    in fp32 from the forward.  Everything else runs ``mae_loss_reference``."""
    if not (pred.is_cuda and pred.dtype == torch.bfloat16):
        return mae_loss_reference(pred, images, ids_restore, keep, norm_pix)
    if images.dtype != torch.bfloat16 or not (images.is_contiguous() or images.is_contiguous(memory_format=torch.channels_last)):
        raise ValueError(f"mae_loss on CUDA needs contiguous or channels_last bf16 images, got {images.dtype}")
    if images.requires_grad and torch.is_grad_enabled():
        raise ValueError("mae_loss gives the images no gradient; pass images that do not require one")
    return _MaeLoss.apply(_aligned16(pred), images, ids_restore.to(torch.int32).contiguous(), int(keep), bool(norm_pix))
