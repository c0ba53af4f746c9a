"""Element-wise error bounds for the native kernels, against a float64 reference of the same operation.

The reference is computed from the kernel's own inputs (bf16 or fp32, so exact in float64) on their device.  Every output
element gets its own bound from the magnitudes that entered it; there is no global norm, so one wrong element, a missing
bias on the last column or a dropped row at a ragged edge fails the check however large the rest of the output is.

GEMM (D = act(A Bᵀ + bias), fp32 accumulation), with P = |A| |B|ᵀ + |bias| and u = 2⁻²⁴:
  accumulation   C_ACC · (K + 1) · u · P        the tensor cores' fp32 accumulate (K products and the bias)
  activation     its Lipschitz constant (1 for none / ReLU, 1.13 for erf-GELU) times the above, plus ERF_ULPS · u · |z|
  output         2⁻⁸ · |ref| for bf16, 2⁻²³ · |ref| for fp32
  floor          FLOOR, far below the data's scale (exact zeros compare against it)

C_ACC is the one measured constant: the worst-case bound of recursive fp32 summation has C_ACC = 1, and the tensor cores'
accumulation (internal alignment of the k16 partial products) is allowed a small multiple of it.  On an H100 80GB HBM3
(700 W power limit) the fp32 outputs of test_gpu_gemm_elementwise.py reach at most 0.019 of the bound at C_ACC = 2.
bf16 outputs reach about 0.99 of theirs: the half-ulp rounding term is exact, so a correct rounding can nearly fill it.

The norms accumulate on the CUDA cores in IEEE fp32, so their sums take the plain worst-case bound n · u · Σ|terms|.

Attention reuses C_ACC for its tensor-core products.  On the same H100, test_gpu_attention_elementwise.py
reaches at most 0.037 of the lse bound at C_ACC = 2 and 0.23 at C_ACC = 0.25, and fails it at C_ACC = 0 (2.2): the lse
has no bf16 rounding to hide behind, so it is what calibrates C_ACC there.  EXP_ULPS = 0 passes as well as 2: no bound
is filled by the exp2 terms, so EXP_ULPS stays at exp2f's documented maximum.  Its bf16 outputs reach 0.95.

ResNet-50 (its own section below).  The convolutions (conv_wgmma.cu, conv_wgrad_wgmma.cu, the stem) are GEMMs on the tensor
cores and take the GEMM bound with the same C_ACC, P being the same convolution of the absolute values:
  fprop   K = R S Cin (the stem: 147; its packed layout only adds exact zero products)
  dgrad   K = R S Cout, plus one term for the fp32 addend the epilogue adds before rounding
  wgrad   K = the pixels one split sums on the tensor cores, plus the fixed-order fp32 reduction of the split partials
          (its longest chain, split lanes + 8, times u P)
then the bf16 rounding of the output.  The epilogue statistics (column sums of the stored bf16 output, and S1 / S2 of the
BatchNorm backward fused into dgrad) are fp32 chains of 32 rows per warp + one add per tile the CTA ran + the 4 epilogue
warps: conv_epilogue_depth().
BatchNorm (batchnorm.cu) sums x and x² (backward: dy* and dy* x̂) per channel in fp32 in an order fixed by its launch path;
D is the longest chain of fp32 additions any term goes through in that order (bn_two_pass_depth here, the resident and
from-partials depths in test_gpu_batchnorm_elementwise.py), so each sum is within D u Σ|terms|.  The forward then forms
mean = Σx / R, var = max(Σx²/R - mean², 0), rstd = rsqrtf(var + eps) (2 ulp), scale = γ rstd, shift = β - mean scale and
y = relu(x scale + shift (+ residual)); the bound carries every rounding at the magnitude it meets: the variance error is
relative to Σx²/R (not to var, which cancels when |mean| >> σ), rstd is bounded over the interval of var, and y's error is
relative to |x scale|, |mean scale| and |β| (not to |x̂|).  The backward takes the kernel's own mean, rstd and ReLU mask
as exact inputs and follows its dx = a dy* + b x + c, a = γ rstd, b = -a rstd S2/R, c = -a (S1/R - mean rstd S2/R), whose
b x and c also cancel when |mean| >> σ.  Max pool 3x3/s2/p1: the forward is exact (bitwise, the first maximum in (ky, kx)
order wins); the backward sums at most four dy per input in fp32.  MSE: dout = 2 (out - t) gscale / n; the loss is a
two-stage fp32 sum.
On an H100 80GB HBM3 (700 W power limit) test_gpu_conv_elementwise.py and test_gpu_batchnorm_elementwise.py reach at most,
at C_ACC = 2: conv fprop 0.992, dgrad 0.993, wgrad 0.994 and stem 0.984 / 0.926 (bf16 outputs, filled by their rounding
term); epilogue statistics 0.065, fused S1 / S2 0.037; BatchNorm y and dx 0.996, mean 0.11, rstd 0.12 (0.061 with every
channel at |mean| = 64σ), running statistics 0.38, dgamma / dbeta 0.073; max pool 0.996; MSE dout 0.996, loss 0.033.

Cross-entropy (the last section; its derivation is in lm_loss_reference's docstring).  The references take the kernels'
own bf16 logits (gemm_nt of the same operands) as exact inputs, so the softmax bounds stay at fp32 level: the error of
each term exp(x_j - m) is carried by __expf's documented 2 + ⌊1.173 |x|⌋ ulp over the arguments along its path (they
add up to m - x_j), the rescales and the fp32 sums in the kernels' order; lse takes Σ p_j ρ_j, __logf and the final add.
The gradients (dh, dw, dbias of the fused head; dlogits of xent_fwd_bwd) take that error times p, the coefficient's
roundings and the GEMM or column-sum bound.  On an H100 80GB HBM3 (700 W power limit) test_gpu_lm_loss_elementwise.py
reaches at most, over two runs: lse 0.34, row_loss 0.70, loss 0.11 (fp32); dh 0.93, dw 0.98, dbias 0.79 (bf16, filled
by their rounding term); xent_fwd_bwd dlogits 0.99 in bf16 and 0.29 in fp32, through autograd with g = 0.7: 0.80 / 0.20;
loss 0.091.  The grouped expert GEMMs of test_gpu_moe.py take the GEMM bound at C_ACC = 2 and reach 0.99.

Set B200DDP_NUMERICS_LOG to a file path to append "<group> <largest error / bound>" for every check, which is how C_ACC
is recalibrated after a kernel change.
"""
import math
import os

import torch
import torch.nn.functional as F

U = 2.0 ** -24                # unit roundoff of fp32
C_ACC = 2.0                   # tensor-core accumulation, in multiples of the recursive-summation bound
GELU_LIPSCHITZ = 1.13         # max |d gelu / dz| = 1.1289...
ERF_ULPS = 8.0                # erff and the two products around it, in units of u relative to |z|
FLOOR = 2.0 ** -60
ROUNDING = {torch.bfloat16: 2.0 ** -8, torch.float32: 2.0 ** -23}


def rounding(dtype):
    """Relative error of rounding a value to `dtype` (round to nearest)."""
    return ROUNDING[dtype]


def activation64(z, epilogue):
    if epilogue == 2:
        return torch.relu(z)
    if epilogue == 3:
        return 0.5 * z * (1.0 + torch.erf(z * (1.0 / math.sqrt(2.0))))
    return z


def gemm_reference(a, b, bias=None, epilogue=0, c_acc=None):
    """fp64 reference of act(a bᵀ + bias) for a [M, K], b [N, K] (bf16, logical layout) and the element-wise bound of the
    fp32 accumulation and activation, both [M, N] float64.  epilogue: 0 none, 1 bias, 2 bias + ReLU, 3 bias + erf-GELU."""
    c_acc = C_ACC if c_acc is None else c_acc
    A, B = a.double(), b.double()
    z = A @ B.t()
    P = A.abs() @ B.abs().t()
    terms = a.shape[1]
    if epilogue >= 1 and bias is not None:
        z = z + bias.double()
        P = P + bias.double().abs()
        terms += 1
    acc = c_acc * terms * U * P
    if epilogue == 3:
        acc = GELU_LIPSCHITZ * acc + ERF_ULPS * U * z.abs()
    return activation64(z, epilogue), acc


def bound(ref, acc, dtype):
    """Total element-wise bound: computation (`acc`) plus rounding the computed value (within `acc` of `ref`) to the output
    dtype, plus the floor."""
    r = rounding(dtype)
    return (1.0 + r) * acc + r * ref.abs() + FLOOR


def _where(idx, shape):
    out = []
    for s in reversed(shape):
        out.append(idx % s)
        idx //= s
    return tuple(reversed(out))


def check(name, got, ref, bnd, group=None):
    """Assert |got - ref| <= bnd element by element (NaN fails).  On failure the message names the worst element (its
    index, value, reference and bound) and how many elements fail.  Returns the largest error / bound."""
    assert got.shape == ref.shape, f"{name}: shape {tuple(got.shape)} != reference {tuple(ref.shape)}"
    err = (got.double() - ref).abs()
    ratio = torch.nan_to_num(err / bnd, nan=math.inf)
    worst = float(ratio.max()) if ratio.numel() else 0.0
    log = os.environ.get("B200DDP_NUMERICS_LOG")
    if log and group is not None:
        with open(log, "a") as f:
            f.write(f"{group} {worst:.6g}\n")
    if not worst <= 1.0:
        bad = int((ratio > 1.0).sum())
        i = int(ratio.reshape(-1).argmax())
        where = _where(i, tuple(ref.shape))
        raise AssertionError(f"{name}: {bad} of {ref.numel()} elements out of bound; worst at {where}: "
                             f"got {float(got.reshape(-1)[i])!r}, reference {float(ref.reshape(-1)[i])!r}, "
                             f"bound {float(bnd.reshape(-1)[i]):.3g} (error / bound {worst:.3g})")
    return worst


def check_gemm(name, got, a, b, bias=None, epilogue=0, group=None, c_acc=None):
    """check() of a GEMM output `got` [M, N] (bf16 or fp32) against gemm_reference."""
    ref, acc = gemm_reference(a, b, bias, epilogue, c_acc)
    return check(name, got, ref, bound(ref, acc, got.dtype), group)


def column_stats_reference(d, group_rows=32):
    """Per-group column sums and sums of squares of the stored output d [M, N] over groups of `group_rows` rows (rows past M
    count as zero): reference [2, G, N] float64 and its bound group_rows · u · Σ|terms| per group."""
    M, N = d.shape
    G = (M + group_rows - 1) // group_rows
    x = torch.zeros(G * group_rows, N, dtype=torch.float64, device=d.device)
    x[:M] = d.double()
    x = x.view(G, group_rows, N)
    sq = x * x
    ref = torch.stack([x.sum(1), sq.sum(1)])
    mag = torch.stack([x.abs().sum(1), sq.sum(1)])
    return ref, group_rows * U * mag + FLOOR


def layernorm_reference(x, gamma, beta, eps, rms=False):
    """fp64 reference of LayerNorm (or RMSNorm: no mean, no beta) over the last dim of x [R, n], and element-wise bounds of
    the fp32 kernel before output rounding: {"y": (ref, acc), "mean": (ref, bnd), "rstd": (ref, bnd)}."""
    X = x.double()
    n = X.shape[1]
    mu = torch.zeros(X.shape[0], dtype=torch.float64, device=X.device) if rms else X.mean(1)
    d = X - mu[:, None]
    ssq = (d * d).sum(1)
    var = ssq / n
    rs = 1.0 / torch.sqrt(var + eps)
    xn = d * rs[:, None]
    g = gamma.double()
    y = xn * g
    if not rms:
        y = y + beta.double()
    # mean: one fp32 sum of n terms; rstd: the sum of squares (n terms, plus the shift by the computed mean), the scale,
    # + eps and rsqrtf (2 ulp)
    d_mu = torch.zeros_like(mu) if rms else n * U * X.abs().mean(1)
    rel_rs = 0.5 * (n * U + 4 * U + n * d_mu ** 2 / torch.clamp(ssq, min=1e-300)) + 8 * U
    acc_y = g.abs() * rs[:, None] * (d_mu[:, None] + d.abs() * (rel_rs[:, None] + 3 * U))
    acc_y = acc_y + 2 * U * (y.abs() + (xn * g).abs())
    return {"y": (y, acc_y), "mean": (mu, d_mu + FLOOR), "rstd": (rs, rs * rel_rs + FLOOR)}


def layernorm_bwd_reference(dy, x, gamma, mean, rstd, rms=False):
    """fp64 reference of the LayerNorm (RMSNorm) backward at the given fp32 mean / rstd (taken as exact inputs) and the
    bounds of the fp32 kernel before output rounding: {"dx": (ref, acc), "dgamma": (ref, acc), "dbeta": (ref, acc)}."""
    X, DY, G = x.double(), dy.double(), gamma.double()
    R, n = X.shape
    m = torch.zeros(R, dtype=torch.float64, device=X.device) if rms else mean.double()
    s = rstd.double()
    xn = (X - m[:, None]) * s[:, None]
    dg = DY * G
    s1 = torch.zeros_like(s) if rms else dg.mean(1)
    t = dg * xn
    s2 = t.mean(1)
    dx = s[:, None] * (dg - s1[:, None] - xn * s2[:, None])
    m1 = dg.abs().mean(1)
    m2 = t.abs().mean(1)
    acc_dx = s[:, None] * (n * U * ((0 if rms else m1[:, None]) + xn.abs() * m2[:, None])
                           + 8 * U * (dg.abs() + s1.abs()[:, None] + m1[:, None] + xn.abs() * (s2.abs() + m2)[:, None]))
    dyxn = DY * xn
    dgamma = dyxn.sum(0)
    dbeta = DY.sum(0)
    acc_dgamma = (R + 4) * U * dyxn.abs().sum(0)
    acc_dbeta = R * U * DY.abs().sum(0)
    return {"dx": (dx, acc_dx), "dgamma": (dgamma, acc_dgamma), "dbeta": (dbeta, acc_dbeta)}


def rel_err(a, b):
    """The global relative error the older GEMM tests assert below 1e-2: it cannot see a local error."""
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-12))


# ---- attention ----------------------------------------------------------------------------------------------------------
# Per (batch row, query head), with scale c, visible set V_i of query i and n_i = |V_i|.  The kernels compute the scores
# s = c q kᵀ in fp32 on the tensor cores, p = exp2(s log2e - m log2e) against the running row maximum m (rescaling the
# accumulators by alpha = exp2((m_old - m) log2e) once per key tile of 128 they visit), round p to bf16 for P V, and
# divide by the fp32 sum of the unrounded p.  The backward recomputes P' = exp(s - lse) from the forward's own lse, forms
# dS = P' (dO vᵀ - D) with D = rowsum(dO o) from the forward's own o, and rounds P' and dS to bf16 before the products
# dV = P'ᵀ dO, dK = c dSᵀ q and dQ = c dS k.  So, with A = C_ACC d u |q||k|ᵀ the score error:
#   rho_ij   relative error of one unnormalised p: c A_ij + u (EXP_ULPS + 3 + 2 (|s_ij| + max_j |s_ij|)) + (EXP_ULPS + 3) u T_i
#            (the exponent's rounding is absolute, so it grows with |s| and the maximum; T_i key tiles rescale the sums)
#   o        (P (2⁻⁸ + rho)) |V| + C_ACC (n_i + 1) u P|V| + |o| (sum_j P_ij rho_ij + (n_i + 2) u), then the bf16 rounding
#   lse      sum_j P_ij rho_ij + (n_i + 2) u + 2 u (|lse| + 1)
#   dS       P' rho' |dP - D| + P' (err dP + err D) + 2 u |dS|, plus 2⁻⁸ for its bf16 rounding (rho': |lse| for the maximum,
#            no rescale), with err dP = C_ACC d u |dO||v|ᵀ and err D = d u sum |dO o|
#   dV dK dQ that error times |dO|, |q| or |k|, plus C_ACC (m + 1) u times the absolute product over the m summed terms,
#            plus u for the multiply by c when c is not a power of two, then the bf16 rounding
# EXP_ULPS is exp2f's documented maximum error; the build does not use --use_fast_math, so exp2f, logf and 1 / l are the
# accurate versions.
EXP_ULPS = 2.0
BF16_U = 2.0 ** -8            # P and dS are rounded to bf16 before their products
ATTN_BLOCK = 1 << 22          # elements of one [B, H, rows, S] block of the attention references (32 MB in float64)
KEY_TILE = 128                # keys per forward tile (one online-softmax rescale each)


def attention_visible(mask, S, causal=False):
    """[B, S, S] bool, query i sees key j.  mask: seq_lens int [B] (key j is visible iff j < len, len clamped to [0, S] as
    the kernels' clamped_len does) or bounds int [B, S, 2] (start clamped to [0, S], end to [start, S] as row_bounds
    does); causal also needs j <= i."""
    j = torch.arange(S, device=mask.device)
    if mask.dim() == 1:
        n = mask.long().clamp(0, S)
        return (j[None, None, :] < n[:, None, None]).expand(-1, S, -1).contiguous()
    b = mask.long().reshape(-1, S, 2)
    start = b[..., 0].clamp(0, S)
    end = torch.maximum(b[..., 1], start).clamp(max=S)
    vis = (j >= start[..., None]) & (j < end[..., None])
    if causal:
        vis &= j[None, None, :] <= j[None, :, None]
    return vis


def _attn_chunks(B, H, S):
    rows = max(16, min(1024, ATTN_BLOCK // (B * H * S)))
    return [(r, min(r + rows, S)) for r in range(0, S, rows)]


def _by_batch_row(fn, tensors, visible, args):
    """fn on one batch row at a time, its (ref, bound) pairs concatenated: keeps the [B, H, S, d] terms of a wide problem
    small."""
    parts = [fn(*(t[b:b + 1] for t in tensors), visible[b:b + 1], *args) for b in range(visible.shape[0])]
    return {key: tuple(torch.cat([p[key][i] for p in parts]) for i in range(2)) for key in parts[0]}


def _kv_per_query_head(t, H):
    """K or V [B, Hkv, S, d] as float64 [B, H, S, d]: query head h reads K/V head h // (H // Hkv)."""
    return t.double().repeat_interleave(H // t.shape[1], dim=1)


def _scale_ulps(scale):
    return 0.0 if math.frexp(scale)[0] == 0.5 else 1.0


def attention_reference(q, k, v, visible, scale, c_acc=None, exp_ulps=None):
    """fp64 softmax attention of q [B, H, S, d] over k, v [B, Hkv, S, d] (bf16) where visible [B, S, S] allows, and the
    element-wise bounds of the kernels' arithmetic: {"o": (ref, acc) [B, H, S, d], "lse": (ref, bnd) [B, H, S]}.  A row
    that sees no key has o = 0 and lse = -inf, with bound 0 (plus bound()'s floor for o)."""
    c_acc = C_ACC if c_acc is None else c_acc
    e = EXP_ULPS if exp_ulps is None else exp_ulps
    B, H, S, d = q.shape
    if B > 1 and B * H * S * d > ATTN_BLOCK:
        return _by_batch_row(attention_reference, (q, k, v), visible, (scale, c_acc, exp_ulps))
    K, V = _kv_per_query_head(k, H), _kv_per_query_head(v, H)
    o = torch.zeros(B, H, S, d, dtype=torch.float64, device=q.device)
    o_acc = torch.zeros_like(o)
    lse = torch.zeros(B, H, S, dtype=torch.float64, device=q.device)
    lse_bnd = torch.zeros_like(lse)
    for r0, r1 in _attn_chunks(B, H, S):
        Q = q[:, :, r0:r1].double()
        vis = visible[:, None, r0:r1]
        s = scale * (Q @ K.transpose(-1, -2))
        A = c_acc * d * U * (Q.abs() @ K.abs().transpose(-1, -2))
        n = vis.sum(-1).double()
        tiles = vis.reshape(B, 1, r1 - r0, S // KEY_TILE, KEY_TILE).any(-1).sum(-1).double()
        l = torch.logsumexp(s.masked_fill(~vis, -math.inf), -1)
        live = torch.isfinite(l)
        P = torch.where(vis, torch.exp(s - torch.where(live, l, 0.0)[..., None]), 0.0)
        smax = torch.where(vis, s.abs(), 0.0).amax(-1, keepdim=True)
        rho = scale * A + U * (e + 3 + 2 * (s.abs() + smax)) + (e + 3) * U * tiles[..., None]
        Prho = P * rho
        sum_prho = Prho.sum(-1)
        oc = P @ V
        o[:, :, r0:r1] = oc
        Va = V.abs()
        o_acc[:, :, r0:r1] = ((BF16_U * P + Prho) @ Va + (c_acc * U * (n + 1))[..., None] * (P @ Va)
                              + oc.abs() * (sum_prho + (n + 2) * U)[..., None])
        lse[:, :, r0:r1] = l
        lse_bnd[:, :, r0:r1] = torch.where(live, sum_prho + (n + 2) * U + 2 * U * (torch.where(live, l, 0.0).abs() + 1), 0.0)
    return {"o": (o, o_acc), "lse": (lse, lse_bnd)}


def attention_bwd_reference(q, k, v, o, lse, dout, visible, scale, c_acc=None, exp_ulps=None):
    """fp64 gradients of attention_reference at the kernel's own o [B, H, S, d] (bf16) and lse [B, H, S] (fp32), taken
    as exact inputs, for the output gradient dout [B, H, S, d] (bf16), and the bounds of the kernels' arithmetic before
    output rounding: {"dq": (ref, acc) [B, H, S, d], "dk": ..., "dv": ... [B, Hkv, S, d]}; dK and dV sum each group of
    query heads.  A query whose lse is -inf has P' = 0."""
    c_acc = C_ACC if c_acc is None else c_acc
    e = EXP_ULPS if exp_ulps is None else exp_ulps
    B, H, S, d = q.shape
    if B > 1 and B * H * S * d > ATTN_BLOCK:
        return _by_batch_row(attention_bwd_reference, (q, k, v, o, lse, dout), visible, (scale, c_acc, exp_ulps))
    Hkv = k.shape[1]
    K, V = _kv_per_query_head(k, H), _kv_per_query_head(v, H)
    su = _scale_ulps(scale)
    dq = torch.zeros(B, H, S, d, dtype=torch.float64, device=q.device)
    dq_acc = torch.zeros_like(dq)
    dk, dk_mag, dk_err, dv, dv_mag, dv_err = (torch.zeros(B, Hkv, S, d, dtype=torch.float64, device=q.device)
                                              for _ in range(6))
    m = torch.zeros(B, Hkv, S, dtype=torch.float64, device=q.device)

    def group(t):                                               # the sum over each group of query heads
        return t.reshape(B, Hkv, H // Hkv, *t.shape[2:]).sum(2)
    for r0, r1 in _attn_chunks(B, H, S):
        Q, dO, O = (t[:, :, r0:r1].double() for t in (q, dout, o))
        L = lse[:, :, r0:r1].double()
        live = torch.isfinite(L)
        Lz = torch.where(live, L, 0.0)[..., None]
        vis = visible[:, None, r0:r1] & live[..., None]
        s = scale * (Q @ K.transpose(-1, -2))
        A = c_acc * d * U * (Q.abs() @ K.abs().transpose(-1, -2))
        P = torch.where(vis, torch.exp(s - Lz), 0.0)
        dP = dO @ V.transpose(-1, -2)
        err_dP = c_acc * d * U * (dO.abs() @ V.abs().transpose(-1, -2))
        D = (dO * O).sum(-1, keepdim=True)
        err_D = d * U * (dO * O).abs().sum(-1, keepdim=True)
        dS = P * (dP - D)
        rho = scale * A + U * (e + 3 + 2 * (s.abs() + Lz.abs()))
        err_dS = P * rho * (dP - D).abs() + P * (err_dP + err_D) + 2 * U * dS.abs()
        err_dS = err_dS + BF16_U * (dS.abs() + err_dS)
        err_P = P * (rho + BF16_U * (1 + rho))
        dSa = dS.abs()
        n = vis.sum(-1).double()
        dq[:, :, r0:r1] = scale * (dS @ K)
        Ka = K.abs()
        dq_acc[:, :, r0:r1] = scale * (err_dS @ Ka + (U * (c_acc * (n + 1) + su))[..., None] * (dSa @ Ka))
        m += group(vis.sum(-2).double())
        Pt, dSt = P.transpose(-1, -2), dS.transpose(-1, -2)
        dv += group(Pt @ dO)
        dv_mag += group(Pt @ dO.abs())
        dv_err += group(err_P.transpose(-1, -2) @ dO.abs())
        dk += group(dSt @ Q)
        dk_mag += group(dSa.transpose(-1, -2) @ Q.abs())
        dk_err += group(err_dS.transpose(-1, -2) @ Q.abs())
    m = m[..., None]
    return {"dq": (dq, dq_acc),
            "dk": (scale * dk, scale * (dk_err + U * (c_acc * (m + 1) + su) * dk_mag)),
            "dv": (dv, dv_err + c_acc * U * (m + 1) * dv_mag)}


def check_lse(name, got, ref, bnd, group=None):
    """check() of an lse [B, H, S]: -inf exactly where the reference is -inf, the finite entries element by element."""
    dead = torch.isneginf(ref)
    wrong = torch.isneginf(got) != dead
    if wrong.any():
        i = int(wrong.reshape(-1).nonzero()[0])
        raise AssertionError(f"{name}: {int(wrong.sum())} of {ref.numel()} entries are -inf where the reference is not or "
                             f"the reverse; first at {_where(i, tuple(ref.shape))}: got {float(got.reshape(-1)[i])!r}, "
                             f"reference {float(ref.reshape(-1)[i])!r}")
    return check(name, torch.where(dead, 0.0, got.double()), torch.where(dead, 0.0, ref), bnd + FLOOR, group)


def check_attention(name, got, ref, group=None):
    """Checks every output in `got` ({"o", "lse"} or {"dq", "dk", "dv"}, kernel outputs in the references' layouts) against
    the (ref, acc) pairs of attention_reference / attention_bwd_reference; groups log as "<group> <output>".  Returns the
    largest error / bound per output."""
    worst = {}
    for key, t in got.items():
        r, a = ref[key]
        g = None if group is None else f"{group} {key}"
        if key == "lse":
            worst[key] = check_lse(f"{name}: lse [b, h, s]", t, r, a, g)
        else:
            worst[key] = check(f"{name}: {key} [b, h, s, d]", t, r, bound(r, a, t.dtype), g)
    return worst


# ---- ResNet-50: convolutions, BatchNorm, max pool, MSE --------------------------------------------------------------------
# (The bounds of this section are documented in the module docstring.)


def _conv64(t):
    return t.double().contiguous()


def conv_reference(direction, a, b, stride=1, pad=0, shape=None, addend=None, k_pixels=None, reduce_depth=0, c_acc=None):
    """fp64 reference and accumulation bound (before output rounding) of one convolution, both float64 in the output's logical
    NCHW shape.  direction "fprop": a = x, b = w; "dgrad": a = dy, b = w, shape = x's shape, optional fp32 addend added
    before rounding; "wgrad": a = dy, b = x, shape = w's shape, k_pixels = the pixels one split sums, reduce_depth = the
    longest fp32 chain of the split reduction."""
    from torch.nn.grad import conv2d_input, conv2d_weight
    c_acc = C_ACC if c_acc is None else c_acc
    A, B = _conv64(a), _conv64(b)
    if direction == "fprop":
        ref = F.conv2d(A, B, None, stride, pad)
        P = F.conv2d(A.abs(), B.abs(), None, stride, pad)
        K = b.shape[1] * b.shape[2] * b.shape[3]
    elif direction == "dgrad":
        ref = conv2d_input(tuple(shape), B, A, stride, pad)
        P = conv2d_input(tuple(shape), B.abs(), A.abs(), stride, pad)
        K = b.shape[0] * b.shape[2] * b.shape[3]
        if addend is not None:
            ref = ref + addend.double()
            P = P + addend.double().abs()
            K += 1
    elif direction == "wgrad":
        ref = conv2d_weight(B, tuple(shape), A, stride, pad)
        P = conv2d_weight(B.abs(), tuple(shape), A.abs(), stride, pad)
        K = k_pixels
    else:
        raise ValueError(direction)
    return ref, (c_acc * (K + 1) + reduce_depth) * U * P


def conv_epilogue_depth(tiles_per_cta):
    """Longest fp32 chain of the conv epilogue's per-CTA column sums: 32 rows per warp, one add per tile, 4 warps."""
    return 32 + tiles_per_cta + 4


SMS = 132                     # kNumSMs: the persistent and two-pass grids are sized for the H100 SXM


def _ceil(a, b):
    return -(-a // b)


def conv_grid_tiles(num_m_tiles, num_n_tiles, stats=True):
    """(grid, tiles per CTA) of conv_grid_size: the persistent conv grid, a multiple of the n-tiles with statistics."""
    tiles = num_m_tiles * num_n_tiles
    grid = min(tiles, SMS)
    if stats and num_n_tiles > 1:
        grid = max((grid // num_n_tiles) * num_n_tiles, num_n_tiles)
    return grid, _ceil(tiles, grid)


def bn_pick_tile(R, C):
    """(cvb, ty, grid_x, grid_y) of batchnorm.cu's pick_tile: channel vectors per block, row lanes, channel tiles, row splits."""
    cv = C // 8
    cvb = min(cv, 8)
    while 256 % cvb:
        cvb -= 1
    ty = 256 // cvb
    grid_x = _ceil(cv, cvb)
    return cvb, ty, grid_x, min(_ceil(4 * SMS, grid_x), max(R // (ty * 4), 1), 256)


def bn_two_pass_depth(R, C, fused=False):
    """Longest fp32 chain of the two-pass (and fused) stats / reduce kernels: rows per thread + row lanes + the finishing
    block's strided split lanes + its combine of the lanes."""
    cvb, ty, grid_x, S = bn_pick_tile(R, C)
    if fused:
        S = min(S, max(1, (2 * SMS) // grid_x))
    lanes = max(1, 256 // (cvb * 8))
    return _ceil(_ceil(R, S), ty) + ty + _ceil(S, lanes) + lanes


def as_rows(t):
    """A channels_last activation [N, C, H, W] as the [N*H*W, C] matrix the BatchNorm kernels see."""
    return t.permute(0, 2, 3, 1).reshape(-1, t.shape[1])


def unpack_mask(mask, C):
    """uint8 [R, C/8] ReLU bitmask (bit i of byte v = channel 8 v + i) as bool [R, C]."""
    bits = torch.arange(8, device=mask.device, dtype=torch.uint8)
    return ((mask.reshape(-1, C // 8, 1) >> bits) & 1).bool().reshape(-1, C)


def batchnorm_reference(x, gamma, beta, eps, depth, residual=None, relu=False, momentum=0.0, running_mean=None,
                        running_var=None):
    """fp64 training BatchNorm of x [R, C] (the stored input) and the bounds of the kernels' fp32 arithmetic, with `depth`
    the longest chain of the per-channel sums: {"y": (ref, acc) [R, C] before output rounding, "mean", "rstd",
    "running_mean", "running_var": (ref, bnd) [C]}."""
    X = x.double()
    R = X.shape[0]
    g, b = gamma.double(), beta.double()
    A1, A2 = X.abs().sum(0), (X * X).sum(0)
    mean = X.sum(0) / R
    E2 = A2 / R
    var = torch.clamp(E2 - mean * mean, min=0.0)
    d_mean = (depth * U * A1 + 3 * U * A1) / R
    d_E2 = (depth * U * A2 + 3 * U * A2) / R
    d_var = d_E2 + (2 * mean.abs() + d_mean) * d_mean + U * (mean.abs() + d_mean) ** 2 + U * (E2 + d_E2)
    rs = 1.0 / torch.sqrt(var + eps)
    v_lo = (torch.clamp(var - d_var, min=0.0) + eps) * (1 - U)
    v_hi = (var + d_var + eps) * (1 + U)
    d_rs = torch.maximum(v_lo.rsqrt() - rs, rs - v_hi.rsqrt()) + 4 * U * v_lo.rsqrt()
    sc = g * rs
    d_sc = g.abs() * d_rs + U * g.abs() * (rs + d_rs)
    ms = mean * sc
    d_ms = mean.abs() * d_sc + sc.abs() * d_mean + d_mean * d_sc + U * (mean.abs() + d_mean) * (sc.abs() + d_sc)
    sh = b - ms
    d_sh = d_ms + U * (b.abs() + ms.abs() + d_ms)
    xs = X * sc
    z = xs + sh
    acc = X.abs() * d_sc + d_sh + U * (X.abs() * (sc.abs() + d_sc) + sh.abs() + d_sh)
    if residual is not None:
        Rr = residual.double()
        z = z + Rr
        acc = acc + U * (z.abs() + acc)
    y = torch.relu(z) if relu else z
    out = {"y": (y, acc), "mean": (mean, d_mean + FLOOR), "rstd": (rs, d_rs + FLOOR)}
    if running_mean is not None:
        m = float(torch.tensor(momentum, dtype=torch.float32))
        rm0, rv0 = running_mean.double(), running_var.double()
        f = R / (R - 1) if R > 1 else 1.0
        rm = (1 - m) * rm0 + m * mean
        rv = (1 - m) * rv0 + m * f * var
        out["running_mean"] = (rm, m * d_mean + 4 * U * ((1 - m) * rm0.abs() + m * mean.abs()) + FLOOR)
        out["running_var"] = (rv, m * f * d_var + 6 * U * ((1 - m) * rv0.abs() + m * f * var) + FLOOR)
    return out


def batchnorm_bwd_reference(dy, x, mask, gamma, mean, rstd, depth):
    """fp64 BatchNorm backward of dy, x [R, C] at the kernel's own fp32 mean / rstd [C] and ReLU mask (bool [R, C] or None),
    all taken as exact inputs, with `depth` the longest chain of the sums S1 = Σ dy*, S2 = Σ dy* x̂ (dy* = dy m), and the bounds
    of the kernels' fp32 arithmetic before output rounding: {"dx": (ref, acc) [R, C], "dgamma": S2, "dbeta": S1 (ref, acc) [C]}."""
    X, DY = x.double(), dy.double()
    R = X.shape[0]
    G = DY if mask is None else torch.where(mask, DY, 0.0)
    m, s, gam = mean.double(), rstd.double(), gamma.double()
    xh = (X - m) * s
    gx = G * xh
    S1, S2 = G.sum(0), gx.sum(0)
    A1, A2 = G.abs().sum(0), gx.abs().sum(0)
    e1 = depth * U * A1
    e2 = (depth + 3) * U * A2
    c1, c2 = S1 / R, S2 / R
    d_c1, d_c2 = (e1 + 3 * U * A1) / R, (e2 + 3 * U * A2) / R
    ka = gam * s
    d_ka = U * ka.abs()
    kr = (ka * s).abs()
    d_kb = kr * d_c2 + 3 * U * kr * (c2.abs() + d_c2)
    mr = (m * s).abs()
    t = m * s * c2
    d_t = mr * d_c2 + 3 * U * mr * (c2.abs() + d_c2)
    inner = (c1 - t).abs()
    d_inner = d_c1 + d_t + U * (c1.abs() + t.abs() + d_c1 + d_t)
    d_kc = ka.abs() * d_inner + 2 * U * ka.abs() * (inner + d_inner)
    kb, kc = -ka * s * c2, -ka * (c1 - t)
    zx = kb * X + kc
    d_z = X.abs() * d_kb + d_kc + U * ((kb * X).abs() + kc.abs() + X.abs() * d_kb + d_kc)
    dx = ka * (G - c1 - xh * c2)
    acc = G.abs() * d_ka + d_z + U * ((ka * G).abs() + zx.abs() + G.abs() * d_ka + d_z)
    return {"dx": (dx, acc * (1 + 8 * U)), "dgamma": (S2, e2 + FLOOR), "dbeta": (S1, e1 + FLOOR)}


def maxpool_reference(x):
    """3x3 / stride 2 / pad 1 max pool of x [N, C, H, W]: (y, slot) with the first maximum in (ky, kx) order winning, exact."""
    N, C, H, W = x.shape
    OH, OW = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    xp = F.pad(x.double(), (1, 1, 1, 1), value=-math.inf)
    best = torch.full((N, C, OH, OW), -math.inf, dtype=torch.float64, device=x.device)
    slot = torch.zeros(N, C, OH, OW, dtype=torch.uint8, device=x.device)
    for ky in range(3):
        for kx in range(3):
            v = xp[:, :, ky:ky + 2 * OH - 1:2, kx:kx + 2 * OW - 1:2]
            take = v > best
            best = torch.where(take, v, best)
            slot = torch.where(take, ky * 3 + kx, slot).to(torch.uint8)
    return best.to(x.dtype), slot


def maxpool_bwd_reference(dy, slot, H, W):
    """fp64 gradient of the max pool at its recorded window slots, and the bound of summing <= 4 dy per input in fp32."""
    N, C, OH, OW = dy.shape
    D = dy.double()
    dx = torch.zeros(N, C, 2 * OH + 1, 2 * OW + 1, dtype=torch.float64, device=dy.device)
    mag = torch.zeros_like(dx)
    for ky in range(3):
        for kx in range(3):
            g = torch.where(slot == ky * 3 + kx, D, 0.0)
            dx[:, :, ky:ky + 2 * OH:2, kx:kx + 2 * OW:2] += g
            mag[:, :, ky:ky + 2 * OH:2, kx:kx + 2 * OW:2] += g.abs()
    dx, mag = dx[:, :, 1:H + 1, 1:W + 1], mag[:, :, 1:H + 1, 1:W + 1]
    return dx, 4 * U * mag


def mse_reference(out, target, gscale, blocks, threads=256):
    """fp64 MSE loss and gradient 2 (out - t) gscale / n of out, target (any shape) and the bounds of the kernel's fp32
    arithmetic before output rounding: {"loss": (ref, bnd), "dout": (ref, acc)}.  The loss is a per-thread chain over a
    grid-stride loop, two warp trees per block, then the last block's chain over the block partials."""
    O, T = out.double(), target.double()
    n = O.numel()
    d = O - T
    dout = 2.0 * gscale / n * d
    stride = blocks * threads
    depth = -(-n // stride) + 8 + 10 + -(-blocks // threads) + 10
    loss = (d * d).sum() / n
    return {"loss": (loss, (depth + 6) * U * loss + FLOOR), "dout": (dout, 6 * U * dout.abs())}


# ---- cross-entropy: the fused LM head (kLmLse / kLmDlogits, lm_lse_combine, column_sum) and xent_fwd_bwd ------------------
# (The bounds of this section are derived in the docstring of lm_loss_reference.)
EXPF_ULPS = 2.0               # __expf(x): 2 + floor(EXPF_SLOPE |x|) ulp (CUDA C++ Programming Guide, intrinsic functions)
EXPF_SLOPE = 1.173
LOGF_ABS = 2.0 ** -21.41      # __logf(x): absolute error 2^-21.41 on [0.5, 2], otherwise 3 ulp
LOGF_ULPS = 3.0
FTZ = 2.0 ** -126             # the intrinsics flush subnormal results: an absolute error below the smallest normal
LM_TILE, LM_CHUNK = 128, 32   # kLmLse: 128-column tiles, four 32-column chunks, one online (max, sum) rescale per chunk
COMBINE_GROUPS = 8            # lm_lse_combine: thread y merges tiles y, y + 8, ..., then the 8 groups are merged
XENT_THREADS = 256            # xent_fwd_bwd: one block of 256 per row (block_max / block_sum)
FINISH_THREADS = 1024         # xent_finish_kernel / count_valid_kernel
COLSUM_ROWS = 128             # column_sum: an fp32 chain of 128 rows per chunk, then one add per chunk
XENT_BLOCK = 1 << 22          # fp64 elements of one row block of the cross-entropy references (32 MB)


def lm_labelled(t, V, ignore_index=-100):
    """bool [N]: the row carries a label (not ignore_index, 0 <= t < V), the kernels' rule."""
    return (t != ignore_index) & (t >= 0) & (t < V)


def xent_row_blocks(N, V):
    rows = max(1, XENT_BLOCK // max(V, 1))
    return [(r, min(r + rows, N)) for r in range(0, N, rows)]


def lm_lse_depths(V):
    """(__expf calls, other fp32 roundings) on one term's path through kLmLse and lm_lse_combine at vocabulary V."""
    tiles = _ceil(V, LM_TILE)
    merges = _ceil(tiles, COMBINE_GROUPS) - 1 + (COMBINE_GROUPS - 1)
    return 1 + (LM_TILE // LM_CHUNK - 1) + merges, LM_CHUNK + 2 * (LM_TILE // LM_CHUNK) + 2 * merges


def xent_depths(cols):
    """(__expf calls, other fp32 roundings) of one term of xent_fwd_bwd's sum: a strided chain per thread, two warp trees."""
    return 1, _ceil(cols, XENT_THREADS) + 10


def _lse64(X, n_exp, n_ops):
    """fp64 lse of the rows of X (float64 [r, V], -inf = no column) and its bound: (lse, bound, P = softmax, M = max)."""
    M = X.amax(1, keepdim=True)
    gap = (M - X).nan_to_num(posinf=0.0)                      # m - x_j: the arguments of a term's __expf calls add up to it
    E = torch.exp(X - M)
    S = E.sum(1, keepdim=True)
    P = E / S
    rho = 2 * U * (EXPF_ULPS * n_exp + EXPF_SLOPE * gap) + U * gap + U * n_ops
    delta = (P * rho).sum(1) + (X.shape[1] + n_exp) * FTZ
    logS = torch.log(S[:, 0])
    lse = M[:, 0] + logS
    bnd = delta / (1 - delta) + LOGF_ABS + 2 * U * LOGF_ULPS * logS.abs() + U * lse.abs() + FLOOR
    return lse, bnd, P, M[:, 0]


def lm_loss_reference(X, t, V, ignore_index=-100, finish=True):
    """fp64 lse [N], row_loss [N] and loss of the fused forward from the kernel's own bf16 logits X [N, V] (gemm_nt of
    the same hidden, weight and bias: the epilogue sees exactly the logits the unfused head GEMM stores), with their
    element-wise bounds: {"lse": (ref, bnd), "row_loss": (ref, bnd), "loss": (ref, bnd)}.

    Judging the softmax from X, not from the fp64 product, keeps the bounds at fp32 level: a dropped or shifted column
    moves lse by p_j, far more than the bound.  With u = 2⁻²⁴, one fp32 ulp is at most 2u of the value, and m the row max:
      one term   exp(x_j - m) carries a relative error ρ_j = 2u (2 n_exp + 1.173 (m - x_j)) + u (m - x_j) + u n_ops: each
                 of its n_exp __expf calls costs 2 + ⌊1.173 |arg|⌋ ulp, and along its path (its chunk, the chunk rescales
                 s · exp(m - m'), the combine merges a.y · exp(a.x - m)) the arguments add up to m - x_j, which also bounds
                 their fp32 rounding; n_ops counts the other roundings (the 32-term chunk chain, the rescale products and
                 adds, two per merge).  lm_lse_depths gives n_exp and n_ops.
      lse        Σ_j p_j ρ_j (+ FTZ per term and merge for flushed results) through log(1 + δ) ≤ δ / (1 - δ), plus __logf
                 (2⁻²¹·⁴¹ + 3 ulp) and the add m + log s
      row_loss   lse - x_t rounded once: the kernel's row_loss equals float32(lse_kernel - X[i, t_i]) bitwise
      loss       the xent_finish_kernel sum (a strided chain of ⌈N / 1024⌉ then two warp trees) and the division by the
                 exact count"""
    X = X.double()
    N = X.shape[0]
    n_exp, n_ops = lm_lse_depths(V)
    lse = torch.zeros(N, dtype=torch.float64, device=X.device)
    bnd = torch.zeros_like(lse)
    for r0, r1 in xent_row_blocks(N, V):
        lse[r0:r1], bnd[r0:r1] = _lse64(X[r0:r1], n_exp, n_ops)[:2]
    return _row_loss_and_loss(X, lse, bnd, t, V, ignore_index, finish)


def _row_loss_and_loss(X, lse, bnd, t, V, ignore_index, finish):
    lab = lm_labelled(t, V, ignore_index)
    xt = X.gather(1, torch.where(lab, t, 0)[:, None])[:, 0]
    rl = torch.where(lab, lse - xt, 0.0)
    rl_bnd = torch.where(lab, bnd + U * rl.abs(), 0.0) + FLOOR
    out = {"lse": (lse, bnd), "row_loss": (rl, rl_bnd)}
    if finish:
        cnt = int(lab.sum())
        N = X.shape[0]
        depth = _ceil(N, FINISH_THREADS) + 10 + 1
        c = max(cnt, 1)
        loss = rl.sum() / c if cnt else rl.sum() * 0
        out["loss"] = (loss, (rl_bnd.sum() + depth * U * rl.abs().sum()) / c + U * loss.abs() + FLOOR)
    return out


def lm_dlogits_reference(X, lse, t, V, coef, ignore_index=-100):
    """fp64 D = (exp(X - lse) - [j = t]) · coef of the labelled rows (0 elsewhere) at the kernel's own fp32 lse [N], coef
    = gscale / valid, and the bound of kLmDlogits' fp32 arithmetic before the bf16 rounding: (D, acc) [N, V].  The
    argument x - lse is rounded once and __expf costs 2 + ⌊1.173 |x - lse|⌋ ulp; the target's - 1, coef = gscale / valid
    and the product are one rounding each."""
    X = X.double()
    L = lse.double()[:, None]
    lab = lm_labelled(t, V, ignore_index)[:, None]
    gap = (X - L).abs()
    P = torch.exp(X - L)
    onehot = torch.zeros_like(X, dtype=torch.bool)
    onehot.scatter_(1, torch.where(lab[:, 0], t, 0)[:, None], lab)
    D = torch.where(lab, (P - onehot.double()) * coef, 0.0)
    acc = torch.where(lab, abs(coef) * (P * (2 * U * (EXPF_ULPS + EXPF_SLOPE * gap) + U * gap) + FTZ) + 3 * U * D.abs(), 0.0)
    return D, acc


def lm_grad_reference(X, lse, t, h, w, V, coef, slice_width, ignore_index=-100, bound_k=None, c_acc=None):
    """fp64 dh [N, H], dw [V, H] and dbias [V] of the fused backward at the kernel's own lse, and their bounds before the
    bf16 rounding: {"dh": (ref, acc), "dw": ..., "dbias": ...}.  With D, δD from lm_dlogits_reference (δD including the
    bf16 rounding of the stored dlogits):
      dh     Σ_j δD_ij |W_j| + (C_ACC (vs + 1) + slices) u |D| |W|: per slice of vs columns a tensor-core sum, accumulated
             in fp32 (one add per slice) into the fp32 buffer that is cast to bf16 once
      dw     Σ_i δD_ij |h_i| + C_ACC (K + 1) u |D|ᵀ |h|, K = N (or, row-bounded, the count rounded up to 64)
      dbias  Σ_i δD_ij + (128 + chunks) u Σ_i |D_ij|: column_sum's chain per 128-row chunk, one add per chunk"""
    c_acc = C_ACC if c_acc is None else c_acc
    N, H = h.shape
    vs = min(slice_width, V)
    slices = _ceil(V, vs)
    K = N if bound_k is None else bound_k
    W, Hm = w.double(), h.double()
    Wa, Ha = W.abs(), Hm.abs()
    dh = torch.zeros(N, H, dtype=torch.float64, device=h.device)
    dh_acc = torch.zeros_like(dh)
    dw, dw_mag, dw_err = (torch.zeros(V, H, dtype=torch.float64, device=h.device) for _ in range(3))
    db, db_mag, db_err = (torch.zeros(V, dtype=torch.float64, device=h.device) for _ in range(3))
    for r0, r1 in xent_row_blocks(N, V):
        D, acc = lm_dlogits_reference(X[r0:r1], lse[r0:r1], t[r0:r1], V, coef, ignore_index)
        dD = acc + BF16_U * (D.abs() + acc)                      # and the bf16 rounding of the stored dlogits
        Da = D.abs()
        dh[r0:r1] = D @ W
        dh_acc[r0:r1] = dD @ Wa + (c_acc * (vs + 1) + slices) * U * (Da @ Wa)
        dw += D.t() @ Hm[r0:r1]
        dw_mag += Da.t() @ Ha[r0:r1]
        dw_err += dD.t() @ Ha[r0:r1]
        db += D.sum(0)
        db_mag += Da.sum(0)
        db_err += dD.sum(0)
    chunks = _ceil(max(K, 1), COLSUM_ROWS)
    return {"dh": (dh, dh_acc), "dw": (dw, dw_err + c_acc * (K + 1) * U * dw_mag),
            "dbias": (db, db_err + (COLSUM_ROWS + chunks) * U * db_mag)}


def xent_reference(x, t, ignore_index=-100, gscale=1.0, g=None):
    """fp64 references of xent_fwd_bwd (either kernel) on logits x [N, C] (bf16 or fp32, exact in fp64): {"row_loss",
    "loss": (ref, bnd), "dlogits": (ref, acc) [N, C] before the output rounding}.  Softmax statistics from block_max (exact)
    and block_sum (xent_depths), dlogits = (exp(x - m) coef - g [j = t]) with coef = (gscale / valid) / s or, in the
    streaming kernel, (exp(x - m) / s - [j = t]) g: at most four roundings after the exponential.  g (autograd's upstream
    gradient): the backward multiplies the stored dlogits by g cast to the logits' dtype and rounds again, so acc then
    holds the first rounding, the rounding of g and the error above times |g|."""
    X = x.double()
    N, C = X.shape
    lab = lm_labelled(t, C, ignore_index)
    cnt = int(lab.sum())
    coef = gscale / cnt if cnt else 0.0
    n_exp, n_ops = xent_depths(C)
    lse = torch.zeros(N, dtype=torch.float64, device=x.device)
    bnd = torch.zeros_like(lse)
    D = torch.zeros_like(X)
    acc = torch.zeros_like(X)
    for r0, r1 in xent_row_blocks(N, C):
        Xb = X[r0:r1]
        lse[r0:r1], bnd[r0:r1], P, M = _lse64(Xb, n_exp, n_ops)
        gap = (M[:, None] - Xb)
        delta = bnd[r0:r1, None]                                 # the sum's relative error is within the lse bound
        lb = lab[r0:r1, None]
        onehot = torch.zeros_like(Xb, dtype=torch.bool)
        onehot.scatter_(1, torch.where(lb[:, 0], t[r0:r1], 0)[:, None], lb)
        d = torch.where(lb, (P - onehot.double()) * coef, 0.0)
        e = P * (2 * U * (EXPF_ULPS + EXPF_SLOPE * gap) + U * gap + 2 * delta) + FTZ
        D[r0:r1] = d
        acc[r0:r1] = torch.where(lb, abs(coef) * e + 4 * U * (d.abs() + abs(coef) * P), 0.0)
    out = _row_loss_and_loss(X, lse, bnd + U * lse.abs(), t, C, ignore_index, True)
    if g is not None:
        r = rounding(x.dtype)
        gq = float(torch.tensor(g, dtype=x.dtype))               # g as the backward casts it
        acc = abs(gq) * (acc + r * (D.abs() + acc)) + abs(gq - g) * D.abs()
        D = D * g
    out["dlogits"] = (D, acc)
    return out
