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

Attention (the last section) reuses C_ACC for its tensor-core products.  On the same H100, test_gpu_attention_elementwise.py
reaches at most 0.037 of the lse bound at C_ACC = 2 and 0.23 at C_ACC = 0.25, and fails it at C_ACC = 0 (2.2): the lse
has no bf16 rounding to hide behind, so it is what calibrates C_ACC there.  EXP_ULPS = 0 passes as well as 2: no bound
is filled by the exp2 terms, so EXP_ULPS stays at exp2f's documented maximum.  Its bf16 outputs reach 0.95.

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
