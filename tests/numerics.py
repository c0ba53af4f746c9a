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
