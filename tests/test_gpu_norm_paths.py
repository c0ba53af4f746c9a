"""Every LayerNorm / RMSNorm launch path, through the raw bindings, checked element by element against fp64.

LayerNorm forward and backward take a fast path when cols % 8 == 0, cols <= 1024 and the pointers are 32-byte aligned,
and a generic path otherwise (its backward: per-block partials plus a finish kernel).  The fast backward's dgamma / dbeta
come from layernorm_param_grad_kernel on the grid `ln_bwd_geometry` computes; `geometry` below mirrors it, and each test id
names the geometry its row reaches: cvb (8-column vectors per block) and ty (rows per block pass), gy (row splits) and
what capped it, whether rows < ty, and whether a block's paired-row loop leaves a remainder row.  RMSNorm runs the fast
kernels up to 1024 columns and the wide kernels above, whose grid of at most 16 * 132 blocks grid-strides over the rows.

The backward gets the reference mean / rstd rounded to fp32, so its check does not inherit the forward's error.
"""
import pytest
import torch

import numerics as nm

pytestmark = pytest.mark.gpu

NUM_SMS = 132
THREADS = 256
EPS = 1e-5
DTYPES = {"fp32": torch.float32, "bf16": torch.bfloat16}


def partial_rows(rows):
    """Mirror of layernorm_partial_rows."""
    return max(2, min((rows + 63) // 64, 2 * NUM_SMS))


def geometry(rows, cols, max_gy):
    """Mirror of ln_bwd_geometry: (cvb, ty, gx, gy, why gy is what it is)."""
    cv = cols // 8
    cvb = min(cv, 32)
    while THREADS % cvb:
        cvb -= 1
    ty = THREADS // cvb
    gx = (cv + cvb - 1) // cvb
    gy0 = (4 * NUM_SMS + gx - 1) // gx
    by_rows = max(1, rows // (ty * 4))
    gy, why = (gy0, "sms") if gy0 <= by_rows else (by_rows, "rows")
    if gy > max_gy:
        gy, why = max(1, max_gy), "partial-buffer"
    return cvb, ty, gx, gy, why


def fast_name(rows, cols, max_gy):
    cvb, ty, gx, gy, why = geometry(rows, cols, max_gy)
    per = (rows + gy - 1) // gy
    tags = ["gy1" if gy == 1 else f"gy{gy}-by-{why}"]
    if rows < ty:
        tags.append("rows<ty")
    if per % (2 * ty):
        tags.append("remainder-loop")
    return f"cvb{cvb}-ty{ty}-gx{gx}-" + "-".join(tags)


def _ln_rows(cols):
    ty = geometry(1, cols, 1)[1]
    return sorted({1, 7, ty - 1, 2 * ty + 1, 8191, 16384})


LN_FAST_COLS = (8, 104, 768, 1024)       # 104: cvb 8; 1024: the widest fast row
LN_CASES = [(c, r) for c in LN_FAST_COLS for r in _ln_rows(c)] + [(1032, r) for r in (1, 7, 8191, 16384)]
RMS_CASES = [(c, r) for c in (64, 1024, 1032, 4096) for r in (1, 7, 2113)]


def _ln_id(case):
    cols, rows = case
    if cols % 8 or cols > 1024:
        return f"cols{cols}-rows{rows}-generic-parts{partial_rows(rows)}"
    return f"cols{cols}-rows{rows}-fast-{fast_name(rows, cols, partial_rows(rows) // 2)}+generic-at-offset-1"


def _rms_id(case):
    cols, rows = case
    grid = min(rows, 16 * NUM_SMS)
    path = "fast" if cols <= 1024 else f"wide-grid{grid}" + ("-wraps" if rows > grid else "")
    return f"cols{cols}-rows{rows}-{path}-dgamma-{fast_name(rows, cols, partial_rows(rows))}"


@pytest.fixture(scope="module")
def C():
    from b200ddp import _ext
    return _ext.get()


def _rand(shape, dtype, g, scale=1.0, shift=0.0):
    return (torch.randn(*shape, device="cuda", generator=g) * scale + shift).to(dtype)


def _offset_copy(t):
    """The same values as a contiguous view one element into a fresh buffer (breaks the 32-byte alignment)."""
    buf = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
    view = buf[1:].view(t.shape)
    view.copy_(t)
    return view


def _check(name, group, got, ref_acc):
    ref, acc = ref_acc
    nm.check(name, got, ref, nm.bound(ref, acc, got.dtype), group=group)


def _agree(name, a, b, ref_acc):
    """Two paths on the same input: within the sum of their bounds, element by element."""
    ref, acc = ref_acc
    nm.check(name, a, b.double(), 2 * nm.bound(ref, acc, a.dtype))


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("case", LN_CASES, ids=[_ln_id(c) for c in LN_CASES])
def test_layernorm_paths_match_fp64(C, dtype, case):
    cols, rows = case
    dt = DTYPES[dtype]
    g = torch.Generator(device="cuda").manual_seed(rows * 7 + cols)
    x = _rand((rows, cols), dt, g, 2.0, 0.5)
    gamma, beta = _rand((cols,), dt, g), _rand((cols,), dt, g)
    dy = _rand((rows, cols), dt, g)
    fwd = nm.layernorm_reference(x, gamma, beta, EPS)
    mean_in, rstd_in = fwd["mean"][0].float(), fwd["rstd"][0].float()
    bwd = nm.layernorm_bwd_reference(dy, x, gamma, mean_in, rstd_in)
    fast = cols % 8 == 0 and cols <= 1024
    outs = {}
    for path, xi, dyi in [("aligned", x, dy)] + ([("offset-1", _offset_copy(x), _offset_copy(dy))] if fast else []):
        name = f"layernorm {dtype} {rows}x{cols} {path}"
        y, mean, rstd = C.layernorm_fwd(xi, gamma, beta, EPS)
        _check(f"{name} y", "layernorm y", y, fwd["y"])
        nm.check(f"{name} mean", mean, *fwd["mean"], group="layernorm mean")
        nm.check(f"{name} rstd", rstd, *fwd["rstd"], group="layernorm rstd")
        dx, dgamma, dbeta = C.layernorm_bwd(dyi, xi, gamma, mean_in, rstd_in)
        _check(f"{name} dx", "layernorm dx", dx, bwd["dx"])
        _check(f"{name} dgamma", "layernorm dgamma", dgamma, bwd["dgamma"])
        _check(f"{name} dbeta", "layernorm dbeta", dbeta, bwd["dbeta"])
        # bitwise repeatable, also right after a call on fewer rows (another geometry, the same counters' job)
        half = max(1, rows // 2)
        C.layernorm_bwd(dyi[:half], xi[:half], gamma, mean_in[:half], rstd_in[:half])
        again = C.layernorm_bwd(dyi, xi, gamma, mean_in, rstd_in)
        for what, first, second in zip(("dx", "dgamma", "dbeta"), (dx, dgamma, dbeta), again):
            assert torch.equal(first, second), f"{name} {what}: not bitwise repeatable"
        outs[path] = (y, dx, dgamma, dbeta)
    if fast:
        for i, (what, ref) in enumerate((("y", fwd["y"]), ("dx", bwd["dx"]), ("dgamma", bwd["dgamma"]), ("dbeta", bwd["dbeta"]))):
            _agree(f"layernorm {dtype} {rows}x{cols} fast vs generic {what}", outs["aligned"][i], outs["offset-1"][i], ref)


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("rows,cols,offset", [(7, 1032, 0), (8191, 1032, 0), (4096, 768, 1)])
def test_layernorm_generic_backward_is_bitwise_repeatable(C, dtype, rows, cols, offset):
    """The generic backward used to add every warp's dgamma / dbeta terms into shared memory with float atomics, so their
    order, and the last bits of dgamma, changed from call to call.  It now sums each column over the block's rows in row
    order."""
    dt = DTYPES[dtype]
    g = torch.Generator(device="cuda").manual_seed(3)
    x, dy = _rand((rows, cols), dt, g, 2.0, 0.5), _rand((rows, cols), dt, g)
    if offset:
        x, dy = _offset_copy(x), _offset_copy(dy)
    gamma = _rand((cols,), dt, g)
    mean, rstd = x.float().mean(1), torch.rsqrt(x.float().var(1, unbiased=False) + EPS)
    first = C.layernorm_bwd(dy, x, gamma, mean, rstd)
    for _ in range(2):
        for what, a, b in zip(("dx", "dgamma", "dbeta"), first, C.layernorm_bwd(dy, x, gamma, mean, rstd)):
            assert torch.equal(a, b), f"{what} differs between two identical calls"


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("case", RMS_CASES, ids=[_rms_id(c) for c in RMS_CASES])
def test_rmsnorm_paths_match_fp64(C, dtype, case):
    cols, rows = case
    dt = DTYPES[dtype]
    g = torch.Generator(device="cuda").manual_seed(rows * 5 + cols)
    x = _rand((rows, cols), dt, g, 2.0, 0.5)
    gamma = _rand((cols,), dt, g)
    dy = _rand((rows, cols), dt, g)
    fwd = nm.layernorm_reference(x, gamma, None, EPS, rms=True)
    rstd_in = fwd["rstd"][0].float()
    bwd = nm.layernorm_bwd_reference(dy, x, gamma, None, rstd_in, rms=True)
    name = f"rmsnorm {dtype} {rows}x{cols}"
    y, rstd = C.rmsnorm_fwd(x, gamma, EPS)
    _check(f"{name} y", "rmsnorm y", y, fwd["y"])
    nm.check(f"{name} rstd", rstd, *fwd["rstd"], group="rmsnorm rstd")
    dx, dgamma = C.rmsnorm_bwd(dy, x, gamma, rstd_in)
    _check(f"{name} dx", "rmsnorm dx", dx, bwd["dx"])
    _check(f"{name} dgamma", "rmsnorm dgamma", dgamma, bwd["dgamma"])
    half = max(1, rows // 2)
    C.rmsnorm_bwd(dy[:half], x[:half], gamma, rstd_in[:half])
    dx2, dgamma2 = C.rmsnorm_bwd(dy, x, gamma, rstd_in)
    assert torch.equal(dx, dx2) and torch.equal(dgamma, dgamma2), f"{name}: backward not bitwise repeatable"
