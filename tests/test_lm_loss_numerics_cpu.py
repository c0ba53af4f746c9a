"""The cross-entropy bounds of numerics.py tested without a GPU.  The fused LM head's fp32 arithmetic is emulated on the CPU
in the kernels' order (kLmLse's four 32-column chunks per 128-column tile with one online rescale each, lm_lse_combine's
eight tile groups, kLmDlogits per vocabulary slice with its column offset, the fp32 `accumulate` chain into dh, the
row-bounded tiles and k-loop, column_sum's 128-row chunks), and so are xent_fwd_bwd's block reductions.  __expf is a float32
exp2(x · log2e), and also that result pushed by its documented 2 + ⌊1.173 |x|⌋ ulp in the adverse direction.  The
emulations stay inside every bound; then each of eleven faults is injected and must fail the check.  The faults that the
older checks (1e-3 relative on the loss, 2e-2 in norm on dh / dw / dbias, 1e-2 in norm per expert for the grouped GEMMs)
let through on their kind of inputs are named in PASS_OLD_CHECK, and test_faults_that_pass_the_old_checks asserts that list."""
import functools
import math

import pytest
import torch

import numerics as nm

WORST = {}                                  # group -> largest error / bound of the fault-free emulations
LOG2E = torch.tensor(math.log2(math.e), dtype=torch.float32)
F32 = torch.float32


def _bf16(t):
    return t.to(torch.bfloat16)


def _rel(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-300))


def _ok(name, got, ref, bnd):
    try:
        w = nm.check(name, got, ref, bnd)
    except AssertionError:
        return False
    WORST[name] = max(WORST.get(name, 0.0), w)
    return True


def expf(x, adverse=0):
    """__expf: float32 exp2(x · log2e), optionally moved by 2 + ⌊1.173 |x|⌋ ulp (adverse = +1 / -1), flushed below 2⁻¹²⁶."""
    y = torch.exp2(x * LOG2E)
    if adverse:
        _, e = torch.frexp(y)
        ulps = 2 + torch.floor(1.173 * x.abs().nan_to_num(posinf=0.0))
        y = torch.where(y > 0, y + adverse * ulps * torch.ldexp(torch.ones_like(y), e - 24), y)
    return torch.where(y < 2.0 ** -126, torch.zeros_like(y), y)


def _merge(a, b, adverse):
    (am, as_), (bm, bs) = a, b
    m = torch.maximum(am, bm)
    s = as_ * expf(am - m, adverse) + bs * expf(bm - m, adverse)
    m = torch.where(bm == -math.inf, am, torch.where(am == -math.inf, bm, m))
    s = torch.where(bm == -math.inf, as_, torch.where(am == -math.inf, bs, s))
    return m, s


def lm_forward_emulate(X, t, V, ignore_index=-100, adverse=0, fault=None):
    """kLmLse + lm_lse_combine + xent_finish on the bf16 logits X [N, V]: (lse, row_loss, loss), float32."""
    N = X.shape[0]
    T = nm._ceil(V, 128)
    Xp = torch.full((N, T * 128), -math.inf)
    Xp[:, :V] = X.float()
    Xt = Xp.view(N, T, 4, 32)
    m = torch.full((N, T), -math.inf)
    s = torch.zeros(N, T)
    for c in range(4):
        live = (torch.arange(T) * 128 + c * 32) < V                  # the kernel breaks at the first chunk past V
        chunk = Xt[:, :, c]
        nm_ = torch.maximum(m, chunk.amax(-1))
        cs = torch.zeros(N, T)
        for i in range(32):
            cs = cs + expf(chunk[..., i] - nm_, adverse)
        new_s = s + cs if fault == "no_rescale" else s * expf(m - nm_, adverse) + cs
        m, s = torch.where(live, nm_, m), torch.where(live, new_s, s)
    tiles = T - 1 if fault == "drop_last_tile" and V % 128 else T
    groups = []
    for y in range(nm.COMBINE_GROUPS):
        acc = (torch.full((N,), -math.inf), torch.zeros(N))
        for i in range(y, tiles, nm.COMBINE_GROUPS):
            acc = _merge(acc, (m[:, i], s[:, i]), adverse)
        groups.append(acc)
    if fault == "combine_skip_last":
        groups = groups[:-1]
    acc = groups[0]
    for g in groups[1:]:
        acc = _merge(acc, g, adverse)
    lse = acc[0] + (torch.log(acc[1]) + adverse * 2.0 ** -22)
    lab = nm.lm_labelled(t, V, -100 if fault == "ignore_in_range" else ignore_index)
    tcol = torch.where(lab, t, 0)
    if fault == "target_off_by_one":
        tcol = torch.where((tcol % 128 == 0) & (tcol > 0), tcol - 1, tcol)
    row_loss = torch.where(lab, lse - X.float().gather(1, tcol[:, None])[:, 0], torch.zeros(N))
    valid = _valid(t, V, ignore_index, fault)
    loss = row_loss.sum() / valid if valid else torch.zeros(())
    return lse, row_loss, loss


def _valid(t, V, ignore_index, fault):
    if fault == "valid_ge_V":
        return int(((t != ignore_index) & (t >= 0)).sum())
    return int(nm.lm_labelled(t, V, -100 if fault == "ignore_in_range" else ignore_index).sum())


def column_sum_emulate(D, rows, fault=None):
    """column_sum of bf16 D [N, vs] over rows < `rows`: an fp32 chain per 128-row chunk, then the chunks in order."""
    chunks = nm._ceil(rows, 128)
    if fault == "colsum_last_chunk":
        chunks -= 1
    out = torch.zeros(D.shape[1])
    for c in range(chunks):
        acc = torch.zeros(D.shape[1])
        for r in range(c * 128, min(rows, c * 128 + 128)):
            acc = acc + D[r].float()
        out = out + acc
    return _bf16(out)


def lm_backward_emulate(X, lse, t, h, w, V, gscale, slice_w, ignore_index=-100, count=None, adverse=0, fault=None):
    """lm_loss_bwd: per slice kLmDlogits (bf16 dlogits at its column offset), dh accumulated in fp32 and cast once, dw per
    slice, dbias from column_sum; `count` = the row-bounded path.  (dh, dw, dbias) bf16."""
    N, H = h.shape
    vs = min(slice_w, V)
    lab = nm.lm_labelled(t, V, -100 if fault == "ignore_in_range" else ignore_index)
    valid = _valid(t, V, ignore_index, fault)
    coef = torch.tensor(gscale, dtype=F32) / torch.tensor(float(valid), dtype=F32) if valid else torch.zeros((), dtype=F32)
    coef = torch.where(lab, coef, torch.zeros(N))
    live = N if count is None else min(N, nm._ceil(count, 128) * 128)
    if fault == "bound_rows_down":
        live = (count // 128) * 128
    kend = N if count is None else min(N, nm._ceil(count, 64) * 64)
    if fault == "boundk_down":
        kend = (count // 64) * 64
    dh32 = torch.zeros(N, H)
    dw = torch.zeros(V, H, dtype=torch.bfloat16)
    db = torch.zeros(V, dtype=torch.bfloat16)
    for v0 in range(0, V, vs):
        n = min(vs, V - v0)
        d = expf(X[:, v0:v0 + n].float() - torch.where(lab, lse, torch.zeros(N))[:, None], adverse)
        base = v0 + (128 if fault == "col_offset" and v0 > 0 else 0)
        tcol = t - base
        hit = lab & (tcol >= 0) & (tcol < n)
        d[hit.nonzero()[:, 0], tcol[hit]] -= 1
        D = _bf16(d * coef[:, None])
        part = D[:live].float() @ w[v0:v0 + n].float()
        dh32[:live] = part if v0 == 0 else dh32[:live] + part
        dw[v0:v0 + n] = _bf16(D[:kend].float().t() @ h[:kend].float())
        db[v0:v0 + n] = column_sum_emulate(D, N if count is None else count, fault)
    return _bf16(dh32), dw, db


def _lm_inputs(N, V, H, slice_w, peaked, seed=0):
    """The new checks' inputs (peaked rows on the edge columns, scale-40 rows) or, peaked=False, the older tests' kind
    (h ~ N(0, 1), w ~ 0.05 N(0, 1)).  Targets: the edge columns, -100, negatives, >= V and 0."""
    g = torch.Generator().manual_seed(seed)
    h = torch.randn(N, H, generator=g)
    w = _bf16(torch.randn(V, H, generator=g) * 0.05)
    t = torch.randint(0, V, (N,), generator=g)
    edges = [c for c in dict.fromkeys([0, 127, 128, 4095, 4096, 4097, V - 1] +
                                      [min(v0 + slice_w, V) - 1 for v0 in range(0, V, slice_w)]) if c < V]
    if peaked:
        h[::5] *= 40
        for r, c in zip(range(1, N, 5), edges * N):
            wc = w[c].float()
            h[r] = wc * (math.log(V) + 0.5) / wc.square().sum()
            t[r] = c
    special = edges + [-100, -7, V, V + 5, 0, 0]
    for r, v in zip([r for r in range(N) if r % 5 not in (0, 1)], special):
        t[r] = v
    h = _bf16(h)
    X = _bf16(h.float() @ w.float().t())                      # the head GEMM's stored logits
    return X, h, w, t


LM = dict(N=256, V=49216, H=64, slice_w=4096)                  # Granite's padded vocabulary: a 64-column last tile / slice


def lm_case(fault=None, peaked=True, ignore_index=-100, gscale=0.3, count=None, adverse=0, **shape):
    """(new check passes, old check passes) of the emulated forward + backward with `fault`."""
    s = dict(LM, **shape)
    N, V, H, slice_w = s["N"], s["V"], s["H"], s["slice_w"]
    X, h, w, t = _lm_inputs(N, V, H, slice_w, peaked)
    if count is not None:                                      # row-bounded: the labelled rows first, then ignored ones
        t = torch.where(torch.arange(N) < count, t.clamp(0, V - 1), torch.full_like(t, -100))
        h = torch.where((torch.arange(N) < count)[:, None], h, torch.zeros_like(h))
        X = _bf16(h.float() @ w.float().t())
    lse, rl, loss = lm_forward_emulate(X, t, V, ignore_index, adverse, fault)
    dh, dw, db = lm_backward_emulate(X, lse, t, h, w, V, gscale, slice_w, ignore_index, count, adverse, fault)
    lab = nm.lm_labelled(t, V, ignore_index)
    cnt = int(lab.sum())
    coef = gscale / cnt if cnt else 0.0
    ref = nm.lm_loss_reference(X, t, V, ignore_index)
    new = _ok("lm lse", lse, *ref["lse"]) and _ok("lm row_loss", rl, *ref["row_loss"])
    new = new and _ok("lm loss", loss.reshape(1), ref["loss"][0].reshape(1), ref["loss"][1].reshape(1))
    bound_k = None if count is None else nm._ceil(count, 64) * 64
    grads = nm.lm_grad_reference(X, lse, t, h, w, V, coef, slice_w, ignore_index, bound_k=bound_k)
    for key, got in (("dh", dh), ("dw", dw), ("dbias", db)):
        new = new and _ok(f"lm {key}", got, grads[key][0], nm.bound(*grads[key], got.dtype))
    new = new and bool((dh[~lab] == 0).all())
    # the older checks: the loss to 1e-3 and the gradients to 2e-2 in norm against the fp64 gradient at the fp64 lse
    true = nm.lm_grad_reference(X, ref["lse"][0], t, h, w, V, coef, slice_w, ignore_index)
    old = abs(float(loss) - float(ref["loss"][0])) <= 1e-3 * abs(float(ref["loss"][0]))
    old = old and all(_rel(got, true[key][0]) < 2e-2 for key, got in (("dh", dh), ("dw", dw), ("dbias", db)))
    return new, old


# ---- unfused xent_fwd_bwd -------------------------------------------------------------------------------------------------
def _warp_tree(v):
    """__shfl_xor butterfly over the last dim (32 lanes): every lane ends with the same sum; lane 0's."""
    lanes = torch.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = v + v[..., lanes ^ o]
    return v[..., 0]


def block_sum_emulate(per_thread):
    """block_sum of [N, 256] per-thread values: a warp tree per warp, then one over the 8 warp sums (padded to 32)."""
    w = _warp_tree(per_thread.view(-1, 8, 32))
    return _warp_tree(torch.cat([w, torch.zeros(w.shape[0], 24)], 1))


def xent_emulate(x, t, gscale, adverse=0, streaming=False):
    """xent_fwd_bwd (shared-memory or streaming kernel) on x [N, C] (values of the logits dtype): (loss, dlogits)."""
    N, C = x.shape
    X = x.float()
    m = X.amax(1)
    k = nm._ceil(C, 256)
    Xp = torch.full((N, k * 256), -math.inf)
    Xp[:, :C] = X
    e = expf(Xp - m[:, None], adverse).view(N, k, 256)
    acc = torch.zeros(N, 256)
    for i in range(k):                                        # thread j: columns j, j + 256, ... in order
        acc = acc + e[:, i]
    s = block_sum_emulate(acc)
    lse = m + (torch.log(s) + adverse * 2.0 ** -22)
    lab = nm.lm_labelled(t, C)
    valid = int(lab.sum())
    g = torch.tensor(gscale, dtype=F32) / valid if valid else torch.zeros((), dtype=F32)
    g = torch.where(lab, g, torch.zeros(N))
    ex = e.view(N, -1)[:, :C]
    onehot = torch.zeros(N, C, dtype=torch.bool)
    onehot[lab.nonzero()[:, 0], t[lab]] = True
    if streaming:
        p = ex * (1 / s)[:, None]
        d = torch.where(onehot, p - 1, p) * g[:, None]
    else:
        p = ex * (g / s)[:, None]
        d = torch.where(onehot, p - g[:, None], p)
    rl = torch.where(lab, lse - X.gather(1, torch.where(lab, t, 0)[:, None])[:, 0], torch.zeros(N))
    loss = rl.sum() / valid if valid else torch.zeros(())
    return loss, d.to(x.dtype)


@pytest.mark.parametrize("adverse", [0, 1, -1], ids=["exp2", "adverse_up", "adverse_down"])
@pytest.mark.parametrize("dtype,cols,streaming", [(torch.bfloat16, 1000, False), (torch.bfloat16, 30522, False),
                                                  (torch.float32, 30522, False), (torch.bfloat16, 151936, True),
                                                  (torch.float32, 60000, True)])
def test_fault_free_xent_emulation_is_within_bounds(dtype, cols, streaming, adverse):
    g = torch.Generator().manual_seed(cols)
    N = 16 if cols > 60000 else 64
    x = torch.randn(N, cols, generator=g)
    x[::4] *= 8
    t = torch.randint(0, cols, (N,), generator=g)
    t[:4] = torch.tensor([-100, cols, 0, cols - 1])
    x = x.to(dtype)
    loss, d = xent_emulate(x, t, 0.3, adverse, streaming)
    ref = nm.xent_reference(x, t, gscale=0.3)
    assert _ok("xent loss", loss.reshape(1), ref["loss"][0].reshape(1), ref["loss"][1].reshape(1))
    D, acc = ref["dlogits"]
    assert _ok(f"xent dlogits {dtype}", d, D, nm.bound(D, acc, dtype))


# ---- grouped expert GEMM (kGrpRows): one tile's expert ---------------------------------------------------------------------
def grouped_fault(fault):
    """Forward of the grouped GEMM on 128-aligned expert segments of the older test's skewed counts; fault "tile_expert":
    the last tile of expert 2's segment multiplies expert 3's weights."""
    counts = [0, 1, 127, 128, 129, 200, 5, 10]
    g = torch.Generator().manual_seed(1)
    K, N = 128, 256
    w = _bf16(torch.randn(len(counts), N, K, generator=g) * 0.1)
    new = old = True
    for e, c in enumerate(counts):
        if c == 0:
            continue
        rows = nm._ceil(c, 128) * 128
        x = torch.zeros(rows, K, dtype=torch.bfloat16)
        x[:c] = _bf16(torch.randn(c, K, generator=g))
        y = x.float() @ w[e].float().t()
        if fault == "tile_expert" and e == 4:
            y[128:] = x[128:].float() @ w[e + 1].float().t()
        y = _bf16(y)
        new = new and _ok("grouped fwd", y, *(lambda r: (r[0], nm.bound(r[0], r[1], torch.bfloat16)))(nm.gemm_reference(x, w[e])))
        old = old and _rel(y, x.float() @ w[e].float().t()) < 1e-2
    return new, old


# ---- the fault table -------------------------------------------------------------------------------------------------------
def _both(fault, **kw):
    """The new check on the new inputs, the old check on the older tests' kind of inputs."""
    return lm_case(fault, **kw)[0], lm_case(fault, peaked=False, **kw)[1]


FAULTS = {
    "1 the last partial tile dropped": lambda: _both("drop_last_tile"),
    "2 the target column off by one at a 128 boundary": lambda: _both("target_off_by_one"),
    "3 the slice col_offset off by 128": lambda: _both("col_offset"),
    "4 the combine skips its last group": lambda: _both("combine_skip_last"),
    "5 a missing chunk rescale": lambda: _both("no_rescale"),
    "6 an in-range ignore_index not ignored": lambda: _both("ignore_in_range", ignore_index=0),
    "7 valid counts targets >= V": lambda: _both("valid_ge_V"),
    "8 the bounded row tile rounded down": lambda: _both("bound_rows_down", count=200),
    "9 kBoundK stops at the count rounded down": lambda: _both("boundk_down", count=200),
    "10 column_sum misses its last chunk": lambda: _both("colsum_last_chunk"),
    "11 one tile_expert off by one": lambda: grouped_fault("tile_expert"),
}
# faults the older checks let through on their kind of inputs (Granite's vocabulary, 256 rows).  A dropped 64-column last
# tile, or a target logit read one column early, moves an unpeaked row's lse or row_loss by about 1/V of the loss: far
# below 1e-3, and the gradients move by as little.  The others change whole gradient columns (a misplaced -1, a missing
# 128-row chunk of dbias), 1/8 of the probability mass, the loss's denominator or whole rows, and fail the old checks too.
PASS_OLD_CHECK = {"1 the last partial tile dropped", "2 the target column off by one at a 128 boundary"}


@functools.cache
def fault_result(fault):
    return FAULTS[fault]()


@pytest.mark.parametrize("fault", sorted(FAULTS, key=lambda f: int(f.split()[0])))
def test_fault_fails_the_new_check(fault):
    new, _ = fault_result(fault)
    assert not new, f"fault {fault!r} passes the element-wise check"


def test_faults_that_pass_the_old_checks():
    passing = {f for f in FAULTS if fault_result(f)[1]}
    assert passing == PASS_OLD_CHECK, (sorted(passing - PASS_OLD_CHECK), sorted(PASS_OLD_CHECK - passing))


@pytest.mark.parametrize("adverse", [0, 1, -1], ids=["exp2", "adverse_up", "adverse_down"])
@pytest.mark.parametrize("kw", [{}, {"ignore_index": 0, "gscale": 1.0}, {"count": 200},
                                {"V": 2176, "slice_w": 128, "N": 300}, {"V": 8, "slice_w": 128, "N": 129}],
                         ids=["granite", "ignore0", "bounded", "slice128", "v8"])
def test_fault_free_lm_emulation_is_within_bounds(kw, adverse):
    assert lm_case(adverse=adverse, **kw)[0]


def test_fault_free_grouped_emulation_is_within_bounds():
    assert grouped_fault(None)[0]


def test_record_largest_ratio():
    """The fault-free emulations' largest error / bound per group (printed with -s; all must be <= 1)."""
    WORST.clear()
    for adverse in (0, 1, -1):
        lm_case(adverse=adverse)
    for k, v in sorted(WORST.items()):
        print(f"{k}: {v:.3g}")
    assert WORST and max(WORST.values()) <= 1.0
