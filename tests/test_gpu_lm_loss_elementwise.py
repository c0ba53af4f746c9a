"""The fused LM-head cross-entropy (`lm_loss_fwd` / `lm_loss_bwd`), the sparse-prediction row kernels and the unfused
`xent_fwd_bwd` kernels, checked element by element against fp64 (numerics.py, cross-entropy section).

The references take the kernel's own bf16 logits X = gemm_nt(h, w, b) as exact inputs; that the fused epilogue sees
exactly these logits is asserted, not assumed: every row's row_loss equals float32(lse - X[i, t_i]) bitwise.  Each case
then checks lse, row_loss, loss, dh, dw and dbias per element, and that dh is exactly zero on ignored rows.

`fwd_kernels` / `bwd_kernels` mirror the dispatch of the two bindings (and launch_xent_fwd_bwd's selection for the unfused
kernels); the coverage tests assert that the parameter tables reach every instantiation.
"""
import math

import pytest
import torch

import numerics as nm

pytestmark = pytest.mark.gpu
DEV = "cuda"

# ---- dispatch mirrors -----------------------------------------------------------------------------------------------------
EVERY_LM = {"kLmLse", "kLmLse+kBoundRows", "lm_lse_combine<false>", "lm_lse_combine<true>", "kLmDlogits",
            "kLmDlogits+kBoundRows", "kBoundRows (dh)", "kBoundK (dw)", "column_sum"}


def fwd_kernels(bounded):
    """launch_gemm_lm_lse + launch_lm_loss_combine."""
    return {"kLmLse+kBoundRows" if bounded else "kLmLse", f"lm_lse_combine<{'true' if bounded else 'false'}>"}


def bwd_kernels(bounded, need_dbias):
    """lm_loss_bwd per slice: the dlogits GEMM, dh (row-bounded or the plain gemm), dw (row-bounded or plain), column_sum."""
    out = {"kLmDlogits+kBoundRows" if bounded else "kLmDlogits"}
    if bounded:
        out |= {"kBoundRows (dh)", "kBoundK (dw)"}
    if need_dbias:
        out.add("column_sum")
    return out


def xent_kernel(dtype, cols, offset):
    """launch_xent_fwd_bwd's choice: the shared-memory kernel when the row fits in 200 KB and logits / dlogits share their
    16-byte phase (dlogits is a fresh allocation, so a logits view at `offset` elements has phase offset * size)."""
    esz = 2 if dtype == torch.bfloat16 else 4
    return "smem" if (cols + 16) * esz <= 200 * 1024 and (offset * esz) % 16 == 0 else "stream"


# ---- cases ----------------------------------------------------------------------------------------------------------------
# (N, V, H, bias, slice, ignore_index, gscales): why.  bias: None, "gpt2" (the constant -1e4 padded-column mask) or "train"
# (a trained bias: dbias through column_sum).  Every case has scale-40 rows (|x - lse| reaches tens) and peaked rows.
DENSE = {
    (129, 8, 72, "train", 128, -100, (1.0, 0.3)): "V = 8: one partial tile; H = 72 is not a multiple of 64; N = 129",
    (1000, 2176, 128, None, 128, -100, (1.0, 0.25, 0.3)): "fewer columns than one 4096 slice; slice = 128: 17 fp32 dh adds",
    (384, 30528, 128, "train", 4096, -100, (1.0,)): "BERT: the last tile is 64 columns",
    (129, 49216, 128, None, 4096, -100, (0.3,)): "Granite: the last tile and the last slice are one 64-column tile",
    (1, 50280, 64, None, 4096, -100, (1.0,)): "Mamba: the last tile is 104 columns; N = 1",
    (1000, 50304, 128, "gpt2", 65536, -100, (1.0,)): "GPT-2's -1e4 padded columns; one slice wider than V",
    (384, 32128, 128, "train", 4096, 0, (0.25,)): "T5; ignore_index = 0 lies inside [0, V) and must be honoured",
    (1024, 151936, 128, None, 4096, -100, (1.0,)): "Qwen: the widest vocabulary, 38 slices",
}
SPARSE_COUNTS = (0, 1, 127, 128, 129, 384)
XENT = {
    (torch.bfloat16, 10, 0): "smem, a row shorter than one 16-byte vector",
    (torch.bfloat16, 1000, 0): "smem",
    (torch.bfloat16, 30522, 0): "smem: BERT's unpadded vocabulary, rows only 4-byte aligned",
    (torch.bfloat16, 50304, 0): "smem: GPT-2",
    (torch.float32, 1000, 0): "smem, fp32",
    (torch.float32, 30522, 0): "smem, fp32",
    (torch.bfloat16, 151936, 0): "streaming: a bf16 row wider than 200 KB (Qwen without --fused_lm_loss)",
    (torch.float32, 60000, 0): "streaming: an fp32 row wider than 200 KB",
    (torch.bfloat16, 30522, 1): "streaming: a logits view one element in, its 16-byte phase unlike dlogits'",
}


def test_parameter_tables_reach_every_instantiation():
    reached = set()
    for _, _, _, bias, *_ in DENSE:
        reached |= fwd_kernels(False) | bwd_kernels(False, bias == "train")
    reached |= fwd_kernels(True) | bwd_kernels(True, True)          # test_sparse_prediction_rows (bias trained)
    assert reached == EVERY_LM, sorted(EVERY_LM - reached)
    assert {xent_kernel(*k) for k in XENT} == {"smem", "stream"}
    assert {(d, xent_kernel(d, c, o)) for d, c, o in XENT} == {(d, k) for d in (torch.bfloat16, torch.float32)
                                                               for k in ("smem", "stream")}


@pytest.fixture(scope="module")
def C():
    from b200ddp import _ext
    return _ext.get()


def _edges(V, slice_w):
    """The columns where a tile, slice or vocabulary edge can go wrong."""
    cols = [0, 127, 128, 4095, 4096, 4097, V - 1] + [min(v0 + slice_w, V) - 1 for v0 in range(0, V, slice_w)]
    return list(dict.fromkeys(c for c in cols if 0 <= c < V))


def _inputs(N, V, H, bias, slice_w, ignore_index, seed):
    """h, w, t, b.  Rows 0, 5, 10, ... are scaled by 40; rows 1, 6, 11, ... are peaked: h = w_c (log V + 0.5) / |w_c|²
    puts p ≈ 0.4 on an edge column c, which is also their target; rows 2, 3, 4, 7, ... carry the special targets."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    h = torch.randn(N, H, device=DEV, generator=g)
    h[::5] *= 40
    w = (torch.randn(V, H, device=DEV, generator=g) * 0.05).to(torch.bfloat16)
    t = torch.randint(0, V, (N,), device=DEV, generator=g)
    edges = _edges(V, slice_w)
    for r, c in zip(range(1, N, 5), edges * N):
        wc = w[c].float()
        h[r] = wc * (math.log(V) + 0.5) / wc.square().sum()
        t[r] = c
    special = edges + [-100, -7, V, V + 5] + ([0, 0, 0] if ignore_index == 0 else [])
    rows = [r for r in range(N) if r % 5 not in (0, 1)]
    for r, v in zip(rows, special):
        t[r] = v
    b = None
    if bias == "gpt2":
        b = torch.zeros(V, device=DEV, dtype=torch.bfloat16)
        b[V - 47:] = -1e4
    elif bias == "train":
        b = torch.randn(V, device=DEV, generator=g).to(torch.bfloat16)
    return h.to(torch.bfloat16), w, t, b


def _logits(C, h, w, b):
    return C.gemm_nt(h, w, b, 1 if b is not None else 0)


def _check_forward(where, C, h, w, t, b, ignore_index, lse, row_loss, loss, rows=None):
    """The bitwise row_loss <-> X consistency and the element-wise forward checks on the first `rows` rows."""
    N, V = h.shape[0], w.shape[0]
    n = N if rows is None else rows
    X = _logits(C, h[:n], w, b) if n else torch.zeros(0, V, device=DEV, dtype=torch.bfloat16)
    lab = nm.lm_labelled(t, V, ignore_index)
    assert float(row_loss[N]) == float(lab.sum()), f"{where}: valid count"
    xt = X.float().gather(1, torch.where(lab[:n], t[:n], 0)[:, None])[:, 0]
    expect = torch.where(lab[:n], lse[:n] - xt, torch.zeros_like(xt))
    bad = (row_loss[:n] != expect).nonzero()
    assert bad.numel() == 0, (f"{where}: row_loss != float32(lse - X[i, t_i]) at {bad.numel()} rows, first {int(bad[0])}: "
                              f"the fused epilogue does not see the logits gemm_nt stores")
    ref = nm.lm_loss_reference(X, t[:n], V, ignore_index, finish=False)
    nm.check(f"{where}: lse [row]", lse[:n], *ref["lse"], group="lm lse")
    nm.check(f"{where}: row_loss [row]", row_loss[:n], *ref["row_loss"], group="lm row_loss")
    rl, rl_bnd = ref["row_loss"]
    cnt = max(int(lab.sum()), 1)
    depth = nm._ceil(N, nm.FINISH_THREADS) + 11
    loss_ref = rl.sum() / cnt
    nm.check(f"{where}: loss", loss.reshape(1), loss_ref.reshape(1),
             ((rl_bnd.sum() + depth * nm.U * rl.abs().sum()) / cnt + nm.U * loss_ref.abs() + nm.FLOOR).reshape(1),
             group="lm loss")
    return X


def _check_backward(where, X, lse, t, h, w, V, ignore_index, gscale, slice_w, dh, dw, db, rows=None):
    N = h.shape[0]
    n = N if rows is None else rows
    lab = nm.lm_labelled(t, V, ignore_index)
    cnt = int(lab.sum())
    coef = gscale / cnt if cnt else 0.0
    bound_k = None if rows is None else nm._ceil(rows, 64) * 64
    ref = nm.lm_grad_reference(X, lse[:n], t[:n], h[:n], w, V, coef, slice_w, ignore_index, bound_k=bound_k)
    nm.check(f"{where}: dh [row, h]", dh[:n], ref["dh"][0], nm.bound(*ref["dh"], dh.dtype), group="lm dh")
    nm.check(f"{where}: dw [vocab, h]", dw, ref["dw"][0], nm.bound(*ref["dw"], dw.dtype), group="lm dw")
    if db is not None:
        nm.check(f"{where}: dbias [vocab]", db, ref["dbias"][0], nm.bound(*ref["dbias"], db.dtype), group="lm dbias")
    assert (dh[~lab] == 0).all(), f"{where}: dh not exactly zero on ignored rows"


def _case_id(case):
    N, V, H, bias, s, ii, gs = case
    return f"N{N}-V{V}-H{H}-{bias or 'nobias'}-slice{s}-ii{ii}"


@pytest.mark.parametrize("case", list(DENSE), ids=[_case_id(c) for c in DENSE])
def test_fused_lm_loss_matches_fp64_elementwise(C, case):
    N, V, H, bias, slice_w, ii, gscales = case
    h, w, t, b = _inputs(N, V, H, bias, slice_w, ii, seed=N + V)
    where = _case_id(case)
    loss, lse, rl = C.lm_loss_fwd(h, w, t, b, ii)
    X = _check_forward(where, C, h, w, t, b, ii, lse, rl, loss)
    for gscale in gscales:
        gs = torch.tensor([gscale], device=DEV)
        dh, dw, db = C.lm_loss_bwd(h, w, t, b, lse, rl, gs, ii, slice_w, True, True, need_dbias=bias == "train")
        _check_backward(f"{where} gscale {gscale}", X, lse, t, h, w, V, ii, gscale, slice_w, dh, dw, db)


def test_all_rows_ignored():
    from b200ddp import _ext
    C = _ext.get()
    h, w, _, b = _inputs(300, 2176, 128, "train", 128, -100, seed=3)
    t = torch.tensor([-100, -1, 2176, 5000] * 75, device=DEV)
    loss, lse, rl = C.lm_loss_fwd(h, w, t, b, -100)
    X = _check_forward("all ignored", C, h, w, t, b, -100, lse, rl, loss)
    assert float(loss) == 0.0 and float(rl[-1]) == 0.0
    dh, dw, db = C.lm_loss_bwd(h, w, t, b, lse, rl, torch.ones(1, device=DEV), -100, 128, True, True, need_dbias=True)
    _check_backward("all ignored", X, lse, t, h, w, 2176, -100, 1.0, 128, dh, dw, db)
    assert (dh == 0).all() and (dw == 0).all() and (db == 0).all()


# ---- sparse prediction: compact / gather / scatter (exact) and the row-bounded GEMMs ----------------------------------------
@pytest.mark.parametrize("count", SPARSE_COUNTS)
def test_sparse_prediction_rows(C, count):
    N, V, H, slice_w = 384, 30528, 128, 4096
    h, w, _, b = _inputs(N, V, H, "train", slice_w, -100, seed=count)
    g = torch.Generator(device=DEV).manual_seed(count + 1)
    t = torch.tensor([-100, -3, V, V + 9], device=DEV).repeat(N // 4)
    lab_rows = torch.randperm(N, device=DEV, generator=g)[:count]
    t[lab_rows] = torch.randint(0, V, (count,), device=DEV, generator=g)
    t[lab_rows[:8]] = torch.tensor([0, 127, 128, 4095, 4096, 4097, V - 64, V - 1], device=DEV)[:len(lab_rows[:8])]
    lab = nm.lm_labelled(t, V)
    index, cnt, tc = C.compact_rows(t, -100, V)
    want = torch.cat([lab.nonzero()[:, 0], (~lab).nonzero()[:, 0]])
    assert int(cnt) == count and torch.equal(index.long(), want), "compact_rows: not the stable partition"
    assert torch.equal(tc[:count], t[want[:count]]) and (tc[count:] == -100).all()
    hc = C.gather_rows(h, index, cnt)
    assert torch.equal(hc[:count], h[want[:count]]) and (hc[count:] == 0).all(), "gather_rows: not exact"

    loss, lse, rl = C.lm_loss_fwd(hc, w, tc, b, -100, rows=cnt)
    assert (lse[count:] == 0).all() and (rl[count:N] == 0).all(), "lse / row_loss past the count are not zero"
    where = f"sparse count {count}"
    X = _check_forward(where, C, hc, w, tc, b, -100, lse, rl, loss, rows=count)
    gscale = 0.3
    dh, dw, db = C.lm_loss_bwd(hc, w, tc, b, lse, rl, torch.tensor([gscale], device=DEV), -100, slice_w, True, True,
                               rows=cnt, need_dbias=True)
    assert (dh[count:] == 0).all(), f"{where}: dh rows past the count are not exactly zero"
    _check_backward(where, X, lse, tc, hc, w, V, -100, gscale, slice_w, dh, dw, db, rows=count)
    dx = C.scatter_rows(dh, index, cnt)
    assert torch.equal(dx[want[:count]], dh[:count]) and (dx[want[count:]] == 0).all(), "scatter_rows: not exact"


def test_rows_past_the_count_with_large_logits_get_zero_gradients(C):
    """The binding only asks that rows at or past the count be ignored ones.  Here they hold hidden states whose logits
    exceed 88.7 (where exp overflows fp32) in the 128-row tile that holds the count: with lse = 0 for those rows, exp(x) *
    0 must not turn into NaN in dh (rows past the count, promised zero) or in dw (kBoundK reads up to the count rounded up
    to 64)."""
    N, V, H, count = 256, 2176, 128, 100
    h, w, t, b = _inputs(N, V, H, "train", 4096, -100, seed=11)
    wc = w[5].float()
    h[count:] = (wc * 120.0 / wc.square().sum()).to(torch.bfloat16)
    t[count:] = -100
    t[:count] = t[:count].clamp(0, V - 1)
    X = _logits(C, h, w, b)
    assert float(X[count:].float().amax()) > 100.0
    cnt = torch.tensor([count], device=DEV, dtype=torch.int32)
    loss, lse, rl = C.lm_loss_fwd(h, w, t, b, -100, rows=cnt)
    dh, dw, db = C.lm_loss_bwd(h, w, t, b, lse, rl, torch.ones(1, device=DEV), -100, 4096, True, True, rows=cnt,
                               need_dbias=True)
    assert torch.isfinite(dh.float()).all() and torch.isfinite(dw.float()).all() and torch.isfinite(db.float()).all()
    assert (dh[count:] == 0).all()
    _check_backward("large logits past the count", X[:count], lse, t, h, w, V, -100, 1.0, 4096, dh, dw, db, rows=count)


# ---- unfused xent_fwd_bwd -------------------------------------------------------------------------------------------------
def _xent_inputs(dtype, cols, offset, seed):
    N = 64 if cols > 60000 else 300
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(N, cols, device=DEV, generator=g)
    x[::4] *= 8                                                   # |x - lse| reaches tens
    t = torch.randint(0, cols, (N,), device=DEV, generator=g)
    special = [c for c in (0, 127, 128, 4095, 4096, cols - 1) if c < cols] + [-100, -5, cols, cols + 3]
    t[1:1 + len(special)] = torch.tensor(special, device=DEV)
    for r in range(1 + len(special), min(N, 1 + len(special) + 6)):   # peaked rows at the special columns
        c = special[r % 6] if special[r % 6] >= 0 and special[r % 6] < cols else 0
        x[r, c] = math.log(cols) + 0.5
        t[r] = c
    buf = torch.empty(N * cols + offset, device=DEV, dtype=dtype)
    view = buf[offset:].view(N, cols)
    view.copy_(x.to(dtype))
    return view, t


@pytest.mark.parametrize("dtype,cols,offset", list(XENT),
                         ids=[f"{'bf16' if d == torch.bfloat16 else 'fp32'}-{c}-off{o}" for d, c, o in XENT])
def test_unfused_cross_entropy_matches_fp64_elementwise(C, dtype, cols, offset):
    x, t = _xent_inputs(dtype, cols, offset, seed=cols + offset)
    where = f"xent {xent_kernel(dtype, cols, offset)} {dtype} {cols} offset {offset}"
    gscale = 0.3
    loss, dl = C.xent_fwd_bwd(x, t, -100, gscale)
    ref = nm.xent_reference(x, t, gscale=gscale)
    nm.check(f"{where}: loss", loss.reshape(1), ref["loss"][0].reshape(1), ref["loss"][1].reshape(1), group="xent loss")
    D, acc = ref["dlogits"]
    nm.check(f"{where}: dlogits [row, col]", dl, D, nm.bound(D, acc, dtype), group=f"xent dlogits {'bf16' if dtype == torch.bfloat16 else 'fp32'}")
    if offset == 0:                                              # through autograd, with a non-unit upstream gradient
        from b200ddp.ops import cross_entropy
        xx = x.clone().requires_grad_(True)
        l2 = cross_entropy(xx, t)
        g = 0.7
        l2.backward(torch.tensor(g, device=DEV))
        ref = nm.xent_reference(x, t, g=g)
        D, acc = ref["dlogits"]
        nm.check(f"{where}: autograd dlogits, g = {g}", xx.grad, D, nm.bound(D, acc, dtype),
                 group=f"xent autograd {'bf16' if dtype == torch.bfloat16 else 'fp32'}")
