"""BatchNorm (csrc/batchnorm.cu), max pool (csrc/pool.cu) and the MSE loss (csrc/loss.cu), element by element against
float64 references (numerics.batchnorm_reference, batchnorm_bwd_reference, maxpool_reference, mse_reference).

Every BatchNorm launch path is covered: the resident kernels (one or two launches per direction), the two-pass stats +
apply kernels in bf16 and fp32, the programmatic-dependent-launch pair, the single-launch fused kernels (a subprocess: the
switch is read once per process), and the from-partials kernels fed by real convolution epilogues.  The tests mirror the
host-side planning (pick_tile, fused_tile, resident_plan) to get each path's summation depth D and launch count, check the
launch count against it, and assert that the cases reach every path."""
import os
import subprocess
import sys

import pytest
import torch

import numerics as nm

pytestmark = pytest.mark.gpu

SMS = nm.SMS
EPS, MOMENTUM = 1e-5, 0.1


def _ceil(a, b):
    return -(-a // b)


def _ext():
    from b200ddp import _ext as e
    return e.get()


@pytest.fixture(autouse=True)
def _peak_memory(request):
    torch.cuda.reset_peak_memory_stats()
    yield
    log = os.environ.get("B200DDP_NUMERICS_LOG")
    if log:
        with open(log, "a") as f:
            f.write(f"peak_gib:{request.node.name} {torch.cuda.max_memory_allocated() / 2 ** 30:.3f}\n")


# ---- mirrors of the host-side planning --------------------------------------------------------------------------------
pick_tile, two_pass_depth = nm.bn_pick_tile, nm.bn_two_pass_depth


def resident_plan(R, C, streams):
    """(launches, depth) of resident_plan, or None where the resident kernels do not fit."""
    prop = torch.cuda.get_device_properties(torch.cuda.current_device())
    sms, optin = prop.multi_processor_count, prop.shared_memory_per_block_optin
    budget = optin - (16 * 8 + (8 * 2 + 2 + 3) * 64 * 4) - 1024
    ntiles = _ceil(C, 64)
    row_bytes = 64 * 2 * streams + (8 if streams == 2 else 0)
    for T in range(ntiles, 0, -1):
        P = min(sms // T, 17 * 8)
        if P < 1:
            continue
        P = min(P, max(1, _ceil(R, 32)))
        need = _ceil(R, P)
        nbox = _ceil(need, 256)
        if nbox > 16:
            continue
        box_rows = _ceil(need, nbox)
        if nbox * box_rows * row_bytes > budget:
            continue
        waves = _ceil(ntiles, T)
        if waves > 4:
            return None
        P = _ceil(R, nbox * box_rows)
        return _ceil(waves, 2), nbox * _ceil(box_rows, 32) + 2 + 8 + _ceil(P, 8) + 8
    return None


def partials_depth(R, C, G, epilogue_depth):
    """The conv epilogue's chain, then the from-partials kernels' chain over the G rows."""
    _, ty, _, _ = pick_tile(R, C)
    return epilogue_depth + _ceil(G, ty) + ty


def path(R, C, dtype, mode, streams):
    """(path name, launches, depth) of one BatchNorm call.  mode: "default", "two_pass", "pdl" or "fused"."""
    if dtype == torch.bfloat16 and mode == "default":
        plan = resident_plan(R, C, streams)
        if plan is not None:
            return f"resident x{plan[0]}", plan[0], plan[1]
    if mode == "fused" and pick_tile(R, C)[2] <= 2 * SMS:
        return "fused", 1, two_pass_depth(R, C, fused=True)
    return ("pdl" if mode == "pdl" else "two-pass"), 2, two_pass_depth(R, C)


# ---- cases --------------------------------------------------------------------------------------------------------------
# (C, H, W, relu, residual) of ResNet-50's BatchNorms at batch 32 (torchvision v1.5: stride on the 3x3 conv)
RESNET50_BN = [(64, 112, 112, True, False), (64, 56, 56, True, False), (256, 56, 56, True, True), (256, 56, 56, False, False),
               (128, 56, 56, True, False), (128, 28, 28, True, False), (512, 28, 28, True, True), (512, 28, 28, False, False),
               (256, 28, 28, True, False), (256, 14, 14, True, False), (1024, 14, 14, True, True), (1024, 14, 14, False, False),
               (512, 14, 14, True, False), (512, 7, 7, True, False), (2048, 7, 7, True, True), (2048, 7, 7, False, False)]
CASES = ([((32, c, h, w), relu, res) for c, h, w, relu, res in RESNET50_BN]
         + [((32, 512, 56, 56), True, True),        # a forward of four resident waves: two launches
            ((8, 520, 60, 60), True, True), ((8, 520, 60, 60), False, False), ((4, 24, 5, 5), True, True),
            ((4, 24, 5, 5), False, False), ((2, 96, 9, 7), True, False)])
CASE_IDS = [f"{'x'.join(map(str, s))}-{'relu' if r else 'id'}{'-res' if q else ''}" for s, r, q in CASES]
# input distributions: per-channel mean and scale; then every channel shifted to |mean| = 8 sigma and 64 sigma; then a constant
# channel and a channel with var ~ eps among otherwise random ones
DISTS = ["randn", "shift8", "shift64", "edge"]
SMALL = [((32, 256, 14, 14), True, True), ((8, 520, 60, 60), True, False), ((2, 96, 9, 7), False, False),
         ((32, 64, 56, 56), True, False)]


def _act(shape, dtype, dist, g):
    N, C, H, W = shape
    sigma = 0.5 + 1.5 * torch.rand(1, C, 1, 1, device="cuda", generator=g)
    mean = torch.rand(1, C, 1, 1, device="cuda", generator=g) * 2 - 1
    if dist.startswith("shift"):
        sign = torch.where(torch.rand(1, C, 1, 1, device="cuda", generator=g) > 0.5, 1.0, -1.0)
        mean = sign * int(dist[5:]) * sigma
    x = torch.randn(shape, device="cuda", generator=g) * sigma + mean
    if dist == "edge":
        x[:, 0] = 1.375                                           # a constant channel: var = 0
        x[:, 1] = torch.randn(N, H, W, device="cuda", generator=g) * EPS ** 0.5    # var ~ eps
    return x.to(dtype).contiguous(memory_format=torch.channels_last)


def _inputs(shape, dtype, dist, residual, seed=0):
    g = torch.Generator("cuda").manual_seed(seed * 131 + sum(shape))
    C = shape[1]
    x = _act(shape, dtype, dist, g)
    res = _act(shape, dtype, "randn", g) if residual else None
    dy = _act(shape, dtype, "randn", g)
    gamma = 0.5 + torch.rand(C, device="cuda", generator=g)
    beta = torch.rand(C, device="cuda", generator=g) - 0.5
    rm = torch.randn(C, device="cuda", generator=g) * 0.1
    rv = 1 + torch.rand(C, device="cuda", generator=g)
    return x, res, dy, gamma, beta, rm, rv


def forward_backward(x, res, dy, gamma, beta, rm0, rv0, relu):
    """bn_forward then bn_backward; returns their outputs, the updated running statistics and the launches of each."""
    C = _ext()
    R, Cc = x.numel() // x.shape[1], x.shape[1]
    pf, cn = C.bn_workspace(R, Cc)
    partial = torch.zeros(pf, device="cuda")
    counters = torch.zeros(cn, device="cuda", dtype=torch.int32)
    rm, rv = rm0.clone(), rv0.clone()
    nbt = torch.full((1,), 7, device="cuda", dtype=torch.int64)
    b0 = C.launch_count()
    y, stats, mask = C.bn_forward(x, res, gamma, beta, rm, rv, nbt, EPS, MOMENTUM, relu, partial, counters)
    b1 = C.launch_count()
    dx, dres, dparams = C.bn_backward(dy, x, mask if relu else None, gamma, stats, relu, True, partial, counters)
    b2 = C.launch_count()
    torch.cuda.synchronize()
    return dict(y=y, stats=stats, mask=mask, rm=rm, rv=rv, nbt=nbt, dx=dx, dres=dres, dparams=dparams, fwd_launches=b1 - b0,
                bwd_launches=b2 - b1)


def check_forward(name, group, out, x, res, gamma, beta, rm0, rv0, relu, depth, nbt0=7):
    X = nm.as_rows(x)
    ref = nm.batchnorm_reference(X, gamma, beta, EPS, depth, None if res is None else nm.as_rows(res), relu, MOMENTUM, rm0, rv0)
    y = nm.as_rows(out["y"])
    worst = {"y": nm.check(f"{name}: y [row, channel]", y, ref["y"][0], nm.bound(*ref["y"], y.dtype), f"{group} y")}
    for key, got in (("mean", out["stats"][0]), ("rstd", out["stats"][1]), ("running_mean", out["rm"]), ("running_var", out["rv"])):
        if got is not None:
            worst[key] = nm.check(f"{name}: {key} [channel]", got, *ref[key], f"{group} {key}")
    if out.get("nbt") is not None:
        assert int(out["nbt"]) == nbt0 + 1, f"{name}: num_batches_tracked {int(out['nbt'])} != {nbt0 + 1}"
    if relu:
        bits = nm.unpack_mask(out["mask"], x.shape[1])
        wrong = bits != (y > 0)
        assert not wrong.any(), f"{name}: {int(wrong.sum())} ReLU mask bits differ from (y > 0), first at " \
                                f"{tuple(int(i) for i in wrong.nonzero()[0])}"
    return worst


def check_backward(name, group, out, dy, x, gamma, relu, depth, dres=None):
    X, DY = nm.as_rows(x), nm.as_rows(dy)
    bits = nm.unpack_mask(out["mask"], x.shape[1]) if relu else None
    st = out["stats"]
    ref = nm.batchnorm_bwd_reference(DY, X, bits, gamma, st[0], st[1], depth)
    dx = nm.as_rows(out["dx"])
    nm.check(f"{name}: dx [row, channel]", dx, ref["dx"][0], nm.bound(*ref["dx"], dx.dtype), f"{group} dx")
    dp = out["dparams"]
    for i, key in enumerate(("dgamma", "dbeta")):
        r, a = ref[key]
        nm.check(f"{name}: {key} [channel]", dp[i], r, nm.bound(r, a, torch.float32), f"{group} {key}")
    if dres is not None:
        want = DY if bits is None else torch.where(bits, DY, torch.zeros_like(DY))
        assert torch.equal(nm.as_rows(dres), want), f"{name}: dres != dy * mask"


def run_case(shape, relu, residual, dtype, dist, mode, group):
    """One forward + backward on the path `mode` selects, checked against the references with the path's depth."""
    R, Cc = shape[0] * shape[2] * shape[3], shape[1]
    x, res, dy, gamma, beta, rm0, rv0 = _inputs(shape, dtype, dist, residual)
    out = forward_backward(x, res, dy, gamma, beta, rm0, rv0, relu)
    fname, flaunch, fdepth = path(R, Cc, dtype, mode, 1)
    bname, blaunch, bdepth = path(R, Cc, dtype, mode, 2)
    assert out["fwd_launches"] == flaunch, (fname, out["fwd_launches"])
    assert out["bwd_launches"] == blaunch, (bname, out["bwd_launches"])
    name = f"{shape} {dtype} {dist} {mode}"
    check_forward(name, f"bn {group} fwd", out, x, res, gamma, beta, rm0, rv0, relu, fdepth)
    check_backward(name, f"bn {group} bwd", out, dy, x, gamma, relu, bdepth, out["dres"])
    if dtype == torch.bfloat16 and mode == "default":
        assert _ext().bn_resident_error() == 0
    return fname, bname


def all_paths():
    """Every (direction, path) the cases below reach, from the planning mirrors."""
    out = set()
    for shape, _, _ in CASES:
        R, Cc = shape[0] * shape[2] * shape[3], shape[1]
        for dtype, mode in ((torch.bfloat16, "default"), (torch.bfloat16, "two_pass"), (torch.float32, "default")):
            out.add(("fwd", dtype, path(R, Cc, dtype, mode, 1)[0]))
            out.add(("bwd", dtype, path(R, Cc, dtype, mode, 2)[0]))
    for shape, _, _ in PDL_CASES:
        R, Cc = shape[0] * shape[2] * shape[3], shape[1]
        for dtype in (torch.bfloat16, torch.float32):
            out.add(("fwd", dtype, path(R, Cc, dtype, "pdl", 1)[0]))
            out.add(("bwd", dtype, path(R, Cc, dtype, "pdl", 2)[0]))
    for shape, _, _, dtype in FUSED_CASES:
        R, Cc = shape[0] * shape[2] * shape[3], shape[1]
        out.add(("fwd", dtype, path(R, Cc, dtype, "fused", 1)[0]))
        out.add(("bwd", dtype, path(R, Cc, dtype, "fused", 2)[0]))
    return out


PDL_CASES = [((32, 64, 56, 56), True, False), ((8, 256, 14, 14), True, True), ((4, 24, 5, 5), False, False)]
FUSED_CASES = [((16, 64, 28, 28), True, True, torch.bfloat16), ((2, 512, 7, 7), False, False, torch.bfloat16),
               ((16, 64, 28, 28), True, False, torch.float32)]


def test_cases_reach_every_batchnorm_path():
    got = all_paths()
    want = {(d, torch.bfloat16, p) for d in ("fwd", "bwd") for p in ("resident x1", "resident x2", "two-pass", "pdl", "fused")}
    want |= {(d, torch.float32, p) for d in ("fwd", "bwd") for p in ("two-pass", "pdl", "fused")}
    assert got == want, (sorted(map(str, want - got)), sorted(map(str, got - want)))


def test_resident_paths_are_the_ones_taken():
    """Launch counts cannot tell resident x2 from two-pass or PDL (2 launches each), nor resident x1 from fused (1 launch):
    on one case per resident path, the statistics (forward) or dgamma / dbeta (backward, from the same stats and mask) must
    differ in their last bits from the two-pass kernels' on the same inputs, i.e. a different summation order ran."""
    C = _ext()
    picks = {}
    for shape, relu, residual in CASES:
        R, Cc = shape[0] * shape[2] * shape[3], shape[1]
        for d, streams in (("fwd", 1), ("bwd", 2)):
            name = path(R, Cc, torch.bfloat16, "default", streams)[0]
            if name.startswith("resident") and R >= 4096:
                picks.setdefault((d, name), (shape, relu, residual))
    assert set(picks) == {(d, f"resident x{k}") for d in ("fwd", "bwd") for k in (1, 2)}, sorted(picks)
    for (d, name), (shape, relu, residual) in sorted(picks.items()):
        x, res, dy, gamma, beta, rm0, rv0 = _inputs(shape, torch.bfloat16, "randn", residual)
        a = forward_backward(x, res, dy, gamma, beta, rm0, rv0, relu)
        C.set_bn_two_pass(1)
        try:
            b = forward_backward(x, res, dy, gamma, beta, rm0, rv0, relu)
            R, Cc = x.numel() // x.shape[1], x.shape[1]
            pf, cn = C.bn_workspace(R, Cc)
            b_bwd = C.bn_backward(dy, x, a["mask"] if relu else None, gamma, a["stats"], relu, True, torch.zeros(pf, device="cuda"),
                                  torch.zeros(cn, device="cuda", dtype=torch.int32))[2]
        finally:
            C.set_bn_two_pass(0)
        if d == "fwd":
            assert b["fwd_launches"] == 2 and not torch.equal(a["stats"][:2], b["stats"][:2]), f"{name} forward at {shape}: same sums"
        else:
            assert not torch.equal(a["dparams"][:2], b_bwd[:2]), f"{name} backward at {shape}: same sums as the two-pass kernels"
        assert C.bn_resident_error() == 0


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("shape,relu,residual", CASES, ids=CASE_IDS)
def test_batchnorm_default_path_elementwise(shape, relu, residual, dtype):
    run_case(shape, relu, residual, dtype, "randn", "default", "bf16" if dtype == torch.bfloat16 else "fp32")


@pytest.mark.parametrize("shape,relu,residual", CASES, ids=CASE_IDS)
def test_batchnorm_two_pass_path_elementwise(shape, relu, residual):
    C = _ext()
    C.set_bn_two_pass(1)
    try:
        run_case(shape, relu, residual, torch.bfloat16, "randn", "two_pass", "two-pass")
    finally:
        C.set_bn_two_pass(0)


@pytest.mark.parametrize("dist", DISTS[1:])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("shape,relu,residual", SMALL, ids=[f"{'x'.join(map(str, s))}" for s, _, _ in SMALL])
def test_batchnorm_shifted_and_degenerate_channels(shape, relu, residual, dtype, dist):
    run_case(shape, relu, residual, dtype, dist, "default", dist)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("shape,relu,residual", PDL_CASES)
def test_batchnorm_pdl_path_elementwise(shape, relu, residual, dtype):
    C = _ext()
    C.set_bn_pdl(1)
    try:
        run_case(shape, relu, residual, dtype, "randn", "pdl", "pdl")
        run_case(shape, relu, residual, dtype, "shift64", "pdl", "pdl")
    finally:
        C.set_bn_pdl(0)


def test_batchnorm_fused_path_elementwise():
    """B200DDP_BN_FUSED=1 is read once per process: the checks run in a subprocess."""
    here = os.path.dirname(os.path.abspath(__file__))
    code = ("import sys, torch; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "import test_gpu_batchnorm_elementwise as t\n"
            "for shape, relu, res, dtype in t.FUSED_CASES:\n"
            "    for dist in ('randn', 'shift64', 'edge'):\n"
            "        t.run_case(shape, relu, res, dtype, dist, 'fused', 'fused')\n"
            "print('ok')\n") % (os.path.dirname(here), here)
    res = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600,
                         env=dict(os.environ, B200DDP_BN_FUSED="1"))
    assert res.returncode == 0 and "ok" in res.stdout, res.stderr[-3000:]


# ---- the from-partials kernels, fed by real convolution epilogues ---------------------------------------------------------
@pytest.mark.parametrize("dist", ["randn", "shift64"])
@pytest.mark.parametrize("n,ci,co,k,h,relu", [(32, 256, 64, 1, 56, True), (32, 64, 64, 3, 56, True), (32, 512, 2048, 1, 7, False),
                                              (8, 128, 192, 3, 28, True), (3, 64, 128, 1, 5, True)])
def test_batchnorm_from_conv_partials_elementwise(n, ci, co, k, h, relu, dist):
    C = _ext()
    g = torch.Generator("cuda").manual_seed(n + ci + co + k)
    cl = torch.channels_last
    xin = _act((n, ci, h, h), torch.bfloat16, dist, g)
    wt = (torch.randn(co, ci, k, k, device="cuda", generator=g) / (ci * k * k) ** 0.5).to(torch.bfloat16).contiguous(memory_format=cl)
    y, st = C.conv_fprop(xin, wt, 1, (k - 1) // 2, -1, 0, 0, True)
    mode = 2 if (k == 3 and ci == 64) else (1 if k == 3 else 0)
    mt = C.conv_tile_plan(n, h, h, k, k, mode)[4]
    bn = 64 if co % 128 else 128
    grid, per = nm.conv_grid_tiles(mt, _ceil(co, bn))
    R = n * h * h
    depth = partials_depth(R, co, st.shape[1], nm.conv_epilogue_depth(per))
    _, _, _, gamma, beta, rm0, rv0 = _inputs((n, co, h, h), torch.bfloat16, "randn", False)
    rm, rv = rm0.clone(), rv0.clone()
    nbt = torch.zeros(1, device="cuda", dtype=torch.int64)
    b0 = C.launch_count()
    z, stats, mask = C.bn_forward_partials(y, None, gamma, beta, rm, rv, nbt, EPS, MOMENTUM, relu, st)
    assert C.launch_count() - b0 == 1
    out = dict(y=z, stats=stats, mask=mask, rm=rm, rv=rv, nbt=nbt)
    check_forward(f"partials fwd {n, ci, co, k, h}", "bn partials fwd", out, y, None, gamma, beta, rm0, rv0, relu, depth, 0)
    # backward: the data gradient of a following convolution (ci = co here) emits S1 / S2 of this BatchNorm's backward
    w2 = (torch.randn(64, co, 1, 1, device="cuda", generator=g) / co ** 0.5).to(torch.bfloat16).contiguous(memory_format=cl)
    dz = _act((n, 64, h, h), torch.bfloat16, "randn", g)
    dy, part = C.conv_dgrad(dz, w2, 1, 0, -1, 0, 0, 0, None, y, mask if relu else None, stats)
    mt2 = C.conv_tile_plan(n, h, h, 1, 1, 0)[4]
    _, per2 = nm.conv_grid_tiles(mt2, _ceil(co, bn))
    bdepth = partials_depth(R, co, part.shape[1], nm.conv_epilogue_depth(per2))
    b0 = C.launch_count()
    dx, dres, dparams = C.bn_backward_partials(dy, y, mask if relu else None, gamma, stats, relu, True, part)
    assert C.launch_count() - b0 == 1
    out.update(dx=dx, dparams=dparams)
    check_backward(f"partials bwd {n, ci, co, k, h}", "bn partials bwd", out, dy, y, gamma, relu, bdepth, dres)


@pytest.mark.parametrize("n", [2, 32])
def test_batchnorm_from_stem_partials_elementwise(n):
    C = _ext()
    g = torch.Generator("cuda").manual_seed(n)
    cl = torch.channels_last
    x = torch.randn(n, 3, 224, 224, device="cuda", generator=g).to(torch.bfloat16).contiguous(memory_format=cl)
    wt = (torch.randn(64, 3, 7, 7, device="cuda", generator=g) / 147 ** 0.5).to(torch.bfloat16).contiguous(memory_format=cl)
    y, st, _ = C.stem_conv_fprop(x, wt, True, True)
    grid, per = nm.conv_grid_tiles(n * 112, 1)
    R = n * 112 * 112
    depth = partials_depth(R, 64, st.shape[1], nm.conv_epilogue_depth(per))
    _, _, _, gamma, beta, rm0, rv0 = _inputs((n, 64, 112, 112), torch.bfloat16, "randn", False)
    rm, rv = rm0.clone(), rv0.clone()
    nbt = torch.zeros(1, device="cuda", dtype=torch.int64)
    z, stats, mask = C.bn_forward_partials(y, None, gamma, beta, rm, rv, nbt, EPS, MOMENTUM, True, st)
    check_forward(f"stem partials n={n}", "bn partials fwd", dict(y=z, stats=stats, mask=mask, rm=rm, rv=rv, nbt=nbt), y, None,
                  gamma, beta, rm0, rv0, True, depth, 0)


# ---- max pool 3x3 / stride 2 / pad 1 ------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("shape", [(32, 64, 112, 112), (2, 16, 9, 7), (3, 8, 11, 13), (1, 24, 2, 3)])
def test_maxpool_elementwise_with_ties(shape, dtype):
    C = _ext()
    g = torch.Generator("cuda").manual_seed(sum(shape))
    cl = torch.channels_last
    # a handful of levels: most windows hold a tied maximum, so the first-maximum rule decides the slot
    x = (torch.randint(-3, 3, shape, device="cuda", generator=g).float() * 0.5).to(dtype).contiguous(memory_format=cl)
    y, idx = C.maxpool3x3s2_fwd(x)
    y_ref, slot_ref = nm.maxpool_reference(x)
    assert torch.equal(y, y_ref), "max pool output differs"
    wrong = idx != slot_ref
    assert not wrong.any(), f"{int(wrong.sum())} window slots differ, first at {tuple(int(i) for i in wrong.nonzero()[0])}"
    dy = torch.randn(y.shape, device="cuda", generator=g).to(dtype).contiguous(memory_format=cl)
    dx = C.maxpool3x3s2_bwd(dy, idx, shape[2], shape[3])
    ref, acc = nm.maxpool_bwd_reference(dy, slot_ref, shape[2], shape[3])
    nm.check(f"maxpool bwd {shape} {dtype}", dx, ref, nm.bound(ref, acc, dtype), "maxpool bwd")


# ---- MSE -----------------------------------------------------------------------------------------------------------------
def mse_blocks(n):
    return min(max(_ceil(n, 256 * 16), 1), 8 * SMS)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("shape,offset", [((32, 1000), 0), ((3, 333), 0), ((32, 1000), 1), ((1024, 4096), 0)])
def test_mse_elementwise(shape, offset, dtype):
    C = _ext()
    g = torch.Generator("cuda").manual_seed(shape[1] + offset)
    n = shape[0] * shape[1]
    out = torch.randn(n + offset, device="cuda", generator=g).to(dtype)[offset:].view(shape)
    tgt = (torch.randn(n + offset, device="cuda", generator=g) + 0.5).to(dtype)[offset:].view(shape)
    for gscale in (1.0, 0.375):
        loss, dout = C.mse_fwd_bwd(out, tgt, gscale)
        ref = nm.mse_reference(out, tgt, gscale, mse_blocks(n))
        nm.check(f"mse dout {shape} offset {offset}", dout, ref["dout"][0], nm.bound(*ref["dout"], dtype), "mse dout")
        nm.check(f"mse loss {shape} offset {offset}", loss, *ref["loss"], "mse loss")
