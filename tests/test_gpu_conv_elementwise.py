"""The wgmma convolutions (csrc/conv_wgmma.cu, csrc/conv_wgrad_wgmma.cu) and the strided stem, element by element against a
float64 reference of the same convolution (numerics.conv_reference): forward, data gradient (plain, with the shortcut
addend, with the fused BatchNorm-backward partial sums), weight gradient at every tiling the planner accepts, the epilogue
BatchNorm statistics, and the stem's operand packing.

launch_conv_tap_gemm has 8 kernel instantiations, <block_n in {64, 128}, filter MN-major, EPI> with (fprop, EPI 0 / 1) and
(dgrad, EPI 0 / 2), and picks the flat / patch / halo tiling at run time.  The tests mirror its choice of tiling, block_n
and ring depth kc (conv_pick_block_n, conv_tile_plan, launch_variant) and assert that the cases reach every combination."""
import math
import os

import pytest
import torch

import numerics as nm

pytestmark = pytest.mark.gpu

SMS = nm.SMS


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
def pick_block_n(nc, want):
    if want == 256:
        return 128                          # a 256-wide request runs as two 128-wide n-tiles
    if want:
        return want
    return 64 if nc % 128 else 128


def tiling(n, h, w, k, kc_channels, mode):
    """(mode, BH, BI, num_m_tiles, a_rows) of conv_tile_plan, with launch_conv_tap_gemm's automatic 3x3 choice."""
    if mode < 0 and k == 3:
        mode = 2 if kc_channels == 64 else 1
    ok, m, bh, bi, mt, dense, acc_rows, a_rows = _ext().conv_tile_plan(n, h, w, k, k, mode)
    assert ok, (n, h, w, k, mode)
    return m, bh, bi, mt, a_rows


def ring_kc(k, kc_channels, block_n, epi, a_rows, want_kc):
    """launch_variant's k chunks per ring stage (flat / patch tilings)."""
    budget = 227 * 1024 - 2 * 128 * 128 - 1024 - 1024 - (4 * 32 * 36 * 4 if epi else 0) - 128 * (block_n + 8) * 4
    chunk = max(_ceil(a_rows * 128, 1024) * 1024, 128 * 128) + block_n * 64 * 2
    chunks = (kc_channels // 64) * k * k
    kc = want_kc if want_kc > 0 else 2
    while kc > 1 and (chunks % kc or budget // (kc * chunk) < 3):
        kc -= 1
    return kc


def ring_kc_values():
    """Every kc some flat / patch launch can run with: three stages of kc chunks must fit the ring."""
    out = set()
    for block_n in (64, 128):
        for epi in (0, 1):
            budget = 227 * 1024 - 2 * 128 * 128 - 2048 - (4 * 32 * 36 * 4 if epi else 0) - 128 * (block_n + 8) * 4
            kc = 1
            while budget // (kc * (128 * 128 + block_n * 128)) >= 3:
                out.add(kc)
                kc += 1
    return out


grid_tiles = nm.conv_grid_tiles


def wgrad_plan(n, h, w, cin, cout, k, split, tile_n):
    """(pixels per k block, k blocks, split) of wgrad_plan, or None where it refuses the tiling."""
    if k == 1:
        kb, nkb = 64, _ceil(n * h * w, 64)
    else:
        bh, bi = 0, 1
        for d in range(1, 17):
            for i in range(1, (4 if d >= h else 1) + 1):
                if (w * d * i) % 16 == 0 and 96 <= w * d * i <= 128:
                    bh, bi = d, i
                    break
            if bh:
                break
        if not bh:
            for d in range(1, h + 16):
                if (w * d) % 16 == 0 and w * d <= 128:
                    bh = d
                    break
            if not bh:
                return None
        if bi > 1 and n % bi:
            return None
        kb, nkb = w * bh * bi, (n // bi) * _ceil(h, bh)
    tn = tile_n or (cin if cin < 128 else 128)
    if tn not in (64, 128) or tn > cin:
        return None
    groups = _ceil(cout, 128) * _ceil(cin, tn) * k * k
    sp = split if split > 0 else SMS // groups
    return kb, nkb, min(max(sp, 1), nkb)


# ---- cases --------------------------------------------------------------------------------------------------------------
RESNET_1X1 = [(64, 64, 56), (256, 64, 56), (64, 256, 56), (256, 128, 56), (128, 512, 28), (512, 128, 28), (512, 256, 28),
              (256, 1024, 14), (1024, 256, 14), (1024, 512, 14), (512, 2048, 7), (2048, 512, 7)]
RESNET_3X3 = [(64, 56), (128, 28), (256, 14), (512, 7)]
SHAPES = ([(32, ci, co, 1, s, s) for ci, co, s in RESNET_1X1] + [(32, c, c, 3, s, s) for c, s in RESNET_3X3] + [
    (3, 64, 128, 1, 5, 7),                  # N*H*W = 105: not a multiple of 128
    (2, 64, 64, 3, 13, 20),                 # H prime: BH = 1 (halo)
    (2, 128, 128, 3, 13, 20),               # H prime: BH = 1 (patch)
    (6, 128, 192, 3, 7, 7),                 # patch with BI = 2, Cout = 192: three 64-wide n-tiles
    (2, 64, 192, 1, 14, 14),                # Cout = 192 on the flat tiling
    (2, 64, 64, 3, 9, 83),                  # the widest halo: W + 2 = 85
    (2, 128, 128, 3, 4, 126),               # W = 126 (patch; a halo tile of W + 2 = 128 columns exceeds a TMA box)
    (1, 64, 64, 3, 8, 8),                   # fewer tiles than SMs
])
SHAPE_IDS = [f"n{n}-{ci}to{co}-k{k}-{h}x{w}" for n, ci, co, k, h, w in SHAPES]


def variants(ci, co, k, h, w, n):
    """(mode, block_n, kc) launches of one shape: the automatic choice, every block_n that tiles both channel counts, the
    other 3x3 tiling, and a forced one-chunk ring stage."""
    out = [(-1, 0, 0)]
    for bn in (64, 128, 256):
        if co % min(bn, 128) == 0 and ci % min(bn, 128) == 0:
            out.append((-1, bn, 0))
    if k == 3:
        for mode in (1, 2):
            ok = _ext().conv_tile_plan(n, h, w, 3, 3, mode)[0]
            if ok and (mode, 0, 0) not in out:
                out.append((mode, 0, 0))
        if _ext().conv_tile_plan(n, h, w, 3, 3, 1)[0]:
            out.append((1, 64, 1))
    else:
        out.append((-1, 64, 1))
    return out


def reached(shapes=SHAPES):
    """(direction, tiling, block_n, epilogue) combinations and kc values the cases launch."""
    combos, kcs = set(), set()
    for n, ci, co, k, h, w in shapes:
        for mode, bn, kc in variants(ci, co, k, h, w, n):
            for direction, kch, nc, epis in (("fprop", ci, co, (0, 1)), ("dgrad", co, ci, (0, 2))):
                m, _, _, _, a_rows = tiling(n, h, w, k, kch, mode)
                block_n = pick_block_n(nc, bn)
                for epi in epis:
                    combos.add((direction, m, block_n, epi))
                    if m != 2:
                        kcs.add(ring_kc(k, kch, block_n, epi, a_rows, kc))
    return combos, kcs


def test_cases_reach_every_instantiation_and_tiling():
    combos, _ = reached()
    allowed = {(d, m, bn, e) for d, epis in (("fprop", (0, 1)), ("dgrad", (0, 2))) for m in (0, 1, 2) for bn in (64, 128)
               for e in epis}
    assert combos == allowed, sorted(allowed - combos)
    assert pick_block_n(512, 256) == 128 and any(256 in [v[1] for v in variants(ci, co, k, h, w, n)]
                                                 for n, ci, co, k, h, w in SHAPES)


def test_cases_reach_every_ring_depth():
    _, kcs = reached()
    assert kcs == ring_kc_values(), (sorted(kcs), sorted(ring_kc_values()))


def _inputs(n, ci, co, k, h, w, shifted, seed=0):
    g = torch.Generator("cuda").manual_seed(seed * 7919 + n * 1000 + ci + co + k + h + w)
    cl = torch.channels_last
    x = torch.randn(n, ci, h, w, device="cuda", generator=g)
    if shifted:                            # every channel its own large mean: the sums no longer cancel
        x = x + 2 + 4 * torch.rand(1, ci, 1, 1, device="cuda", generator=g)
    x = x.to(torch.bfloat16).contiguous(memory_format=cl)
    wt = (torch.randn(co, ci, k, k, device="cuda", generator=g) / math.sqrt(ci * k * k)).to(torch.bfloat16).contiguous(memory_format=cl)
    dy = torch.randn(n, co, h, w, device="cuda", generator=g)
    if shifted:
        dy = dy + 1 + torch.rand(1, co, 1, 1, device="cuda", generator=g)
    dy = dy.to(torch.bfloat16).contiguous(memory_format=cl)
    return x, wt, dy


def _column_sums(t):
    """Σ and Σ of squares over the rows of the stored output, and Σ| |, in float64 [C]."""
    r = nm.as_rows(t).double()
    return r.sum(0), (r * r).sum(0), r.abs().sum(0)


def _check_stats(name, st, y, depth, group):
    s, q, a = _column_sums(y)
    tot = st.double().sum(1)
    nm.check(f"{name}: column sums", tot[0], s, depth * nm.U * a + nm.FLOOR, group + " stats")
    nm.check(f"{name}: column sums of squares", tot[1], q, depth * nm.U * q + nm.FLOOR, group + " stats")


@pytest.mark.parametrize("shifted", [False, True], ids=["randn", "shifted"])
@pytest.mark.parametrize("n,ci,co,k,h,w", SHAPES, ids=SHAPE_IDS)
def test_forward_and_statistics_elementwise(n, ci, co, k, h, w, shifted):
    C = _ext()
    x, wt, _ = _inputs(n, ci, co, k, h, w, shifted)
    pad = (k - 1) // 2
    ref, acc = nm.conv_reference("fprop", x, wt, 1, pad)
    bnd = nm.bound(ref, acc, torch.bfloat16)
    for mode, bn, kc in variants(ci, co, k, h, w, n):
        name = f"fprop mode {mode} block_n {bn} kc {kc}"
        y0 = C.conv_fprop(x, wt, 1, pad, mode, bn, 0, False, None, kc)[0]
        nm.check(name, y0, ref, bnd, "conv fprop")
        y, st = C.conv_fprop(x, wt, 1, pad, mode, bn, 0, True, None, kc)
        assert torch.equal(y, y0), f"{name}: the statistics epilogue changed the output"
        m, _, _, mt, _ = tiling(n, h, w, k, ci, mode)
        nn = _ceil(co, pick_block_n(co, bn))
        grid, per = grid_tiles(mt, nn)
        assert st.shape == (2, grid // nn, co)
        _check_stats(name, st, y, nm.conv_epilogue_depth(per), "conv fprop")
        y2, st2 = C.conv_fprop(x, wt, 1, pad, mode, bn, 0, True, None, kc)
        assert torch.equal(y2, y) and torch.equal(st2, st), f"{name}: not repeatable"


@pytest.mark.parametrize("shifted", [False, True], ids=["randn", "shifted"])
@pytest.mark.parametrize("n,ci,co,k,h,w", SHAPES, ids=SHAPE_IDS)
def test_data_gradient_and_fused_partial_sums_elementwise(n, ci, co, k, h, w, shifted):
    C = _ext()
    x, wt, dy = _inputs(n, ci, co, k, h, w, shifted)
    pad = (k - 1) // 2
    g = torch.Generator("cuda").manual_seed(3)
    addend = torch.randn(x.shape, device="cuda", generator=g).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    bn_x = (torch.randn(x.shape, device="cuda", generator=g) * 2 + 1).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    mask_bits = torch.rand(n * h * w, ci, device="cuda", generator=g) > 0.4
    packed = (mask_bits.view(-1, ci // 8, 8).to(torch.uint8) << torch.arange(8, device="cuda", dtype=torch.uint8)).sum(-1).to(torch.uint8)
    mean = torch.randn(ci, device="cuda", generator=g) * 0.5 + 1
    rstd = torch.rand(ci, device="cuda", generator=g) + 0.5
    stats = torch.stack([mean, rstd]).contiguous()
    ref, acc = nm.conv_reference("dgrad", dy, wt, 1, pad, shape=x.shape)
    ref_a, acc_a = nm.conv_reference("dgrad", dy, wt, 1, pad, shape=x.shape, addend=addend)
    bnd, bnd_a = nm.bound(ref, acc, torch.bfloat16), nm.bound(ref_a, acc_a, torch.bfloat16)
    for mode, bn, kc in variants(ci, co, k, h, w, n):
        name = f"dgrad mode {mode} block_n {bn} kc {kc}"
        dx = C.conv_dgrad(dy, wt, 1, pad, mode, bn, 0, kc)[0]
        nm.check(name, dx, ref, bnd, "conv dgrad")
        only_add = C.conv_dgrad(dy, wt, 1, pad, mode, bn, 0, kc, addend)[0]
        nm.check(name + " + addend", only_add, ref_a, bnd_a, "conv dgrad")
        _, _, _, mt, _ = tiling(n, h, w, k, co, mode)
        nn = _ceil(ci, pick_block_n(ci, bn))
        grid, per = grid_tiles(mt, nn)
        depth = nm.conv_epilogue_depth(per)
        for use_mask in (True, False):
            m = packed if use_mask else None
            dxf, part = C.conv_dgrad(dy, wt, 1, pad, mode, bn, 0, kc, addend, bn_x, m, stats)
            assert torch.equal(dxf, only_add), f"{name}: the BatchNorm partial sums changed dx"
            assert part.shape == (2, grid // nn, ci)
            d = nm.as_rows(dxf).double()
            if use_mask:
                d = torch.where(mask_bits, d, 0.0)
            t = d * (nm.as_rows(bn_x).double() - mean.double()) * rstd.double()
            tot = part.double().sum(1)
            nm.check(f"{name} mask {use_mask}: S1", tot[0], d.sum(0), depth * nm.U * d.abs().sum(0) + nm.FLOOR, "conv dgrad S1")
            nm.check(f"{name} mask {use_mask}: S2", tot[1], t.sum(0), (depth + 3) * nm.U * t.abs().sum(0) + nm.FLOOR,
                     "conv dgrad S2")
        assert torch.equal(C.conv_dgrad(dy, wt, 1, pad, mode, bn, 0, kc)[0], dx), f"{name}: not repeatable"


@pytest.mark.parametrize("shifted", [False, True], ids=["randn", "shifted"])
@pytest.mark.parametrize("n,ci,co,k,h,w", SHAPES, ids=SHAPE_IDS)
def test_weight_gradient_elementwise(n, ci, co, k, h, w, shifted):
    C = _ext()
    x, wt, dy = _inputs(n, ci, co, k, h, w, shifted)
    pad = (k - 1) // 2
    ref, acc1 = nm.conv_reference("wgrad", dy, x, 1, pad, shape=wt.shape, k_pixels=0, c_acc=1.0)
    P = acc1 / nm.U                                            # the same gradient of the absolute values
    ran = 0
    for split in (0, 1, 7, SMS):
        for tile_n in (0, 64, 128):
            plan = wgrad_plan(n, h, w, ci, co, k, split, tile_n)
            if plan is None:
                with pytest.raises(RuntimeError):
                    C.conv_wgrad(dy, x, k, 1, pad, split, 0, tile_n)
                continue
            kb, nkb, sp = plan
            dw = C.conv_wgrad(dy, x, k, 1, pad, split, 0, tile_n)
            acc = (nm.C_ACC * (_ceil(nkb, sp) * kb + 1) + _ceil(sp, 8) + 8) * nm.U * P
            nm.check(f"wgrad split {split} ({sp}) tile_n {tile_n}", dw, ref, nm.bound(ref, acc, dw.dtype), "conv wgrad")
            assert torch.equal(dw, C.conv_wgrad(dy, x, k, 1, pad, split, 0, tile_n)), "wgrad is not repeatable"
            ran += 1
    assert ran or wgrad_plan(n, h, w, ci, co, k, 0, 0) is None      # W = 83: no pixel block is a multiple of 16


# ---- the strided 7x7 stem -----------------------------------------------------------------------------------------------
STEM_SHAPES = [(2, 224, 224), (3, 64, 96), (1, 32, 256), (32, 224, 224)]


def _stem_inputs(n, h, w, shifted):
    g = torch.Generator("cuda").manual_seed(n + h + w)
    cl = torch.channels_last
    x = torch.randn(n, 3, h, w, device="cuda", generator=g) + (2.0 if shifted else 0.0)
    x = x.to(torch.bfloat16).contiguous(memory_format=cl)
    wt = (torch.randn(64, 3, 7, 7, device="cuda", generator=g) / 147 ** 0.5).to(torch.bfloat16).contiguous(memory_format=cl)
    dy = (torch.randn(n, 64, h // 2, w // 2, device="cuda", generator=g) + (1.0 if shifted else 0.0)).to(torch.bfloat16)
    return x, wt, dy.contiguous(memory_format=cl)


def stem_pack_input_reference(x):
    """xp[n, i, wp] = (x[n, :, 2i - 3, wp - 4], 0, x[n, :, 2i - 2, wp - 4], 0), zero outside the image."""
    n, _, h, w = x.shape
    xp = torch.zeros(n, h + 6, w + 8, 4, dtype=x.dtype, device=x.device)
    xp[:, 3:3 + h, 4:4 + w, :3] = x.permute(0, 2, 3, 1)
    return xp.view(n, h // 2 + 3, 2, w + 8, 4).permute(0, 1, 3, 2, 4).reshape(n, h // 2 + 3, w + 8, 8)


def stem_pack_weight_reference(wt):
    """w2[co, t, p, 4 rr + c] = w[co, c, 2t + rr, p - 1] (zero where r = 7, p = 0 or c = 3)."""
    w8 = torch.zeros(wt.shape[0], 8, 8, 4, dtype=wt.dtype, device=wt.device)     # [co, r, p, c]
    w8[:, :7, 1:, :3] = wt.permute(0, 2, 3, 1)
    return w8.view(-1, 4, 2, 8, 4).permute(0, 1, 3, 2, 4).reshape(-1, 256)


@pytest.mark.parametrize("shifted", [False, True], ids=["randn", "shifted"])
@pytest.mark.parametrize("n,h,w", STEM_SHAPES)
def test_stem_elementwise(n, h, w, shifted):
    C = _ext()
    x, wt, dy = _stem_inputs(n, h, w, shifted)
    xp_ref, w2_ref = stem_pack_input_reference(x), stem_pack_weight_reference(wt)
    assert torch.equal(C.stem_pack_input(x), xp_ref)
    assert torch.equal(C.stem_pack_weight(wt), w2_ref)
    ref, acc = nm.conv_reference("fprop", x, wt, 2, 3)
    bnd = nm.bound(ref, acc, torch.bfloat16)
    ho = h // 2
    grid, per = grid_tiles(n * ho, 1)
    outs = []
    for stats in (False, True):
        for resident in (True, False):
            y, part, xp = C.stem_conv_fprop(x, wt, stats, resident)
            assert torch.equal(xp, xp_ref)
            nm.check(f"stem fprop stats {stats} resident {resident}", y, ref, bnd, "stem fprop")
            if stats:
                assert part.shape == (2, grid, 64)
                _check_stats(f"stem resident {resident}", part, y, nm.conv_epilogue_depth(per), "stem fprop")
            outs.append(y)
    assert all(torch.equal(o, outs[0]) for o in outs)
    # weight gradient: split over pixels, fixed-order reduction of at most SMS partials
    red = _ceil(SMS, 8) + 8
    ref_w, acc_w = nm.conv_reference("wgrad", dy, x, 2, 3, shape=wt.shape, k_pixels=n * ho * (w // 2), reduce_depth=red)
    # the packed gradient also covers the structural-zero filter slots: the same windows over the padded 4-channel image
    x4 = torch.zeros(n, 4, h + 6, w + 7, dtype=x.dtype, device=x.device)
    x4[:, :3, 3:3 + h, 4:4 + w] = x
    ref8, acc8 = nm.conv_reference("wgrad", dy, x4, 2, 0, shape=(64, 4, 8, 8), k_pixels=n * ho * (w // 2), reduce_depth=red)

    def pack(t):                                               # [co, c, r, p] -> [co, 256]
        return t.permute(0, 2, 3, 1).reshape(-1, 4, 2, 8, 4).permute(0, 1, 3, 2, 4).reshape(-1, 256)
    for variant in (0, 1):
        dw = C.stem_conv_wgrad(dy, xp_ref, h, w, variant, True)
        nm.check(f"stem wgrad variant {variant}", dw, ref_w, nm.bound(ref_w, acc_w, torch.bfloat16), "stem wgrad")
        dw2 = C.stem_conv_wgrad(dy, xp_ref, h, w, variant, False)
        dw2 = dw2.t() if variant == 0 else dw2
        nm.check(f"stem wgrad variant {variant} packed", dw2, pack(ref8), nm.bound(pack(ref8), pack(acc8), torch.bfloat16),
                 "stem wgrad")
