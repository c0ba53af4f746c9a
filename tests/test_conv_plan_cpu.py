"""Host-side checks for the wgmma convolution kernels (csrc/conv_wgmma.cu): the kernels need a GPU
(tests/test_gpu_conv.py); what can be pinned down here is their *index plan* - tile shapes, tap -> TMA coordinates, halo row
offsets, mirrored taps of the data gradient, filter column order, accumulator row -> pixel.  ``emulate`` walks exactly the
indices the kernel walks, with zero fill standing in for the TMA unit's out-of-bounds behaviour."""
import pytest
import torch
import torch.nn.functional as F

from b200ddp import _ext

pytestmark = pytest.mark.skipif(not _ext.available(), reason="native extension not built")


def plan(N, H, W, k, mode):
    ok, mode, BH, BI, tiles, dense, acc, a_rows = _ext.get().conv_tile_plan(N, H, W, k, k, mode)
    return ok, dict(mode=mode, BH=BH, BI=BI, tiles=tiles, dense=dense, acc=acc, a_rows=a_rows)


@pytest.mark.parametrize("N,H,W,mode,expect", [
    (32, 56, 56, 2, dict(BH=2, BI=1, dense=112, acc=116, a_rows=232)),
    (32, 28, 28, 2, dict(BH=4, BI=1, dense=112, acc=120, a_rows=180)),
    (32, 14, 14, 2, dict(BH=7, BI=1, dense=98, acc=112, a_rows=144)),
    (32, 7, 7, 2, dict(BH=7, BI=1, dense=49, acc=63, a_rows=81)),
    (32, 56, 56, 1, dict(BH=2, BI=1, dense=112, acc=112, a_rows=112)),
    (32, 14, 14, 1, dict(BH=7, BI=1, dense=98, acc=98, a_rows=98)),
    (32, 7, 7, 1, dict(BH=7, BI=2, dense=98, acc=98, a_rows=98)),
])
def test_tile_plans_of_the_resnet_maps(N, H, W, mode, expect):
    ok, p = plan(N, H, W, 3, mode)
    assert ok and p["mode"] == mode
    for key, val in expect.items():
        assert p[key] == val, (key, p)
    assert p["acc"] <= 128 and H % p["BH"] == 0 and N % p["BI"] == 0


def test_flat_plan_for_pointwise_and_rejections():
    ok, p = plan(32, 56, 56, 1, -1)
    assert ok and p["mode"] == 0 and p["tiles"] == 32 * 56 * 56 // 128 and p["dense"] == 128
    assert not plan(1, 8, 300, 3, -1)[0]                    # rows wider than a tile
    assert not plan(1, 8, 8, 1, 2)[0]                       # no halo tiling for 1x1


def emulate(a, w, mode, dgrad):
    """a [N,C,H,W] (x, or dy for the data gradient), w [K,C,3,3] (fp32 here).  Mirrors conv_tap_gemm_kernel."""
    N, Ca, H, W = a.shape
    K, C = w.shape[0], w.shape[1]
    Kc, Nc = (K, C) if dgrad else (C, K)
    assert Ca == Kc
    ok, p = plan(N, H, W, 3, mode)
    assert ok
    BH, BI = p["BH"], p["BI"]
    Wp = W + 2
    an = a.permute(0, 2, 3, 1).contiguous()                       # NHWC
    wk = w.permute(0, 2, 3, 1).reshape(K, 9 * C)                  # [K][r][s][C] == row-major [K, 9C]
    out = torch.zeros(N, H, W, Nc)
    tiles_h = H // BH
    for mt in range(p["tiles"]):
        img0, h0 = (mt // tiles_h) * BI, (mt % tiles_h) * BH
        acc = torch.zeros(128 + 2 * Wp + 2, Nc)[:128]
        for cb in range(Kc // 64):
            if mode == 2:                                         # halo: ONE load per channel block, box {64, Wp, BH+2, 1} at (c0, -1, h0-1, img)
                halo = torch.zeros((BH + 2) * Wp + 128 + 2 * Wp + 2, 64)
                for hh in range(BH + 2):
                    for ww in range(Wp):
                        hs, ws_ = h0 - 1 + hh, ww - 1
                        if 0 <= hs < H and 0 <= ws_ < W:
                            halo[hh * Wp + ww] = an[img0, hs, ws_, cb * 64:(cb + 1) * 64]
            for tap in range(9):
                r, s = tap // 3, tap % 3
                if mode == 2:
                    rr, sc = (2 - r, 2 - s) if dgrad else (r, s)
                    off = rr * Wp + sc                            # descriptor start advanced by whole 128-byte rows
                    atile = halo[off:off + 128]
                else:                                             # patch: box {64, W, BH, BI} at (c0, dw, h0 + dh, img0)
                    dh, dw = (1 - r, 1 - s) if dgrad else (r - 1, s - 1)
                    atile = torch.zeros(128, 64)
                    for bi in range(BI):
                        for hh in range(BH):
                            for ww in range(W):
                                hs, ws_ = h0 + hh + dh, ww + dw
                                if 0 <= hs < H and 0 <= ws_ < W:
                                    atile[(bi * BH + hh) * W + ww] = an[img0 + bi, hs, ws_, cb * 64:(cb + 1) * 64]
                if dgrad:     # B read MN-major: rows = Cout (reduction), columns = Cin at offset tap * Cin
                    b = wk[cb * 64:(cb + 1) * 64, tap * C: tap * C + Nc].t()          # [Nc, 64]
                else:         # B K-major: box at column tap * Cin + cb * 64
                    b = wk[:, tap * C + cb * 64: tap * C + (cb + 1) * 64]             # [Nc, 64]
                acc += atile @ b.t()
        row0 = (img0 * H + h0) * W
        flat = out.view(N * H * W, Nc)
        for i in range(128):                                      # epilogue: accumulator row -> dense row of the output tile
            if mode == 2:
                hh, ww = divmod(i, Wp)
                valid, dense = hh < BH and ww < W, hh * W + ww
            else:
                valid, dense = i < p["dense"], i
            if valid:
                flat[row0 + dense] = acc[i]
    return out.permute(0, 3, 1, 2)


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("N,C,H,W,K", [(2, 64, 8, 8, 64), (4, 64, 7, 7, 128), (1, 128, 6, 10, 64)])
def test_tap_gemm_plan_equals_the_convolution(N, C, H, W, K, mode):
    torch.manual_seed(0)
    x = torch.randn(N, C, H, W)
    w = torch.randn(K, C, 3, 3) * 0.1
    ref = F.conv2d(x, w, padding=1)
    assert torch.allclose(emulate(x, w, mode, False), ref, atol=1e-3, rtol=1e-4)


@pytest.mark.parametrize("mode", [1, 2])
def test_mirrored_taps_give_the_data_gradient(mode):
    torch.manual_seed(1)
    N, C, H, W, K = 2, 64, 8, 6, 128
    x = torch.randn(N, C, H, W, requires_grad=True)
    w = torch.randn(K, C, 3, 3) * 0.1
    dy = torch.randn(N, K, H, W)
    F.conv2d(x, w, padding=1).backward(dy)
    assert torch.allclose(emulate(dy, w, mode, True), x.grad, atol=1e-3, rtol=1e-4)


def test_conv_module_falls_back_on_cpu_and_keeps_parameter_layout():
    from b200ddp.ops import Conv3x3, PointwiseConv2d
    m = Conv3x3(8, 6)
    ref = torch.nn.Conv2d(8, 6, 3, padding=1, bias=False)
    ref.load_state_dict(m.state_dict())
    x = torch.randn(2, 8, 5, 5)
    assert torch.allclose(m(x), ref(x))
    y, part = PointwiseConv2d(8, 4, stride=2).forward_with_stats(x)
    assert part is None and y.shape == (2, 4, 3, 3)


def test_stem_window_algebra_and_geometry():
    """The layout contract of the wgmma stem (csrc/conv.h): with the input repacked into a zero-bordered image of ROW PAIRS
    (16-byte pixels: padded rows 2i and 2i+1, 4 channels each), the 64-element window starting every 16 elements (32 bytes)
    of pair row oh + t IS the im2col row of filter rows 2t, 2t+1 - for forward and weight gradient.  Checked here in plain
    PyTorch against F.conv2d; the host-side geometry predicate too."""
    import torch
    import torch.nn.functional as F
    from b200ddp import _ext
    C = _ext.get()
    assert C.stem_conv_supported(224, 224) and C.stem_conv_supported(64, 96)
    assert not C.stem_conv_supported(224, 225) and not C.stem_conv_supported(224, 512) and not C.stem_conv_supported(224, 40)
    torch.manual_seed(0)
    n, h, w, k = 2, 32, 64, 64
    x, wt = torch.randn(n, 3, h, w), torch.randn(k, 3, 7, 7)
    ho, wo, hp2, wp = h // 2, w // 2, h // 2 + 3, w + 8
    pad = torch.zeros(n, 2 * hp2, wp, 4)                       # padded image: pixel (h, w) at (h + 3, w + 4), 4th channel zero
    pad[:, 3:3 + h, 4:4 + w, :3] = x.permute(0, 2, 3, 1)
    xp = torch.cat([pad[:, 0::2], pad[:, 1::2]], dim=3)         # [n, hp2, wp, 8]: rows 2i | 2i+1
    w2 = torch.zeros(k, 4, 8, 8)                                # [co, t, p, j]: r = 2t + j // 4, s = p - 1, c = j % 4
    wr = torch.zeros(k, 8, 7, 4)
    wr[:, :7, :, :3] = wt.permute(0, 2, 3, 1)
    for t in range(4):
        for half in range(2):
            w2[:, t, 1:8, 4 * half:4 * half + 4] = wr[:, 2 * t + half]
    w2 = w2.reshape(k, 256)
    flat = xp.reshape(n, hp2, wp * 8)
    dy = torch.randn(n, ho, wo, k)
    y = torch.zeros(n, ho, wo, k)
    dw2 = torch.zeros(k, 4, 64)
    for t in range(4):
        win = flat[:, t:t + ho, :].unfold(2, 64, 16)[:, :, :wo, :]
        y += win @ w2[:, t * 64:(t + 1) * 64].t()
        dw2[:, t, :] = torch.einsum("nhwk,nhwe->ke", dy, win)
    wg = wt.clone().requires_grad_(True)
    ref = F.conv2d(x, wg, None, 2, 3)
    ref.backward(dy.permute(0, 3, 1, 2))
    assert torch.allclose(y, ref.detach().permute(0, 2, 3, 1), atol=1e-3)
    d = dw2.reshape(k, 4, 8, 2, 4)                               # [co, t, p, half, c]
    dw = torch.stack([d[:, r // 2, 1:8, r % 2, :3] for r in range(7)], dim=1).permute(0, 3, 1, 2)   # [co, c, r, s]
    assert torch.allclose(dw, wg.grad, atol=2e-3, rtol=1e-4)


def test_conv_modules_fall_back_to_stock_on_cpu_and_keep_stock_state_dicts():
    """StemConv7x7 / PointwiseConv2d / Conv3x3 are nn.Conv2d subclasses: same parameter names and shapes (checkpoints and DDP
    bucket layouts are unchanged), stock computation on CPU, and no epilogue statistics there."""
    import torch
    import torch.nn as nn
    from b200ddp.ops import Conv3x3, PointwiseConv2d, StemConv7x7
    torch.manual_seed(0)
    for ours, stock, x in ((StemConv7x7(), nn.Conv2d(3, 64, 7, 2, 3, bias=False), torch.randn(2, 3, 32, 32)),
                           (PointwiseConv2d(64, 128), nn.Conv2d(64, 128, 1, bias=False), torch.randn(2, 64, 8, 8)),
                           (Conv3x3(64, 64, stride=2), nn.Conv2d(64, 64, 3, 2, 1, bias=False), torch.randn(2, 64, 8, 8))):
        assert list(ours.state_dict().keys()) == list(stock.state_dict().keys()) == ["weight"]
        stock.load_state_dict(ours.state_dict())
        y, part = ours.forward_with_stats(x)
        assert part is None and torch.allclose(y, stock(x), atol=1e-6)
        assert torch.allclose(ours(x), stock(x), atol=1e-6)
