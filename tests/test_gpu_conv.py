"""wgmma convolution kernels (csrc/conv_wgmma.cu, csrc/conv_wgrad_wgmma.cu) against a plain PyTorch fp32 reference of
the same op: forward, data gradient, weight gradient, epilogue BatchNorm statistics, every tiling, ResNet's map sizes."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return float((a.float() - b.float()).norm() / (b.float().norm() + 1e-12))


def _mk(n, ci, co, k, h, w):
    torch.manual_seed(n * 1000 + ci + co + k + h)
    dev = "cuda"
    x = torch.randn(n, ci, h, w, device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    wt = (torch.randn(co, ci, k, k, device=dev) / (ci * k * k) ** 0.5).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    dy = torch.randn(n, co, h, w, device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    return x, wt, dy


def _ref(x, wt, dy, k):
    xf = x.float().requires_grad_(True)
    wf = wt.float().requires_grad_(True)
    y = F.conv2d(xf, wf, padding=(k - 1) // 2)
    y.backward(dy.float())
    return y.detach(), xf.grad, wf.grad


SHAPES = [  # n, cin, cout, k, h, w
    (4, 64, 64, 1, 56, 56), (2, 256, 64, 1, 56, 56), (3, 64, 256, 1, 28, 28), (5, 512, 128, 1, 14, 14), (6, 128, 512, 1, 7, 7),
    (1, 2048, 512, 1, 7, 7), (2, 64, 64, 3, 56, 56), (3, 128, 128, 3, 28, 28), (4, 256, 256, 3, 14, 14), (6, 512, 512, 3, 7, 7),
    (2, 64, 128, 3, 9, 12), (1, 64, 64, 1, 5, 3),
]


@pytest.mark.parametrize("n,ci,co,k,h,w", SHAPES)
def test_forward_and_data_gradient_match_fp32_reference(n, ci, co, k, h, w):
    from b200ddp import _ext
    C = _ext.get()
    x, wt, dy = _mk(n, ci, co, k, h, w)
    y_ref, dx_ref, _ = _ref(x, wt, dy, k)
    pad = (k - 1) // 2
    modes = [-1] if k == 1 else [1, 2]
    for mode in modes:
        for bn in (0, 64, 128, 256):                      # 256 runs as two 128-wide n-tiles (csrc/conv.h)
            if bn and (co % bn or ci % bn):
                continue
            y = C.conv_fprop(x, wt, 1, pad, mode, bn, 0, False)[0]
            dx = C.conv_dgrad(dy, wt, 1, pad, mode, bn, 0)[0]
            assert y.shape == y_ref.shape and y.is_contiguous(memory_format=torch.channels_last)
            assert _rel(y, y_ref) < 6e-3, (mode, bn, _rel(y, y_ref))
            assert _rel(dx, dx_ref) < 6e-3, (mode, bn, _rel(dx, dx_ref))


@pytest.mark.parametrize("n,ci,co,k,h,w", SHAPES)
def test_weight_gradient_matches_fp32_reference(n, ci, co, k, h, w):
    from b200ddp import _ext
    C = _ext.get()
    x, wt, dy = _mk(n, ci, co, k, h, w)
    _, _, dw_ref = _ref(x, wt, dy, k)
    pad = (k - 1) // 2
    for (split, tm, tn) in [(0, 0, 0), (1, 0, 0), (3, 128, 64)]:
        dw = C.conv_wgrad(dy, x, k, 1, pad, split, tm, tn)
        assert dw.shape == dw_ref.shape
        assert _rel(dw, dw_ref) < 6e-3, (split, tm, tn, _rel(dw, dw_ref))
    # deterministic: fixed-order reduction of the split partials
    a = C.conv_wgrad(dy, x, k, 1, pad, 0, 0, 0)
    b = C.conv_wgrad(dy, x, k, 1, pad, 0, 0, 0)
    assert torch.equal(a, b)


@pytest.mark.parametrize("n,ci,co,k,h,w", [(4, 64, 256, 1, 56, 56), (3, 256, 128, 1, 28, 28), (2, 64, 64, 3, 56, 56), (5, 256, 256, 3, 14, 14),
                                           (7, 512, 2048, 1, 7, 7)])
def test_epilogue_statistics_equal_the_column_sums_of_the_stored_output(n, ci, co, k, h, w):
    from b200ddp import _ext
    C = _ext.get()
    x, wt, _ = _mk(n, ci, co, k, h, w)
    y, st = C.conv_fprop(x, wt, 1, (k - 1) // 2, -1, 0, 0, True)
    assert st.shape[0] == 2 and st.shape[2] == co
    y2 = y.permute(0, 2, 3, 1).reshape(-1, co).float()
    s, q = st[0].sum(0), st[1].sum(0)
    assert torch.allclose(s, y2.sum(0), rtol=2e-3, atol=2e-2 * float(y2.abs().sum(0).max()) / y2.shape[0] + 1e-2)
    assert torch.allclose(q, (y2 * y2).sum(0), rtol=2e-3, atol=1e-2)
    # identical output with and without the statistics epilogue, and run to run
    assert torch.equal(y, C.conv_fprop(x, wt, 1, (k - 1) // 2, -1, 0, 0, False)[0])
    assert torch.equal(st, C.conv_fprop(x, wt, 1, (k - 1) // 2, -1, 0, 0, True)[1])


def test_bottleneck_matches_stock_modules_forward_and_backward(monkeypatch):
    """Conv2dTC + FusedBatchNormAct2d with statistics from the epilogue vs nn.Conv2d + nn.BatchNorm2d in fp32."""
    import torch.nn as nn
    monkeypatch.setenv("B200DDP_CONV", "native")
    from b200ddp.models.resnet import Bottleneck
    from b200ddp.utils import to_mixed_bf16
    torch.manual_seed(0)
    blk = to_mixed_bf16(Bottleneck(256, 64).cuda()).to(memory_format=torch.channels_last)
    ref = nn.Sequential(nn.Conv2d(256, 64, 1, bias=False), nn.BatchNorm2d(64), nn.ReLU(), nn.Conv2d(64, 64, 3, padding=1, bias=False), nn.BatchNorm2d(64),
                        nn.ReLU(), nn.Conv2d(64, 256, 1, bias=False), nn.BatchNorm2d(256)).cuda()
    with torch.no_grad():
        for a, b in ((blk.conv1, ref[0]), (blk.conv2, ref[3]), (blk.conv3, ref[6])):
            b.weight.copy_(a.weight.float())
    x = torch.randn(8, 256, 28, 28, device="cuda").to(torch.bfloat16).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    xr = x.detach().float().requires_grad_(True)
    y = blk(x)
    yr = torch.relu(ref(xr) + xr)
    assert _rel(y, yr) < 3e-2
    g = torch.randn_like(yr)
    y.backward(g.to(torch.bfloat16).contiguous(memory_format=torch.channels_last))
    yr.backward(g)
    assert _rel(x.grad, xr.grad) < 6e-2
    for a, b in ((blk.conv1, ref[0]), (blk.conv2, ref[3]), (blk.conv3, ref[6])):
        assert _rel(a.weight.grad, b.weight.grad) < 1e-1      # bf16 activations through three BatchNorms vs an fp32 chain
        assert a.weight.grad.stride() == a.weight.stride()
    assert torch.allclose(blk.bn1.running_mean, ref[1].running_mean, atol=2e-2)


@pytest.mark.parametrize("n,ci,co,k,h,w", [(4, 64, 256, 1, 56, 56), (3, 128, 128, 3, 28, 28), (2, 64, 64, 3, 56, 56), (5, 1024, 256, 1, 14, 14)])
def test_data_gradient_epilogue_fusion_addend_and_batchnorm_partial_sums(n, ci, co, k, h, w):
    """conv_dgrad(+ addend)(+ S1/S2 of the BatchNorm backward that consumes dx) vs the same quantities computed by hand."""
    from b200ddp import _ext
    C = _ext.get()
    x, wt, dy = _mk(n, ci, co, k, h, w)
    pad = (k - 1) // 2
    torch.manual_seed(3)
    addend = torch.randn_like(x)
    bn_x = torch.randn_like(x)                             # input of the (imaginary) BatchNorm whose output fed this convolution
    mask_bits = torch.rand(n, h, w, ci, device="cuda") > 0.4
    packed = (mask_bits.view(-1, ci // 8, 8).to(torch.uint8) << torch.arange(8, device="cuda", dtype=torch.uint8)).sum(-1).to(torch.uint8)
    mean = torch.randn(ci, device="cuda") * 0.1
    rstd = torch.rand(ci, device="cuda") + 0.5
    stats = torch.stack([mean, rstd]).contiguous()
    plain = C.conv_dgrad(dy, wt, 1, pad, -1, 0, 0)[0]
    dx, part = C.conv_dgrad(dy, wt, 1, pad, -1, 0, 0, 0, addend, bn_x, packed.contiguous(), stats)
    ref = (plain.float() + addend.float()).to(torch.bfloat16)
    assert _rel(dx, ref) < 1e-2
    d2 = dx.permute(0, 2, 3, 1).reshape(-1, ci).float()
    m2 = mask_bits.reshape(-1, ci).float()
    xh = (bn_x.permute(0, 2, 3, 1).reshape(-1, ci).float() - mean) * rstd
    s1, s2 = (d2 * m2).sum(0), (d2 * m2 * xh).sum(0)
    assert part.shape[0] == 2 and part.shape[2] == ci
    assert torch.allclose(part[0].sum(0), s1, rtol=2e-3, atol=0.5), float((part[0].sum(0) - s1).abs().max())
    assert torch.allclose(part[1].sum(0), s2, rtol=2e-3, atol=0.5), float((part[1].sum(0) - s2).abs().max())
    only_add = C.conv_dgrad(dy, wt, 1, pad, -1, 0, 0, 0, addend)[0]
    assert torch.equal(only_add, dx)


@pytest.mark.parametrize("with_downsample", [False, True])
def test_fused_bottleneck_node_equals_the_per_layer_composition(with_downsample, monkeypatch):
    """ops/bottleneck.py (one autograd node, epilogue-fused backward) vs the same block composed of per-layer autograd ops."""
    import copy
    import torch.nn as nn
    from b200ddp.models.resnet import Bottleneck
    from b200ddp.ops import FusedBatchNormAct2d, PointwiseConv2d
    from b200ddp.utils import to_mixed_bf16
    monkeypatch.setenv("B200DDP_CONV", "native")
    torch.manual_seed(0)
    inpl = 64 if with_downsample else 256
    ds = nn.Sequential(PointwiseConv2d(64, 256), FusedBatchNormAct2d(256)) if with_downsample else None
    a = to_mixed_bf16(Bottleneck(inpl, 64, 1, ds).cuda()).to(memory_format=torch.channels_last)
    b = copy.deepcopy(a)
    x = torch.randn(8, inpl, 28, 28, device="cuda").to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    xa, xb = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
    g = torch.randn(8, 256, 28, 28, device="cuda").to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    monkeypatch.setenv("B200DDP_BLOCK_FUSE", "1")
    ya = a(xa)
    ya.backward(g)
    monkeypatch.setenv("B200DDP_BLOCK_FUSE", "0")
    yb = b(xb)
    yb.backward(g)
    assert ya.grad_fn.__class__.__name__.startswith("_BottleneckFn")
    assert _rel(ya, yb) < 1e-3
    assert _rel(xa.grad, xb.grad) < 3e-2
    for (n, p), q in zip(a.named_parameters(), b.parameters()):
        assert p.grad is not None and q.grad is not None, n
        assert _rel(p.grad, q.grad) < 3e-2, (n, _rel(p.grad, q.grad))
        assert p.grad.stride() == p.stride(), n
    for (n, u), v in zip(a.named_buffers(), b.buffers()):
        assert torch.allclose(u.float(), v.float(), atol=1e-3), n


# ---- the strided 7x7 stem ------------------------------------------------------------------------------------------
STEM_SHAPES = [(2, 224, 224), (3, 64, 96), (1, 32, 256), (32, 224, 224)]   # n, h, w   (w / 2 a multiple of 16, <= 128)


def _stem_mk(n, h, w):
    torch.manual_seed(n + h + w)
    x = torch.randn(n, 3, h, w, device="cuda").to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    wt = (torch.randn(64, 3, 7, 7, device="cuda") / 147 ** 0.5).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    dy = torch.randn(n, 64, h // 2, w // 2, device="cuda").to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    return x, wt, dy


@pytest.mark.parametrize("n,h,w", STEM_SHAPES)
def test_stem_forward_statistics_and_weight_gradient_match_fp32_reference(n, h, w):
    from b200ddp import _ext
    C = _ext.get()
    x, wt, dy = _stem_mk(n, h, w)
    wf = wt.float().requires_grad_(True)
    y_ref = F.conv2d(x.float(), wf, None, 2, 3)
    y_ref.backward(dy.float())
    for stats in (False, True):
        for resident in (True, False):
            y, part, xp = C.stem_conv_fprop(x, wt, stats, resident)
            assert y.shape == y_ref.shape and y.is_contiguous(memory_format=torch.channels_last)
            assert _rel(y, y_ref) < 6e-3, (stats, resident, _rel(y, y_ref))
            if stats:
                s = part.sum(dim=1)
                yf = y.float()
                assert torch.allclose(s[0], yf.sum(dim=(0, 2, 3)), rtol=2e-3, atol=2e-2 * (n * h * w) ** 0.5)
                assert torch.allclose(s[1], (yf * yf).sum(dim=(0, 2, 3)), rtol=2e-3, atol=1e-2)
    for variant in (0, 1):                                   # dedicated kernel / generic split-pixel kernel
        dw = C.stem_conv_wgrad(dy, xp, h, w, variant)
        assert dw.shape == wt.shape and dw.is_contiguous(memory_format=torch.channels_last)
        assert _rel(dw, wf.grad) < 6e-3, (variant, _rel(dw, wf.grad))


def test_stem_module_matches_stock_conv_through_autograd():
    """ops.StemConv7x7 (native path) against nn.Conv2d with the same weights: output, weight gradient, and the BatchNorm that
    consumes the epilogue statistics against the same BatchNorm computing its own."""
    import torch.nn as nn
    from b200ddp.ops import FusedBatchNormAct2d, StemConv7x7
    x, wt, dy = _stem_mk(4, 224, 224)
    ours = StemConv7x7().cuda().to(torch.bfloat16).to(memory_format=torch.channels_last)
    stock = nn.Conv2d(3, 64, 7, 2, 3, bias=False).cuda().to(torch.bfloat16).to(memory_format=torch.channels_last)
    with torch.no_grad():
        ours.weight.copy_(wt); stock.weight.copy_(wt)
    assert ours._native(x)
    bn_a, bn_b = FusedBatchNormAct2d(64, relu=True).cuda(), FusedBatchNormAct2d(64, relu=True).cuda()
    y, part = ours.forward_with_stats(x)
    za = bn_a(y, partials=part)
    zb = bn_b(stock(x))
    assert part is not None and _rel(za, zb) < 1e-2, _rel(za, zb)
    assert torch.allclose(bn_a.running_mean, bn_b.running_mean, atol=2e-3) and torch.allclose(bn_a.running_var, bn_b.running_var, rtol=1e-2, atol=1e-3)
    za.backward(dy)
    zb.backward(dy)
    assert ours.weight.grad.stride() == ours.weight.stride()
    assert _rel(ours.weight.grad, stock.weight.grad) < 2e-2, _rel(ours.weight.grad, stock.weight.grad)
