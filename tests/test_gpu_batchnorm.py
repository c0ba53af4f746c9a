"""Fused BatchNorm(+residual)(+ReLU) channels_last kernels vs a plain fp32 PyTorch reference."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _reference(x, res, w, b, relu, eps=1e-5):
    xr = x.detach().float().requires_grad_()
    rr = res.detach().float().requires_grad_() if res is not None else None
    wr, br = w.detach().clone().requires_grad_(), b.detach().clone().requires_grad_()
    rm, rv = torch.zeros_like(w), torch.ones_like(w)
    y = F.batch_norm(xr, rm, rv, wr, br, True, 0.1, eps)
    if rr is not None:
        y = y + rr
    if relu:
        y = torch.relu(y)
    return xr, rr, wr, br, rm, rv, y


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("shape", [(32, 64, 56, 56), (32, 2048, 7, 7), (4, 24, 5, 5), (8, 256, 14, 14), (1, 8, 1, 3)])
@pytest.mark.parametrize("relu,residual", [(False, False), (True, False), (True, True), (False, True)])
def test_fused_batchnorm_fwd_bwd(dtype, shape, relu, residual):
    from b200ddp import _ext
    from b200ddp.ops import FusedBatchNormAct2d
    C = _ext.get()
    torch.manual_seed(0)
    dev = "cuda"
    x = (torch.randn(*shape, device=dev) * 2 + 0.5).to(dtype).contiguous(memory_format=torch.channels_last).requires_grad_()
    res = torch.randn(*shape, device=dev).to(dtype).contiguous(memory_format=torch.channels_last).requires_grad_() if residual else None
    bn = FusedBatchNormAct2d(shape[1], relu=relu).to(dev)
    with torch.no_grad():
        bn.weight.uniform_(0.5, 1.5)
        bn.bias.uniform_(-0.5, 0.5)
    before = C.launch_count()
    y = bn(x, residual=res) if residual else bn(x)
    assert C.launch_count() - before in (1, 2), "forward = one fused launch (or stats + apply)"
    assert y.dtype == dtype and y.is_contiguous(memory_format=torch.channels_last)
    dy = torch.randn_like(y)
    y.backward(dy)
    assert C.launch_count() - before in (2, 4)
    xr, rr, wr, br, rm, rv, yr = _reference(x, res, bn.weight, bn.bias, relu)
    yr.backward(dy.float())
    tol = 2e-4 if dtype == torch.float32 else 4e-2
    assert torch.allclose(y.float(), yr, atol=tol, rtol=tol), (y.float() - yr).abs().max()
    gscale = max(1.0, float(xr.grad.abs().max()))
    assert torch.allclose(x.grad.float(), xr.grad, atol=tol * gscale, rtol=tol), (x.grad.float() - xr.grad).abs().max()
    if residual:
        assert torch.allclose(res.grad.float(), rr.grad, atol=tol, rtol=tol)
    n = x.numel() / shape[1]
    ptol = tol * max(1.0, n ** 0.5)
    assert torch.allclose(bn.weight.grad, wr.grad, atol=ptol, rtol=tol * 4), (bn.weight.grad - wr.grad).abs().max()
    assert torch.allclose(bn.bias.grad, br.grad, atol=ptol, rtol=tol * 4)
    assert torch.allclose(bn.running_mean, rm, atol=tol, rtol=tol) and torch.allclose(bn.running_var, rv, atol=tol, rtol=tol)
    assert int(bn.num_batches_tracked) == 1
    # reproducible: no float atomics anywhere
    bn2 = FusedBatchNormAct2d(shape[1], relu=relu).to(dev)
    bn2.load_state_dict(bn.state_dict())
    y1 = bn2(x.detach(), residual=res.detach() if residual else None)
    bn2.load_state_dict(bn.state_dict())
    y2 = bn2(x.detach(), residual=res.detach() if residual else None)
    assert torch.equal(y1, y2)


def test_resnet50_fused_matches_stock_modules():
    """Whole network, fp32 channels_last: fused-BN ResNet-50 vs torchvision's (same weights) - outputs and grads agree."""
    import torchvision
    from b200ddp.models import resnet50
    torch.manual_seed(1)
    ours = resnet50().cuda().to(memory_format=torch.channels_last)
    stock = torchvision.models.resnet50().cuda().to(memory_format=torch.channels_last)
    stock.load_state_dict(ours.state_dict())
    x = torch.randn(8, 3, 96, 96, device="cuda").contiguous(memory_format=torch.channels_last)
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        a, b = ours(x), stock(x)
        a.square().mean().backward()
        b.square().mean().backward()
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
    assert torch.allclose(a, b, atol=2e-3, rtol=2e-3), (a - b).abs().max()
    for (n, p), q in zip(ours.named_parameters(), stock.parameters()):
        # 53 normalisation layers deep, a different (but fixed) summation order flips a few ReLU masks: compare in norm
        rel = float((p.grad - q.grad).norm() / (q.grad.norm() + 1e-12))
        assert rel < 3e-2, (n, rel)
    for (n, p), q in zip(ours.named_buffers(), stock.buffers()):
        assert torch.allclose(p.float(), q.float(), atol=1e-3, rtol=1e-3), n


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("shape", [(32, 64, 112, 112), (2, 8, 7, 9), (3, 16, 6, 6), (1, 8, 1, 1)])
def test_maxpool3x3s2_matches_torch(dtype, shape):
    from b200ddp.ops import MaxPool3x3s2
    torch.manual_seed(0)
    x = torch.randn(*shape, device="cuda").to(dtype).contiguous(memory_format=torch.channels_last).requires_grad_()
    y = MaxPool3x3s2()(x)
    dy = torch.randn_like(y)
    y.backward(dy)
    xr = x.detach().clone().requires_grad_()
    yr = F.max_pool2d(xr, 3, stride=2, padding=1)
    yr.backward(dy)
    assert torch.equal(y, yr)
    assert torch.allclose(x.grad.float(), xr.grad.float(), atol=1e-2 if dtype == torch.bfloat16 else 1e-6)


# ---- the two kept experiment paths (default off) ---------------------------------------------------------------------
def _bn_fwd_bwd(shape, relu, residual, seed=0):
    from b200ddp.ops import FusedBatchNormAct2d
    torch.manual_seed(seed)
    x = (torch.randn(*shape, device="cuda") * 2 + 0.5).to(torch.bfloat16).contiguous(memory_format=torch.channels_last).requires_grad_()
    res = torch.randn(*shape, device="cuda").to(torch.bfloat16).contiguous(memory_format=torch.channels_last).requires_grad_() if residual else None
    bn = FusedBatchNormAct2d(shape[1], relu=relu).cuda()
    with torch.no_grad():
        bn.weight.uniform_(0.5, 1.5)
        bn.bias.uniform_(-0.5, 0.5)
    y = bn(x, residual=res) if residual else bn(x)
    dy = torch.randn(*shape, device="cuda", generator=torch.Generator("cuda").manual_seed(seed + 1)).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    y.backward(dy)
    out = [y.detach(), x.grad, bn.weight.grad, bn.bias.grad, bn.running_mean.clone(), bn.running_var.clone()]
    if residual:
        out.append(res.grad)
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("shape,relu,residual", [((32, 64, 56, 56), True, False), ((8, 256, 14, 14), True, True), ((4, 24, 5, 5), False, False)])
def test_programmatic_dependent_launch_path_matches_default(shape, relu, residual):
    """B200DDP_PDL=1 / set_bn_pdl(1): statistics -> apply and reduce -> apply as programmatic dependent launches (same arithmetic,
    earlier scheduling of the dependent grid): outputs agree with the default path."""
    from b200ddp import _ext
    C = _ext.get()
    ref = _bn_fwd_bwd(shape, relu, residual)
    C.set_bn_pdl(1)
    try:
        got = _bn_fwd_bwd(shape, relu, residual)
    finally:
        C.set_bn_pdl(0)
    for a, b in zip(got, ref):
        assert torch.allclose(a.float(), b.float(), atol=1e-2, rtol=1e-2), float((a.float() - b.float()).abs().max())


def test_single_launch_batchnorm_path_matches_default():
    """B200DDP_BN_FUSED=1 (one launch per direction with a tile barrier, kept selectable): same results as
    the default 2 + 2 launches.  The switch is read once per process, hence the subprocess."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = ("import sys, torch; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "from test_gpu_batchnorm import _bn_fwd_bwd\n"
            "outs = _bn_fwd_bwd((16, 64, 28, 28), True, True) + _bn_fwd_bwd((2, 512, 7, 7), False, False)\n"
            "torch.save([o.cpu() for o in outs], sys.argv[1])\n") % (root, os.path.join(root, "tests"))
    import tempfile
    with tempfile.TemporaryDirectory() as td:
        files = {}
        for mode in ("0", "1"):
            files[mode] = os.path.join(td, f"bn_{mode}.pt")
            res = subprocess.run([sys.executable, "-c", code, files[mode]], capture_output=True, text=True, timeout=300,
                                 env=dict(os.environ, B200DDP_BN_FUSED=mode))
            assert res.returncode == 0, res.stderr[-2000:]
        a, b = torch.load(files["0"]), torch.load(files["1"])
    for u, v in zip(a, b):
        assert torch.allclose(u.float(), v.float(), atol=4e-2, rtol=4e-2), float((u.float() - v.float()).abs().max())
