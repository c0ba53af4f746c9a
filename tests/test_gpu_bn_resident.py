"""Single-read (resident) BatchNorm kernels: every ResNet-50 BatchNorm shape at batch 32 against an fp32 reference and
against the two-pass kernels (``set_bn_two_pass``), bitwise reproducibility, launch counts and CUDA-graph replay."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

# (C, H, W, relu, residual) of ResNet-50's BatchNorms at batch 32 (torchvision v1.5: stride on the 3x3 conv)
RESNET50_BN = [
    (64, 112, 112, True, False),      # stem (its forward takes statistics from the conv epilogue in the net)
    (64, 56, 56, True, False),        # layer1 bn1 / bn2
    (256, 56, 56, True, True),        # layer1 bn3
    (256, 56, 56, False, False),      # layer1 downsample
    (128, 56, 56, True, False),       # layer2 block-0 bn1
    (128, 28, 28, True, False),       # layer2 bn2, bn1
    (512, 28, 28, True, True),        # layer2 bn3
    (512, 28, 28, False, False),      # layer2 downsample
    (256, 28, 28, True, False),       # layer3 block-0 bn1
    (256, 14, 14, True, False),       # layer3 bn2, bn1
    (1024, 14, 14, True, True),       # layer3 bn3
    (1024, 14, 14, False, False),     # layer3 downsample
    (512, 14, 14, True, False),       # layer4 block-0 bn1
    (512, 7, 7, True, False),         # layer4 bn2, bn1
    (2048, 7, 7, True, True),         # layer4 bn3
    (2048, 7, 7, False, False),       # layer4 downsample
]
CASES = [((32, c, h, w), relu, res) for c, h, w, relu, res in RESNET50_BN] + [((4, 24, 5, 5), True, True), ((4, 24, 5, 5), False, False),
                                                                               ((2, 96, 9, 7), True, False)]


def _ext():
    from b200ddp import _ext as e
    return e.get()


def _inputs(shape, residual, seed=0):
    g = torch.Generator("cuda").manual_seed(seed)
    mk = lambda scale, shift: (torch.randn(*shape, device="cuda", generator=g) * scale + shift).to(torch.bfloat16).contiguous(  # noqa: E731
        memory_format=torch.channels_last)
    x = mk(2.0, 0.5)
    res = mk(1.0, 0.0) if residual else None
    dy = mk(1.0, 0.0)
    return x, res, dy


def _run(shape, relu, residual, two_pass, seed=0):
    """One forward + backward through FusedBatchNormAct2d; returns outputs, side effects and launch counts."""
    from b200ddp.ops import FusedBatchNormAct2d
    C = _ext()
    x, res, dy = _inputs(shape, residual, seed)
    x = x.requires_grad_()
    if res is not None:
        res = res.requires_grad_()
    torch.manual_seed(seed)
    bn = FusedBatchNormAct2d(shape[1], relu=relu).cuda()
    with torch.no_grad():
        bn.weight.uniform_(0.5, 1.5)
        bn.bias.uniform_(-0.5, 0.5)
    C.set_bn_two_pass(1 if two_pass else 0)
    try:
        n0 = C.launch_count()
        y = bn(x, residual=res)
        n1 = C.launch_count()
        y.backward(dy)
        n2 = C.launch_count()
    finally:
        C.set_bn_two_pass(0)
    torch.cuda.synchronize()
    out = {"y": y.detach(), "dx": x.grad, "dgamma": bn.weight.grad, "dbeta": bn.bias.grad, "running_mean": bn.running_mean.clone(),
           "running_var": bn.running_var.clone(), "num_batches": int(bn.num_batches_tracked)}
    if res is not None:
        out["dres"] = res.grad
    return out, (n1 - n0, n2 - n1), (x, res, dy, bn)


def _expected_launches(shape):
    # one launch per direction on every ResNet-50 shape at batch 32, except: the stem (its 51 MB activation does not fit
    # the CTAs' shared memory) and the backward of [100352, 256] (dy + x would need 4 waves), which keep the two-pass kernels
    if shape == (32, 64, 112, 112):
        return (2, 2)
    if shape == (32, 256, 56, 56):
        return (1, 2)
    return (1, 1)


def _ulp_band(a, b):
    """|a - b| <= one bf16 ulp at the larger magnitude (plus a floor far below the data's scale for values near zero)."""
    a, b = a.float(), b.float()
    mag = torch.maximum(a.abs(), b.abs())
    ulp = torch.exp2(torch.floor(torch.log2(mag.clamp_min(1e-30))) - 7)
    floor = 1e-5 * float(b.abs().max())
    return (a - b).abs() <= ulp + floor


@pytest.mark.parametrize("shape,relu,residual", CASES)
def test_resident_matches_reference_and_two_pass(shape, relu, residual):
    got, launches, (x, res, dy, bn) = _run(shape, relu, residual, two_pass=False)
    ref, ref_launches, _ = _run(shape, relu, residual, two_pass=True)
    assert launches == _expected_launches(shape), launches
    assert ref_launches == (2, 2)
    assert _ext().bn_resident_error() == 0

    # fp32 reference (tolerances of test_gpu_batchnorm.py for bf16)
    xr = x.detach().float().requires_grad_()
    rr = res.detach().float().requires_grad_() if res is not None else None
    wr = bn.weight.detach().clone().requires_grad_()
    br = bn.bias.detach().clone().requires_grad_()
    rm, rv = torch.zeros_like(wr), torch.ones_like(wr)
    yr = F.batch_norm(xr, rm, rv, wr, br, True, 0.1, 1e-5)
    if rr is not None:
        yr = yr + rr
    if relu:
        yr = torch.relu(yr)
    yr.backward(dy.float())
    tol = 4e-2
    assert torch.allclose(got["y"].float(), yr, atol=tol, rtol=tol), float((got["y"].float() - yr).abs().max())
    gscale = max(1.0, float(xr.grad.abs().max()))
    assert torch.allclose(got["dx"].float(), xr.grad, atol=tol * gscale, rtol=tol), float((got["dx"].float() - xr.grad).abs().max())
    if res is not None:
        assert torch.allclose(got["dres"].float(), rr.grad, atol=tol, rtol=tol)
    n = x.numel() / shape[1]
    ptol = tol * max(1.0, n ** 0.5)
    assert torch.allclose(got["dgamma"], wr.grad, atol=ptol, rtol=tol * 4), float((got["dgamma"] - wr.grad).abs().max())
    assert torch.allclose(got["dbeta"], br.grad, atol=ptol, rtol=tol * 4)
    assert torch.allclose(got["running_mean"], rm, atol=tol, rtol=tol) and torch.allclose(got["running_var"], rv, atol=tol, rtol=tol)
    assert got["num_batches"] == 1

    # two-pass kernels: same arithmetic, fp32 sums in another order
    for k in ("y", "dx") + (("dres",) if res is not None else ()):
        ok = _ulp_band(got[k], ref[k])
        assert bool(ok.all()), (k, int((~ok).sum()), float((got[k].float() - ref[k].float()).abs().max()))
    R = x.numel() // shape[1]
    for k in ("dgamma", "dbeta"):
        # a sum of R terms in a different order: within R * 2^-24 of the terms' scale (|dy*| and |dy* xhat| are O(1) here)
        assert torch.allclose(got[k], ref[k], atol=R * 2.0 ** -24 * 4, rtol=1e-4), (k, float((got[k] - ref[k]).abs().max()))
    for k in ("running_mean", "running_var"):
        assert torch.allclose(got[k], ref[k], atol=1e-5, rtol=1e-5), (k, float((got[k] - ref[k]).abs().max()))
    assert got["num_batches"] == ref["num_batches"]


@pytest.mark.parametrize("shape,relu,residual", [((32, 256, 56, 56), True, True), ((32, 128, 56, 56), True, False), ((32, 512, 28, 28), True, True),
                                                 ((32, 2048, 7, 7), False, False), ((4, 24, 5, 5), True, True)])
def test_resident_is_bitwise_reproducible(shape, relu, residual):
    a, la, _ = _run(shape, relu, residual, two_pass=False, seed=3)
    b, lb, _ = _run(shape, relu, residual, two_pass=False, seed=3)
    assert la == lb == _expected_launches(shape)
    for k in a:
        if isinstance(a[k], torch.Tensor):
            assert torch.equal(a[k], b[k]), k
        else:
            assert a[k] == b[k], k


def test_fp32_keeps_two_pass_kernels():
    from b200ddp.ops import FusedBatchNormAct2d
    C = _ext()
    x = torch.randn(8, 64, 14, 14, device="cuda").contiguous(memory_format=torch.channels_last).requires_grad_()
    bn = FusedBatchNormAct2d(64, relu=True).cuda()
    n0 = C.launch_count()
    y = bn(x)
    n1 = C.launch_count()
    y.backward(torch.randn_like(y))
    assert (n1 - n0, C.launch_count() - n1) == (2, 2)


def _resnet_steps(use_graph, steps=5):
    from b200ddp.engine.step import TrainStep
    from b200ddp.models import resnet50
    from b200ddp.ops import MSELoss
    from b200ddp.optim import FusedSGD
    from b200ddp.utils import to_mixed_bf16
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    net = to_mixed_bf16(resnet50().to(dev)).to(memory_format=torch.channels_last)
    opt = FusedSGD(net.parameters(), lr=1e-3, max_grad_norm=1000.0)
    step = TrainStep(net, MSELoss(), opt, dev, use_graph=use_graph)
    g = torch.Generator().manual_seed(7)
    batches = [(torch.randn(32, 3, 224, 224, generator=g).to(torch.bfloat16).contiguous(memory_format=torch.channels_last),
                torch.randn(32, 1000, generator=g).to(torch.bfloat16)) for _ in range(2)]
    losses = []
    for i in range(steps):
        x, y = batches[i % 2]
        losses.append(float(step(x.to(dev), y.to(dev))))
    torch.cuda.synchronize()
    state = {k: v.detach().float().clone() for k, v in net.state_dict().items()}
    return losses, state, step


def test_resnet50_graph_replay_matches_eager():
    """Batch 32, 224x224: the captured step (cooperative BatchNorm launches inside the CUDA graph) agrees with the eager one."""
    eager_losses, eager_state, _ = _resnet_steps(False)
    graph_losses, graph_state, step = _resnet_steps(True)
    assert step.graph is not None
    assert _ext().bn_resident_error() == 0
    for a, b in zip(eager_losses, graph_losses):
        assert abs(a - b) <= 1e-3 * max(1.0, abs(a)), (eager_losses, graph_losses)
    for k, a in eager_state.items():
        b = graph_state[k]
        if a.dtype.is_floating_point and a.numel() > 1:
            rel = float((a - b).norm() / (a.norm() + 1e-12))
            assert rel < 1e-2, (k, rel)
        else:
            assert torch.equal(a, b), k
