"""Multi-wave resident BatchNorm: shapes whose slabs need two or more waves (and the backward of [100352, 256], which runs as
two launches of two waves) against an fp32 reference and the two-pass kernels, a ragged last wave with a partial last
channel tile, bitwise reproducibility, and back-to-back modules captured in one CUDA graph and replayed."""
import pytest
import torch
import torch.nn.functional as F

from test_gpu_bn_resident import _ext, _inputs, _run, _ulp_band

pytestmark = pytest.mark.gpu

# (shape, relu, residual).  (8, 520, 60, 60): 9 channel tiles, the last one 8 channels wide, over 2+ waves.
MULTI_WAVE = [((32, 256, 56, 56), True, True), ((32, 256, 56, 56), False, False), ((32, 128, 56, 56), True, False),
              ((32, 512, 28, 28), True, True), ((32, 512, 28, 28), False, False), ((8, 520, 60, 60), True, True),
              ((8, 520, 60, 60), False, False)]


def _min_waves(shape, streams):
    """A lower bound on the waves of the resident plan: one wave holds at most every SM's shared memory of slabs."""
    p = torch.cuda.get_device_properties(0)
    n, c, h, w = shape
    tiles = (c + 63) // 64
    row_bytes = 64 * 2 * streams
    total = tiles * n * h * w * row_bytes
    per_wave = p.multi_processor_count * p.shared_memory_per_block_optin
    return -(-total // per_wave)


@pytest.mark.parametrize("shape,relu,residual", MULTI_WAVE)
def test_multi_wave_matches_reference_and_two_pass(shape, relu, residual):
    assert max(_min_waves(shape, 1), _min_waves(shape, 2)) >= 2
    got, launches, (x, res, dy, bn) = _run(shape, relu, residual, two_pass=False)
    ref, ref_launches, _ = _run(shape, relu, residual, two_pass=True)
    assert ref_launches == (2, 2)
    assert launches[0] == 1 and launches[1] in (1, 2), launches      # resident in both directions
    assert _ext().bn_resident_error() == 0

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
    R = x.numel() // shape[1]
    ptol = tol * max(1.0, R ** 0.5)
    assert torch.allclose(got["dgamma"], wr.grad, atol=ptol, rtol=tol * 4), float((got["dgamma"] - wr.grad).abs().max())
    assert torch.allclose(got["dbeta"], br.grad, atol=ptol, rtol=tol * 4)
    assert torch.allclose(got["running_mean"], rm, atol=tol, rtol=tol) and torch.allclose(got["running_var"], rv, atol=tol, rtol=tol)
    assert got["num_batches"] == 1

    for k in ("y", "dx") + (("dres",) if res is not None else ()):
        ok = _ulp_band(got[k], ref[k])
        assert bool(ok.all()), (k, int((~ok).sum()), float((got[k].float() - ref[k].float()).abs().max()))
    for k in ("dgamma", "dbeta"):
        assert torch.allclose(got[k], ref[k], atol=R * 2.0 ** -24 * 4, rtol=1e-4), (k, float((got[k] - ref[k]).abs().max()))
    for k in ("running_mean", "running_var"):
        assert torch.allclose(got[k], ref[k], atol=1e-5, rtol=1e-5), (k, float((got[k] - ref[k]).abs().max()))
    assert got["num_batches"] == ref["num_batches"]


@pytest.mark.parametrize("shape,relu,residual", MULTI_WAVE)
def test_multi_wave_is_bitwise_reproducible(shape, relu, residual):
    a, la, _ = _run(shape, relu, residual, two_pass=False, seed=5)
    b, lb, _ = _run(shape, relu, residual, two_pass=False, seed=5)
    assert la == lb
    for k in a:
        if isinstance(a[k], torch.Tensor):
            assert torch.equal(a[k], b[k]), k
        else:
            assert a[k] == b[k], k


def test_back_to_back_modules_graph_replay_matches_eager():
    """Modules of different shapes (one and two waves, one and two backward launches) run back to back, then the same
    sequence captured in one CUDA graph and replayed 3 times: every replay equals the eager run, so the tile barriers'
    counter words are back at rest after each launch."""
    from b200ddp.ops import FusedBatchNormAct2d
    specs = [((32, 256, 56, 56), True, True), ((32, 64, 56, 56), True, False), ((32, 512, 28, 28), True, True),
             ((8, 520, 60, 60), False, False), ((32, 1024, 14, 14), True, True), ((32, 128, 56, 56), True, False)]
    torch.manual_seed(0)
    mods, data = [], []
    for i, (shape, relu, residual) in enumerate(specs):
        bn = FusedBatchNormAct2d(shape[1], relu=relu).cuda()
        with torch.no_grad():
            bn.weight.uniform_(0.5, 1.5)
            bn.bias.uniform_(-0.5, 0.5)
        mods.append(bn)
        data.append(_inputs(shape, residual, seed=i))

    def run():
        outs = []
        for bn, (x, res, dy) in zip(mods, data):
            y = bn(x, residual=res)
            xg = x.detach().requires_grad_()
            rg = res.detach().requires_grad_() if res is not None else None
            yg = bn(xg, residual=rg)
            gx, gw = torch.autograd.grad(yg, (xg, bn.weight), dy)
            outs += [y.detach(), gx, gw]
        return outs

    state = [(bn.running_mean.clone(), bn.running_var.clone(), bn.num_batches_tracked.clone()) for bn in mods]

    def reset():
        with torch.no_grad():
            for bn, (m, v, n) in zip(mods, state):
                bn.running_mean.copy_(m)
                bn.running_var.copy_(v)
                bn.num_batches_tracked.copy_(n)

    eager = run()                                   # also allocates every module's workspace outside the capture
    torch.cuda.synchronize()
    eager_stats = [(bn.running_mean.clone(), bn.running_var.clone()) for bn in mods]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        reset()
        run()                                       # warm-up on the capture stream
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = run()
    for _ in range(3):
        reset()
        graph.replay()
        torch.cuda.synchronize()
        assert _ext().bn_resident_error() == 0
        for a, b in zip(eager, captured):
            assert torch.equal(a, b)
        for bn, (m, v) in zip(mods, eager_stats):
            assert torch.equal(bn.running_mean, m) and torch.equal(bn.running_var, v)
