"""Numerics of every single-GPU sm_90a kernel against a plain PyTorch fp32 reference."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def C():
    from b200ddp import _ext
    return _ext.get()


def dev():
    return torch.device("cuda", 0)


def test_extension_loaded_is_in_tree(C):
    import b200ddp
    import os
    assert os.path.dirname(C.__file__) == os.path.dirname(b200ddp.__file__)
    assert C.launch_count() >= 0


@pytest.mark.parametrize("M,N,K,relu", [(32, 10, 10, True), (32, 5, 10, False), (7, 3, 17, True), (128, 64, 48, False)])
def test_small_linear_fwd_bwd(C, M, N, K, relu):
    from b200ddp.ops import linear
    torch.manual_seed(0)
    x = torch.randn(M, K, device=dev(), requires_grad=True)
    w = torch.randn(N, K, device=dev(), requires_grad=True)
    b = torch.randn(N, device=dev(), requires_grad=True)
    before = C.launch_count()
    y = linear(x, w, b, "relu" if relu else None)
    g = torch.randn_like(y)
    y.backward(g)
    assert C.launch_count() - before == 2                 # one fwd + one bwd launch
    xr, wr, br = (t.detach().double().requires_grad_() for t in (x, w, b))
    yr = F.linear(xr, wr, br)
    yr = torch.relu(yr) if relu else yr
    yr.backward(g.double())
    assert torch.allclose(y.double(), yr, atol=1e-4)
    for a, r in ((x, xr), (w, wr), (b, br)):
        assert torch.allclose(a.grad.double(), r.grad, atol=1e-3), (a.grad.double() - r.grad).abs().max()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("shape", [(32, 5), (32, 1000), (3, 7, 11), (4096, 513)])
def test_mse_fused(C, dtype, shape):
    from b200ddp.ops import mse_loss
    torch.manual_seed(1)
    o = torch.randn(*shape, device=dev(), dtype=dtype, requires_grad=True)
    t = torch.randn(*shape, device=dev(), dtype=dtype)
    loss = mse_loss(o, t)
    (loss * 3.0).backward()
    orf = o.detach().float().requires_grad_()
    ref = F.mse_loss(orf, t.float())
    (ref * 3.0).backward()
    tol = 1e-5 if dtype == torch.float32 else 2e-2
    assert torch.allclose(loss.float(), ref, rtol=tol, atol=tol)
    assert torch.allclose(o.grad.float(), orf.grad, rtol=tol, atol=tol * max(1e-3, float(orf.grad.abs().max())))
    # determinism of the two-stage reduction
    assert float(mse_loss(o, t)) == float(mse_loss(o, t))


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("rows,cols", [(16, 10), (64, 1000), (33, 30522)])
def test_cross_entropy_fused(C, dtype, rows, cols):
    from b200ddp.ops import cross_entropy
    torch.manual_seed(2)
    x = (torch.randn(rows, cols, device=dev()) * 3).to(dtype).requires_grad_()
    t = torch.randint(0, cols, (rows,), device=dev())
    t[::5] = -100
    loss = cross_entropy(x, t)
    loss.backward()
    xr = x.detach().float().requires_grad_()
    ref = F.cross_entropy(xr, t, ignore_index=-100)
    ref.backward()
    tol = 1e-4 if dtype == torch.float32 else 2e-2
    assert torch.allclose(loss, ref, rtol=tol, atol=tol)
    assert torch.allclose(x.grad.float(), xr.grad, atol=tol * 0.1 + 1e-6, rtol=tol)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("rows,cols", [(8, 768), (1000, 768), (37, 100), (4, 4096)])
def test_layernorm(C, dtype, rows, cols):
    from b200ddp.ops import layer_norm
    torch.manual_seed(3)
    x = torch.randn(rows, cols, device=dev(), dtype=dtype, requires_grad=True)
    g = torch.randn(cols, device=dev(), dtype=dtype, requires_grad=True)
    b = torch.randn(cols, device=dev(), dtype=dtype, requires_grad=True)
    y = layer_norm(x, g, b, 1e-5)
    dy = torch.randn_like(y)
    y.backward(dy)
    xr, gr, br = (t.detach().float().requires_grad_() for t in (x, g, b))
    yr = F.layer_norm(xr, (cols,), gr, br, 1e-5)
    yr.backward(dy.float())
    tol = 1e-4 if dtype == torch.float32 else 3e-2
    assert torch.allclose(y.float(), yr, atol=tol, rtol=tol)
    assert torch.allclose(x.grad.float(), xr.grad, atol=tol, rtol=tol)
    scale = max(1.0, float(gr.grad.abs().max()))
    assert torch.allclose(g.grad.float(), gr.grad, atol=tol * scale, rtol=tol)
    assert torch.allclose(b.grad.float(), br.grad, atol=tol * scale, rtol=tol)


@pytest.mark.parametrize("dtype,momentum,wd,nesterov", [(torch.float32, 0.0, 0.0, False), (torch.float32, 0.9, 1e-2, True),
                                                         (torch.bfloat16, 0.0, 0.0, False), (torch.bfloat16, 0.9, 1e-2, False)])
def test_fused_sgd_clip_matches_torch(C, dtype, momentum, wd, nesterov):
    from b200ddp.optim import FusedSGD
    torch.manual_seed(4)
    shapes = [(10, 10), (10,), (5, 10), (5,), (300, 77), (64, 3, 7, 7), (20000,)]
    params = [torch.nn.Parameter(torch.randn(*s, device=dev()).to(dtype)) for s in shapes]
    params[5].data = params[5].data.contiguous(memory_format=torch.channels_last)
    ref = [torch.nn.Parameter(p.detach().float().clone()) for p in params]
    opt = FusedSGD(params, lr=0.05, momentum=momentum, weight_decay=wd, nesterov=nesterov, max_grad_norm=0.5)
    ropt = torch.optim.SGD(ref, lr=0.05, momentum=momentum, weight_decay=wd, nesterov=nesterov)
    for it in range(4):
        for p, r in zip(params, ref):
            g = torch.randn_like(r) * (0.1 if it % 2 else 3.0)
            if p.dim() == 4:
                g = g.contiguous(memory_format=torch.channels_last)
            p.grad = g.to(dtype)
            r.grad = p.grad.float().clone()
        total = torch.nn.utils.clip_grad_norm_(ref, 0.5)
        opt.step(); ropt.step()
        assert math.isclose(opt.grad_norm(), float(total), rel_tol=2e-3)
    tol = 1e-5 if dtype == torch.float32 else 2e-2
    for p, r in zip(params, ref):
        assert torch.allclose(p.detach().float(), r.detach(), atol=tol, rtol=tol)
    if dtype == torch.bfloat16:                            # fp32 masters track the reference far tighter than bf16 can
        off = opt._groups[0].offsets[4]
        assert torch.allclose(opt._master[off:off + 300 * 77].view(300, 77), ref[4].detach(), atol=1e-4)


def test_normalize_to_channels_last(C):
    x = torch.randn(4, 3, 32, 40, device=dev())
    mean = torch.tensor([0.1, 0.2, 0.3], device=dev())
    istd = torch.tensor([2.0, 0.5, 1.5], device=dev())
    for src, out_dt in ((x, torch.bfloat16), (x, torch.float32), ((x * 40 + 128).clamp(0, 255).to(torch.uint8), torch.bfloat16)):
        dst = torch.empty(src.shape, device=dev(), dtype=out_dt).contiguous(memory_format=torch.channels_last)
        C.normalize_to_channels_last(src, dst, mean, istd, 1.0)
        ref = ((src.float() - mean.view(1, 3, 1, 1)) * istd.view(1, 3, 1, 1)).to(out_dt)
        assert dst.is_contiguous(memory_format=torch.channels_last)
        assert torch.allclose(dst.float(), ref.float(), atol=1e-6 if out_dt == torch.float32 else 1e-2, rtol=1e-2)


def test_foo_training_graph_matches_eager_and_cpu(C):
    """Same seed, same data: CUDA-graph step == eager CUDA step == CPU step (fp32 workload of the reference)."""
    from b200ddp.engine.step import TrainStep
    from b200ddp.models import FooModel
    from b200ddp.ops import MSELoss
    from b200ddp.optim import FusedSGD
    torch.manual_seed(5)
    base = FooModel()
    X, Y = torch.randn(10, 32, 10), torch.randn(10, 32, 5)
    finals = []
    for device, graph in ((torch.device("cpu"), False), (dev(), False), (dev(), True)):
        m = FooModel()
        m.load_state_dict(base.state_dict())
        m = m.to(device)
        opt = FusedSGD(m.parameters(), lr=0.05, max_grad_norm=1.0)
        step = TrainStep(m, MSELoss(), opt, device, use_graph=graph)
        for i in range(10):
            step(X[i].to(device), Y[i].to(device))
        if graph:
            assert step.graph is not None and step.captured_native_launches >= 6
        finals.append([p.detach().cpu() for p in m.parameters()] + [torch.tensor(step.read_loss_sum())])
    for a, b in zip(finals[0], finals[1]):
        assert torch.allclose(a, b, atol=1e-5)
    for a, b in zip(finals[1], finals[2]):
        assert torch.allclose(a, b, atol=1e-6)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("n", [5, 4096, 100003])
def test_gelu_fwd_bwd(C, dtype, n):
    torch.manual_seed(6)
    pre = (torch.randn(n, device=dev()) * 2).to(dtype)
    dy = torch.randn(n, device=dev()).to(dtype)
    y = C.gelu_fwd(pre)
    dx = C.gelu_bwd(dy, pre)
    pr = pre.float().requires_grad_()
    yr = F.gelu(pr)
    yr.backward(dy.float())
    tol = 1e-5 if dtype == torch.float32 else 2e-2
    assert torch.allclose(y.float(), yr, atol=tol, rtol=tol)
    assert torch.allclose(dx.float(), pr.grad, atol=tol, rtol=tol)


def test_bert_tiny_gpu_matches_cpu_reference():
    """bf16 BERT on the native kernels (fused-QKV wgmma GEMMs, LayerNorm, GELU, cross-entropy) vs the same weights in
    fp32 on the CPU path: loss and every parameter gradient agree to bf16 accuracy."""
    from b200ddp.models.bert import BertConfig, BertForMaskedLM
    from b200ddp.ops import cross_entropy
    torch.manual_seed(7)
    cfg = BertConfig(vocab_size=1000, hidden=128, layers=2, heads=4, intermediate=256, max_position=64, pad_vocab_to=64)
    ref = BertForMaskedLM(cfg)
    gpu = BertForMaskedLM(cfg)
    gpu.load_state_dict(ref.state_dict())
    gpu = gpu.to(dev(), torch.bfloat16)
    ids = torch.randint(0, 1000, (4, 64))
    labels = torch.where(torch.rand(4, 64) < 0.3, torch.randint(0, 1000, (4, 64)), torch.full((4, 64), -100))
    lr = cross_entropy(ref(ids), labels)
    lr.backward()
    lg = cross_entropy(gpu(ids.to(dev())), labels.to(dev()))
    lg.backward()
    assert abs(float(lg) - float(lr)) < 5e-2 * max(1.0, abs(float(lr)))
    worst = 0.0
    for (n, p), q in zip(gpu.named_parameters(), ref.parameters()):
        if float(q.grad.norm()) < 1e-4:      # e.g. key.bias: softmax is shift-invariant, its true gradient is exactly 0
            assert float(p.grad.float().norm()) < 5e-2, n
            continue
        rel = float((p.grad.float().cpu() - q.grad).norm() / (q.grad.norm() + 1e-8))
        worst = max(worst, rel)
        assert rel < 0.15, (n, rel)


def test_normalize_pads_channels_with_zeros():
    """normalize_to_channels_last may write into a destination with more channels than the source: the extra ones are zeros."""
    from b200ddp import _ext
    C = _ext.get()
    x = torch.randn(4, 3, 32, 40, device="cuda")
    mean = torch.tensor([0.1, 0.2, 0.3], device="cuda")
    istd = torch.tensor([2.0, 0.5, 1.5], device="cuda")
    dst = torch.full((4, 8, 32, 40), 7.0, device="cuda", dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)
    C.normalize_to_channels_last(x, dst, mean, istd, 1.0)
    ref = ((x - mean.view(1, 3, 1, 1)) * istd.view(1, 3, 1, 1)).to(torch.bfloat16)
    assert torch.allclose(dst[:, :3].float(), ref.float(), atol=1e-2, rtol=1e-2)
    assert float(dst[:, 3:].abs().max()) == 0.0
