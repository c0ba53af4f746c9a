"""FP8 linears on one H100: the quantiser against the CPU cast, the FP8 GEMM's accuracy against torch._scaled_mm on the
same bytes, Linear(fp8=True) against the CPU emulation of the recipe, no host synchronisation, a tiny FP8 BERT against
the fp32 CPU model, and FP8 training under a CUDA graph."""
import math

import pytest
import torch

from b200ddp.ops import functional as Fn

pytestmark = pytest.mark.gpu


def dev():
    return torch.device("cuda", 0)


def C():
    from b200ddp import _ext
    return _ext.get()


@pytest.mark.parametrize("fmt", ["e4m3", "e5m2"])
@pytest.mark.parametrize("shape", [(8192, 768), (8192, 3072), (1040, 768), (1001, 64), (256, 128)])
def test_quantize_matches_the_cpu_cast_bitwise(fmt, shape):
    g = torch.Generator().manual_seed(shape[0] + shape[1])
    if shape == (256, 128):
        t = torch.zeros(shape, dtype=torch.bfloat16)                  # all zeros: s = 1
    else:
        t = (torch.randn(shape, generator=g) * 3.0).to(torch.bfloat16)
        t[5, 7] = -1000.0 if fmt == "e4m3" else 70000.0                # amax above fmax: s < 1
    want_t = shape[0] % 16 == 0
    q, qt, scale_inv, colsum = C().fp8_quantize(t.to(dev()), fmt, want_t, True)
    q_ref, s = Fn.fp8_quantize_reference(t, fmt)
    assert q.dtype == q_ref.dtype and q.shape == t.shape
    assert torch.equal(q.cpu().view(torch.uint8), q_ref.view(torch.uint8))
    if want_t:
        assert torch.equal(qt.cpu().view(torch.uint8), q_ref.t().contiguous().view(torch.uint8))
    else:
        assert qt is None
    assert float(scale_inv.cpu()) == 1.0 / s
    amax = C().fp8_amax(t.to(dev()))
    assert float(amax.cpu()) == float(t.float().abs().max())
    ref_sum = t.double().sum(0)
    assert torch.allclose(colsum.cpu().double(), ref_sum, rtol=1e-5, atol=1e-5 * float(t.double().abs().sum(0).max()) + 1e-6)
    again = C().fp8_quantize(t.to(dev()), fmt, want_t, True)[3]
    assert torch.equal(colsum, again)


def _operands(M, N, K, layout, seed):
    """(a, b) FP8 operands with their scale factors for one of the three GEMMs of an FP8 linear with x [M,K], W [N,K]."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(M, K, generator=g).to(torch.bfloat16).to(dev())
    w = (torch.randn(N, K, generator=g) * 0.05).to(torch.bfloat16).to(dev())
    dy = (torch.randn(M, N, generator=g) * 1e-3).to(torch.bfloat16).to(dev())
    if layout == "fwd":
        xq, _, xs, _ = C().fp8_quantize(x, "e4m3")
        wq, _, ws, _ = C().fp8_quantize(w, "e4m3")
        return xq, wq, xs, ws
    if layout == "dgrad":
        dq, _, ds, _ = C().fp8_quantize(dy, "e5m2")
        _, wqt, ws, _ = C().fp8_quantize(w, "e4m3", True)
        return dq, wqt, ds, ws
    _, dqt, ds, _ = C().fp8_quantize(dy, "e5m2", True)
    _, xqt, xs, _ = C().fp8_quantize(x, "e4m3", True)
    return dqt, xqt, ds, xs


_SHAPES = [(2304, 768), (768, 768), (3072, 768), (768, 3072)]


@pytest.mark.parametrize("layout", ["fwd", "dgrad", "wgrad"])
@pytest.mark.parametrize("M, N, K", [(8192, n, k) for n, k in _SHAPES] + [(1040, 768, 3072), (1040, 2304, 768)])
def test_fp8_gemm_is_as_accurate_as_scaled_mm(layout, M, N, K):
    """M = 1040 is ragged against the 128-row tiles (and still a multiple of 16, which the transposed copies need)."""
    a, b, sa, sb = _operands(M, N, K, layout, seed=M + N + K)
    out = C().gemm_fp8(a, b, sa, sb, None, 0)
    assert out.dtype == torch.bfloat16 and out.shape == (a.shape[0], b.shape[0])
    ref = (a.double() @ b.double().t()) * (sa.double() * sb.double())
    lib = torch._scaled_mm(a, b.t(), scale_a=sa, scale_b=sb, out_dtype=torch.bfloat16, use_fast_accum=False)
    err = float((out.double() - ref).norm() / ref.norm())
    err_lib = float((lib.double() - ref).norm() / ref.norm())
    assert err <= 1.25 * err_lib, (err, err_lib)
    assert torch.equal(out, C().gemm_fp8(a, b, sa, sb, None, 0))


def test_fp8_gemm_bias_gelu_epilogue():
    a, b, sa, sb = _operands(512, 768, 768, "fwd", seed=3)
    bias = (torch.randn(768) * 0.1).to(torch.bfloat16).to(dev())
    pre = (a.float() @ b.float().t()) * (sa * sb) + bias.float()
    assert torch.allclose(C().gemm_fp8(a, b, sa, sb, bias, 1).float(), pre, rtol=1e-2, atol=1e-2)
    gelu = torch.nn.functional.gelu(pre)
    assert torch.allclose(C().gemm_fp8(a, b, sa, sb, bias, 3).float(), gelu, rtol=1e-2, atol=1e-2)


@pytest.mark.parametrize("activation", [None, "gelu"])
def test_fp8_linear_matches_the_cpu_emulation(activation):
    from b200ddp.ops import Linear
    torch.manual_seed(0)
    lin = Linear(768, 3072, activation=activation, fp8=True).to(torch.bfloat16)
    with torch.no_grad():
        lin.bias.normal_(0, 0.1)
    x = torch.randn(4, 256, 768).to(torch.bfloat16)
    dy = (torch.randn(4, 256, 3072) * 1e-2).to(torch.bfloat16)
    outs = []
    for d in ("cpu", dev()):
        m = Linear(768, 3072, activation=activation, fp8=True).to(d, torch.bfloat16)
        m.load_state_dict(lin.state_dict())
        xi = x.detach().to(d).requires_grad_(True)
        y = m(xi)
        y.backward(dy.to(d))
        outs.append([t.detach().float().cpu() for t in (y, xi.grad, m.weight.grad, m.bias.grad)])
        if d != "cpu":
            assert m.weight.grad.stride() == m.weight.stride() and m.weight.grad.dtype == torch.bfloat16
    for name, c, g in zip(("y", "dx", "dW", "db"), *outs):
        if activation == "gelu" and name in ("dx", "dW"):
            # GELU' from the CUDA and the CPU math libraries can differ in the last bit, which moves a bf16 rounding of
            # dy * GELU'(pre) and then, now and then, an E5M2 rounding (a quarter of that element): compare norms
            assert float((g - c).norm() / c.norm()) < 2 ** -7, name
            continue
        # identical FP8 bytes on both sides: only the fp32 summation order differs, then bf16 output rounding
        tol = 2 ** -7 * float(c.abs().max())
        bad = ~torch.isclose(g, c, rtol=2 ** -7, atol=tol)
        assert not bad.any(), (name, int(bad.sum()), float((g - c).abs().max()), tol, g[bad][:4].tolist(), c[bad][:4].tolist())


def test_fp8_linear_rejects_unsupported_input():
    from b200ddp.ops import Linear
    m = Linear(64, 64, fp8=True).to(dev())
    with pytest.raises(ValueError, match="bf16"):
        m(torch.randn(32, 64, device=dev()))                            # fp32 on CUDA
    m = m.to(torch.bfloat16)
    with pytest.raises(ValueError, match=r"\(40, 64\)"):
        m(torch.randn(40, 64, device=dev(), dtype=torch.bfloat16))     # a backward over 40 rows
    with torch.no_grad():
        assert m(torch.randn(40, 64, device=dev(), dtype=torch.bfloat16)).shape == (40, 64)


def _tiny_cfg(**kw):
    from b200ddp.models.bert import BertConfig
    return BertConfig(vocab_size=1000, hidden=128, layers=2, heads=4, intermediate=256, max_position=64, pad_vocab_to=64, **kw)


def test_fp8_bert_step_has_no_host_synchronisation():
    from b200ddp.models.bert import BertForMaskedLM
    from b200ddp.ops import cross_entropy
    torch.manual_seed(1)
    model = BertForMaskedLM(_tiny_cfg(fp8=True)).to(dev(), torch.bfloat16)
    ids = torch.randint(0, 1000, (4, 64), device=dev())
    labels = torch.randint(0, 1000, (4, 64), device=dev())
    cross_entropy(model(ids), labels).backward()   # first calls: module loading, tensor maps
    model.zero_grad(set_to_none=True)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        loss = cross_entropy(model(ids), labels)
        loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert math.isfinite(float(loss))


def test_fp8_bert_tiny_gpu_matches_cpu_reference():
    """The bf16 test's setup (test_gpu_kernels.py) with fp8=True: the GPU loss and every parameter gradient against the
    fp32 CPU model.  Tolerances are the bf16 test's, except the gradient bound, which FP8 (E5M2 gradients) needs wider."""
    from b200ddp.models.bert import BertForMaskedLM
    from b200ddp.ops import cross_entropy
    torch.manual_seed(7)
    ref = BertForMaskedLM(_tiny_cfg())
    gpu = BertForMaskedLM(_tiny_cfg(fp8=True))
    gpu.load_state_dict(ref.state_dict())
    gpu = gpu.to(dev(), torch.bfloat16)
    ids = torch.randint(0, 1000, (4, 64))
    labels = torch.where(torch.rand(4, 64) < 0.3, torch.randint(0, 1000, (4, 64)), torch.full((4, 64), -100))
    lr = cross_entropy(ref(ids), labels)
    lr.backward()
    lg = cross_entropy(gpu(ids.to(dev())), labels.to(dev()))
    lg.backward()
    assert abs(float(lg) - float(lr)) < 5e-2 * max(1.0, abs(float(lr)))
    for (n, p), q in zip(gpu.named_parameters(), ref.parameters()):
        if float(q.grad.norm()) < 1e-4:
            assert float(p.grad.float().norm()) < 5e-2, n
            continue
        rel = float((p.grad.float().cpu() - q.grad).norm() / (q.grad.norm() + 1e-8))
        assert rel < 0.2, (n, rel)


def _train(fp8, graph, steps=60):
    from b200ddp.engine.step import TrainStep
    from b200ddp.models.bert import BertConfig, BertForMaskedLM
    from b200ddp.ops import CrossEntropyLoss
    from b200ddp.optim import FusedAdamW, weight_decay_groups
    from b200ddp.utils import to_mixed_bf16
    torch.manual_seed(0)
    cfg = BertConfig(vocab_size=2048, hidden=256, layers=2, heads=4, intermediate=1024, max_position=128, pad_vocab_to=64, fp8=fp8)
    model = to_mixed_bf16(BertForMaskedLM(cfg).to(dev()))
    opt = FusedAdamW(weight_decay_groups(model, 0.01), lr=1e-3, max_grad_norm=1.0)
    step = TrainStep(model, CrossEntropyLoss(), opt, dev(), use_graph=graph)
    g = torch.Generator().manual_seed(3)
    base = torch.randint(0, 2048, (16, 128), generator=g)
    losses = []
    for i in range(steps):
        ids = torch.where(torch.rand(16, 128, generator=g) < 0.15, torch.randint(0, 2048, (16, 128), generator=g), base)
        losses.append(float(step(ids.to(dev()), base.to(dev()))))
    torch.cuda.synchronize()
    return losses, step


def test_fp8_bert_trains_under_a_cuda_graph_like_bf16():
    l8, step8 = _train(True, True)
    assert step8.graph is not None
    l16, _ = _train(False, True)
    l8_eager, _ = _train(True, False)
    assert all(math.isfinite(v) for v in l8)
    assert sum(l8[-10:]) / 10 < sum(l8[:5]) / 5 - 0.5, l8
    m8, m16 = sum(l8[-10:]) / 10, sum(l16[-10:]) / 10
    assert abs(m8 - m16) <= 0.05 * m16, (m8, m16)
    for a, b in zip(l8, l8_eager):
        assert abs(a - b) <= 2e-2 * max(1.0, abs(b)), (a, b)


def test_fp8_bert_base_graph_training_lowers_the_loss(tmp_path):
    """What `python ddp.py --model bert-base --fp16 --fp8 --optimizer adamw --cuda_graph --max_steps 30 --seq_len 128` runs."""
    from b200ddp.engine import cli
    from b200ddp.engine.trainer import Trainer
    from b200ddp.models import build_model
    from b200ddp.ops import Linear
    args = cli.build_parser().parse_args(["--model", "bert-base", "--fp16", "--fp8", "--optimizer", "adamw", "--cuda_graph",
                                          "--max_steps", "30", "--seq_len", "128", "--per_gpu_train_batch_size", "16",
                                          "--lr", "5e-4", "--warmup_steps", "5", "--weight_decay", "0.01",
                                          "--save_steps", "0", "--logging_steps", "10", "--no_tensorboard",
                                          "--output_dir", str(tmp_path / "out")])
    cli.setup(args)
    trainer = Trainer(args, build_model("bert-base", fp8=True), cli.log)
    assert sum(isinstance(m, Linear) and m.fp8 for m in trainer.model.modules()) == 48
    before = trainer.evaluate(max_batches=4)["eval_loss"]
    trainer.train()
    after = trainer.evaluate(max_batches=4)["eval_loss"]
    assert trainer.step_fn.graph is not None
    assert math.isfinite(after) and after < before - 0.05, (before, after)
