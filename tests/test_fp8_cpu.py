"""FP8 linears without a GPU: the power-of-two scale rule, the CPU emulation of the recipe against fp32 math, checkpoint
interchange between bf16 and FP8 BERT, and the --fp8 flag's checks."""
import math

import pytest
import torch
import torch.nn.functional as F

from b200ddp.ops import functional as Fn


@pytest.mark.parametrize("fmt", ["e4m3", "e5m2"])
def test_scale_is_the_largest_power_of_two_that_fits(fmt):
    fmax = Fn.FP8_FORMATS[fmt][1]
    g = torch.Generator().manual_seed(0)
    amaxes = [1.0, fmax, fmax / 2, fmax * 0.875, fmax * 1.0000001, 3e-30, 1e-40, 3e38, 0.3, 1e5]
    amaxes += [float(v) for v in torch.rand(200, generator=g).double() * 10.0 ** torch.randint(-20, 20, (200,), generator=g)]
    for amax in amaxes:
        amax = float(torch.tensor(amax, dtype=torch.float32))          # fp32 values, as on the device
        s = Fn.fp8_scale(amax, fmt)
        m, e = math.frexp(s)
        assert m == 0.5 and -126 <= e - 1 <= 127, (amax, s)
        if -126 < e - 1 < 127:                                          # not clamped
            assert amax * s <= fmax < amax * 2 * s, (amax, s)
    assert Fn.fp8_scale(0.0, fmt) == 1.0


@pytest.mark.parametrize("fmt", ["e4m3", "e5m2"])
def test_reference_quantisation_never_saturates_and_round_trips_within_format_precision(fmt):
    torch.manual_seed(1)
    t = (torch.randn(64, 48) * 3.7).to(torch.bfloat16)
    q, s = Fn.fp8_quantize_reference(t, fmt)
    assert q.dtype == Fn.FP8_FORMATS[fmt][0]
    assert torch.isfinite(q.float()).all()
    assert float(q.float().abs().max()) <= Fn.FP8_FORMATS[fmt][1]
    rel = 2.0 ** (-4 if fmt == "e4m3" else -3)                          # half an ulp of a 3- / 2-bit mantissa
    big = t.float().abs() > float(t.float().abs().max()) / 64             # away from the subnormal range
    err = ((q.float() / s - t.float()).abs() / t.float().abs())[big]
    assert float(err.max()) <= rel


def _rel(a, b):
    a, b = a.detach().float(), b.detach().float()
    return float((a - b).norm() / (b.norm() + 1e-12))


@pytest.mark.parametrize("activation", [None, "gelu", "relu"])
def test_cpu_fp8_linear_matches_fp32_linear_to_fp8_accuracy(activation):
    torch.manual_seed(2)
    M, K, N = 96, 64, 48
    x = torch.randn(M, K, requires_grad=True)
    w = (torch.randn(N, K) * 0.1).requires_grad_(True)
    b = (torch.randn(N) * 0.1).requires_grad_(True)
    dy = torch.randn(M, N)
    y8 = Fn.linear(x, w, b, activation, fp8=True)
    y8.backward(dy)
    g8 = (x.grad, w.grad, b.grad)
    x.grad = w.grad = b.grad = None
    y = F.linear(x, w, b)
    y = {None: y, "gelu": F.gelu(y) if activation == "gelu" else y, "relu": F.relu(y)}[activation]
    y.backward(dy)
    # E4M3 keeps 3 mantissa bits (relative rounding error <= 1/16), E5M2 2 bits (<= 1/8); a ReLU mask also flips
    # where the FP8 pre-activation changes sign
    assert _rel(y8, y) < 0.05
    assert _rel(g8[0], x.grad) < 0.2
    assert _rel(g8[1], w.grad) < 0.2
    # without an activation the bias gradient is the exact column sum of dy; with one, dy * act'(pre) sees the FP8 pre
    assert _rel(g8[2], b.grad) < (1e-6 if activation is None else 0.2)
    assert not torch.equal(y8, y)                         # it did quantise


def test_cpu_fp8_linear_bf16_outputs_keep_dtypes_and_shapes():
    torch.manual_seed(3)
    lin = Fn.linear
    x = torch.randn(2, 16, 32, dtype=torch.bfloat16, requires_grad=True)
    w = torch.randn(64, 32, dtype=torch.bfloat16, requires_grad=True)
    b = torch.zeros(64, dtype=torch.bfloat16, requires_grad=True)
    y = lin(x, w, b, "gelu", fp8=True)
    assert y.shape == (2, 16, 64) and y.dtype == torch.bfloat16
    y.float().sum().backward()
    assert x.grad.shape == x.shape and w.grad.shape == w.shape and b.grad.shape == b.shape
    assert x.grad.dtype == w.grad.dtype == b.grad.dtype == torch.bfloat16


def test_fp8_linear_module_checks_feature_counts():
    from b200ddp.ops import Linear
    Linear(32, 48, fp8=True)
    with pytest.raises(ValueError, match="divisible by 16"):
        Linear(30, 48, fp8=True)
    with pytest.raises(ValueError, match="divisible by 16"):
        Linear(32, 40, fp8=True)
    Linear(30, 40)                                        # bf16 / fp32 linears have no such rule


def _tiny(fp8):
    from b200ddp.models.bert import BertConfig, BertForMaskedLM
    torch.manual_seed(7)
    return BertForMaskedLM(BertConfig(vocab_size=1000, hidden=128, layers=2, heads=4, intermediate=256, max_position=64,
                                      pad_vocab_to=64, fp8=fp8))


def test_fp8_bert_has_the_bf16_state_dict_and_loads_it_both_ways():
    from b200ddp.ops import Linear
    a, b = _tiny(False), _tiny(True)
    sa, sb = a.state_dict(), b.state_dict()
    assert list(sa) == list(sb)
    assert all(sa[k].shape == sb[k].shape for k in sa)
    b.load_state_dict(sa, strict=True)
    a.load_state_dict(b.state_dict(), strict=True)
    n8 = [n for n, m in b.named_modules() if isinstance(m, Linear) and m.fp8]
    assert len(n8) == 4 * 2 and all(n.rsplit(".", 1)[1] in ("qkv", "attn_out", "ffn_in", "ffn_out") for n in n8)
    assert not b.transform.fp8


def test_fp8_bert_cpu_emulation_tracks_fp32():
    """The FP8 recipe (CPU emulation) against the same weights in fp32: the loss and the gradients stay close.  This is
    the accuracy the GPU comparison of the FP8 model against the fp32 CPU model allows on top of bf16's."""
    from b200ddp.ops import cross_entropy
    ref, m8 = _tiny(False), _tiny(True)
    m8.load_state_dict(ref.state_dict())
    ids = torch.randint(0, 1000, (4, 64), generator=torch.Generator().manual_seed(1))
    labels = torch.where(torch.rand(4, 64, generator=torch.Generator().manual_seed(2)) < 0.3, ids, torch.full((4, 64), -100))
    lr = cross_entropy(ref(ids), labels)
    lr.backward()
    l8 = cross_entropy(m8(ids), labels)
    l8.backward()
    assert abs(float(l8) - float(lr)) < 2e-2 * abs(float(lr))
    for (n, p), q in zip(m8.named_parameters(), ref.parameters()):
        if float(q.grad.norm()) < 1e-4:
            continue
        assert _rel(p.grad, q.grad) < 0.15, n


def _args(tmp_path, *extra):
    from b200ddp.engine import cli
    return cli.build_parser().parse_args(["--no_tensorboard", "--output_dir", str(tmp_path / "out"), *extra])


def test_fp8_flag_parses_and_defaults_off(tmp_path):
    assert _args(tmp_path).fp8 is False
    assert _args(tmp_path, "--fp8", "--model", "bert-base", "--fp16").fp8 is True


@pytest.mark.parametrize("extra, message", [
    (["--model", "bert-base", "--fp16", "--no_cuda"], "CUDA device"),
    (["--model", "bert-base", "--no_cuda"], "--fp16"),
    (["--model", "resnet50", "--fp16", "--no_cuda"], "bert-base"),
])
def test_fp8_flag_is_rejected_outside_bf16_bert_on_a_gpu(tmp_path, extra, message):
    from b200ddp.engine import cli
    args = _args(tmp_path, "--fp8", *extra)
    with pytest.raises(ValueError, match=message):
        cli.setup(args)


def test_fp8_bert_base_builds_through_the_registry():
    from b200ddp.models import build_model
    from b200ddp.ops import Linear
    m = build_model("bert-base", fp8=True)
    assert sum(isinstance(x, Linear) and x.fp8 for x in m.modules()) == 48
    assert m.bert.config.padded_vocab % 64 == 0
