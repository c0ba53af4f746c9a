"""Key-padding attention kernels (csrc/attention.cu) on the GPU: accuracy against fp64 beside SDPA's own bf16 error,
zero gradients at padding, determinism, bounds, CUDA-graph replay with new lengths, input checks, and BERT training."""
import math

import pytest
import torch
import torch.nn.functional as F

from b200ddp.ops import functional as Fn

pytestmark = pytest.mark.gpu

HEADS, HD = 12, 64


def dev():
    return torch.device("cuda", 0)


def C():
    from b200ddp import _ext
    return _ext.get()


def _inputs(B, S, lens, seed=0, heads=HEADS):
    g = torch.Generator(device="cuda").manual_seed(seed)
    qkv = torch.randn(B * S, 3 * heads * HD, device=dev(), generator=g).to(torch.bfloat16)
    dout = torch.randn(B * S, heads * HD, device=dev(), generator=g).to(torch.bfloat16)
    return qkv, dout, torch.tensor(lens, dtype=torch.int32, device=dev())


def _split(t, B, S, heads=HEADS):
    """[B*S, 3*heads*64] -> q, k, v [B, heads, S, 64]"""
    return [x.reshape(B, S, heads, HD).transpose(1, 2) for x in t.reshape(B, S, 3 * heads * HD).split(heads * HD, dim=-1)]


def _merge(q, k, v, B, S):
    return torch.cat([x.transpose(1, 2).reshape(B * S, -1) for x in (q, k, v)], dim=1)


def _reference(qkv, dout, lens, B, S):
    """fp64 o [B*S, H*64], lse [B, H, S], dqkv [B*S, 3*H*64] on the same bf16 inputs."""
    x = qkv.double().requires_grad_(True)
    q, k, v = _split(x, B, S)
    keep = (torch.arange(S, device=dev())[None, :] < lens.long().clamp(0, S)[:, None])[:, None, None, :]
    s = (q @ k.transpose(-1, -2)) / 8.0
    s = s.masked_fill(~keep, -math.inf)
    lse = torch.logsumexp(s, dim=-1)
    o = (torch.softmax(s, dim=-1) @ v).transpose(1, 2).reshape(B * S, -1)
    o.backward(dout.double())
    return o.detach(), lse.detach(), x.grad


def _sdpa(qkv, dout, lens, B, S, full):
    """SDPA in bf16 on the same inputs: flash when every key is visible, the boolean key mask otherwise."""
    x = qkv.detach().clone().requires_grad_(True)
    q, k, v = _split(x, B, S)
    mask = None if full else (torch.arange(S, device=dev())[None, :] < lens.long()[:, None])[:, None, None, :]
    o = F.scaled_dot_product_attention(q, k, v, attn_mask=mask).transpose(1, 2).reshape(B * S, -1)
    o.backward(dout)
    return o.detach(), x.grad


def _rms(t):
    return float(t.double().pow(2).mean().sqrt())


def _lengths(kind, B, S, seed):
    if kind == "full":
        return [S] * B
    if kind == "random":
        g = torch.Generator().manual_seed(seed)
        return torch.randint(1, S + 1, (B,), generator=g).tolist()
    edges = [1, 63, 64, 65, 127, 128, 129, S]
    return [min(edges[i % len(edges)], S) for i in range(B)]


@pytest.mark.parametrize("kind", ["full", "random", "edges"])
@pytest.mark.parametrize("S", [128, 512])
@pytest.mark.parametrize("B", [1, 4, 16])
def test_attention_is_as_accurate_as_sdpa(B, S, kind):
    lens = _lengths(kind, B, S, seed=B * 1000 + S)
    qkv, dout, lt = _inputs(B, S, lens, seed=B + S)
    o, lse = C().attention_fwd(qkv, lt, HEADS)
    dqkv = C().attention_bwd(dout, qkv, o, lse, lt, HEADS)
    o_ref, lse_ref, d_ref = _reference(qkv, dout, lt, B, S)
    o_lib, d_lib = _sdpa(qkv, dout, lt, B, S, full=kind == "full")
    assert torch.isfinite(o.float()).all() and torch.isfinite(dqkv.float()).all()
    assert torch.allclose(lse.double(), lse_ref, rtol=0, atol=2e-3), float((lse.double() - lse_ref).abs().max())
    W = HEADS * HD
    for name, ours, lib, ref in (("o", o, o_lib, o_ref), ("dq", dqkv[:, :W], d_lib[:, :W], d_ref[:, :W]),
                                 ("dk", dqkv[:, W:2 * W], d_lib[:, W:2 * W], d_ref[:, W:2 * W]),
                                 ("dv", dqkv[:, 2 * W:], d_lib[:, 2 * W:], d_ref[:, 2 * W:])):
        err, lib_err = _rms(ours.double() - ref), _rms(lib.double() - ref)
        assert err <= 1.5 * lib_err + 2e-3 * _rms(ref), (name, err, lib_err, _rms(ref))


def test_padding_gets_zero_gradients_and_empty_sequences_are_zero():
    B, S = 4, 256
    lens = [0, 1, 200, 256]
    qkv, dout, lt = _inputs(B, S, lens, seed=5)
    o, lse = C().attention_fwd(qkv, lt, HEADS)
    dqkv = C().attention_bwd(dout, qkv, o, lse, lt, HEADS)
    W = HEADS * HD
    assert torch.isfinite(o.float()).all() and torch.isfinite(dqkv.float()).all()
    o3, d3 = o.view(B, S, W), dqkv.view(B, S, 3 * W)
    for b, n in enumerate(lens):
        assert (d3[b, n:, W:] == 0).all(), b                   # dK, dV rows at or beyond the length
    assert (o3[0] == 0).all() and (d3[0] == 0).all()            # length 0: zeros everywhere, not NaN
    assert torch.isinf(lse[0]).all() and (lse[0] < 0).all()
    assert (d3[1, :, :W].abs().sum() > 0) and (d3[3, :, W:].abs().sum() > 0)


def test_attention_is_deterministic():
    B, S = 8, 512
    qkv, dout, lt = _inputs(B, S, _lengths("random", B, S, 11), seed=9)
    runs = []
    for _ in range(2):
        o, lse = C().attention_fwd(qkv, lt, HEADS)
        runs.append((o, lse, C().attention_bwd(dout, qkv, o, lse, lt, HEADS)))
    for a, b in zip(*runs):
        assert torch.equal(a, b)


def test_attention_stays_in_bounds():
    B, S = 3, 256
    qkv, dout, lt = _inputs(B, S, [0, 100, 256], seed=2)
    W = HEADS * HD
    sentinel = -12345.0
    pad = 64                                                    # elements before and after: keeps 16-byte alignment
    o_buf = torch.full((B * S * W + 2 * pad,), sentinel, device=dev(), dtype=torch.bfloat16)
    lse_buf = torch.full((B * HEADS * S + 2 * pad,), sentinel, device=dev())
    d_buf = torch.full((B * S * 3 * W + 2 * pad,), sentinel, device=dev(), dtype=torch.bfloat16)
    o = o_buf[pad:pad + B * S * W].view(B * S, W)
    lse = lse_buf[pad:pad + B * HEADS * S].view(B, HEADS, S)
    dqkv = d_buf[pad:pad + B * S * 3 * W].view(B * S, 3 * W)
    C().attention_fwd(qkv, lt, HEADS, o, lse)
    C().attention_bwd(dout, qkv, o, lse, lt, HEADS, dqkv)
    o_ref, lse_ref = C().attention_fwd(qkv, lt, HEADS)
    assert torch.equal(o, o_ref) and torch.equal(lse, lse_ref)
    assert torch.equal(dqkv, C().attention_bwd(dout, qkv, o_ref, lse_ref, lt, HEADS))
    for buf in (o_buf, lse_buf, d_buf):
        assert (buf[:pad] == sentinel).all() and (buf[-pad:] == sentinel).all()


def test_graph_replay_with_new_lengths_matches_eager():
    B, S = 4, 512
    qkv, dout, lt = _inputs(B, S, [512, 300, 17, 129], seed=4)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                                  # warm-up: tensor maps, kernel attributes
        o, lse = C().attention_fwd(qkv, lt, HEADS)
        C().attention_bwd(dout, qkv, o, lse, lt, HEADS)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        o_g, lse_g = C().attention_fwd(qkv, lt, HEADS)
        d_g = C().attention_bwd(dout, qkv, o_g, lse_g, lt, HEADS)
    for lens in ([64, 512, 0, 1], [129, 128, 127, 500]):
        lt.copy_(torch.tensor(lens, dtype=torch.int32))
        graph.replay()
        o, lse = C().attention_fwd(qkv, lt, HEADS)
        d = C().attention_bwd(dout, qkv, o, lse, lt, HEADS)
        torch.cuda.synchronize()
        assert torch.equal(o_g, o) and torch.equal(lse_g, lse) and torch.equal(d_g, d), lens


def test_attention_rejects_unsupported_input():
    lens = torch.tensor([100, 128], device=dev())
    good = torch.randn(2, 128, 3 * 128, device=dev()).to(torch.bfloat16)
    Fn.attention(good, lens, 2)                                 # head dim 64, S = 128: accepted
    with pytest.raises(ValueError):
        Fn.attention(good.half(), lens, 2)                      # not bf16
    with pytest.raises(ValueError):
        Fn.attention(good, lens, 4)                             # head dim 32
    with pytest.raises(ValueError):
        Fn.attention(torch.randn(2, 192, 3 * 128, device=dev()).to(torch.bfloat16), lens, 2)   # S % 128 != 0
    with pytest.raises(ValueError):
        Fn.attention(torch.randn(2, 128, 6 * 128, device=dev()).to(torch.bfloat16)[..., :3 * 128], lens, 2)  # non-contiguous


def test_attention_op_matches_its_cpu_body():
    B, S, H = 3, 128, 2
    torch.manual_seed(0)
    qkv = torch.randn(B, S, 3 * H * HD).to(torch.bfloat16)
    lens = torch.tensor([5, 128, 0])
    dy = torch.randn(B, S, H * HD).to(torch.bfloat16)
    xc = qkv.clone().requires_grad_(True)
    Fn.attention(xc, lens, H).backward(dy)
    yc = Fn.attention_reference(qkv, lens, H)
    xg = qkv.to(dev()).requires_grad_(True)
    yg = Fn.attention(xg, lens.to(dev()), H)
    yg.backward(dy.to(dev()))
    assert torch.allclose(yg.float().cpu(), yc.float(), rtol=2e-2, atol=2e-2)
    assert torch.allclose(xg.grad.float().cpu(), xc.grad.float(), rtol=5e-2, atol=5e-2)


# ---- BERT --------------------------------------------------------------------------------------------------------------
def _tiny_cfg(**kw):
    from b200ddp.models.bert import BertConfig
    return BertConfig(vocab_size=1000, hidden=128, layers=2, heads=2, intermediate=256, max_position=128, pad_vocab_to=64, **kw)


def _padded_batch(B, S, lens, seed):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(1, 1000, (B, S), generator=g)
    labels = torch.where(torch.rand(B, S, generator=g) < 0.3, torch.randint(0, 1000, (B, S), generator=g), torch.full((B, S), -100))
    pad = torch.arange(S)[None, :] >= torch.tensor(lens)[:, None]
    return ids.masked_fill(pad, 0), labels.masked_fill(pad, -100)


def test_padded_bert_tiny_gpu_matches_cpu_reference():
    """bf16 GPU model (native attention) against the fp32 CPU model with the same weights; tolerances of the FP8 test."""
    from b200ddp.models.bert import BertForMaskedLM
    from b200ddp.ops import cross_entropy
    torch.manual_seed(7)
    ref = BertForMaskedLM(_tiny_cfg(pad_token_id=0))
    gpu = BertForMaskedLM(_tiny_cfg(pad_token_id=0))
    gpu.load_state_dict(ref.state_dict())
    gpu = gpu.to(dev(), torch.bfloat16)
    ids, labels = _padded_batch(4, 128, [128, 77, 1, 64], seed=1)
    lr = cross_entropy(ref(ids), labels)
    lr.backward()
    lg = cross_entropy(gpu(ids.to(dev())), labels.to(dev()))
    lg.backward()
    lg, lr = float(lg.detach()), float(lr.detach())
    assert abs(lg - lr) < 5e-2 * max(1.0, abs(lr))
    for (n, p), q in zip(gpu.named_parameters(), ref.parameters()):
        if float(q.grad.norm()) < 1e-4:
            assert float(p.grad.float().norm()) < 5e-2, n
            continue
        rel = float((p.grad.float().cpu() - q.grad).norm() / (q.grad.norm() + 1e-8))
        assert rel < 0.2, (n, rel)


def test_padded_bert_step_has_no_host_synchronisation():
    from b200ddp.models.bert import BertForMaskedLM
    from b200ddp.ops import cross_entropy
    torch.manual_seed(1)
    model = BertForMaskedLM(_tiny_cfg(pad_token_id=0)).to(dev(), torch.bfloat16)
    ids, labels = _padded_batch(4, 128, [100, 128, 3, 50], seed=2)
    ids, labels = ids.to(dev()), labels.to(dev())
    cross_entropy(model(ids), labels).backward()
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


@pytest.mark.parametrize("fp8", [False, True])
def test_padded_bert_base_graph_training_lowers_the_loss(tmp_path, fp8):
    """What `python ddp.py --model bert-base --fp16 --optimizer adamw --cuda_graph --max_steps 30 --seq_len 128
    --min_seq_len 32 [--fp8]` runs."""
    from b200ddp.engine import cli
    from b200ddp.engine.trainer import Trainer
    from b200ddp.models import build_model
    argv = ["--model", "bert-base", "--fp16", "--optimizer", "adamw", "--cuda_graph", "--max_steps", "30", "--seq_len", "128",
            "--min_seq_len", "32", "--per_gpu_train_batch_size", "16", "--lr", "5e-4", "--warmup_steps", "5",
            "--weight_decay", "0.01", "--save_steps", "0", "--logging_steps", "10", "--no_tensorboard",
            "--output_dir", str(tmp_path / "out")] + (["--fp8"] if fp8 else [])
    args = cli.build_parser().parse_args(argv)
    cli.setup(args)
    kwargs = {"pad_token_id": 0, **({"fp8": True} if fp8 else {})}
    trainer = Trainer(args, build_model("bert-base", **kwargs), cli.log)
    assert trainer.dataset.lengths is not None and int(trainer.dataset.lengths.min()) < 128
    before = trainer.evaluate(max_batches=4)["eval_loss"]
    trainer.train()
    after = trainer.evaluate(max_batches=4)["eval_loss"]
    assert trainer.step_fn.graph is not None
    assert math.isfinite(after) and after < before - 0.05, (before, after)
