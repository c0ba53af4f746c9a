"""Causal document attention (csrc/attention.cu, causal mode) on the GPU: accuracy against fp64 beside SDPA's own bf16
error with the dense causal block-diagonal mask, causality, padding rows, determinism, bounds, CUDA-graph replay with a
new packing, input checks, the op against its CPU body, and GPT-2 models and training."""
import math

import pytest
import torch
import torch.nn.functional as F

from b200ddp.ops import functional as Fn

pytestmark = pytest.mark.gpu

HEADS, HD = 12, 64
W = HEADS * HD
BOS, PAD = 50256, 0


def dev():
    return torch.device("cuda", 0)


def C():
    from b200ddp import _ext
    return _ext.get()


def _bounds(layout, S):
    """layout: one list of document lengths per row (the rest of a row is padding) -> int32 [B, S, 2] on the GPU."""
    b = torch.zeros(len(layout), S, 2, dtype=torch.int32)
    for r, docs in enumerate(layout):
        at = 0
        for n in docs:
            b[r, at:at + n, 0], b[r, at:at + n, 1] = at, at + n
            at += n
        assert at <= S
    return b.to(dev())


def _inputs(B, S, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    qkv = torch.randn(B * S, 3 * W, device=dev(), generator=g).to(torch.bfloat16)
    dout = torch.randn(B * S, W, device=dev(), generator=g).to(torch.bfloat16)
    return qkv, dout


def _split(t, B, S):
    return [x.reshape(B, S, HEADS, HD).transpose(1, 2) for x in t.reshape(B, S, 3 * W).split(W, dim=-1)]


def _mask(bounds, S):
    j = torch.arange(S, device=dev())
    inside = (j >= bounds[..., :1].long()) & (j < bounds[..., 1:].long())
    return (inside & (j[None, :] <= j[:, None]))[:, None]      # [B, 1, S, S]


def _reference(qkv, dout, bounds, B, S):
    """fp64 o, lse, dqkv; rows that see no key give zeros and lse = -inf."""
    x = qkv.double().requires_grad_(True)
    q, k, v = _split(x, B, S)
    keep = _mask(bounds, S)
    s = ((q @ k.transpose(-1, -2)) / 8.0).masked_fill(~keep, -math.inf)
    lse = torch.logsumexp(s, dim=-1)
    p = torch.softmax(s.masked_fill(~keep, torch.finfo(torch.float64).min), dim=-1) * keep
    o = (p @ v).transpose(1, 2).reshape(B * S, -1)
    o.backward(dout.double())
    return o.detach(), lse.detach(), x.grad


def _sdpa(qkv, dout, bounds, B, S):
    """SDPA in bf16 with the dense causal block-diagonal boolean mask.  A padding row would be NaN there, so it sees its
    own key instead and its output is zeroed (as its reference is): its dO is then zero, which adds nothing."""
    x = qkv.detach().clone().requires_grad_(True)
    q, k, v = _split(x, B, S)
    live = bounds[..., 1] > bounds[..., 0]
    mask = _mask(bounds, S) | (~live[:, None, :, None] & torch.eye(S, dtype=torch.bool, device=dev()))
    o = F.scaled_dot_product_attention(q, k, v, attn_mask=mask).transpose(1, 2).reshape(B * S, -1)
    o = torch.where(live.reshape(B * S, 1), o, torch.zeros_like(o))
    o.backward(dout)
    return o.detach(), x.grad


def _rms(t):
    return float(t.double().pow(2).mean().sqrt())


def _random_packing(S, seed, lo=1):
    g = torch.Generator().manual_seed(seed)
    docs, at = [], 0
    while True:
        n = int(torch.randint(lo, S + 1, (1,), generator=g))
        if at + n > S:
            return docs
        docs.append(n)
        at += n


LAYOUTS = {                                                     # S -> document lengths per row
    "full_rows": lambda S: [[S], [S], [S]],
    "right_padded": lambda S: [[S // 2 + 3], [S - 1], [1]],
    "tile_edges": lambda S: ([[1, 63, 64, 65, 63], [127, 129], [128, 128]] if S == 256 else
                             [[1, 63, 64, 65, 127, 128, 64], [129, 127, 1, 128, 127], [129, 129, 129, 125]]),
    "many_one_token_docs": lambda S: [[1] * S, [1] * (S // 2) + [S // 4]],
    "docs_and_tail_padding": lambda S: [[100, 5, 40], _random_packing(S, 3, 16), [S // 2]],
    "all_padding_row": lambda S: [[], [70, 30], [S]],
}


@pytest.mark.parametrize("layout", sorted(LAYOUTS))
@pytest.mark.parametrize("S", [256, 512])
def test_causal_attention_is_as_accurate_as_sdpa(layout, S):
    docs = LAYOUTS[layout](S)
    B = len(docs)
    bounds = _bounds(docs, S)
    qkv, dout = _inputs(B, S, seed=S + len(layout))
    o, lse = C().causal_attention_fwd(qkv, bounds, HEADS)
    dqkv = C().causal_attention_bwd(dout, qkv, o, lse, bounds, HEADS)
    o_ref, lse_ref, d_ref = _reference(qkv, dout, bounds, B, S)
    o_lib, d_lib = _sdpa(qkv, dout, bounds, B, S)
    assert torch.isfinite(o.float()).all() and torch.isfinite(dqkv.float()).all()
    live = torch.isfinite(lse_ref)
    assert torch.equal(torch.isfinite(lse), live)
    assert torch.allclose(lse.double()[live], lse_ref[live], rtol=0, atol=2e-3), float((lse.double() - lse_ref)[live].abs().max())
    for name, ours, lib, ref in (("o", o, o_lib, o_ref), ("dq", dqkv[:, :W], d_lib[:, :W], d_ref[:, :W]),
                                 ("dk", dqkv[:, W:2 * W], d_lib[:, W:2 * W], d_ref[:, W:2 * W]),
                                 ("dv", dqkv[:, 2 * W:], d_lib[:, 2 * W:], d_ref[:, 2 * W:])):
        err, lib_err = _rms(ours.double() - ref), _rms(lib.double() - ref)
        assert err <= 1.5 * lib_err + 2e-3 * _rms(ref), (name, err, lib_err, _rms(ref))


@pytest.mark.parametrize("t", [0, 1, 63, 64, 127, 128, 200, 383])
def test_perturbing_token_t_leaves_every_earlier_row_bit_identical(t):
    """Rows before t never see token t: their output, lse and dQ (same dO) stay bit-identical."""
    B, S = 2, 384
    bounds = _bounds([[S], [100, 150, 134]], S)
    qkv, dout = _inputs(B, S, seed=31)
    o, lse = C().causal_attention_fwd(qkv, bounds, HEADS)
    d = C().causal_attention_bwd(dout, qkv, o, lse, bounds, HEADS)
    qkv2 = qkv.clone()
    for r in range(B):
        qkv2[r * S + t] = torch.randn(3 * W, device=dev()).to(torch.bfloat16) * 4
    o2, lse2 = C().causal_attention_fwd(qkv2, bounds, HEADS)
    d2 = C().causal_attention_bwd(dout, qkv2, o2, lse2, bounds, HEADS)
    o3, o23 = o.view(B, S, W), o2.view(B, S, W)
    assert torch.equal(o3[:, :t], o23[:, :t])
    assert torch.equal(lse[:, :, :t], lse2[:, :, :t])
    assert torch.equal(d.view(B, S, 3 * W)[:, :t, :W], d2.view(B, S, 3 * W)[:, :t, :W])
    assert not torch.equal(o3[0, t], o23[0, t])


def test_padding_rows_get_zeros_minus_inf_and_zero_gradients():
    S = 256
    docs = [[], [1, 40], [256]]
    bounds = _bounds(docs, S)
    qkv, dout = _inputs(3, S, seed=5)
    o, lse = C().causal_attention_fwd(qkv, bounds, HEADS)
    d = C().causal_attention_bwd(dout, qkv, o, lse, bounds, HEADS)
    assert torch.isfinite(o.float()).all() and torch.isfinite(d.float()).all() and not torch.isnan(lse).any()
    o3, d3, lse3 = o.view(3, S, W), d.view(3, S, 3 * W), lse.view(3, HEADS, S)
    for r, fill in ((0, 0), (1, 41)):
        assert (o3[r, fill:] == 0).all() and (d3[r, fill:] == 0).all(), r
        assert torch.isinf(lse3[r, :, fill:]).all() and (lse3[r, :, fill:] < 0).all(), r
    assert torch.isfinite(lse3[1, :, :41]).all() and torch.isfinite(lse3[2]).all()
    # a one-token document sees only itself: its output is its own value row
    assert torch.equal(o3[1, 0], qkv.view(3, S, 3 * W)[1, 0, 2 * W:])
    assert d3[1, :41].abs().sum() > 0


def test_causal_attention_is_deterministic():
    S = 512
    docs = [_random_packing(S, s) for s in range(8)]
    bounds = _bounds(docs, S)
    qkv, dout = _inputs(8, S, seed=9)
    runs = []
    for _ in range(2):
        o, lse = C().causal_attention_fwd(qkv, bounds, HEADS)
        runs.append((o, lse, C().causal_attention_bwd(dout, qkv, o, lse, bounds, HEADS)))
    for a, b in zip(*runs):
        assert torch.equal(a, b)


def test_causal_attention_stays_in_bounds():
    B, S = 3, 256
    bounds = _bounds([[], [100, 56], [256]], S)
    # out-of-range bounds are clamped on the device: they may give any values, but never touch memory outside
    bounds[1, 200:, 0], bounds[1, 200:, 1] = -50, 10 ** 6
    bounds[2, :5, 0], bounds[2, :5, 1] = 300, 200
    bounds[2, 10:20, 0] = 15                                    # start after the row itself: the row sees no key
    qkv, dout = _inputs(B, S, seed=2)
    sentinel, pad = -12345.0, 64
    o_buf = torch.full((B * S * W + 2 * pad,), sentinel, device=dev(), dtype=torch.bfloat16)
    lse_buf = torch.full((B * HEADS * S + 2 * pad,), sentinel, device=dev())
    d_buf = torch.full((B * S * 3 * W + 2 * pad,), sentinel, device=dev(), dtype=torch.bfloat16)
    o = o_buf[pad:pad + B * S * W].view(B * S, W)
    lse = lse_buf[pad:pad + B * HEADS * S].view(B, HEADS, S)
    dqkv = d_buf[pad:pad + B * S * 3 * W].view(B * S, 3 * W)
    C().causal_attention_fwd(qkv, bounds, HEADS, o, lse)
    C().causal_attention_bwd(dout, qkv, o, lse, bounds, HEADS, dqkv)
    o_ref, lse_ref = C().causal_attention_fwd(qkv, bounds, HEADS)
    assert torch.equal(o, o_ref) and torch.equal(lse, lse_ref)
    assert torch.equal(dqkv, C().causal_attention_bwd(dout, qkv, o_ref, lse_ref, bounds, HEADS))
    assert torch.isfinite(o.float()).all() and torch.isfinite(dqkv.float()).all()
    for buf in (o_buf, lse_buf, d_buf):
        assert (buf[:pad] == sentinel).all() and (buf[-pad:] == sentinel).all()


def test_graph_replay_with_a_new_packing_matches_eager():
    B, S = 4, 512
    bounds = _bounds([_random_packing(S, s, 16) for s in range(B)], S)
    qkv, dout = _inputs(B, S, seed=4)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                                  # warm-up: tensor maps, kernel attributes
        o, lse = C().causal_attention_fwd(qkv, bounds, HEADS)
        C().causal_attention_bwd(dout, qkv, o, lse, bounds, HEADS)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        o_g, lse_g = C().causal_attention_fwd(qkv, bounds, HEADS)
        d_g = C().causal_attention_bwd(dout, qkv, o_g, lse_g, bounds, HEADS)
    for layout in ([[512], [1] * 100, [], [300, 200]], [_random_packing(S, 40 + s, 8) for s in range(B)]):
        bounds.copy_(_bounds(layout, S))
        graph.replay()
        o, lse = C().causal_attention_fwd(qkv, bounds, HEADS)
        d = C().causal_attention_bwd(dout, qkv, o, lse, bounds, HEADS)
        torch.cuda.synchronize()
        assert torch.equal(o_g, o) and torch.equal(lse_g, lse) and torch.equal(d_g, d), layout


def test_causal_attention_rejects_unsupported_input():
    good = torch.randn(2, 128, 3 * 128, device=dev()).to(torch.bfloat16)
    bounds = _bounds([[100], [28, 100]], 128)
    Fn.causal_attention(good, bounds, 2)                        # head dim 64, S = 128: accepted
    with pytest.raises(ValueError):
        Fn.causal_attention(good.half(), bounds, 2)             # not bf16
    with pytest.raises(ValueError):
        Fn.causal_attention(good, bounds, 4)                    # head dim 32
    with pytest.raises(ValueError):
        Fn.causal_attention(torch.randn(2, 192, 3 * 128, device=dev()).to(torch.bfloat16), _bounds([[1], [1]], 192), 2)
    with pytest.raises(ValueError):
        Fn.causal_attention(torch.randn(2, 128, 6 * 128, device=dev()).to(torch.bfloat16)[..., :3 * 128], bounds, 2)
    with pytest.raises(ValueError):
        Fn.causal_attention(good, bounds[:, :64], 2)            # bounds not [B, S, 2]
    with pytest.raises(ValueError):
        Fn.causal_attention(good, bounds.float(), 2)            # bounds not integer


def test_causal_op_matches_its_cpu_body():
    B, S, H = 2, 128, 2
    torch.manual_seed(0)
    qkv = torch.randn(B, S, 3 * H * HD).to(torch.bfloat16)
    bounds = _bounds([[5, 60, 63], [30]], S).cpu()
    dy = torch.randn(B, S, H * HD).to(torch.bfloat16)
    xc = qkv.clone().requires_grad_(True)
    Fn.causal_attention(xc, bounds, H).backward(dy)
    yc = Fn.causal_attention_reference(qkv, bounds, H)
    xg = qkv.to(dev()).requires_grad_(True)
    yg = Fn.causal_attention(xg, bounds.to(dev()), H)
    yg.backward(dy.to(dev()))
    assert torch.allclose(yg.float().cpu(), yc.float(), rtol=2e-2, atol=2e-2)
    assert torch.allclose(xg.grad.float().cpu(), xc.grad.float(), rtol=5e-2, atol=5e-2)


def test_gelu_tanh_kernels_match_torch():
    from b200ddp.ops import Linear
    torch.manual_seed(3)
    pre = (torch.randn(64, 3072, device=dev()) * 3).to(torch.bfloat16)
    dy = torch.randn_like(pre)
    y = C().gelu_fwd(pre, True)
    g = C().gelu_bwd(dy, pre, True)
    x = pre.float().requires_grad_(True)
    ref = F.gelu(x, approximate="tanh")
    ref.backward(dy.float())
    assert torch.allclose(y.float(), ref.detach(), rtol=1e-2, atol=1e-2)
    assert torch.allclose(g.float(), x.grad, rtol=2e-2, atol=2e-2)
    assert torch.equal(C().gelu_fwd(pre), C().gelu_fwd(pre, False))  # the erf form is the default
    for fp8 in (False, True):
        lin = Linear(256, 512, activation="gelu_tanh", fp8=fp8)
        cpu = Linear(256, 512, activation="gelu_tanh", fp8=fp8)
        cpu.load_state_dict(lin.state_dict())
        lin = lin.to(dev(), torch.bfloat16)
        cpu = cpu.to(torch.bfloat16)
        xb = torch.randn(128, 256).to(torch.bfloat16)
        xg, xc = xb.to(dev()).requires_grad_(True), xb.clone().requires_grad_(True)
        yg, yc = lin(xg), cpu(xc)
        yg.float().square().mean().backward()
        yc.float().square().mean().backward()
        rel = float((yg.detach().float().cpu() - yc.detach().float()).norm() / yc.detach().float().norm())
        rel_g = float((xg.grad.float().cpu() - xc.grad.float()).norm() / xc.grad.float().norm())
        assert rel < 2e-2 and rel_g < 5e-2, (fp8, rel, rel_g)


# ---- GPT-2 -------------------------------------------------------------------------------------------------------------
def _tiny_cfg(**kw):
    from b200ddp.models.gpt import GPTConfig
    return GPTConfig(vocab_size=1000, hidden=128, layers=2, heads=2, intermediate=512, max_position=256, **kw)


def _packed_batch(rows, S, seed, bos=999):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(1, 999, (len(rows), S), generator=g)
    labels = torch.full(ids.shape, -100)
    for r, docs in enumerate(rows):
        at = 0
        for n in docs:
            ids[r, at] = bos
            labels[r, at:at + n - 1] = ids[r, at + 1:at + n]
            at += n
        ids[r, at:] = PAD
    return ids, labels


@pytest.mark.parametrize("mode", ["sdpa", "padded", "packed"])
def test_gpt_tiny_gpu_matches_cpu_reference(mode):
    """bf16 GPU model (SDPA is_causal, or the native causal kernel) against the fp32 CPU model with the same weights."""
    from b200ddp.models.gpt import GPTLMHeadModel
    from b200ddp.ops import cross_entropy
    kw = {"sdpa": {}, "padded": {"pad_token_id": PAD}, "packed": {"pad_token_id": PAD, "bos_token_id": 999}}[mode]
    torch.manual_seed(7)
    ref = GPTLMHeadModel(_tiny_cfg(**kw))
    gpu = GPTLMHeadModel(_tiny_cfg(**kw))
    gpu.load_state_dict(ref.state_dict())
    gpu = gpu.to(dev(), torch.bfloat16)
    rows = {"sdpa": [[128]] * 4, "padded": [[128], [100], [1], [64]], "packed": [[40, 1, 57, 30], [128], [64, 63], []]}[mode]
    ids, labels = _packed_batch(rows, 128, seed=1)
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


def test_gpt2_step_has_no_host_synchronisation():
    from b200ddp.models.gpt import GPTLMHeadModel
    from b200ddp.ops import cross_entropy
    torch.manual_seed(1)
    model = GPTLMHeadModel(_tiny_cfg(pad_token_id=PAD, bos_token_id=999)).to(dev(), torch.bfloat16)
    ids, labels = _packed_batch([[100, 28], [1, 1, 126], [50], [128]], 128, seed=2)
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
def test_packed_gpt2_graph_training_lowers_the_loss(tmp_path, fp8):
    """What `python ddp.py --model gpt2 --fp16 --optimizer adamw --cuda_graph --max_steps 30 --seq_len 256
    --min_seq_len 32 --pack [--fp8]` runs."""
    from b200ddp.engine import cli
    from b200ddp.engine.trainer import Trainer
    from b200ddp.models import build_model
    argv = ["--model", "gpt2", "--fp16", "--optimizer", "adamw", "--cuda_graph", "--max_steps", "30", "--seq_len", "256",
            "--min_seq_len", "32", "--pack", "--per_gpu_train_batch_size", "8", "--lr", "5e-4", "--warmup_steps", "5",
            "--weight_decay", "0.01", "--save_steps", "0", "--logging_steps", "10", "--no_tensorboard",
            "--output_dir", str(tmp_path / "out")] + (["--fp8"] if fp8 else [])
    args = cli.build_parser().parse_args(argv)
    cli.setup(args)
    kwargs = {"pad_token_id": PAD, "bos_token_id": BOS, **({"fp8": True} if fp8 else {})}
    model = build_model("gpt2", **kwargs)
    assert sum(getattr(m, "fp8", False) is True for m in model.modules()) == (48 if fp8 else 0)
    # uniform tokens over 50257 ids leave almost nothing to learn (the loss floor is ln 50256): fold the document tokens
    # into 64 ids, keeping BOS, padding and the next-token labels consistent
    from b200ddp.data import SyntheticTokens
    from b200ddp.engine.trainer import build_dataset
    ds = build_dataset(args)
    assert isinstance(ds, SyntheticTokens) and ds.bos_token_id == BOS
    ds.X = torch.where((ds.X != PAD) & (ds.X != BOS), ds.X % 64 + 1, ds.X)
    ds.Y = torch.where(ds.Y >= 0, ds.Y % 64 + 1, ds.Y)
    trainer = Trainer(args, model, cli.log, dataset=ds)
    assert trainer.dataset.doc_lengths is not None and max(len(r) for r in trainer.dataset.doc_lengths) > 1
    before = trainer.evaluate(max_batches=4)["eval_loss"]
    trainer.train()
    after = trainer.evaluate(max_batches=4)["eval_loss"]
    assert trainer.step_fn.graph is not None
    assert math.isfinite(after) and after < before - 0.05, (before, after)
