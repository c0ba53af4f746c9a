"""Llama / SmolLM kernels on the GPU: grouped-query causal attention against fp64 beside SDPA's own bf16 error, its
determinism and CUDA-graph replay with a new packing, rotary / RMSNorm / SwiGLU against fp64, the model against its CPU
body, a training step without host synchronisation, and CUDA-graph AdamW training on padded and packed rows."""
import math

import pytest
import torch
import torch.nn.functional as F

from b200ddp.ops import functional as Fn

pytestmark = pytest.mark.gpu
HD = 64


def dev():
    return torch.device("cuda", 0)


def C():
    from b200ddp import _ext
    return _ext.get()


def _bounds(layout, S):
    b = torch.zeros(len(layout), S, 2, dtype=torch.int32)
    for r, docs in enumerate(layout):
        at = 0
        for n in docs:
            b[r, at:at + n, 0], b[r, at:at + n, 1] = at, at + n
            at += n
    return b.to(dev())


def _packing(S, seed, lo=1):
    g = torch.Generator().manual_seed(seed)
    docs, at = [], 0
    while True:
        n = int(torch.randint(lo, S + 1, (1,), generator=g))
        if at + n > S:
            return docs
        docs.append(n)
        at += n


def _split(qkv, B, S, H, Hkv):
    q, k, v = qkv.reshape(B, S, -1).split([H * HD, Hkv * HD, Hkv * HD], -1)
    return [t.reshape(B, S, -1, HD).transpose(1, 2) for t in (q, k, v)]


def _mask(bounds, S):
    j = torch.arange(S, device=dev())
    inside = (j >= bounds[..., :1].long()) & (j < bounds[..., 1:].long())
    return (inside & (j[None, :] <= j[:, None]))[:, None]


def _reference(qkv, dout, bounds, B, S, H, Hkv):
    x = qkv.double().requires_grad_(True)
    q, k, v = _split(x, B, S, H, Hkv)
    k, v = (t.repeat_interleave(H // Hkv, dim=1) for t in (k, v))
    keep = _mask(bounds, S)
    s = ((q @ k.transpose(-1, -2)) / 8.0).masked_fill(~keep, -math.inf)
    lse = torch.logsumexp(s, dim=-1)
    p = torch.softmax(s.masked_fill(~keep, torch.finfo(torch.float64).min), dim=-1) * keep
    o = (p @ v).transpose(1, 2).reshape(B * S, -1)
    o.backward(dout.double())
    return o.detach(), lse.detach(), x.grad


def _sdpa(qkv, dout, bounds, B, S, H, Hkv):
    x = qkv.detach().clone().requires_grad_(True)
    q, k, v = _split(x, B, S, H, Hkv)
    live = bounds[..., 1] > bounds[..., 0]
    mask = _mask(bounds, S) | (~live[:, None, :, None] & torch.eye(S, dtype=torch.bool, device=dev()))
    o = F.scaled_dot_product_attention(q, k, v, attn_mask=mask, enable_gqa=True).transpose(1, 2).reshape(B * S, -1)
    o = torch.where(live.reshape(B * S, 1), o, torch.zeros_like(o))
    o.backward(dout)
    return o.detach(), x.grad


def _rms(t):
    return float(t.double().pow(2).mean().sqrt())


LAYOUTS = {
    "fixed": lambda S: [[S], [S]],
    "right_padded": lambda S: [[S // 2 + 3], [S - 1], [1]],
    "packed": lambda S: [_packing(S, 3, 16), [100, 5, 40], _packing(S, 5)],
    "all_padding_row": lambda S: [[], [70, 30], [S]],
}


@pytest.mark.parametrize("layout", sorted(LAYOUTS))
@pytest.mark.parametrize("H,Hkv,S", [(4, 4, 256), (9, 3, 512), (8, 2, 256), (4, 1, 384), (9, 3, 2048)])
def test_gqa_attention_is_as_accurate_as_sdpa(layout, H, Hkv, S):
    if S == 2048 and layout != "packed":
        pytest.skip("one long-row layout keeps the fp64 reference affordable")
    docs = LAYOUTS[layout](S)
    B = len(docs)
    bounds = _bounds(docs, S)
    g = torch.Generator(device="cuda").manual_seed(S + H + Hkv)
    qkv = torch.randn(B * S, (H + 2 * Hkv) * HD, device=dev(), generator=g).to(torch.bfloat16)
    dout = torch.randn(B * S, H * HD, device=dev(), generator=g).to(torch.bfloat16)
    o, lse = C().causal_gqa_attention_fwd(qkv, bounds, H, Hkv)
    dqkv = C().causal_gqa_attention_bwd(dout, qkv, o, lse, bounds, H, Hkv)
    o_ref, lse_ref, d_ref = _reference(qkv, dout, bounds, B, S, H, Hkv)
    o_lib, d_lib = _sdpa(qkv, dout, bounds, B, S, H, Hkv)
    live = torch.isfinite(lse_ref)
    assert torch.equal(torch.isfinite(lse), live)
    assert torch.allclose(lse.double()[live], lse_ref[live], rtol=0, atol=2e-3)
    W, K = H * HD, Hkv * HD
    for name, sl in (("dq", slice(0, W)), ("dk", slice(W, W + K)), ("dv", slice(W + K, W + 2 * K))):
        err, lib_err = _rms(dqkv[:, sl].double() - d_ref[:, sl]), _rms(d_lib[:, sl].double() - d_ref[:, sl])
        assert err <= 1.5 * lib_err + 2e-3 * _rms(d_ref[:, sl]), (name, err, lib_err)
    err, lib_err = _rms(o.double() - o_ref), _rms(o_lib.double() - o_ref)
    assert err <= 1.5 * lib_err + 2e-3 * _rms(o_ref), ("o", err, lib_err)
    if layout == "all_padding_row":
        assert (o.view(B, S, -1)[0] == 0).all() and (dqkv.view(B, S, -1)[0] == 0).all()


def test_gqa_gradients_are_bitwise_deterministic():
    S, H, Hkv = 512, 9, 3
    bounds = _bounds([_packing(S, s, 8) for s in range(4)], S)
    qkv = torch.randn(4 * S, (H + 2 * Hkv) * HD, device=dev()).to(torch.bfloat16)
    dout = torch.randn(4 * S, H * HD, device=dev()).to(torch.bfloat16)
    runs = []
    for _ in range(2):
        o, lse = C().causal_gqa_attention_fwd(qkv, bounds, H, Hkv)
        runs.append((o, lse, C().causal_gqa_attention_bwd(dout, qkv, o, lse, bounds, H, Hkv)))
    for a, b in zip(*runs):
        assert torch.equal(a, b)


def test_gqa_graph_replay_with_a_new_packing_matches_eager():
    B, S, H, Hkv = 3, 512, 9, 3
    bounds = _bounds([_packing(S, s, 16) for s in range(B)], S)
    qkv = torch.randn(B * S, (H + 2 * Hkv) * HD, device=dev()).to(torch.bfloat16)
    dout = torch.randn(B * S, H * HD, device=dev()).to(torch.bfloat16)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        o, lse = C().causal_gqa_attention_fwd(qkv, bounds, H, Hkv)
        C().causal_gqa_attention_bwd(dout, qkv, o, lse, bounds, H, Hkv)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        o_g, lse_g = C().causal_gqa_attention_fwd(qkv, bounds, H, Hkv)
        d_g = C().causal_gqa_attention_bwd(dout, qkv, o_g, lse_g, bounds, H, Hkv)
    for layout in ([[512], [1] * 100, []], [_packing(S, 40 + r, 8) for r in range(B)]):
        bounds.copy_(_bounds(layout, S))
        graph.replay()
        o, lse = C().causal_gqa_attention_fwd(qkv, bounds, H, Hkv)
        d = C().causal_gqa_attention_bwd(dout, qkv, o, lse, bounds, H, Hkv)
        torch.cuda.synchronize()
        assert torch.equal(o_g, o) and torch.equal(lse_g, lse) and torch.equal(d_g, d), layout


def test_gqa_op_rejects_bad_input_and_matches_its_cpu_body():
    bounds = _bounds([[100], [28, 100]], 128)
    with pytest.raises(ValueError):
        Fn.causal_attention(torch.randn(2, 128, 7 * 64, device=dev()).to(torch.bfloat16), bounds, 4, 2)   # wrong width
    with pytest.raises(ValueError):
        Fn.causal_attention(torch.randn(2, 128, 8 * 64, device=dev()), bounds, 4, 2)                       # not bf16
    torch.manual_seed(0)
    qkv = torch.randn(2, 128, 8 * 64).to(torch.bfloat16)
    dy = torch.randn(2, 128, 4 * 64).to(torch.bfloat16)
    xc = qkv.clone().requires_grad_(True)
    yc = Fn.causal_attention(xc, bounds.cpu(), 4, 2)
    yc.backward(dy)
    xg = qkv.to(dev()).requires_grad_(True)
    yg = Fn.causal_attention(xg, bounds, 4, 2)
    yg.backward(dy.to(dev()))
    assert torch.allclose(yg.float().cpu(), yc.float(), rtol=2e-2, atol=2e-2)
    assert torch.allclose(xg.grad.float().cpu(), xc.grad.float(), rtol=5e-2, atol=5e-2)


def test_rotary_rms_norm_and_swiglu_match_fp64():
    torch.manual_seed(3)
    H, Hkv, B, S = 9, 3, 2, 2048
    qkv = torch.randn(B, S, (H + 2 * Hkv) * HD, device=dev()).to(torch.bfloat16)
    pos = torch.stack([torch.arange(S), torch.arange(S) % 300]).to(dev())
    table = Fn.rotary_cos_sin(2048)
    y = Fn.rotary(qkv, pos, table, H, Hkv)
    ref = Fn._rotary_reference(qkv.double().cpu(), pos.cpu(), Fn.rotary_cos_sin(2048).double(), H, Hkv)
    assert (y.double().cpu() - ref).abs().max() <= 2 ** -7 * ref.abs().max()
    dy = torch.randn_like(y)
    dx = C().rotary(dy.view(B * S, -1), pos.reshape(-1).int(), table.to(dev()), H, Hkv, True).view(B, S, -1)
    dref = Fn._rotary_reference(dy.double().cpu(), pos.cpu(), Fn.rotary_cos_sin(2048).double(), H, Hkv, inverse=True)
    assert (dx.double().cpu() - dref).abs().max() <= 2 ** -7 * dref.abs().max()
    # RMSNorm: output, dx, and a dgamma that is the same on every run
    x = torch.randn(4096, 576, device=dev()).to(torch.bfloat16)
    w = (torch.rand(576, device=dev()) + 0.5).to(torch.bfloat16)
    g = torch.randn_like(x)
    xa, wa = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    ya = Fn.rms_norm(xa, wa, 1e-5)
    ya.backward(g)
    x64, w64 = x.double().requires_grad_(True), w.double().requires_grad_(True)
    r64 = x64 * torch.rsqrt(x64.pow(2).mean(-1, keepdim=True) + 1e-5) * w64
    r64.backward(g.double())
    assert _rms(ya.double() - r64.detach()) < 1e-2 * _rms(r64.detach())
    assert _rms(xa.grad.double() - x64.grad) < 2e-2 * _rms(x64.grad)
    assert _rms(wa.grad.double() - w64.grad) < 2e-2 * _rms(w64.grad)
    dws = [torch.autograd.grad(Fn.rms_norm(x, wb, 1e-5), wb, g)[0] for wb in (w.clone().requires_grad_(True) for _ in range(2))]
    assert torch.equal(dws[0], dws[1])
    # SwiGLU
    gu = (torch.randn(4096, 2 * 1536, device=dev()) * 2).to(torch.bfloat16).requires_grad_(True)
    s = Fn.swiglu(gu)
    ds = torch.randn_like(s)
    s.backward(ds)
    g64 = gu.detach().double().requires_grad_(True)
    a, b = g64.chunk(2, -1)
    s64 = F.silu(a) * b
    s64.backward(ds.double())
    assert _rms(s.double() - s64.detach()) < 1e-2 * _rms(s64.detach())
    assert _rms(gu.grad.double() - g64.grad) < 1e-2 * _rms(g64.grad)


def _tiny_cfg(**kw):
    from b200ddp.models.llama import LlamaConfig
    return LlamaConfig(vocab_size=1024, max_position=256, hidden=192, layers=2, heads=3, kv_heads=1, intermediate=256, **kw)


def _batch(rows, S, seed, bos=1):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(2, 1024, (len(rows), S), generator=g)
    labels = torch.full(ids.shape, -100)
    for r, docs in enumerate(rows):
        at = 0
        for n in docs:
            ids[r, at] = bos
            labels[r, at:at + n - 1] = ids[r, at + 1:at + n]
            at += n
        ids[r, at:] = 0
    return ids, labels


@pytest.mark.parametrize("mode", ["fixed", "padded", "packed"])
def test_llama_tiny_gpu_matches_cpu_body(mode):
    from b200ddp.models.llama import LlamaForCausalLM
    from b200ddp.ops import cross_entropy
    kw = {"fixed": {}, "padded": {"pad_token_id": 0}, "packed": {"pad_token_id": 0, "bos_token_id": 1}}[mode]
    torch.manual_seed(7)
    ref = LlamaForCausalLM(_tiny_cfg(**kw))
    gpu = LlamaForCausalLM(_tiny_cfg(**kw))
    gpu.load_state_dict(ref.state_dict())
    gpu = gpu.to(dev(), torch.bfloat16)
    rows = {"fixed": [[128]] * 3, "padded": [[128], [100], [1]], "packed": [[40, 1, 57, 30], [128], []]}[mode]
    ids, labels = _batch(rows, 128, seed=1)
    if mode == "fixed":
        ids[ids == 0] = 5
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


def test_llama_step_has_no_host_synchronisation():
    from b200ddp.models.llama import LlamaForCausalLM
    from b200ddp.ops import cross_entropy
    torch.manual_seed(1)
    model = LlamaForCausalLM(_tiny_cfg(pad_token_id=0, bos_token_id=1)).to(dev(), torch.bfloat16)
    ids, labels = _batch([[100, 28], [1, 1, 126], [50]], 128, seed=2)
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


@pytest.mark.parametrize("pack,fp8", [(False, False), (True, False), (False, True), (True, True)])
def test_smollm_graph_training_lowers_the_loss(tmp_path, pack, fp8):
    """What `python ddp.py --model smollm-135m --fp16 --optimizer adamw --cuda_graph --max_steps 30 --seq_len 256
    --min_seq_len 32 [--pack] [--fp8]` runs."""
    from b200ddp.data import SyntheticTokens
    from b200ddp.engine import cli
    from b200ddp.engine.trainer import Trainer, build_dataset
    from b200ddp.models import build_model
    argv = ["--model", "smollm-135m", "--fp16", "--optimizer", "adamw", "--cuda_graph", "--max_steps", "30", "--seq_len",
            "256", "--min_seq_len", "32", "--per_gpu_train_batch_size", "8", "--lr", "5e-4", "--warmup_steps", "5",
            "--weight_decay", "0.01", "--save_steps", "0", "--logging_steps", "10", "--no_tensorboard",
            "--output_dir", str(tmp_path / "out")] + (["--pack"] if pack else []) + (["--fp8"] if fp8 else [])
    args = cli.build_parser().parse_args(argv)
    cli.setup(args)
    kwargs = {"pad_token_id": 0, **({"bos_token_id": 1} if pack else {}), **({"fp8": True} if fp8 else {})}
    model = build_model("smollm-135m", **kwargs)
    ds = build_dataset(args)
    assert isinstance(ds, SyntheticTokens) and ds.bos_token_id == (1 if pack else None)
    ds.X = torch.where(ds.X > 1, ds.X % 64 + 2, ds.X)
    ds.Y = torch.where(ds.Y > 1, ds.Y % 64 + 2, ds.Y)
    trainer = Trainer(args, model, cli.log, dataset=ds)
    before = trainer.evaluate(max_batches=4)["eval_loss"]
    trainer.train()
    after = trainer.evaluate(max_batches=4)["eval_loss"]
    assert trainer.step_fn.graph is not None
    assert math.isfinite(after) and after < before - 0.05, (before, after)
