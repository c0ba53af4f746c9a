"""Qwen2.5-1.5B kernels on the GPU: head-dim-128 causal attention (grouped-query and multi-head) against fp64 beside
SDPA's own bf16 error, padding rows, determinism, writes confined to the outputs, CUDA-graph replay with a new packing,
rejected input, rotary at d = 128 with theta 1e6 up to position 32767, wide RMSNorm, a tiny Qwen-shaped model against its
CPU body, a training step without host synchronisation, CUDA-graph AdamW training and one step of the full preset."""
import math

import pytest
import torch
import torch.nn.functional as F

from b200ddp.ops import functional as Fn

pytestmark = pytest.mark.gpu
HD = 128


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
    s = ((q @ k.transpose(-1, -2)) / math.sqrt(HD)).masked_fill(~keep, -math.inf)
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


def _inputs(B, S, H, Hkv, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    qkv = torch.randn(B * S, (H + 2 * Hkv) * HD, device=dev(), generator=g).to(torch.bfloat16)
    dout = torch.randn(B * S, H * HD, device=dev(), generator=g).to(torch.bfloat16)
    return qkv, dout


LAYOUTS = {
    "full": lambda S: [[S], [S]],
    "right_padded": lambda S: [[S // 2 + 3], [S - 1], [1]],
    "packed": lambda S: [_packing(S, 3, 16), _packing(S, 5), _packing(S, 8, S // 8)],
}


@pytest.mark.parametrize("layout", sorted(LAYOUTS))
@pytest.mark.parametrize("S", [128, 512, 2048, 4096])
@pytest.mark.parametrize("H,Hkv", [(12, 2), (8, 8), (4, 1), (6, 3)])
def test_d128_attention_is_as_accurate_as_sdpa(layout, S, H, Hkv):
    if S == 4096 and (H, Hkv) != (12, 2):
        pytest.skip("the Qwen2.5 head layout alone at 4096 keeps the fp64 reference affordable")
    docs = LAYOUTS[layout](S)
    B = len(docs)
    bounds = _bounds(docs, S)
    qkv, dout = _inputs(B, S, H, Hkv, S + H + Hkv)
    o, lse = C().causal_attention_d128_fwd(qkv, bounds, H, Hkv)
    dqkv = C().causal_attention_d128_bwd(dout, qkv, o, lse, bounds, H, Hkv)
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


def test_d128_all_padding_row_gives_zeros_and_empty_lse():
    S, H, Hkv = 256, 12, 2
    bounds = _bounds([[], [70, 30], [S]], S)
    qkv, dout = _inputs(3, S, H, Hkv, 11)
    o, lse = C().causal_attention_d128_fwd(qkv, bounds, H, Hkv)
    dqkv = C().causal_attention_d128_bwd(dout, qkv, o, lse, bounds, H, Hkv)
    assert (o.view(3, S, -1)[0] == 0).all() and (dqkv.view(3, S, -1)[0] == 0).all()
    assert torch.isneginf(lse[0]).all() and torch.isfinite(lse[1:, :, :100]).all() and torch.isneginf(lse[1, :, 100:]).all()
    assert (dqkv.view(3, S, -1)[1, 100:] == 0).all()


def test_d128_gradients_are_bitwise_deterministic():
    S, H, Hkv = 1024, 12, 2
    bounds = _bounds([_packing(S, s, 8) for s in range(3)] + [[S]], S)
    qkv, dout = _inputs(4, S, H, Hkv, 2)
    runs = []
    for _ in range(2):
        o, lse = C().causal_attention_d128_fwd(qkv, bounds, H, Hkv)
        runs.append((o, lse, C().causal_attention_d128_bwd(dout, qkv, o, lse, bounds, H, Hkv)))
    for a, b in zip(*runs):
        assert torch.equal(a, b)


def test_d128_writes_stay_inside_the_outputs():
    B, S, H, Hkv, pad = 2, 384, 6, 3, 64
    bounds = _bounds([_packing(S, 1, 8), [S - 5]], S)
    qkv, dout = _inputs(B, S, H, Hkv, 4)
    rows = B * S

    def framed(cols, dtype):
        buf = torch.full((rows + 2 * pad, cols), -7.0, device=dev(), dtype=dtype)
        return buf, buf[pad:pad + rows]

    o_buf, o = framed(H * HD, torch.bfloat16)
    lse_buf = torch.full((B * H * S + 2 * 256,), -7.0, device=dev())
    lse = lse_buf[256:256 + B * H * S]
    C().causal_attention_d128_fwd(qkv, bounds, H, Hkv, o=o, lse=lse)
    d_buf, dqkv = framed((H + 2 * Hkv) * HD, torch.bfloat16)
    C().causal_attention_d128_bwd(dout, qkv, o, lse.view(B, H, S), bounds, H, Hkv, dqkv=dqkv)
    torch.cuda.synchronize()
    for buf in (o_buf, d_buf):
        assert (buf[:pad] == -7.0).all() and (buf[pad + rows:] == -7.0).all()
    assert (lse_buf[:256] == -7.0).all() and (lse_buf[256 + B * H * S:] == -7.0).all()
    o_ref, lse_ref = C().causal_attention_d128_fwd(qkv, bounds, H, Hkv)
    assert torch.equal(o, o_ref) and torch.equal(lse.view(B, H, S), lse_ref)
    assert torch.equal(dqkv, C().causal_attention_d128_bwd(dout, qkv, o_ref, lse_ref, bounds, H, Hkv))


def test_d128_graph_replay_with_a_new_packing_matches_eager():
    B, S, H, Hkv = 3, 512, 12, 2
    bounds = _bounds([_packing(S, s, 16) for s in range(B)], S)
    qkv, dout = _inputs(B, S, H, Hkv, 6)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        o, lse = C().causal_attention_d128_fwd(qkv, bounds, H, Hkv)
        C().causal_attention_d128_bwd(dout, qkv, o, lse, bounds, H, Hkv)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        o_g, lse_g = C().causal_attention_d128_fwd(qkv, bounds, H, Hkv)
        d_g = C().causal_attention_d128_bwd(dout, qkv, o_g, lse_g, bounds, H, Hkv)
    for layout in ([[512], [1] * 100, []], [_packing(S, 40 + r, 8) for r in range(B)]):
        bounds.copy_(_bounds(layout, S))
        graph.replay()
        o, lse = C().causal_attention_d128_fwd(qkv, bounds, H, Hkv)
        d = C().causal_attention_d128_bwd(dout, qkv, o, lse, bounds, H, Hkv)
        torch.cuda.synchronize()
        assert torch.equal(o_g, o) and torch.equal(lse_g, lse) and torch.equal(d_g, d), layout


def test_d128_op_routes_multi_head_and_gqa_and_rejects_bad_input():
    bounds = _bounds([[100], [28, 100]], 128)
    bf = lambda *s: torch.randn(*s, device=dev()).to(torch.bfloat16)   # noqa: E731
    with pytest.raises(ValueError):
        Fn.causal_attention(bf(2, 128, 16 * 128 + 64), bounds, 12, 2)            # head dim neither 64 nor 128
    with pytest.raises(ValueError):
        Fn.causal_attention(torch.randn(2, 128, 16 * 128, device=dev()), bounds, 12, 2)   # not bf16
    with pytest.raises(ValueError):
        Fn.causal_attention(bf(2, 192, 16 * 128), _bounds([[1], [1]], 192), 12, 2)   # S not a multiple of 128
    with pytest.raises(ValueError):
        Fn.causal_attention(bf(2, 128, 32 * 128)[..., :16 * 128], bounds, 12, 2)   # not contiguous
    with pytest.raises(ValueError):
        Fn.causal_attention(bf(2, 128, 21 * 128), bounds, 9, 6)                  # kv_heads does not divide heads
    with pytest.raises(ValueError):
        Fn.causal_attention(bf(2, 128, 16 * 128), bounds[:, :64], 12, 2)        # bounds not [B, S, 2]
    with pytest.raises(ValueError):
        Fn.attention(bf(2, 128, 3 * 256), torch.tensor([5, 128], device=dev()), 2)   # key padding stays d = 64
    with pytest.raises(ValueError):
        Fn.packed_attention(bf(2, 128, 3 * 256), bounds, 2)                      # so does the segment mode
    # multi-head (kv_heads None or == heads) and GQA all reach the d = 128 kernels and match their CPU body
    for heads, kv in ((2, None), (2, 2), (4, 2)):
        torch.manual_seed(heads)
        width = (heads + 2 * (kv or heads)) * HD
        qkv = torch.randn(2, 128, width).to(torch.bfloat16)
        dy = torch.randn(2, 128, heads * HD).to(torch.bfloat16)
        xc = qkv.clone().requires_grad_(True)
        Fn.causal_attention(xc, bounds.cpu(), heads, kv).backward(dy)
        yc = Fn.causal_attention(xc.detach(), bounds.cpu(), heads, kv)
        xg = qkv.to(dev()).requires_grad_(True)
        yg = Fn.causal_attention(xg, bounds, heads, kv)
        yg.backward(dy.to(dev()))
        assert yg.shape == (2, 128, heads * HD)
        assert torch.allclose(yg.float().cpu(), yc.float(), rtol=2e-2, atol=2e-2)
        assert torch.allclose(xg.grad.float().cpu(), xc.grad.float(), rtol=5e-2, atol=5e-2)


def _fp64_table(max_pos, d, theta):
    inv = theta ** (-torch.arange(0, d, 2, dtype=torch.float64) / d)
    ang = torch.arange(max_pos, dtype=torch.float64)[:, None] * inv[None, :]
    return torch.stack([ang.cos(), ang.sin()], 1)


def test_rotary_d128_matches_fp64_at_long_positions():
    torch.manual_seed(5)
    H, Hkv, B, S, P = 12, 2, 2, 2048, 32768
    qkv = torch.randn(B, S, (H + 2 * Hkv) * HD, device=dev()).to(torch.bfloat16)
    pos = torch.stack([torch.arange(P - S, P), torch.randint(0, P, (S,))]).to(dev())
    pos[1, :3] = torch.tensor([0, 1, P - 1])
    table = Fn.rotary_cos_sin(P, HD, 1e6)
    assert table.shape == (P, 2, 64)
    ref_table = _fp64_table(P, HD, 1e6)
    y = Fn.rotary(qkv, pos, table, H, Hkv)
    ref = Fn._rotary_reference(qkv.double().cpu(), pos.cpu(), ref_table, H, Hkv)
    assert (y.double().cpu() - ref).abs().max() <= 2 ** -7 * ref.abs().max()
    assert torch.equal(y[..., (H + Hkv) * HD:], qkv[..., (H + Hkv) * HD:])        # value heads copied
    dy = torch.randn_like(y)
    dx = C().rotary(dy.view(B * S, -1), pos.reshape(-1).int(), table.to(dev()), H, Hkv, True).view(B, S, -1)
    dref = Fn._rotary_reference(dy.double().cpu(), pos.cpu(), ref_table, H, Hkv, inverse=True)
    assert (dx.double().cpu() - dref).abs().max() <= 2 ** -7 * dref.abs().max()
    with pytest.raises(ValueError):
        Fn.rotary(torch.randn(B, S, 16 * 96, device=dev()).to(torch.bfloat16), pos, Fn.rotary_cos_sin(64, 96), H, Hkv)


@pytest.mark.parametrize("hidden,dtype", [(1536, torch.bfloat16), (2048, torch.bfloat16), (3072, torch.bfloat16),
                                          (4096, torch.bfloat16), (3072, torch.float32), (1032, torch.bfloat16)])
def test_wide_rms_norm_matches_fp64_with_deterministic_dgamma(hidden, dtype):
    torch.manual_seed(hidden)
    x = torch.randn(4096, hidden, device=dev()).to(dtype)
    w = (torch.rand(hidden, device=dev()) + 0.5).to(dtype)
    g = torch.randn_like(x)
    xa, wa = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    ya = Fn.rms_norm(xa, wa, 1e-6)
    ya.backward(g)
    x64, w64 = x.double().requires_grad_(True), w.double().requires_grad_(True)
    r64 = x64 * torch.rsqrt(x64.pow(2).mean(-1, keepdim=True) + 1e-6) * w64
    r64.backward(g.double())
    tol = 1e-2 if dtype == torch.bfloat16 else 1e-5
    assert _rms(ya.double() - r64.detach()) < tol * _rms(r64.detach())
    assert _rms(xa.grad.double() - x64.grad) < 2 * tol * _rms(x64.grad)
    assert _rms(wa.grad.double() - w64.grad) < 2 * tol * _rms(w64.grad)
    dws = [torch.autograd.grad(Fn.rms_norm(x, wb, 1e-6), wb, g)[0] for wb in (w.clone().requires_grad_(True) for _ in range(2))]
    assert torch.equal(dws[0], dws[1])


def test_rms_norm_still_rejects_rows_wider_than_4096():
    with pytest.raises(ValueError):
        Fn.rms_norm(torch.randn(4, 4104, device=dev()), torch.ones(4104, device=dev()))


def _tiny_cfg(**kw):
    from b200ddp.models.llama import LlamaConfig
    return LlamaConfig(vocab_size=1024, max_position=256, hidden=256, layers=2, heads=2, kv_heads=1, intermediate=384, eps=1e-6,
                       rope_theta=1e6, attention_bias=True, **kw)


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
def test_qwen_tiny_gpu_matches_cpu_body(mode):
    from b200ddp.models.llama import LlamaForCausalLM
    from b200ddp.ops import cross_entropy
    kw = {"fixed": {}, "padded": {"pad_token_id": 0}, "packed": {"pad_token_id": 0, "bos_token_id": 1}}[mode]
    torch.manual_seed(7)
    ref = LlamaForCausalLM(_tiny_cfg(**kw))
    with torch.no_grad():
        for layer in ref.model.layers:
            layer.qkv.bias.normal_(std=0.5)
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


def test_qwen_step_has_no_host_synchronisation():
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
def test_qwen_graph_training_lowers_the_loss(tmp_path, pack, fp8):
    """What `python ddp.py --model qwen2.5-1.5b --fp16 --optimizer adamw --cuda_graph --max_steps 30 --seq_len 256
    --min_seq_len 32 [--pack] [--fp8]` runs, on a two-layer Qwen-shaped model (head dim 128, q / k / v bias)."""
    from b200ddp.data import SyntheticTokens
    from b200ddp.engine import cli
    from b200ddp.engine.trainer import Trainer, build_dataset
    from b200ddp.models.llama import LlamaForCausalLM
    argv = ["--model", "qwen2.5-1.5b", "--fp16", "--optimizer", "adamw", "--cuda_graph", "--max_steps", "30", "--seq_len",
            "256", "--min_seq_len", "32", "--per_gpu_train_batch_size", "8", "--lr", "5e-4", "--warmup_steps", "5",
            "--weight_decay", "0.01", "--save_steps", "0", "--logging_steps", "10", "--no_tensorboard",
            "--output_dir", str(tmp_path / "out")] + (["--pack"] if pack else []) + (["--fp8"] if fp8 else [])
    args = cli.build_parser().parse_args(argv)
    cli.setup(args)
    ds = build_dataset(args)
    assert isinstance(ds, SyntheticTokens) and ds.bos_token_id == (SyntheticTokens.QWEN_BOS_ID if pack else None)
    # a small alphabet leaves something to learn; the start id maps to the small model's 1
    ds.X = torch.where(ds.X == SyntheticTokens.QWEN_BOS_ID, torch.ones_like(ds.X), torch.where(ds.X > 0, ds.X % 64 + 2, ds.X))
    ds.Y = torch.where(ds.Y > 0, ds.Y % 64 + 2, ds.Y)
    if pack:
        ds.bos_token_id = 1
    model = LlamaForCausalLM(_tiny_cfg(pad_token_id=0, fp8=fp8, **({"bos_token_id": 1} if pack else {})))
    trainer = Trainer(args, model, cli.log, dataset=ds)
    before = trainer.evaluate(max_batches=4)["eval_loss"]
    trainer.train()
    after = trainer.evaluate(max_batches=4)["eval_loss"]
    assert trainer.step_fn.graph is not None
    assert math.isfinite(after) and after < before - 0.05, (before, after)


def test_qwen2_5_1_5b_full_preset_step(capsys):
    from b200ddp.models import build_model
    from b200ddp.ops import cross_entropy
    from b200ddp.optim import FusedAdamW, weight_decay_groups
    torch.manual_seed(0)
    torch.cuda.reset_peak_memory_stats()
    model = build_model("qwen2.5-1.5b").to(dev(), torch.bfloat16)
    opt = FusedAdamW(weight_decay_groups(model, 0.01), lr=1e-4, max_grad_norm=1.0)
    ids = torch.randint(1, 151936, (1, 2048), device=dev())
    loss = cross_entropy(model(ids), torch.roll(ids, -1, 1))
    loss.backward()
    opt.step()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    with capsys.disabled():
        print(f"\nqwen2.5-1.5b batch 1 x 2048 on {torch.cuda.get_device_name(dev())}: loss {float(loss):.4f}, "
              f"peak memory {peak:.1f} GiB")
    assert math.isfinite(float(loss)) and abs(float(loss) - math.log(151936)) < 1.0
