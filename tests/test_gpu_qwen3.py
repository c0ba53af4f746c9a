"""Qwen3-0.6B on the GPU: the fused per-head q / k RMSNorm + rotary op against fp64 beside Hugging Face's bf16 expression,
its gradients against fp64 autograd, value heads copied bitwise, deterministic weight gradients, CUDA-graph replay with
new positions, rejected input, a tiny Qwen3-shaped model against its CPU body, a training step without host
synchronisation and one AdamW step of the full preset with the fused LM-head loss."""
import math

import pytest
import torch

from b200ddp.ops import functional as Fn

pytestmark = pytest.mark.gpu
HD = 128
BOS = 1


def dev():
    return torch.device("cuda", 0)


def C():
    from b200ddp import _ext
    return _ext.get()


def _fp64_table(max_pos, theta=1e6):
    inv = theta ** (-torch.arange(0, HD, 2, dtype=torch.float64) / HD)
    ang = torch.arange(max_pos, dtype=torch.float64)[:, None] * inv[None, :]
    return torch.stack([ang.cos(), ang.sin()], 1)


def _positions(layout, B, S, seed):
    """position ids of document_bounds for fixed-length rows, right-padded rows or packed documents"""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(2, 1000, (B, S), generator=g)
    if layout == "right_padded":
        for r in range(B):
            ids[r, int(torch.randint(1, S + 1, (1,), generator=g)):] = 0
        return Fn.document_bounds(ids.to(dev()), None, 0)[1]
    if layout == "packed":
        for r in range(B):
            at = 0
            while at < S:
                ids[r, at] = BOS
                at += int(torch.randint(1, S // 2 + 1, (1,), generator=g))
        ids[:, -S // 8:] = 0
        return Fn.document_bounds(ids.to(dev()), BOS, 0)[1]
    return Fn.document_bounds(ids.to(dev()), None, None)[1]


def _inputs(rows, H, Hkv, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    qkv = (torch.randn(rows, (H + 2 * Hkv) * HD, device=dev(), generator=g) * 2).to(torch.bfloat16)
    wq = (torch.rand(HD, device=dev(), generator=g) + 0.5).to(torch.bfloat16)
    wk = (torch.rand(HD, device=dev(), generator=g) + 0.5).to(torch.bfloat16)
    dy = torch.randn(rows, (H + 2 * Hkv) * HD, device=dev(), generator=g).to(torch.bfloat16)
    return qkv, wq, wk, dy


def _hf_bf16(qkv, wq, wk, pos, table, H, Hkv, eps):
    """Hugging Face's Qwen3Attention in bf16: Qwen3RMSNorm (fp32 statistics, rounded to bf16, times the bf16 weight), then
    apply_rotary_pos_emb with bf16 cos / sin"""
    B, S, _ = qkv.shape
    x = qkv.view(B, S, -1, HD)

    def norm(t, w):
        tf = t.float()
        return w * (tf * torch.rsqrt(tf.pow(2).mean(-1, keepdim=True) + eps)).to(torch.bfloat16)
    cs = table[pos.long()]
    cos = torch.cat([cs[:, :, 0]] * 2, -1)[:, :, None].to(torch.bfloat16)
    sin = torch.cat([cs[:, :, 1]] * 2, -1)[:, :, None].to(torch.bfloat16)

    def rope(t):
        return t * cos + torch.cat([-t[..., HD // 2:], t[..., :HD // 2]], -1) * sin
    q, k, v = x[:, :, :H], x[:, :, H:H + Hkv], x[:, :, H + Hkv:]
    return torch.cat([rope(norm(q, wq)), rope(norm(k, wk)), v], 2).reshape(B, S, -1)


def _ulp(t):
    return 2.0 ** (math.floor(math.log2(float(t.abs().max()))) - 7)


@pytest.mark.parametrize("layout", ["full", "right_padded", "packed"])
@pytest.mark.parametrize("rows", [128, 16384])
@pytest.mark.parametrize("H,Hkv", [(16, 8), (12, 2), (4, 1)])
def test_qk_norm_rotary_matches_fp64_at_least_as_well_as_hugging_face_bf16(layout, rows, H, Hkv):
    B = 2 if rows == 128 else 8
    S, eps = rows // B, 1e-6
    qkv, wq, wk, dy = _inputs(rows, H, Hkv, rows + H + Hkv)
    pos = _positions(layout, B, S, seed=H)
    table = Fn.rotary_cos_sin(S, HD, 1e6).to(dev())
    ins = [t.clone().requires_grad_(True) for t in (qkv.view(B, S, -1), wq, wk)]
    y = Fn.qk_norm_rotary(*ins, pos, table, H, Hkv, eps)
    y.backward(dy.view(B, S, -1))
    ref_in = [t.double().requires_grad_(True) for t in (qkv.view(B, S, -1), wq, wk)]
    ref = Fn._qk_norm_rotary_reference(*ref_in, pos, _fp64_table(S).to(dev()), H, Hkv, eps)
    ref.backward(dy.view(B, S, -1).double())
    ref = ref.detach()
    W = (H + Hkv) * HD
    assert torch.equal(y[..., W:], qkv.view(B, S, -1)[..., W:])                      # value heads copied
    assert torch.equal(ins[0].grad[..., W:], dy.view(B, S, -1)[..., W:])              # and their gradient passes through
    hf = _hf_bf16(qkv.view(B, S, -1), wq, wk, pos, table, H, Hkv, eps)
    err, hf_err = float((y.detach().double() - ref).abs().max()), float((hf.double() - ref).abs().max())
    assert err <= hf_err + _ulp(ref), (err, hf_err)
    dx, dx_ref = ins[0].grad.double(), ref_in[0].grad
    assert float((dx - dx_ref).pow(2).mean().sqrt()) <= 5e-3 * float(dx_ref.pow(2).mean().sqrt())
    assert float((dx - dx_ref).abs().max()) <= 2 * _ulp(dx_ref)
    for name, a, b in (("dw_q", ins[1], ref_in[1]), ("dw_k", ins[2], ref_in[2])):
        assert float((a.grad.double() - b.grad).abs().max()) <= 2 ** -7 * float(b.grad.abs().max()), name


def test_qk_norm_rotary_backward_is_bitwise_deterministic():
    H, Hkv, rows = 16, 8, 16384
    qkv, wq, wk, dy = _inputs(rows, H, Hkv, 3)
    pos = _positions("packed", 8, rows // 8, 4).reshape(-1).int()
    table = Fn.rotary_cos_sin(4096, HD, 1e6).to(dev())
    y, rstd = C().qk_norm_rotary_fwd(qkv, wq, wk, pos, table, H, Hkv, 1e-6)
    y2, rstd2 = C().qk_norm_rotary_fwd(qkv, wq, wk, pos, table, H, Hkv, 1e-6)
    assert torch.equal(y, y2) and torch.equal(rstd, rstd2) and rstd.shape == (rows, H + Hkv)
    runs = [C().qk_norm_rotary_bwd(dy, qkv, rstd, wq, wk, pos, table, H, Hkv) for _ in range(2)]
    for a, b in zip(*runs):
        assert torch.equal(a, b)


def test_qk_norm_rotary_graph_replay_with_new_positions_matches_eager():
    B, S, H, Hkv = 4, 512, 16, 8
    qkv, wq, wk, dy = _inputs(B * S, H, Hkv, 6)
    qkv, dy = qkv.view(B, S, -1).clone().requires_grad_(True), dy.view(B, S, -1)
    wq, wk = wq.requires_grad_(True), wk.requires_grad_(True)
    pos = _positions("packed", B, S, 1).int()
    table = Fn.rotary_cos_sin(S, HD, 1e6).to(dev())

    def step():
        y = Fn.qk_norm_rotary(qkv, wq, wk, pos, table, H, Hkv, 1e-6)
        return (y, *torch.autograd.grad(y, (qkv, wq, wk), dy))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = step()
    for layout, seed in (("full", 2), ("right_padded", 3), ("packed", 4)):
        pos.copy_(_positions(layout, B, S, seed))
        graph.replay()
        eager = step()
        torch.cuda.synchronize()
        assert all(torch.equal(a, b) for a, b in zip(outs, eager)), layout


def test_qk_norm_rotary_rejects_bad_input():
    B, S, H, Hkv = 2, 64, 4, 2
    pos = torch.zeros(B, S, dtype=torch.int32, device=dev())
    table = Fn.rotary_cos_sin(S, HD, 1e6).to(dev())
    w = torch.ones(HD, device=dev(), dtype=torch.bfloat16)
    qkv = torch.randn(B, S, (H + 2 * Hkv) * HD, device=dev()).to(torch.bfloat16)
    with pytest.raises(ValueError):
        Fn.qk_norm_rotary(qkv.float(), w, w, pos, table, H, Hkv)                      # not bf16
    with pytest.raises(ValueError):                                                    # head dim 64
        Fn.qk_norm_rotary(qkv[..., :(H + 2 * Hkv) * 64].contiguous(), w[:64], w[:64], pos, Fn.rotary_cos_sin(S, 64).to(dev()), H, Hkv)
    buf = torch.empty(qkv.numel() + 1, device=dev(), dtype=torch.bfloat16)
    with pytest.raises(ValueError):                                                    # 2-byte aligned
        Fn.qk_norm_rotary(buf[1:].view_as(qkv), w, w, pos, table, H, Hkv)
    with pytest.raises(ValueError):
        Fn.qk_norm_rotary(qkv, torch.ones(2 * HD, device=dev(), dtype=torch.bfloat16), w, pos, table, H, Hkv)   # weight shape
    with pytest.raises(ValueError):
        Fn.qk_norm_rotary(qkv, w.float(), w, pos, table, H, Hkv)                      # weight dtype
    with pytest.raises(ValueError):
        Fn.qk_norm_rotary(qkv, w.cpu(), w, pos, table, H, Hkv)                        # weight device
    with pytest.raises(RuntimeError, match="eps"):
        C().qk_norm_rotary_fwd(qkv.view(B * S, -1), w, w, pos.view(-1), table, H, Hkv, 0.0)


def _tiny_cfg(**kw):
    from b200ddp.models.llama import LlamaConfig
    return LlamaConfig(vocab_size=1024, max_position=256, hidden=256, layers=2, heads=4, kv_heads=2, intermediate=384, eps=1e-6,
                       rope_theta=1e6, explicit_head_dim=128, qk_norm=True, **kw)


def _batch(rows, S, seed):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(2, 1024, (len(rows), S), generator=g)
    labels = torch.full(ids.shape, -100)
    for r, docs in enumerate(rows):
        at = 0
        for n in docs:
            ids[r, at] = BOS
            labels[r, at:at + n - 1] = ids[r, at + 1:at + n]
            at += n
        ids[r, at:] = 0
    return ids, labels


@pytest.mark.parametrize("mode", ["fixed", "padded", "packed"])
def test_qwen3_tiny_gpu_matches_cpu_body(mode):
    from b200ddp.models.llama import LlamaForCausalLM
    from b200ddp.ops import cross_entropy
    kw = {"fixed": {}, "padded": {"pad_token_id": 0}, "packed": {"pad_token_id": 0, "bos_token_id": BOS}}[mode]
    torch.manual_seed(7)
    ref = LlamaForCausalLM(_tiny_cfg(**kw))
    with torch.no_grad():
        for layer in ref.model.layers:
            layer.q_norm.weight.uniform_(0.5, 1.5)
            layer.k_norm.weight.uniform_(0.5, 1.5)
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


def test_qwen3_step_has_no_host_synchronisation():
    from b200ddp.models.llama import LlamaForCausalLM
    from b200ddp.ops import cross_entropy
    torch.manual_seed(1)
    model = LlamaForCausalLM(_tiny_cfg(pad_token_id=0, bos_token_id=BOS)).to(dev(), torch.bfloat16)
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
    assert all(layer.q_norm.weight.grad is not None and layer.k_norm.weight.grad is not None for layer in model.model.layers)


def test_qwen3_0_6b_full_preset_adamw_step_with_fused_lm_loss(capsys):
    from b200ddp.models import build_model
    from b200ddp.optim import FusedAdamW, weight_decay_groups
    torch.manual_seed(0)
    model = build_model("qwen3-0.6b", fused_lm_loss=True).to(dev(), torch.bfloat16)
    opt = FusedAdamW(weight_decay_groups(model, 0.01), lr=1e-4, max_grad_norm=1.0)
    crit = model.lm_head_loss()
    ids = torch.randint(1, 151936, (8, 2048), device=dev())
    torch.cuda.reset_peak_memory_stats()
    loss = crit(model(ids), torch.roll(ids, -1, 1))
    loss.backward()
    norm_grads = [layer.k_norm.weight.grad.float().clone() for layer in model.model.layers]
    opt.step()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    with capsys.disabled():
        print(f"\nqwen3-0.6b batch 8 x 2048, fused LM-head loss, on {torch.cuda.get_device_name(dev())}: loss {float(loss):.4f}, "
              f"peak memory {peak:.1f} GiB")
    assert math.isfinite(float(loss)) and abs(float(loss) - math.log(151936)) < 1.0
    assert all(bool(torch.isfinite(g).all()) and float(g.abs().max()) > 0 for g in norm_grads)
    assert all(bool(torch.isfinite(p.float()).all()) for p in model.parameters())
