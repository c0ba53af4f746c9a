"""Mixture of experts on the H100: routing, the expert sort, the grouped wgmma GEMMs (forward, data and weight gradient) on
skewed routing, the MoE layer against fp32, determinism, a training step without host synchronisation, CUDA-graph replay
with new routing, a tiny Granite-shaped model against its CPU body, and an AdamW step of the full preset."""
import pytest
import torch

import numerics as nm
from b200ddp.ops import functional as Fn

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _C():
    from b200ddp import _ext
    return _ext.get()


def _rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm().clamp(min=1e-30))


@pytest.mark.parametrize("T,E,k", [(512, 32, 8), (200, 8, 2), (64, 64, 8), (96, 8, 1)])
def test_router_and_permutation_match_the_reference(T, E, k):
    g = torch.Generator(device=DEV).manual_seed(T + E)
    logits = torch.randn(T, E, device=DEV, generator=g).to(torch.bfloat16)
    logits[: T // 4] = logits[: T // 4].round()               # many exact ties
    ids, gates, probsum = _C().moe_route(logits, k, True)
    ref_ids, ref_gates = Fn.moe_route_reference(logits.float().cpu(), k)
    assert torch.equal(ids.cpu().long(), ref_ids)
    assert torch.allclose(gates.float().cpu(), ref_gates.to(torch.bfloat16).float(), atol=4e-3, rtol=0)
    assert torch.allclose(probsum.cpu(), torch.softmax(logits.float().cpu(), -1).sum(0), rtol=1e-4, atol=1e-4)
    for got, want in zip(_C().moe_permute(ids, E), Fn.moe_permute_reference(ref_ids, E)):
        assert torch.equal(got.cpu(), want), (got, want)


def _skewed_ids(counts, k=1):
    ids = torch.cat([torch.full((c,), e, dtype=torch.int32) for e, c in enumerate(counts)])
    return ids[torch.randperm(len(ids), generator=torch.Generator().manual_seed(0))].view(-1, k).to(DEV)


EVERY_GROUPED = {"kGrpRows, B K-major", "kGrpRows, B MN-major", "kGrpWgrad"}
GROUPED_CALLS = [("moe_gemm", False), ("moe_gemm", True), ("moe_gemm_wgrad", None)]   # what every grouped case runs


def grouped_kernel(op, dgrad):
    """Mirror of launch_gemm_grouped (B MN-major exactly for the data gradient) and launch_gemm_grouped_wgrad."""
    if op == "moe_gemm_wgrad":
        return "kGrpWgrad"
    return "kGrpRows, B MN-major" if dgrad else "kGrpRows, B K-major"
# routing: the skewed counts of the older cases, Granite's (32 experts, top-8 of random router logits), and segments that
# end exactly on 128-row boundaries
ROUTINGS = [[0, 1, 127, 128, 129, 200, 5, 10], [0, 0, 600, 0, 0, 0, 0, 0], "granite", [256, 128, 0, 384]]


def test_grouped_cases_reach_every_grouped_gemm():
    assert {grouped_kernel(op, d) for op, d in GROUPED_CALLS} == EVERY_GROUPED


@pytest.mark.parametrize("counts", ROUTINGS)
@pytest.mark.parametrize("N,K", [(256, 128), (192, 64), (64, 64)])
def test_grouped_gemms_against_per_expert_fp32(counts, N, K):
    """Each expert segment of the forward, data-gradient and weight-gradient outputs against fp64, element by element:
    forward and dgrad take the GEMM bound with K from the weight, wgrad with K = the segment's rows."""
    C = _C()
    if counts == "granite":
        logits = torch.randn(512, 32, generator=torch.Generator().manual_seed(2))
        ids = logits.topk(8, -1).indices.to(torch.int32).to(DEV)
        counts = torch.bincount(ids.reshape(-1).cpu().long(), minlength=32).tolist()
    else:
        ids = _skewed_ids(counts)
    E = len(counts)
    T = ids.shape[0]
    cnt, offsets, fwd, inv, tiles = C.moe_permute(ids, E)
    assert cnt.tolist() == counts
    g = torch.Generator(device=DEV).manual_seed(1)
    x = torch.randn(T, K, device=DEV, generator=g).to(torch.bfloat16)
    w = (torch.randn(E, N, K, device=DEV, generator=g) * 0.1).to(torch.bfloat16)
    xp = C.moe_gather(x, fwd, ids.shape[1])
    pad = fwd < 0
    assert (xp[pad] == 0).all()
    cap = xp.shape[0]
    off = offsets.tolist()
    used = off[-1]                                            # rows of unused tiles are not written
    SENT = -7.0                                               # every output sits inside a sentinel-filled buffer with margins

    def fenced(*shape):
        buf = torch.full((shape[0] + 2, *shape[1:]), SENT, device=DEV, dtype=torch.bfloat16)
        return buf, buf[1:-1]

    def untouched(buf, inner_rows):
        assert (buf[0] == SENT).all() and (buf[-1] == SENT).all()
        assert (buf[1 + inner_rows:-1] == SENT).all()

    ybuf, y = fenced(cap, N)
    C.moe_gemm(xp, w, tiles, False, y)                        # [cap, N]
    dy = torch.randn(cap, N, device=DEV, generator=g).to(torch.bfloat16)
    dy[pad] = 0
    dxbuf, dx = fenced(cap, K)
    C.moe_gemm(dy, w, tiles, True, dx)                        # [cap, K]
    dwbuf, dw = fenced(E, N, K)
    C.moe_gemm_wgrad(dy, xp, offsets, dw)                     # [E, N, K]
    untouched(ybuf, used)
    untouched(dxbuf, used)
    untouched(dwbuf, E)
    dw2 = C.moe_gemm_wgrad(dy, xp, offsets)
    assert torch.equal(dw, dw2) and torch.equal(y[:used], C.moe_gemm(xp, w, tiles, False)[:used])
    for e in range(E):
        seg = slice(off[e], off[e + 1])
        if off[e + 1] == off[e]:
            assert (dw[e] == 0).all()
            continue
        where = f"expert {e} rows {off[e]}:{off[e + 1]}"
        nm.check_gemm(f"{where}: forward [row, n]", y[seg], xp[seg], w[e], group="moe grouped")
        nm.check_gemm(f"{where}: dgrad [row, k]", dx[seg], dy[seg], w[e].t(), group="moe grouped")
        nm.check_gemm(f"{where}: wgrad [n, k]", dw[e], dy[seg].t(), xp[seg].t(), group="moe grouped")
        assert (y[seg][pad[seg]] == 0).all() and (dx[seg][pad[seg]] == 0).all()


def _layer(T=256, H=256, I=128, E=8, k=2, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(T, H, device=DEV, generator=g).to(torch.bfloat16)
    wr = (torch.randn(E, H, device=DEV, generator=g) * 0.2).to(torch.bfloat16)
    wgu = (torch.randn(E, 2 * I, H, device=DEV, generator=g) * 0.1).to(torch.bfloat16)
    wd = (torch.randn(E, H, I, device=DEV, generator=g) * 0.1).to(torch.bfloat16)
    return x, wr, wgu, wd, k


def _run(x, wr, wgu, wd, k, dout, dprob):
    ts = [t.detach().clone().requires_grad_(True) for t in (x, wr, wgu, wd)]
    out, probsum, counts = Fn.moe(*ts, k, aux=True)
    (out.float() * dout.float()).sum().add((probsum * dprob).sum()).backward()
    return out, probsum, counts, [t.grad for t in ts]


@pytest.mark.parametrize("E,k", [(8, 2), (32, 8)])
def test_moe_layer_forward_and_backward_against_fp32(E, k):
    x, wr, wgu, wd, k = _layer(E=E, k=k)
    g = torch.Generator(device=DEV).manual_seed(5)
    dout = torch.randn(x.shape, device=DEV, generator=g).to(torch.bfloat16)
    dprob = torch.randn(E, device=DEV, generator=g)
    out, probsum, counts, grads = _run(x, wr, wgu, wd, k, dout, dprob)
    # fp32 reference that takes the GPU's routing decisions (made on bf16 router logits), so both sides pick the same experts
    rx, rwr, rwgu, rwd = (t.detach().float().cpu().requires_grad_(True) for t in (x, wr, wgu, wd))
    ids = Fn.moe_route_reference(Fn.linear(x, wr).float().cpu(), k)[0]
    logits = rx @ rwr.t()
    gates = torch.softmax(logits.gather(1, ids), -1)
    I = rwd.shape[2]
    ref = torch.zeros_like(rx)
    for t in range(rx.shape[0]):
        for j, e in enumerate(ids[t].tolist()):
            h = torch.nn.functional.silu(rwgu[e, :I] @ rx[t]) * (rwgu[e, I:] @ rx[t])
            ref[t] = ref[t] + gates[t, j] * (rwd[e] @ h)
    rprob, rcounts = torch.softmax(logits, -1).sum(0), torch.bincount(ids.reshape(-1), minlength=E).to(torch.int32)
    (ref * dout.float().cpu()).sum().add((rprob * dprob.cpu()).sum()).backward()
    assert torch.equal(counts.cpu(), rcounts)
    assert _rel(out.cpu(), ref.detach()) < 2e-2
    assert _rel(probsum.cpu(), rprob.detach()) < 5e-3            # bf16 router logits on the GPU
    for got, want in zip(grads, (rx.grad, rwr.grad, rwgu.grad, rwd.grad)):
        assert _rel(got.cpu(), want) < 5e-2
    again = _run(x, wr, wgu, wd, k, dout, dprob)              # bitwise reproducible
    assert torch.equal(out, again[0]) and torch.equal(probsum, again[1])
    assert all(torch.equal(a, b) for a, b in zip(grads, again[3]))


def test_moe_rejects_unsupported_shapes():
    x, wr, wgu, wd, k = _layer()
    with pytest.raises(ValueError, match="multiples of 64"):
        Fn.moe(x[:, :200], wr[:, :200], wgu[..., :200], wd[:, :200], k)
    with pytest.raises(ValueError, match="bf16"):
        Fn.moe(x.float(), wr, wgu, wd, k)
    with pytest.raises(ValueError, match="top_k"):
        Fn.moe(x, wr, wgu, wd, 9)


def _tiny_model(**kw):
    from b200ddp.models.llama import LlamaConfig, LlamaForCausalLM
    cfg = dict(vocab_size=1000, max_position=512, hidden=256, layers=2, heads=4, kv_heads=2, intermediate=128, eps=1e-6,
               num_experts=8, experts_per_token=2, router_aux_loss_coef=0.01, embedding_multiplier=12.0,
               attention_multiplier=0.015625, residual_multiplier=0.22, logits_scaling=6.0, pad_vocab_to=64)
    cfg.update(kw)
    torch.manual_seed(0)
    return LlamaForCausalLM(LlamaConfig(**cfg))


def test_tiny_granite_model_matches_its_cpu_body(monkeypatch):
    import copy
    m = _tiny_model(pad_token_id=0, bos_token_id=1)
    with torch.no_grad():                                     # the same (bf16-representable) weights on both sides
        for p in m.parameters():
            p.copy_(p.bfloat16().float())
    cpu = copy.deepcopy(m)
    ids = torch.randint(2, 1000, (2, 256), generator=torch.Generator().manual_seed(1))
    ids[0, [0, 100]] = 1
    ids[1, 200:] = 0
    labels = torch.cat([ids[:, 1:], torch.full((2, 1), -100)], 1)
    # the GPU run, keeping each layer's bf16 router logits: the routing decisions the CPU body then takes
    g = m.to(DEV, torch.bfloat16)
    routing = []
    hooks = [layer.moe.register_forward_pre_hook(
        lambda mod, inp: routing.append(Fn.linear(inp[0].reshape(-1, inp[0].shape[-1]), mod.router.weight).float().cpu()))
        for layer in g.model.layers]
    logits = g(ids.to(DEV))
    for h in hooks:
        h.remove()
    loss = Fn.cross_entropy(logits, labels.to(DEV)) + 0.01 * g.router_aux_loss()
    loss.backward()
    reference = Fn._moe_reference
    monkeypatch.setattr(Fn, "_moe_reference", lambda *a, **kw: reference(*a, **kw, routing_logits=routing.pop(0)))
    ref_logits = cpu(ids)
    ref = Fn.cross_entropy(ref_logits, labels) + 0.01 * cpu.router_aux_loss()
    ref.backward()
    assert not routing
    assert _rel(logits.float().cpu()[..., :1000], ref_logits.detach()[..., :1000]) < 2e-2
    assert abs(float(loss) - float(ref)) < 5e-3 * float(ref)
    worst = max(((_rel(p.grad.float().cpu(), q.grad), n) for (n, p), (_, q) in zip(g.named_parameters(), cpu.named_parameters())))
    assert worst[0] < 5e-2, worst


def test_training_steps_without_host_sync_and_graph_replay_with_new_routing():
    from b200ddp.engine.step import TrainStep
    from b200ddp.engine.trainer import RouterAuxLoss
    from b200ddp.ops import CrossEntropyLoss
    from b200ddp.optim import FusedAdamW, weight_decay_groups

    def batch(seed):
        gen = torch.Generator().manual_seed(seed)
        x = torch.randint(2, 1000, (2, 256), generator=gen)
        return x.to(DEV), torch.cat([x[:, 1:], torch.full((2, 1), -100)], 1).to(DEV)

    def make(use_graph):
        m = _tiny_model().to(DEV, torch.bfloat16)
        opt = FusedAdamW(weight_decay_groups(m, 0.01), lr=1e-3, max_grad_norm=1.0)
        return TrainStep(m, RouterAuxLoss(CrossEntropyLoss(), m, 0.01), opt, torch.device(DEV), use_graph=use_graph), m

    eager, me = make(False)
    graph, mg = make(True)
    losses = []
    for seed in range(6):                   # three eager warm-up steps, the capture at the fourth, replays on new routing after
        x, y = batch(seed)
        if seed >= 4:                       # eager and replayed steps alike: no host synchronisation anywhere in a step
            torch.cuda.set_sync_debug_mode("error")
        try:
            losses.append((eager(x, y), graph(x, y)))
        finally:
            torch.cuda.set_sync_debug_mode(0)
    losses = [(float(a), float(b)) for a, b in losses]
    for a, b in losses:
        assert abs(a - b) < 1e-3 * abs(a), losses
    for (n, a), (_, b) in zip(me.named_parameters(), mg.named_parameters()):
        assert torch.equal(a, b), n


def test_full_preset_adamw_step():
    from b200ddp.models import build_model
    from b200ddp.optim import FusedAdamW, weight_decay_groups
    from b200ddp.utils import to_mixed_bf16
    torch.manual_seed(0)
    m = to_mixed_bf16(build_model("granite-3.0-1b-a400m").to(DEV))
    opt = FusedAdamW(weight_decay_groups(m, 0.01), lr=1e-4, max_grad_norm=1.0)
    x = torch.randint(1, 49155, (1, 2048), device=DEV)
    y = torch.roll(x, -1, 1)
    crit = lambda: Fn.cross_entropy(m(x), y) + 0.001 * m.router_aux_loss()
    first = crit()
    first.backward()
    opt.step()
    opt.zero_grad(set_to_none=True)
    with torch.no_grad():
        second = crit()
    assert torch.isfinite(first) and torch.isfinite(second) and float(second) < float(first)
