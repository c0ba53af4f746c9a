"""Fused LM-head cross-entropy on the H100: ``ops.linear_cross_entropy`` against an fp32 torch reference and the unfused
native path at the three vocabularies, ignore rules, scaling, determinism, framed outputs, no host synchronisation, CUDA-graph
replay, the memory it saves at Qwen's head shape, and training runs of tiny models with ``--fused_lm_loss``."""
import math

import pytest
import torch

from b200ddp.ops import cross_entropy, linear, linear_cross_entropy
from b200ddp.ops.functional import LM_LOSS_SLICE

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")


def _rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm().clamp(min=1e-30))


def _case(N, V, H, bias, seed=0, scale=1.0):
    g = torch.Generator(device=dev).manual_seed(seed)
    h = (torch.randn(N, H, device=dev, generator=g) * scale).to(torch.bfloat16)
    w = (torch.randn(V, H, device=dev, generator=g) * 0.05).to(torch.bfloat16)
    t = torch.randint(0, V, (N,), device=dev, generator=g)
    special = [0, 127, 128, LM_LOSS_SLICE - 1, LM_LOSS_SLICE, V - 1, -100, V, -7, V + 5]
    t[:len(special)] = torch.tensor(special, device=dev)
    b = None
    if bias:                                                       # GPT-2's padded-vocabulary mask
        b = torch.zeros(V, device=dev, dtype=torch.bfloat16)
        b[V - 47:] = -1e4
    return h, w, t, b


def _fused(h, w, t, b, scale=1.0):
    hh, ww = h.clone().requires_grad_(True), w.clone().requires_grad_(True)
    loss = linear_cross_entropy(hh, ww, t, b)
    (loss * scale).backward()
    return loss.detach(), hh.grad, ww.grad


def _unfused(h, w, t, b):
    hh, ww = h.clone().requires_grad_(True), w.clone().requires_grad_(True)
    loss = cross_entropy(linear(hh, ww, b), t)
    loss.backward()
    return loss.detach(), hh.grad, ww.grad


def _reference(h, w, t, b):
    """fp32 autograd, with the logits rounded to bf16 in the forward (as both native paths store or use them) and the
    rounding passed straight through in the backward."""
    hh, ww = h.float().requires_grad_(True), w.float().requires_grad_(True)
    x = hh @ ww.t() + (0 if b is None else b.float())
    x = x + (x.to(torch.bfloat16).float() - x).detach()
    valid = (t != -100) & (t >= 0) & (t < x.shape[1])
    picked = x.gather(1, torch.where(valid, t, 0)[:, None])[:, 0]
    loss = torch.where(valid, torch.logsumexp(x, -1) - picked, 0.0).sum() / valid.sum().clamp(min=1)
    loss.backward()
    return loss.detach(), hh.grad, ww.grad


@pytest.mark.parametrize("V,H,bias,scale", [(151936, 256, False, 1.0), (49152, 192, False, 1.0), (50304, 256, True, 1.0),
                                            (49152, 192, False, 40.0)])
def test_matches_fp32_reference_and_unfused_native_path(V, H, bias, scale):
    h, w, t, b = _case(1024, V, H, bias, scale=scale)
    loss, dh, dw = _fused(h, w, t, b)
    rl, rh, rw = _reference(h, w, t, b)
    ul, uh, uw = _unfused(h, w, t, b)
    assert torch.isfinite(loss) and torch.isfinite(dh.float()).all() and torch.isfinite(dw.float()).all()
    assert abs(float(loss) - float(rl)) <= 1e-3 * abs(float(rl)), (float(loss), float(rl))
    assert abs(float(loss) - float(ul)) <= 1e-3 * abs(float(ul)), (float(loss), float(ul))
    assert _rel(dh, rh) < 2e-2 and _rel(dw, rw) < 2e-2, (_rel(dh, rh), _rel(dw, rw))
    assert _rel(dh, uh) < 2e-2 and _rel(dw, uw) < 2e-2, (_rel(dh, uh), _rel(dw, uw))
    ignored = (t == -100) | (t < 0) | (t >= V)
    assert (dh[ignored] == 0).all()


def test_all_rows_ignored_gives_zero_loss_and_gradients():
    h, w, _, _ = _case(256, 4096, 128, False)
    loss, dh, dw = _fused(h, w, torch.full((256,), -100, device=dev), None)
    assert float(loss) == 0.0 and (dh == 0).all() and (dw == 0).all()


def test_upstream_gradient_scales_and_runs_are_bitwise_identical():
    h, w, t, b = _case(512, 20000, 128, True, seed=3)
    l1, h1, w1 = _fused(h, w, t, b)
    l2, h2, w2 = _fused(h, w, t, b)
    assert torch.equal(l1, l2) and torch.equal(h1, h2) and torch.equal(w1, w2)
    _, hq, wq = _fused(h, w, t, b, scale=0.25)
    assert _rel(hq, 0.25 * h1.float()) < 1e-2 and _rel(wq, 0.25 * w1.float()) < 1e-2


def test_writes_stay_inside_framed_outputs():
    from b200ddp import _ext
    C = _ext.get()
    N, V, H = 384, 2176, 128
    h, w, t, b = _case(N, V, H, True, seed=5)
    lse_f = torch.full((N + 64,), 7.0, device=dev)
    rl_f = torch.full((N + 65,), 7.0, device=dev)
    loss, lse, rl = C.lm_loss_fwd(h, w, t, b, -100, lse_f[32:32 + N], rl_f[32:33 + N])
    assert (lse_f[:32] == 7).all() and (lse_f[32 + N:] == 7).all() and (rl_f[:32] == 7).all() and (rl_f[33 + N:] == 7).all()
    dh_f = torch.full((N + 2, H), 3.0, device=dev, dtype=torch.bfloat16)
    dw_f = torch.full((V + 2, H), 3.0, device=dev, dtype=torch.bfloat16)
    g = torch.ones(1, device=dev)
    C.lm_loss_bwd(h, w, t, b, lse, rl, g, -100, 1024, True, True, dh_f[1:N + 1], dw_f[1:V + 1])
    for f in (dh_f, dw_f):
        assert (f[0] == 3).all() and (f[-1] == 3).all()
    _, rh, rw = _fused(h, w, t, b)
    assert _rel(dh_f[1:N + 1], rh) < 1e-2 and _rel(dw_f[1:V + 1], rw) < 1e-2


def test_no_host_synchronisation():
    h, w, t, b = _case(512, 8192, 128, True, seed=6)
    _fused(h, w, t, b)                                             # first calls: module load, tensor maps
    hh, ww = h.clone().requires_grad_(True), w.clone().requires_grad_(True)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        linear_cross_entropy(hh, ww, t, b).backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert hh.grad is not None and ww.grad is not None


def test_cuda_graph_replay_with_new_targets_equals_eager():
    h, w, t, b = _case(512, 16384, 128, True, seed=7)
    hh, ww = h.clone().requires_grad_(True), w.clone().requires_grad_(True)
    st = t.clone()

    def step():
        loss = linear_cross_entropy(hh, ww, st, b)
        return (loss,) + torch.autograd.grad(loss, (hh, ww))
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step()
    t2 = torch.randint(0, 16384, t.shape, device=dev)
    t2[:5] = -100
    st.copy_(t2)
    graph.replay()
    ref = _fused(h, w, t2, b)
    for a, e in zip(out, ref):
        assert torch.equal(a, e)


def test_memory_at_qwen_head_shape_stays_below_one_logits_tensor():
    N, V, H = 8192, 151936, 1536
    h, w, t, _ = _case(N, V, H, False, seed=8)
    logits_bytes = N * V * 2

    def rise(fn):
        hh, ww = h.clone().requires_grad_(True), w.clone().requires_grad_(True)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        loss = fn(hh, ww)
        loss.backward()
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - base
    fused = rise(lambda a, c: linear_cross_entropy(a, c, t))
    unfused = rise(lambda a, c: cross_entropy(linear(a, c), t))
    print(f"\n[lm-loss memory] {N} x {V} x {H}: fwd+bwd rise fused {fused / 1e9:.2f} GB, unfused {unfused / 1e9:.2f} GB, "
          f"logits {logits_bytes / 1e9:.2f} GB")
    assert fused < logits_bytes, (fused, logits_bytes)


# ---- tiny models through the trainer: --fused_lm_loss --cuda_graph (+ --pack, + --fp8) -----------------------------------
def _tiny(family, fused, **kw):
    if family == "gpt2":
        from b200ddp.models.gpt import GPTConfig, GPTLMHeadModel
        return GPTLMHeadModel(GPTConfig(vocab_size=1000, max_position=256, hidden=128, layers=2, heads=2, intermediate=256,
                                        fused_lm_loss=fused, **kw))
    from b200ddp.models.llama import LlamaConfig, LlamaForCausalLM
    if family == "smollm":
        return LlamaForCausalLM(LlamaConfig(vocab_size=1024, max_position=256, hidden=128, layers=2, heads=2, kv_heads=1,
                                            intermediate=256, fused_lm_loss=fused, **kw))
    return LlamaForCausalLM(LlamaConfig(vocab_size=1024, max_position=256, hidden=256, layers=2, heads=2, kv_heads=1,
                                        intermediate=256, eps=1e-6, rope_theta=1e6, attention_bias=True, fused_lm_loss=fused, **kw))


_MODEL = {"gpt2": "gpt2", "smollm": "smollm-135m", "qwen": "qwen2.5-1.5b"}


@pytest.mark.parametrize("family,extra", [("gpt2", []), ("smollm", []), ("qwen", []), ("gpt2", ["--pack"]),
                                          ("smollm", ["--fp8"]), ("qwen", ["--pack", "--fp8"])])
def test_tiny_models_train_with_fused_lm_loss_and_cuda_graph(tmp_path, family, extra):
    from b200ddp.engine import cli
    from b200ddp.engine.trainer import Trainer, build_dataset
    from b200ddp.ops import CrossEntropyLoss
    from b200ddp.utils import to_mixed_bf16
    pack = "--pack" in extra
    flags = ["--no_tensorboard", "--output_dir", str(tmp_path / "out"), "--model", _MODEL[family], "--fp16", "--cuda_graph",
             "--fused_lm_loss", "--seq_len", "256", "--optimizer", "adamw", "--lr", "3e-3", "--max_steps", "40",
             "--per_gpu_train_batch_size", "8", "--warmup_steps", "2", "--save_steps", "0", "--logging_steps", "10"]
    flags += ["--min_seq_len", "32", "--pack"] if pack else []
    flags += ["--fp8"] if "--fp8" in extra else []
    args = cli.build_parser().parse_args(flags)
    cli.setup(args)
    ds = build_dataset(args)
    bos = getattr(ds, "bos_token_id", None)
    is_bos = ds.X == bos if bos is not None else torch.zeros_like(ds.X, dtype=torch.bool)
    ds.X = torch.where(is_bos, torch.ones_like(ds.X), torch.where(ds.X > 0, ds.X % 16 + 2, ds.X))
    ds.Y = torch.where(ds.Y > 0, ds.Y % 16 + 2, ds.Y)
    kw = dict(fp8="--fp8" in extra)
    if pack:
        ds.bos_token_id = 1
        kw.update(pad_token_id=0, bos_token_id=1)
    torch.manual_seed(0)
    model = _tiny(family, True, **kw)
    plain = _tiny(family, False, **kw)
    plain.load_state_dict(model.state_dict())
    plain = to_mixed_bf16(plain.to(dev))
    trainer = Trainer(args, model, cli.log, dataset=ds)
    x, y = ds.X[:8].to(dev), ds.Y[:8].to(dev)
    with torch.no_grad():                                          # first-step loss: fused equals unfused
        lf = float(trainer.criterion(trainer.model(x), y))
        lp = float(CrossEntropyLoss()(plain(x), y))
    assert abs(lf - lp) < 2e-3 * abs(lp), (lf, lp)
    before = trainer.evaluate(max_batches=4)["eval_loss"]
    trainer.train()
    after = trainer.evaluate(max_batches=4)["eval_loss"]
    assert trainer.step_fn.graph is not None
    assert math.isfinite(after) and after < before - 0.1, (before, after)


def test_full_qwen_preset_step_with_fused_lm_loss_prints_peak_memory():
    from b200ddp.models import build_model
    from b200ddp.utils import to_mixed_bf16
    model = to_mixed_bf16(build_model("qwen2.5-1.5b", fused_lm_loss=True).to(dev))
    crit = model.lm_head_loss()
    ids = torch.randint(0, 151936, (4, 2048), device=dev)
    torch.cuda.reset_peak_memory_stats()
    loss = crit(model(ids), torch.roll(ids, -1, 1))
    loss.backward()
    loss = loss.detach()
    torch.cuda.synchronize()
    print(f"\n[lm-loss qwen2.5-1.5b 4 x 2048 fwd+bwd, fused head] loss {float(loss):.4f}, peak "
          f"{torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")
    assert math.isfinite(float(loss)) and model.model.embed_tokens.weight.grad is not None
