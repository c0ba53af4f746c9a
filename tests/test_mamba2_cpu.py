"""Mamba-2 on the CPU: parameter counts, state dict and initialisation against transformers' ``Mamba2ForCausalLM``, fp32
agreement with its ``torch_forward``, the document resets of packed and right-padded rows, the reference ops, a two-rank
gloo DDP step, and the CLI."""
import math

import pytest
import torch
import torch.nn.functional as F

transformers = pytest.importorskip("transformers")

from b200ddp.models import MODEL_REGISTRY, build_model  # noqa: E402
from b200ddp.models.mamba2 import Mamba2Config, Mamba2ForCausalLM  # noqa: E402
from b200ddp.ops import causal_conv1d_window, document_bounds, gated_rms_norm, ssd_scan  # noqa: E402
from b200ddp.utils.precision import to_mixed_bf16  # noqa: E402

VOCAB, HIDDEN, LAYERS, HEADS = 96, 128, 2, 4


def _hf(hidden=HIDDEN, layers=LAYERS, heads=HEADS, vocab=VOCAB):
    cfg = transformers.Mamba2Config(hidden_size=hidden, num_hidden_layers=layers, num_heads=heads, head_dim=64, state_size=128, n_groups=1,
                                    expand=2, conv_kernel=4, use_bias=False, use_conv_bias=True, residual_in_fp32=True, vocab_size=vocab,
                                    layer_norm_epsilon=1e-5, tie_word_embeddings=True)
    return transformers.Mamba2ForCausalLM(cfg).eval()


def _ours(**kw):
    return Mamba2ForCausalLM(Mamba2Config(**{"vocab_size": VOCAB, "hidden": HIDDEN, "layers": LAYERS, "heads": HEADS, **kw}))


def _pair(seed=0):
    torch.manual_seed(seed)
    ours = _ours()
    with torch.no_grad():                      # away from the initial values, so every parameter's gradient is exercised
        for p in ours.parameters():
            if p.dim() == 1:
                p.add_(0.1 * torch.randn_like(p))
    hf = _hf()
    sd = ours.state_dict()
    hf.load_state_dict({**sd, "lm_head.weight": sd["backbone.embeddings.weight"]}, strict=True)
    return ours, hf


@pytest.mark.parametrize("name,count,entries", [("mamba2-130m", 128_989_632, 219), ("mamba2-370m", 368_346_624, 435)])
def test_parameter_counts_and_state_dict_match_transformers(name, count, entries):
    c = MODEL_REGISTRY[name].config
    with torch.device("meta"):
        hf = _hf(c.hidden, c.layers, c.heads, c.vocab_size)
        ours = build_model(name)
    assert sum(p.numel() for p in hf.parameters()) == count
    assert sum(p.numel() for p in ours.parameters()) == count
    hsd = hf.state_dict()
    assert len(hsd) == entries and set(hsd) - set(ours.state_dict()) == {"lm_head.weight"}
    for k, v in ours.state_dict().items():
        assert tuple(hsd[k].shape) == tuple(v.shape), k
    E, N, H = 2 * c.hidden, 128, c.heads
    assert tuple(ours.state_dict()["backbone.layers.0.mixer.in_proj.weight"].shape) == (2 * E + 2 * N + H, c.hidden)
    assert 2 * E + 2 * N + H == {"mamba2-130m": 3352, "mamba2-370m": 4384}[name]


def test_registry_entries():
    for name, hidden, layers, heads in (("mamba2-130m", 768, 24, 24), ("mamba2-370m", 1024, 48, 32)):
        e = MODEL_REGISTRY[name]
        c = e.config
        assert e.kind == "causal" and e.start_id == 1 and not e.fp8 and not e.moe and c.max_position == 2048
        assert (c.hidden, c.layers, c.heads, c.head_dim, c.state, c.n_groups, c.vocab_size) == (hidden, layers, heads, 64, 128, 1, 50288)
        with pytest.raises(TypeError):
            e.build(fp8=True)


def test_load_hf_state_dict_is_strict():
    torch.manual_seed(1)
    hf = _hf()
    ours = _ours()
    ours.load_hf_state_dict(hf.state_dict())
    for k, v in ours.state_dict().items():
        assert torch.equal(v, hf.state_dict()[k]), k
    bad = dict(hf.state_dict())
    bad.pop("backbone.layers.1.mixer.D")
    with pytest.raises(RuntimeError):
        ours.load_hf_state_dict(bad)
    bad = dict(hf.state_dict())
    bad["lm_head.weight"] = bad["lm_head.weight"] + 1
    with pytest.raises(ValueError, match="lm_head"):
        ours.load_hf_state_dict(bad)


def test_initialisation_scheme():
    torch.manual_seed(0)
    m = Mamba2ForCausalLM(Mamba2Config(hidden=256, layers=2, heads=8, vocab_size=512))
    mix = m.backbone.layers[0].mixer
    E, H = 512, 8
    assert torch.equal(mix.A_log, torch.log(torch.arange(1, H + 1.0))) and torch.equal(mix.D, torch.ones(H))
    assert torch.equal(mix.norm.weight, torch.ones(E)) and torch.equal(mix.conv1d.bias, torch.zeros(E + 256))
    dt = F.softplus(mix.dt_bias)
    assert dt.min() >= 1e-3 * 0.999 and dt.max() <= 0.1 * 1.001
    assert mix.conv1d.weight.abs().max() <= 1 / math.sqrt(4) and mix.out_proj.weight.abs().max() <= 1 / math.sqrt(E)
    for w in (mix.in_proj.weight, m.backbone.embeddings.weight):
        assert abs(w.std().item() - 0.1) < 0.01 and abs(w.mean().item()) < 0.01
    bf = to_mixed_bf16(m)
    assert mix.A_log.dtype == mix.D.dtype == mix.dt_bias.dtype == torch.float32
    assert mix.in_proj.weight.dtype == mix.norm.weight.dtype == torch.bfloat16 and bf is m


def _rel(a, b):
    return float((a - b).norm() / b.norm())


@pytest.mark.parametrize("seed,S", [(0, 200), (1, 37)])
def test_fp32_model_matches_transformers(seed, S):
    ours, hf = _pair(seed)
    ids = torch.randint(1, VOCAB, (2, S))
    w = torch.randn(2, S, VOCAB)
    lo = ours(ids)
    lh = hf(ids).logits
    assert _rel(lo, lh) < 1e-5
    (lo * w).sum().backward()
    (lh * w).sum().backward()
    hp = dict(hf.named_parameters())
    for k, p in ours.named_parameters():
        assert _rel(p.grad, hp[k].grad) < 1e-5, k


def test_packed_rows_equal_each_document_alone():
    ours, hf = _pair(2)
    ours.config.bos_token_id, ours.config.pad_token_id = 1, 0
    ids = torch.randint(2, VOCAB, (2, 150))
    starts0 = [0, 13, 64, 65, 140]            # at and just after a chunk boundary, one-token documents, one over several chunks
    ids[0, starts0] = 1
    ids[1, [0, 21]] = 1
    ids[1, 133:] = 0
    with torch.no_grad():
        lo = ours(ids)
        for b, starts, end in ((0, starts0, 150), (1, [0, 21], 133)):
            for s, e in zip(starts, starts[1:] + [end]):
                alone = hf(ids[b:b + 1, s:e]).logits[0]
                assert _rel(lo[b, s:e], alone) < 1e-5, (b, s)


def test_right_padded_rows_equal_transformers_at_real_positions():
    ours, hf = _pair(3)
    ours.config.pad_token_id = 0
    ids = torch.randint(1, VOCAB, (3, 130))
    lens = [130, 71, 5]
    for b, n in enumerate(lens):
        ids[b, n:] = 0
    with torch.no_grad():
        lo = ours(ids)
        for b, n in enumerate(lens):
            assert _rel(lo[b, :n], hf(ids[b:b + 1, :n]).logits[0]) < 1e-5, b


def _ssd_inputs(B, S, H, dtype=torch.float64, seed=4):
    g = torch.Generator().manual_seed(seed)
    E, N = 64 * H, 128
    W = 2 * E + 2 * N + H
    zx = torch.randn(B, S, W, dtype=dtype, generator=g)
    w, bias = torch.randn(E + 2 * N, 1, 4, dtype=dtype, generator=g), torch.randn(E + 2 * N, dtype=dtype, generator=g)
    A_log, D, dtb = torch.rand(H, dtype=dtype, generator=g), torch.randn(H, dtype=dtype, generator=g), torch.randn(H, dtype=dtype, generator=g)
    return zx, w, bias, A_log, D, dtb


def test_reference_ops_reset_at_document_starts_and_check_shapes():
    B, S, H = 2, 90, 2
    E = 64 * H
    zx, w, bias, A_log, D, dtb = _ssd_inputs(B, S, H)
    ids = torch.full((B, S), 5)
    ids[0, 70] = 1
    ids[1, 75:] = 0
    bounds, _ = document_bounds(ids, 1, 0)
    xbc = causal_conv1d_window(zx, w, bias, bounds, col=E)
    y = ssd_scan(xbc, zx[..., -H:], A_log, D, dtb, bounds)
    o = gated_rms_norm(y, zx[..., :E], torch.randn(E, dtype=torch.float64), 1e-5)
    assert xbc.dtype == y.dtype == o.dtype == torch.float64
    assert (xbc[1, 75:] == 0).all() and (y[1, 75:] == 0).all()
    one = document_bounds(torch.full((1, S - 70), 5), None, None)[0]
    x1 = causal_conv1d_window(zx[:1, 70:], w, bias, one, col=E)
    y1 = ssd_scan(x1, zx[:1, 70:, -H:], A_log, D, dtb, one)
    assert torch.allclose(xbc[0, 70:], x1[0]) and torch.allclose(y[0, 70:], y1[0])
    # the chunked reference equals the sequential recurrence
    dt = F.softplus(zx[0, :70, -H:] + dtb)
    x, Bm, Cm = xbc[0, :70, :E].reshape(70, H, 64), xbc[0, :70, E:E + 128], xbc[0, :70, E + 128:]
    h = torch.zeros(H, 64, 128, dtype=torch.float64)
    for t in range(70):
        h = torch.exp(dt[t] * -torch.exp(A_log))[:, None, None] * h + dt[t][:, None, None] * x[t][..., None] * Bm[t]
        assert torch.allclose(y[0, t], ((h * Cm[t]).sum(-1) + D[:, None] * x[t]).reshape(-1), atol=1e-10), t
    with pytest.raises(ValueError):
        ssd_scan(xbc, zx[..., -H:], A_log, D, dtb, bounds, head_dim=32)
    with pytest.raises(ValueError):
        ssd_scan(xbc, zx[..., -H:], A_log, D, dtb, bounds, state_size=64)
    with pytest.raises(ValueError):
        ssd_scan(xbc, zx[..., -H:], A_log, D, dtb, bounds, n_groups=2)
    with pytest.raises(ValueError):
        ssd_scan(xbc[..., :-1], zx[..., -H:], A_log, D, dtb, bounds)
    with pytest.raises(ValueError):
        ssd_scan(xbc, zx[..., -H:], A_log[:1], D, dtb, bounds)
    with pytest.raises(ValueError):
        causal_conv1d_window(zx, w, bias, bounds, col=zx.shape[-1] - 8)
    with pytest.raises(ValueError):
        causal_conv1d_window(zx, w[:, :, :3], bias, bounds, col=E)
    with pytest.raises(ValueError):
        gated_rms_norm(y, zx[..., :E - 1], torch.ones(E), 1e-5)
    with pytest.raises(ValueError):
        gated_rms_norm(y, zx[..., :E], torch.ones(E + 1), 1e-5)


def test_config_rejects_unsupported_shapes():
    for kw in ({"state": 64}, {"n_groups": 2}, {"head_dim": 32}, {"heads": 3}):
        with pytest.raises(ValueError):
            _ours(**kw)


def _cli_args(tmp_path, model, *flags):
    from b200ddp.engine import cli
    return cli.build_parser().parse_args(["--no_tensorboard", "--output_dir", str(tmp_path / "out"), "--model", model, "--no_cuda", *flags])


@pytest.mark.parametrize("flags", [[], ["--min_seq_len", "32", "--seq_len", "128"], ["--pack", "--min_seq_len", "32", "--seq_len", "128"],
                                   ["--fused_lm_loss"], ["--cuda_graph"], ["--optimizer", "adamw", "--gradient_accumulation_steps", "2"],
                                   ["--seq_len", "2048"]])
@pytest.mark.parametrize("model", ["mamba2-130m", "mamba2-370m"])
def test_cli_accepts(tmp_path, model, flags):
    from b200ddp.engine import cli
    cli.setup(_cli_args(tmp_path, model, *flags))


@pytest.mark.parametrize("flags,match", [(["--fp8", "--fp16"], "--fp8"), (["--seq_len", "2049"], "2048")])
@pytest.mark.parametrize("model", ["mamba2-130m", "mamba2-370m"])
def test_cli_rejects(tmp_path, model, flags, match):
    from b200ddp.engine import cli
    with pytest.raises(ValueError, match=match):
        cli.setup(_cli_args(tmp_path, model, *flags))


def test_short_cpu_training_run_resumes(tmp_path, monkeypatch):
    from b200ddp import models
    from b200ddp.engine import cli
    from b200ddp.engine.trainer import Trainer
    from b200ddp.models import mamba2 as mm
    tiny = Mamba2Config(hidden=32, layers=1, heads=1, vocab_size=128)
    monkeypatch.setitem(models.MODEL_REGISTRY, "mamba2-130m", models.ModelEntry(
        lambda **kw: mm._build(tiny, kw.get("pad_token_id"), kw.get("bos_token_id"), kw.get("fused_lm_loss", False)),
        "causal", tiny, start_id=1))
    flags = ["--per_gpu_train_batch_size", "2", "--max_steps", "2", "--logging_steps", "1", "--save_steps", "2", "--optimizer", "adamw",
             "--lr", "1e-4", "--dataset_size", "8", "--seq_len", "64", "--min_seq_len", "16", "--pack"]
    args = _cli_args(tmp_path, "mamba2-130m", *flags)
    cli.setup(args)
    step, loss = Trainer(args, build_model("mamba2-130m", pad_token_id=0, bos_token_id=1), cli.log).train()
    assert step == 3 and math.isfinite(loss) and loss > 0
    args = _cli_args(tmp_path, "mamba2-130m", *flags[:5], "4", *flags[6:], "--resume_from", "latest")
    cli.setup(args)
    step, loss = Trainer(args, build_model("mamba2-130m", pad_token_id=0, bos_token_id=1), cli.log).train()
    assert step >= 3 and math.isfinite(loss)


def _free_port():
    import socket
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _gloo_model():
    torch.manual_seed(0)
    return Mamba2ForCausalLM(Mamba2Config(vocab_size=VOCAB, hidden=32, layers=1, heads=1)).double()


def _gloo_data():
    g = torch.Generator().manual_seed(3)
    return torch.randint(1, VOCAB, (4, 24), generator=g)


def _gloo_loss(model, x):
    logits = model(x[:, :-1])
    return F.cross_entropy(logits.reshape(-1, logits.shape[-1]), x[:, 1:].reshape(-1))


def _ddp_worker(rank, world, port, path):
    import os
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from b200ddp.parallel import DistributedDataParallel
        model = _gloo_model()
        ddp = DistributedDataParallel(model, backend="gloo")
        x = _gloo_data()
        n = len(x) // world
        _gloo_loss(ddp, x[rank * n:(rank + 1) * n]).backward()
        grads = {k: p.grad.clone() for k, p in model.named_parameters()}
        torch.optim.SGD(model.parameters(), lr=0.1).step()
        torch.save({"grads": grads, "params": {k: p.detach().clone() for k, p in model.named_parameters()}}, f"{path}.{rank}")
    finally:
        dist.destroy_process_group()


def test_gloo_world_2_keeps_ranks_identical_and_averages_gradients(tmp_path):
    import torch.multiprocessing as mp
    path = str(tmp_path / "rank")
    mp.spawn(_ddp_worker, args=(2, _free_port(), path), nprocs=2, join=True)
    r0, r1 = torch.load(f"{path}.0"), torch.load(f"{path}.1")
    x = _gloo_data()
    single = []
    for half in (slice(0, 2), slice(2, 4)):
        m = _gloo_model()
        _gloo_loss(m, x[half]).backward()
        single.append({k: p.grad for k, p in m.named_parameters()})
    for k in single[0]:
        want = (single[0][k] + single[1][k]) / 2
        assert torch.allclose(r0["grads"][k], want, rtol=1e-9, atol=1e-12), k
        assert torch.equal(r0["params"][k], r1["params"][k]), k
