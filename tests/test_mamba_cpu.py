"""Mamba on the CPU: parameter counts, state dict and initialisation against transformers' ``MambaForCausalLM``, fp32
agreement with its ``slow_forward``, the document resets of packed and right-padded rows, the reference ops, a two-rank
gloo DDP step, and the CLI."""
import math

import pytest
import torch
import torch.nn.functional as F

transformers = pytest.importorskip("transformers")

from b200ddp.models import MODEL_REGISTRY, build_model  # noqa: E402
from b200ddp.models.mamba import MambaConfig, MambaForCausalLM  # noqa: E402
from b200ddp.ops import causal_conv1d, document_bounds, selective_scan  # noqa: E402
from b200ddp.utils.precision import to_mixed_bf16  # noqa: E402

VOCAB, HIDDEN, LAYERS = 96, 64, 2


def _hf(hidden=HIDDEN, layers=LAYERS, vocab=VOCAB):
    cfg = transformers.MambaConfig(hidden_size=hidden, num_hidden_layers=layers, vocab_size=vocab, layer_norm_epsilon=1e-5)
    return transformers.MambaForCausalLM(cfg).eval()


def _pair(seed=0):
    torch.manual_seed(seed)
    ours = MambaForCausalLM(MambaConfig(vocab_size=VOCAB, hidden=HIDDEN, layers=LAYERS))
    hf = _hf()
    sd = ours.state_dict()
    hf.load_state_dict({**sd, "lm_head.weight": sd["backbone.embeddings.weight"]}, strict=True)
    return ours, hf


@pytest.mark.parametrize("name,count", [("mamba-130m", 129_135_360), ("mamba-370m", 371_516_416)])
def test_parameter_counts_match_transformers(name, count):
    entry = MODEL_REGISTRY[name]
    c = entry.config
    with torch.device("meta"):
        hf = _hf(c.hidden, c.layers, c.vocab_size)
    assert sum(p.numel() for p in hf.parameters()) == count
    with torch.device("meta"):
        ours = build_model(name)
    assert sum(p.numel() for p in ours.parameters()) == count
    assert set(hf.state_dict()) - set(ours.state_dict()) == {"lm_head.weight"}
    for k, v in ours.state_dict().items():
        assert tuple(hf.state_dict()[k].shape) == tuple(v.shape), k
    assert tuple(ours.state_dict()["backbone.layers.0.mixer.conv1d.weight"].shape) == (2 * c.hidden, 1, 4)


def test_registry_entries():
    for name, hidden, layers in (("mamba-130m", 768, 24), ("mamba-370m", 1024, 48)):
        e = MODEL_REGISTRY[name]
        c = e.config
        assert e.kind == "causal" and e.start_id == 1 and not e.fp8 and not e.moe and c.max_position == 2048
        assert (c.hidden, c.layers, c.intermediate, c.rank, c.state, c.vocab_size) == (hidden, layers, 2 * hidden,
                                                                                     math.ceil(hidden / 16), 16, 50280)
        with pytest.raises(TypeError):
            e.build(fp8=True)


def test_load_hf_state_dict_is_strict():
    torch.manual_seed(1)
    hf = _hf()
    ours = MambaForCausalLM(MambaConfig(vocab_size=VOCAB, hidden=HIDDEN, layers=LAYERS))
    ours.load_hf_state_dict(hf.state_dict())
    for k, v in ours.state_dict().items():
        assert torch.equal(v, hf.state_dict()[k]), k
    bad = dict(hf.state_dict())
    bad.pop("backbone.layers.1.mixer.D")
    with pytest.raises(RuntimeError):
        ours.load_hf_state_dict(bad)


def test_initialisation_scheme():
    torch.manual_seed(0)
    m = MambaForCausalLM(MambaConfig(hidden=256, layers=2, vocab_size=512))
    mix = m.backbone.layers[0].mixer
    E, R = 512, 16
    assert torch.equal(mix.A_log, torch.log(torch.arange(1, 17.0)).repeat(E, 1)) and torch.equal(mix.D, torch.ones(E))
    dt = F.softplus(mix.dt_proj.bias)
    assert dt.min() >= 1e-3 * 0.999 and dt.max() <= 0.1 * 1.001
    assert mix.dt_proj.weight.abs().max() <= R ** -0.5
    assert torch.equal(mix.conv1d.bias, torch.zeros(E))
    assert mix.conv1d.weight.abs().max() <= 1 / math.sqrt(4) and mix.out_proj.weight.abs().max() <= 1 / math.sqrt(E)
    for w in (mix.in_proj.weight, mix.x_proj.weight, m.backbone.embeddings.weight):
        assert abs(w.std().item() - 0.1) < 0.01 and abs(w.mean().item()) < 0.01
    bf = to_mixed_bf16(m)
    assert mix.A_log.dtype == mix.D.dtype == mix.dt_proj.bias.dtype == torch.float32
    assert mix.in_proj.weight.dtype == mix.dt_proj.weight.dtype == torch.bfloat16 and bf is m


def _rel(a, b):
    return float((a - b).norm() / b.norm())


@pytest.mark.parametrize("seed", [0, 1])
def test_fp32_model_matches_transformers(seed):
    ours, hf = _pair(seed)
    ids = torch.randint(1, VOCAB, (2, 37))
    w = torch.randn(2, 37, VOCAB)
    lo = ours(ids)
    lh = hf(ids).logits
    assert _rel(lo, lh) < 1e-5
    (lo * w).sum().backward()
    (lh * w).sum().backward()
    hp = dict(hf.named_parameters())
    for k, p in ours.named_parameters():
        assert _rel(p.grad, hp[k].grad) < 1e-5, k


def test_packed_rows_equal_each_document_alone():
    torch.manual_seed(2)
    ours, hf = _pair(2)
    ours.config.bos_token_id, ours.config.pad_token_id = 1, 0
    ids = torch.randint(2, VOCAB, (2, 40))
    ids[0, [0, 13, 29]] = 1
    ids[1, [0, 21]] = 1
    ids[1, 33:] = 0
    with torch.no_grad():
        lo = ours(ids)
        for b, starts, end in ((0, [0, 13, 29], 40), (1, [0, 21], 33)):
            for s, e in zip(starts, starts[1:] + [end]):
                alone = hf(ids[b:b + 1, s:e]).logits[0]
                assert _rel(lo[b, s:e], alone) < 1e-5, (b, s)


def test_right_padded_rows_equal_transformers_at_real_positions():
    ours, hf = _pair(3)
    ours.config.pad_token_id = 0
    ids = torch.randint(1, VOCAB, (3, 30))
    lens = [30, 17, 5]
    for b, n in enumerate(lens):
        ids[b, n:] = 0
    with torch.no_grad():
        lo = ours(ids)
        for b, n in enumerate(lens):
            assert _rel(lo[b, :n], hf(ids[b:b + 1, :n]).logits[0]) < 1e-5, b


def test_reference_ops_reset_at_document_starts_and_check_shapes():
    torch.manual_seed(4)
    B, S, E, R = 2, 19, 8, 4
    xz = torch.randn(B, S, 2 * E, dtype=torch.float64)
    xbc = torch.randn(B, S, R + 32, dtype=torch.float64)
    dr = torch.randn(B, S, E, dtype=torch.float64)
    w, bias = torch.randn(E, 1, 4, dtype=torch.float64), torch.randn(E, dtype=torch.float64)
    A_log, D, dtb = torch.rand(E, 16, dtype=torch.float64), torch.randn(E, dtype=torch.float64), torch.randn(E, dtype=torch.float64)
    ids = torch.full((B, S), 5)
    ids[0, 7] = 1
    ids[1, 15:] = 0
    bounds, _ = document_bounds(ids, 1, 0)
    u = causal_conv1d(xz, w, bias, bounds)
    y = selective_scan(u, dr, xbc, xz, A_log, D, dtb, bounds)
    assert u.dtype == y.dtype == torch.float64
    assert (u[1, 15:] == 0).all() and (y[1, 15:] == 0).all()
    one = document_bounds(torch.full((1, S - 7), 5), None, None)[0]
    u1 = causal_conv1d(xz[:1, 7:], w, bias, one)
    y1 = selective_scan(u1, dr[:1, 7:], xbc[:1, 7:], xz[:1, 7:], A_log, D, dtb, one)
    assert torch.allclose(u[0, 7:], u1[0]) and torch.allclose(y[0, 7:], y1[0])
    with pytest.raises(ValueError):
        causal_conv1d(xz[..., :-1], w, bias, bounds)
    with pytest.raises(ValueError):
        selective_scan(u, dr, xbc[..., :20], xz, A_log, D, dtb, bounds)
    with pytest.raises(ValueError):
        selective_scan(u, dr, xbc, xz, A_log[:, :8], D, dtb, bounds)


def _cli_args(tmp_path, model, *flags):
    from b200ddp.engine import cli
    return cli.build_parser().parse_args(["--no_tensorboard", "--output_dir", str(tmp_path / "out"), "--model", model, "--no_cuda", *flags])


@pytest.mark.parametrize("flags", [[], ["--min_seq_len", "32", "--seq_len", "128"], ["--pack", "--min_seq_len", "32", "--seq_len", "128"],
                                   ["--fused_lm_loss"], ["--cuda_graph"], ["--optimizer", "adamw", "--gradient_accumulation_steps", "2"],
                                   ["--seq_len", "2048"]])
@pytest.mark.parametrize("model", ["mamba-130m", "mamba-370m"])
def test_cli_accepts(tmp_path, model, flags):
    from b200ddp.engine import cli
    cli.setup(_cli_args(tmp_path, model, *flags))


@pytest.mark.parametrize("flags,match", [(["--fp8", "--fp16"], "--fp8"), (["--seq_len", "2049"], "2048")])
def test_cli_rejects(tmp_path, flags, match):
    from b200ddp.engine import cli
    with pytest.raises(ValueError, match=match):
        cli.setup(_cli_args(tmp_path, "mamba-130m", *flags))


def test_short_cpu_training_run_resumes(tmp_path, monkeypatch):
    from b200ddp import models
    from b200ddp.engine import cli
    from b200ddp.engine.trainer import Trainer
    from b200ddp.models import mamba as mm
    tiny = MambaConfig(hidden=32, layers=1, vocab_size=128)
    monkeypatch.setitem(models.MODEL_REGISTRY, "mamba-130m", models.ModelEntry(
        lambda **kw: mm._build(tiny, kw.get("pad_token_id"), kw.get("bos_token_id"), kw.get("fused_lm_loss", False)),
        "causal", tiny, start_id=1))
    flags = ["--per_gpu_train_batch_size", "2", "--max_steps", "2", "--logging_steps", "1", "--save_steps", "2", "--optimizer", "adamw",
             "--lr", "1e-4", "--dataset_size", "8", "--seq_len", "64", "--min_seq_len", "16", "--pack"]
    args = _cli_args(tmp_path, "mamba-130m", *flags)
    cli.setup(args)
    step, loss = Trainer(args, build_model("mamba-130m", pad_token_id=0, bos_token_id=1), cli.log).train()
    assert step == 3 and math.isfinite(loss) and loss > 0
    args = _cli_args(tmp_path, "mamba-130m", *flags[:5], "4", *flags[6:], "--resume_from", "latest")
    cli.setup(args)
    step, loss = Trainer(args, build_model("mamba-130m", pad_token_id=0, bos_token_id=1), cli.log).train()
    assert step >= 3 and math.isfinite(loss)


def _free_port():
    import socket
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _gloo_model():
    torch.manual_seed(0)
    return MambaForCausalLM(MambaConfig(vocab_size=VOCAB, hidden=32, layers=1)).double()


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
