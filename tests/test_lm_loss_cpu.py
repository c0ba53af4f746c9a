"""Fused LM-head cross-entropy (``ops.linear_cross_entropy``, ``--fused_lm_loss``) on the CPU: the op against
``cross_entropy(linear(...))``, the three causal LMs with and without the flag, the CLI, a training run, checkpoints across
the flag, and a gloo world-2 DDP run."""
import copy
import math
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from b200ddp.ops import CrossEntropyLoss, LinearCrossEntropyLoss, cross_entropy, linear, linear_cross_entropy


def _grads(fn, *ts):
    ts = [t.detach().clone().requires_grad_(True) for t in ts]
    loss = fn(*ts)
    loss.backward()
    return loss.detach(), [t.grad for t in ts]


@pytest.mark.parametrize("with_bias", [False, True])
def test_op_equals_cross_entropy_of_linear(with_bias):
    g = torch.Generator().manual_seed(0)
    h, w = torch.randn(3, 7, 32, generator=g), torch.randn(96, 32, generator=g) * 0.3
    b = torch.randn(96, generator=g) if with_bias else None
    t = torch.randint(0, 96, (3, 7), generator=g)
    t[0, :3] = -100
    loss, (dh, dw) = _grads(lambda h_, w_: linear_cross_entropy(h_, w_, t, b), h, w)
    ref, (rh, rw) = _grads(lambda h_, w_: cross_entropy(linear(h_, w_, b), t), h, w)
    assert torch.allclose(loss, ref, atol=1e-5) and torch.allclose(dh, rh, atol=1e-6) and torch.allclose(dw, rw, atol=1e-6)


def test_op_ignore_rules_and_all_ignored():
    g = torch.Generator().manual_seed(1)
    h, w = torch.randn(6, 16, generator=g), torch.randn(40, 16, generator=g)
    t = torch.tensor([3, -100, 40, -5, 39, 7])                # -100, >= V and negative targets are ignored
    loss, (dh, dw) = _grads(lambda h_, w_: linear_cross_entropy(h_, w_, t), h, w)
    keep = torch.tensor([0, 4, 5])
    ref, (rh, rw) = _grads(lambda h_, w_: cross_entropy(linear(h_[keep], w_), t[keep]), h, w)
    assert torch.allclose(loss, ref, atol=1e-5) and torch.allclose(dh, rh, atol=1e-6) and torch.allclose(dw, rw, atol=1e-6)
    assert (dh[[1, 2, 3]] == 0).all()
    loss0, (dh0, dw0) = _grads(lambda h_, w_: linear_cross_entropy(h_, w_, torch.full((6,), 5), ignore_index=5), h, w)
    assert float(loss0) == 0.0 and (dh0 == 0).all() and (dw0 == 0).all()
    with pytest.raises(ValueError, match="hidden"):
        linear_cross_entropy(h, w[:, :8], t)
    with pytest.raises(ValueError, match="integer"):
        linear_cross_entropy(h, w, t.float())


def _tiny(family, fused, **kw):
    if family == "gpt2":
        from b200ddp.models.gpt import GPTConfig, GPTLMHeadModel
        return GPTLMHeadModel(GPTConfig(vocab_size=500, max_position=64, hidden=64, layers=2, heads=2, intermediate=128,
                                        fused_lm_loss=fused, **kw))   # 500 rows padded to 512, the extra ones masked by the bias
    from b200ddp.models.llama import LlamaConfig, LlamaForCausalLM
    if family == "smollm":
        c = LlamaConfig(vocab_size=384, max_position=64, hidden=64, layers=2, heads=2, kv_heads=1, intermediate=96,
                        fused_lm_loss=fused, **kw)
    else:
        c = LlamaConfig(vocab_size=512, max_position=64, hidden=256, layers=1, heads=2, kv_heads=1, intermediate=128, eps=1e-6,
                        rope_theta=1e6, attention_bias=True, fused_lm_loss=fused, **kw)
    return LlamaForCausalLM(c)


@pytest.mark.parametrize("family", ["gpt2", "smollm", "qwen"])
def test_fused_model_matches_unfused_loss_and_gradients(family):
    torch.manual_seed(0)
    plain = _tiny(family, False)
    fused = _tiny(family, True)
    fused.load_state_dict(plain.state_dict())
    assert set(fused.state_dict()) == set(plain.state_dict())
    ids = torch.randint(1, 500 if family == "gpt2" else 384, (2, 24))
    labels = torch.cat([ids[:, 1:], torch.full((2, 1), -100)], 1)
    loss_p = CrossEntropyLoss()(plain(ids), labels)
    loss_p.backward()
    hidden = fused(ids)
    assert hidden.shape == (2, 24, fused.config.hidden)
    loss_f = fused.lm_head_loss()(hidden, labels)
    loss_f.backward()
    assert torch.allclose(loss_f, loss_p, atol=1e-5), (float(loss_f), float(loss_p))
    gp = dict(plain.named_parameters())
    for n, p in fused.named_parameters():
        assert torch.allclose(p.grad, gp[n].grad, atol=1e-5, rtol=1e-4), n


def test_criterion_follows_casts_of_the_model():
    m = _tiny("gpt2", True)
    crit = m.lm_head_loss()
    assert isinstance(crit, LinearCrossEntropyLoss) and list(crit.parameters()) == []
    m.to(torch.float64)
    w, b = crit.head()
    assert w is m.transformer.wte.weight and w.dtype == torch.float64 and b.dtype == torch.float64
    assert float(b[-1]) == -1e4 and float(b[499]) == 0.0


def _args(tmp_path, *extra):
    from b200ddp.engine import cli
    return cli.build_parser().parse_args(["--no_tensorboard", "--output_dir", str(tmp_path / "out"), *extra])


def test_cli_accepts_and_rejects(tmp_path):
    from b200ddp.engine import cli
    for model in ("gpt2", "smollm-135m", "qwen2.5-1.5b"):
        cli.setup(_args(tmp_path, "--model", model, "--no_cuda", "--fused_lm_loss", "--seq_len", "256", "--min_seq_len", "64",
                        "--pack", "--gradient_accumulation_steps", "2", "--loss", "ce"))
    with pytest.raises(ValueError, match="causal LM"):
        cli.setup(_args(tmp_path, "--model", "bert-base", "--no_cuda", "--fused_lm_loss"))
    with pytest.raises(ValueError, match="--loss ce"):
        cli.setup(_args(tmp_path, "--model", "gpt2", "--no_cuda", "--fused_lm_loss", "--loss", "mse"))
    # the GPU-only rules, checked on an args object that looks like a GPU run
    args = _args(tmp_path, "--model", "gpt2", "--fused_lm_loss")
    args.device, args.local_rank, args.n_gpu = torch.device("cuda"), -1, 1
    with pytest.raises(ValueError, match="--fp16"):
        cli.check_fused_lm_loss_args(args)
    args.fp16 = True
    cli.check_fused_lm_loss_args(args)
    args.n_gpu = 2
    with pytest.raises(ValueError, match="DataParallel"):
        cli.check_fused_lm_loss_args(args)
    args.local_rank = 0                                            # one process per GPU is fine
    cli.check_fused_lm_loss_args(args)


def _train(tmp_path, fused, steps):
    from b200ddp.engine import cli
    from b200ddp.engine.trainer import Trainer, build_dataset
    flags = ["--model", "smollm-135m", "--no_cuda", "--seq_len", "32", "--optimizer", "adamw", "--lr", "3e-3", "--max_steps",
             str(steps), "--per_gpu_train_batch_size", "4", "--warmup_steps", "2", "--logging_steps", "10",
             "--save_steps", "0", "--seed", "3"]
    args = _args(tmp_path, *flags, *(["--fused_lm_loss"] if fused else []))
    cli.setup(args)
    ds = build_dataset(args)
    ds.X, ds.Y = ds.X % 16, ds.Y % 16                              # a small alphabet leaves something to learn
    torch.manual_seed(0)
    model = _tiny("smollm", fused)
    return Trainer(args, model, cli.log, dataset=ds), model


def test_short_cpu_training_run_with_the_flag_lowers_the_loss(tmp_path):
    trainer, _ = _train(tmp_path, True, 30)
    assert isinstance(trainer.criterion, LinearCrossEntropyLoss)
    before = trainer.evaluate(max_batches=4)["eval_loss"]
    trainer.train()
    after = trainer.evaluate(max_batches=4)["eval_loss"]
    assert math.isfinite(after) and after < before - 0.1, (before, after)


@pytest.mark.parametrize("save_fused", [True, False])
def test_checkpoint_loads_across_the_flag(tmp_path, save_fused):
    from b200ddp.utils.checkpoint import latest_checkpoint, load_checkpoint
    trainer, model = _train(tmp_path, save_fused, 4)
    trainer.train()
    trainer.save(0, 0)
    path = latest_checkpoint(str(tmp_path / "out"))
    other = _tiny("smollm", not save_fused)
    load_checkpoint(path, other)
    for (n, a), (_, b) in zip(model.state_dict().items(), other.state_dict().items()):
        assert torch.equal(a, b), n
    ids = torch.randint(0, 16, (2, 32))
    labels = torch.roll(ids, -1, 1)
    plain, fused = (other, model) if save_fused else (model, other)
    with torch.no_grad():
        a, b = CrossEntropyLoss()(plain(ids), labels), fused.lm_head_loss()(fused(ids), labels)
    assert torch.allclose(a, b, atol=1e-5)


def _spawn(fn, world, port, *args):
    mp.spawn(_entry, args=(fn, world, port, args), nprocs=world, join=True)


def _entry(rank, fn, world, port, args):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.set_num_threads(1)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        fn(rank, world, *args)
    finally:
        dist.destroy_process_group()


def _check_ddp(rank, world):
    from b200ddp.parallel import DistributedDataParallel
    torch.manual_seed(0)
    model = _tiny("gpt2", True)
    ref = copy.deepcopy(model)
    ids = torch.randint(1, 500, (2 * world, 16), generator=torch.Generator().manual_seed(7))
    labels = torch.cat([ids[:, 1:], torch.full((2 * world, 1), -100)], 1)
    ref.lm_head_loss()(ref(ids), labels).backward()             # single process, global batch
    ddp = DistributedDataParallel(model, backend="gloo", find_unused_parameters=True)
    crit = model.lm_head_loss()
    crit(ddp(ids[rank::world]), labels[rank::world]).backward()  # equal valid rows per rank: the mean of the means
    expect = dict(ref.named_parameters())
    for n, p in model.named_parameters():
        assert p.grad is not None and torch.allclose(p.grad, expect[n].grad, atol=1e-5, rtol=1e-4), n


def test_ddp_gloo_world2_gradients_match_single_process(free_port):
    _spawn(_check_ddp, 2, free_port)
