"""Sparse masked-LM prediction (``linear_cross_entropy(sparse=True)``, ``--sparse_prediction``) on the CPU: the op against
``sparse=False`` including a trained bias, ``compact_rows``, tiny BERT and ModernBERT with and without the flag, Hugging
Face's ``ModernBertForMaskedLM(sparse_prediction=True)``, the CLI, checkpoints across the flag, a training run and a gloo
world-2 DDP run."""
import math
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from b200ddp.ops import CrossEntropyLoss, LinearCrossEntropyLoss, compact_rows, linear_cross_entropy


def _grads(fn, *ts):
    ts = [t.detach().clone().requires_grad_(True) for t in ts]
    loss = fn(*ts)
    loss.backward()
    return loss.detach(), [t.grad for t in ts]


@pytest.mark.parametrize("case", ["mixed", "all_ignored", "none_ignored"])
def test_sparse_op_equals_dense_in_loss_and_gradients_of_hidden_weight_and_bias(case):
    g = torch.Generator().manual_seed(0)
    h, w, b = torch.randn(3, 11, 32, generator=g), torch.randn(96, 32, generator=g) * 0.3, torch.randn(96, generator=g)
    t = torch.randint(0, 96, (3, 11), generator=g)
    if case == "mixed":
        t[0, :3] = -100
        t[1, 4], t[2, 7], t[2, 8] = 96, -5, 200                   # >= V and negative targets are ignored too
    elif case == "all_ignored":
        t[:] = -100
    dense, dg = _grads(lambda h_, w_, b_: linear_cross_entropy(h_, w_, t, b_), h, w, b)
    sparse, sg = _grads(lambda h_, w_, b_: linear_cross_entropy(h_, w_, t, b_, sparse=True), h, w, b)
    assert torch.allclose(sparse, dense, atol=1e-6), (float(sparse), float(dense))
    for a, e in zip(sg, dg):
        assert torch.allclose(a, e, atol=1e-6)
    ignored = (t == -100) | (t < 0) | (t >= 96)
    assert (sg[0][ignored] == 0).all()
    if case == "all_ignored":
        assert float(sparse) == 0.0 and all((x == 0).all() for x in sg)


def test_compact_rows_is_a_stable_partition_with_ignored_targets_after_the_count():
    t = torch.tensor([5, -100, 7, 40, 3, -1, -100, 0, 39])        # V = 40: 40 and -1 are unlabelled as well
    index, count, out = compact_rows(t, -100, 40)
    assert index.dtype == torch.int32 and count.dtype == torch.int32 and out.dtype == torch.int64
    assert int(count) == 5 and index.tolist() == [0, 2, 4, 7, 8, 1, 3, 5, 6]
    assert out.tolist() == [5, 7, 3, 0, 39, -100, -100, -100, -100]
    index, count, out = compact_rows(torch.tensor([2, 5, 2]), ignore_index=2)   # ignore_index inside the vocabulary
    assert int(count) == 1 and index.tolist() == [1, 0, 2] and out.tolist() == [5, 2, 2]
    with pytest.raises(ValueError, match="integer"):
        compact_rows(t.float())


def _tiny(family, sparse, **kw):
    if family == "bert":
        from b200ddp.models.bert import BertConfig, BertForMaskedLM
        return BertForMaskedLM(BertConfig(vocab_size=300, hidden=64, layers=2, heads=2, intermediate=128, max_position=64,
                                          pad_vocab_to=64, sparse_prediction=sparse, **kw))
    from b200ddp.models.modernbert import ModernBertConfig, ModernBertForMaskedLM
    return ModernBertForMaskedLM(ModernBertConfig(vocab_size=320, hidden=128, layers=4, heads=2, intermediate=192, max_position=64,
                                                  local_attention=16, sparse_prediction=sparse, **kw))


def _batch(vocab, seed=3):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(3, vocab, (2, 40), generator=g)
    labels = torch.where(torch.rand(2, 40, generator=g) < 0.15, ids, -100)
    return ids, labels


@pytest.mark.parametrize("family", ["bert", "modernbert"])
def test_sparse_model_matches_unfused_loss_and_every_gradient(family):
    torch.manual_seed(0)
    plain = _tiny(family, False)
    sparse = _tiny(family, True)
    assert set(sparse.state_dict()) == set(plain.state_dict())
    sparse.load_state_dict(plain.state_dict())
    with torch.no_grad():                                          # a non-zero decoder bias, so its use is checked too
        for m in (plain, sparse):
            bias = m.decoder_bias if family == "bert" else m.decoder.bias
            bias.copy_(torch.linspace(-0.5, 0.5, bias.numel()))
    ids, labels = _batch(300)
    loss_p = CrossEntropyLoss()(plain(ids), labels)
    loss_p.backward()
    head = sparse(ids)
    assert head.shape == (2, 40, 64 if family == "bert" else 128)
    crit = sparse.lm_head_loss()
    assert isinstance(crit, LinearCrossEntropyLoss) and crit.sparse and list(crit.parameters()) == []
    loss_s = crit(head, labels)
    loss_s.backward()
    assert torch.allclose(loss_s, loss_p, atol=1e-5), (float(loss_s), float(loss_p))
    gp = dict(plain.named_parameters())
    for n, p in sparse.named_parameters():
        assert p.grad is not None and torch.allclose(p.grad, gp[n].grad, atol=1e-5, rtol=1e-4), n


def test_sparse_modernbert_matches_hugging_face_sparse_prediction():
    transformers = pytest.importorskip("transformers")
    from b200ddp.models.modernbert import ModernBertConfig, ModernBertForMaskedLM
    torch.manual_seed(0)
    cfg = transformers.ModernBertConfig(vocab_size=512, hidden_size=128, intermediate_size=192, num_hidden_layers=4,
                                        num_attention_heads=2, max_position_embeddings=256, local_attention=16,
                                        pad_token_id=0, bos_token_id=1, eos_token_id=2, cls_token_id=1, sep_token_id=2,
                                        sparse_prediction=True, sparse_pred_ignore_index=-100)
    cfg._attn_implementation = "eager"
    hf = transformers.ModernBertForMaskedLM(cfg).eval()
    with torch.no_grad():
        hf.decoder.bias.uniform_(-0.5, 0.5)
    ours = ModernBertForMaskedLM(ModernBertConfig(vocab_size=512, hidden=128, layers=4, heads=2, intermediate=192, max_position=256,
                                                  local_attention=16, sparse_prediction=True)).eval()
    ours.load_hf_state_dict(hf.state_dict())
    ids, labels = _batch(512, seed=5)
    ref = hf(ids, labels=labels).loss
    ref.backward()
    loss = ours.lm_head_loss()(ours(ids), labels)
    loss.backward()
    loss, ref = float(loss.detach()), float(ref.detach())
    assert abs(loss - ref) < 1e-4, (loss, ref)
    theirs = dict(hf.named_parameters())
    for n, p in ours.named_parameters():
        assert torch.allclose(p.grad, theirs[n].grad, atol=1e-5, rtol=1e-3), n


def _args(tmp_path, *extra):
    from b200ddp.engine import cli
    return cli.build_parser().parse_args(["--no_tensorboard", "--output_dir", str(tmp_path / "out"), *extra])


def test_cli_accepts_and_rejects(tmp_path):
    from b200ddp.engine import cli
    for model in ("bert-base", "modernbert-base", "modernbert-large"):
        cli.setup(_args(tmp_path, "--model", model, "--no_cuda", "--sparse_prediction", "--seq_len", "256", "--min_seq_len", "64",
                        "--pack", "--gradient_accumulation_steps", "2", "--loss_scale", "128", "--loss", "ce"))
    for model in ("gpt2", "smollm-135m", "resnet50", "foo"):
        with pytest.raises(ValueError, match="masked-LM encoder"):
            cli.setup(_args(tmp_path, "--model", model, "--no_cuda", "--sparse_prediction"))
    with pytest.raises(ValueError, match="--loss ce"):
        cli.setup(_args(tmp_path, "--model", "bert-base", "--no_cuda", "--sparse_prediction", "--loss", "mse"))
    with pytest.raises(ValueError, match="sparse_prediction"):                # --fused_lm_loss stays causal-only, with a pointer
        cli.setup(_args(tmp_path, "--model", "bert-base", "--no_cuda", "--fused_lm_loss"))
    # the GPU-only rules, checked on an args object that looks like a GPU run (with --fp8, --cuda_graph and --min_seq_len)
    args = _args(tmp_path, "--model", "modernbert-base", "--sparse_prediction", "--fp8", "--cuda_graph", "--seq_len", "1024",
                 "--min_seq_len", "128")
    args.device, args.local_rank, args.n_gpu = torch.device("cuda"), -1, 1
    with pytest.raises(ValueError, match="--fp16"):
        cli.check_sparse_prediction_args(args)
    args.fp16 = True
    cli.check_sparse_prediction_args(args)
    cli.check_fp8_args(args)
    cli.check_min_seq_len_args(args)
    args.n_gpu = 2
    with pytest.raises(ValueError, match="DataParallel"):
        cli.check_sparse_prediction_args(args)
    args.local_rank = 0                                            # one process per GPU is fine
    cli.check_sparse_prediction_args(args)


def test_main_builds_the_model_with_the_flag(tmp_path, monkeypatch):
    from b200ddp.engine import cli
    seen = {}

    def fake_build(name, **kw):
        seen.update(kw, name=name)
        raise SystemExit(0)
    monkeypatch.setattr(cli, "build_model", fake_build)
    with pytest.raises(SystemExit):
        cli.main(["--no_tensorboard", "--output_dir", str(tmp_path / "out"), "--model", "bert-base", "--no_cuda",
                  "--sparse_prediction"])
    assert seen == {"name": "bert-base", "sparse_prediction": True}


def _train(tmp_path, sparse, steps, family="modernbert"):
    from b200ddp.engine import cli
    from b200ddp.engine.trainer import Trainer, build_dataset
    model_name = "modernbert-base" if family == "modernbert" else "bert-base"
    flags = ["--model", model_name, "--no_cuda", "--seq_len", "64", "--min_seq_len", "8", "--pack", "--optimizer", "adamw",
             "--lr", "3e-3", "--max_steps", str(steps), "--per_gpu_train_batch_size", "4", "--warmup_steps", "2",
             "--logging_steps", "10", "--save_steps", "0", "--seed", "3"]
    args = _args(tmp_path, *flags, *(["--sparse_prediction"] if sparse else []))
    cli.setup(args)
    ds = build_dataset(args)
    cls = ds.X == ds.cls_token_id                                  # a small alphabet leaves something to learn
    ds.X = torch.where(cls, torch.ones_like(ds.X), torch.where(ds.X > 0, ds.X % 16 + 2, ds.X))
    ds.Y = torch.where(ds.Y > 0, ds.Y % 16 + 2, ds.Y)
    ds.cls_token_id = 1
    torch.manual_seed(0)
    model = _tiny(family, sparse, pad_token_id=0, cls_token_id=1)
    return Trainer(args, model, cli.log, dataset=ds), model


def test_short_cpu_training_run_with_sparse_prediction_and_pack_lowers_the_loss(tmp_path):
    trainer, _ = _train(tmp_path, True, 30)
    assert isinstance(trainer.criterion, LinearCrossEntropyLoss) and trainer.criterion.sparse
    before = trainer.evaluate(max_batches=4)["eval_loss"]
    trainer.train()
    after = trainer.evaluate(max_batches=4)["eval_loss"]
    assert math.isfinite(after) and after < before - 0.1, (before, after)


@pytest.mark.parametrize("family", ["bert", "modernbert"])
@pytest.mark.parametrize("save_sparse", [True, False])
def test_checkpoint_loads_across_the_flag(tmp_path, family, save_sparse):
    from b200ddp.utils.checkpoint import latest_checkpoint, load_checkpoint
    trainer, model = _train(tmp_path, save_sparse, 3, family)
    trainer.train()
    trainer.save(0, 0)
    path = latest_checkpoint(str(tmp_path / "out"))
    other = _tiny(family, not save_sparse, pad_token_id=0, cls_token_id=1)
    load_checkpoint(path, other)
    for (n, a), (_, b) in zip(model.state_dict().items(), other.state_dict().items()):
        assert torch.equal(a, b), n
    ids, labels = _batch(18)
    plain, sparse = (other, model) if save_sparse else (model, other)
    with torch.no_grad():
        a, b = CrossEntropyLoss()(plain(ids), labels), sparse.lm_head_loss()(sparse(ids), labels)
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
    model = _tiny("bert", True)
    ddp = DistributedDataParallel(model, backend="gloo", find_unused_parameters=True)
    crit = model.lm_head_loss()
    opt = torch.optim.SGD(model.parameters(), lr=0.1)
    ids, labels = _batch(300, seed=11 + rank)                      # each rank its own batch and its own labelled rows
    crit(ddp(ids), labels).backward()
    grad = model.decoder_bias.grad
    assert grad is not None and float(grad.abs().sum()) > 0
    opt.step()
    for t in (grad, model.decoder_bias.detach(), model.bert.embeddings.word_embeddings.weight.detach()):
        got = [torch.empty_like(t) for _ in range(world)]
        dist.all_gather(got, t.contiguous())
        assert all(torch.equal(got[0], x) for x in got[1:])


def test_ddp_gloo_world2_leaves_identical_decoder_bias_gradients_and_parameters(free_port):
    _spawn(_check_ddp, 2, free_port)
