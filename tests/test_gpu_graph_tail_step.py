"""A CUDA-graph training step that meets an odd-shaped batch (the last, partial batch of an epoch) runs it eagerly between
two replays.  bert-base at seq 512, right-padded and packed: through the trainer (pinned loader, device prefetcher, graph),
and at the TrainStep level, where the replay after the eager step must compute the loss an eager forward computes."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("packed", [False, True])
def test_trainer_replays_after_an_eager_tail_batch(tmp_path, packed):
    """512 right-padded rows in batches of 24, or 351 packed rows in batches of 16: each epoch ends with a partial batch
    (8 or 15 rows) that runs eagerly after the graph was captured, and the next epoch's batches replay the graph."""
    from b200ddp.engine import cli
    from b200ddp.engine.trainer import Trainer
    from b200ddp.models import build_model
    argv = ["--model", "bert-base", "--fp16", "--optimizer", "adamw", "--cuda_graph", "--max_steps", "26", "--seq_len", "512",
            "--min_seq_len", "128", "--per_gpu_train_batch_size", "16" if packed else "24", "--weight_decay", "0.01",
            "--save_steps", "0", "--logging_steps", "25", "--no_tensorboard", "--output_dir", str(tmp_path / "out")]
    args = cli.build_parser().parse_args(argv + (["--pack"] if packed else []))
    cli.setup(args)
    kwargs = {"pad_token_id": 0, **({"cls_token_id": 101} if packed else {})}
    trainer = Trainer(args, build_model("bert-base", **kwargs), cli.log)
    assert len(trainer.dataset) % args.train_batch_size and len(trainer.loader) == 22
    steps, loss = trainer.train()
    torch.cuda.synchronize()
    assert trainer.step_fn.graph is not None and trainer.step_fn._eager_iters == 4   # 3 warm-up steps + the tail batch
    assert steps == 27 and math.isfinite(loss)
    assert math.isfinite(trainer.evaluate(max_batches=2)["eval_loss"])


@pytest.mark.parametrize("packed", [False, True])
def test_replay_after_an_eager_step_computes_the_eager_loss(packed):
    from b200ddp.data import SyntheticTokens
    from b200ddp.engine.step import TrainStep
    from b200ddp.models import bert_base
    from b200ddp.ops import CrossEntropyLoss
    from b200ddp.optim import FusedAdamW, weight_decay_groups
    from b200ddp.utils import to_mixed_bf16
    torch.manual_seed(0)
    ds = SyntheticTokens(samples=64, seq_len=512, min_len=128, pack=packed)
    dev = torch.device("cuda", 0)
    x, y = ds.X[:16].to(dev), ds.Y[:16].to(dev)
    xt, yt = ds.X[16:31].to(dev), ds.Y[16:31].to(dev)           # 15 rows
    model = to_mixed_bf16(bert_base(pad_token_id=ds.pad_token_id, cls_token_id=ds.cls_token_id).to(dev))
    opt = FusedAdamW(weight_decay_groups(model, 0.01), lr=1e-4, max_grad_norm=1.0)
    crit = CrossEntropyLoss()
    step = TrainStep(model, crit, opt, dev, use_graph=True)
    for _ in range(5):                                           # three eager warm-up steps, the capture, one replay
        step(x, y)
    assert step.graph is not None
    step(xt, yt)                                                 # odd shape: eager, between replays
    torch.cuda.synchronize()
    with torch.no_grad():
        expect = float(crit(model(x), y))
    step(x, y)                                                   # replay after the eager step
    torch.cuda.synchronize()
    got = float(step._static_loss)
    assert math.isfinite(got) and abs(got - expect) < 1e-3 * abs(expect), (got, expect)
    assert all(torch.isfinite(p.float()).all() for p in model.parameters())
