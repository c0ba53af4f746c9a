"""FusedAdamW on the CPU path: parity with torch.optim.AdamW + clip_grad_norm_, static loss scaling, checkpoint
interchange with torch.optim.AdamW in both directions, and the --optimizer adamw training run with resume."""
import copy
import os

import pytest
import torch

from b200ddp.engine import cli
from b200ddp.engine.step import TrainStep
from b200ddp.engine.trainer import Trainer
from b200ddp.models import FooModel
from b200ddp.ops import MSELoss
from b200ddp.optim import FusedAdamW, weight_decay_groups

HYPER = dict(lr=0.05, betas=(0.8, 0.99), eps=1e-6)


def _pair(seed=0):
    torch.manual_seed(seed)
    a, b = FooModel(), FooModel()
    b.load_state_dict(a.state_dict())
    return a, b


def _step(models_opts, x, y, clip=None):
    for m, o in models_opts:
        o.zero_grad()
        torch.nn.functional.mse_loss(m(x), y).backward()
    if clip is not None:
        torch.nn.utils.clip_grad_norm_(models_opts[1][0].parameters(), clip)
    for _, o in models_opts:
        o.step()


def test_weight_decay_groups_split_by_ndim():
    groups = weight_decay_groups(FooModel(), 0.1)
    assert [tuple(p.shape) for p in groups[0]["params"]] == [(10, 10), (5, 10)]
    assert [tuple(p.shape) for p in groups[1]["params"]] == [(10,), (5,)]
    assert groups[0]["weight_decay"] == 0.1 and groups[1]["weight_decay"] == 0.0


def test_fused_adamw_cpu_matches_torch_adamw_with_clip():
    a, b = _pair()
    oa = FusedAdamW(weight_decay_groups(a, 0.1), max_grad_norm=0.05, **HYPER)
    ob = torch.optim.AdamW(weight_decay_groups(b, 0.1), **HYPER)
    for _ in range(5):
        _step([(a, oa), (b, ob)], torch.randn(16, 10), torch.randn(16, 5), clip=0.05)
    assert oa.grad_norm() is not None
    for pa, pb in zip(a.parameters(), b.parameters()):
        assert torch.allclose(pa, pb, atol=1e-6), float((pa - pb).abs().max())


def test_fused_adamw_static_loss_scale_is_transparent():
    a, b = _pair()
    sa = TrainStep(a, MSELoss(), FusedAdamW(weight_decay_groups(a, 0.1), max_grad_norm=0.5, **HYPER), torch.device("cpu"))
    sb = TrainStep(b, MSELoss(), FusedAdamW(weight_decay_groups(b, 0.1), max_grad_norm=0.5, **HYPER), torch.device("cpu"),
                   loss_scale=1024.0)
    for _ in range(5):
        x, y = torch.randn(16, 10), torch.randn(16, 5)
        la, lb = sa(x, y), sb(x, y)
        assert torch.allclose(la, lb, atol=1e-6)
    for p, q in zip(a.parameters(), b.parameters()):
        assert torch.allclose(p, q, atol=1e-6)


@pytest.mark.parametrize("direction", ["fused_to_torch", "torch_to_fused"])
def test_fused_adamw_state_dict_interchanges_with_torch(direction):
    a, b = _pair(1)
    make_fused = lambda m: FusedAdamW(weight_decay_groups(m, 0.1), **HYPER)          # noqa: E731
    make_torch = lambda m: torch.optim.AdamW(weight_decay_groups(m, 0.1), **HYPER)   # noqa: E731
    first, second = (make_fused, make_torch) if direction == "fused_to_torch" else (make_torch, make_fused)
    oa = first(a)
    for _ in range(3):
        _step([(a, oa)], torch.randn(16, 10), torch.randn(16, 5))
    b.load_state_dict(a.state_dict())
    ob = second(b)
    ob.load_state_dict(copy.deepcopy(oa.state_dict()))
    for _ in range(3):
        x, y = torch.randn(16, 10), torch.randn(16, 5)
        _step([(a, oa), (b, ob)], x, y)
    for pa, pb in zip(a.parameters(), b.parameters()):
        assert torch.allclose(pa, pb, atol=1e-6), float((pa - pb).abs().max())


def test_fused_adamw_rejects_amsgrad_and_maximize():
    with pytest.raises(ValueError, match="amsgrad"):
        FusedAdamW(FooModel().parameters(), amsgrad=True)
    with pytest.raises(ValueError, match="maximize"):
        FusedAdamW(FooModel().parameters(), maximize=True)


def _run(tmp_path, *flags):
    args = cli.build_parser().parse_args(["--no_cuda", "--no_tensorboard", "--output_dir", str(tmp_path / "out"),
                                          "--dataset_size", "640", *flags])
    cli.setup(args)
    trainer = Trainer(args, FooModel(), cli.log)
    return trainer, trainer.train()


def test_adamw_run_checkpoints_and_resumes(tmp_path):
    common = ["--optimizer", "adamw", "--lr", "1e-2", "--weight_decay", "0.01", "--adam_beta2", "0.98", "--seed", "3",
              "--warmup_steps", "2"]
    t1, (gs, avg) = _run(tmp_path, "--max_steps", "10", "--save_steps", "10", *common)
    assert isinstance(t1.optimizer, FusedAdamW) and gs == 11 and avg > 0
    assert [g["weight_decay"] for g in t1.optimizer.param_groups] == [0.01, 0.0]
    assert t1.optimizer.param_groups[0]["betas"] == (0.9, 0.98)
    saved = torch.load(tmp_path / "out" / "checkpoint-10" / "optimizer.pt", weights_only=False)
    assert float(saved["state"][0]["step"]) == 9 and set(saved["state"][0]) == {"step", "exp_avg", "exp_avg_sq"}
    w_after_10 = torch.load(tmp_path / "out" / "checkpoint-10" / "model.bin")["net1.weight"]
    t2, (gs, _) = _run(tmp_path, "--max_steps", "14", "--save_steps", "0", "--resume_from", "latest", *common)
    assert t2._resume_state["global_step"] == 10 and gs == 15
    assert float(t2.optimizer.state[t2.model.net1.weight]["step"]) == 9 + 5      # 9 steps before the save + 5 after resume
    assert not torch.equal(t2.model.net1.weight.detach(), w_after_10)
    assert os.listdir(tmp_path / "out") == ["checkpoint-10"]
