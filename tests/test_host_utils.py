"""Sampler / schedule / logger / CLI parity with the reference behaviour."""
import logging
import math
import re
import warnings

import pytest
import torch
from torch.utils.data.distributed import DistributedSampler

from b200ddp.engine.cli import build_parser
from b200ddp.optim import FusedSGD, get_linear_schedule_with_warmup, warmup_decay_factor
from b200ddp.parallel import ShardedSampler
from b200ddp.utils import get_logger_with_rank, redirect_warnings_to_logger


class _Sized:
    def __init__(self, n):
        self.n = n

    def __len__(self):
        return self.n


@pytest.mark.parametrize("n,world", [(10, 2), (17, 4), (100, 8), (3, 2), (100000, 8)])
@pytest.mark.parametrize("drop_last", [False, True])
def test_sampler_matches_torch(n, world, drop_last):
    if drop_last and n < world:
        pytest.skip("degenerate")
    for epoch in (0, 3):
        seen = []
        for r in range(world):
            a = ShardedSampler(_Sized(n), world, r, seed=7, drop_last=drop_last)
            b = DistributedSampler(_Sized(n), world, r, seed=7, drop_last=drop_last)
            a.set_epoch(epoch)
            b.set_epoch(epoch)
            la = list(a)
            assert la == list(b) and len(a) == len(b)
            seen += la
        if not drop_last:
            assert set(seen) == set(range(n))           # partition (with wrap-around padding)
            assert len(seen) == math.ceil(n / world) * world


def test_sampler_resume_skips_prefix():
    s = ShardedSampler(_Sized(50), 2, 1, seed=1)
    s.set_epoch(2)
    full = list(s)
    s.set_start_index(7)
    assert list(s) == full[7:]
    assert list(s) == full                              # one-shot


def test_schedule_values_match_reference_lambda():
    from torch import optim
    p = torch.nn.Parameter(torch.zeros(1))
    warm, total = 10, 50

    def lr_lambda(step):                                # reference ddp.py:53-59 semantics
        if step < warm:
            return float(step) / float(max(1, warm))
        return max(0.0, float(total - step) / float(max(1, total - warm)))

    ref_opt = optim.SGD([p], lr=1e-3)
    ref = optim.lr_scheduler.LambdaLR(ref_opt, lr_lambda)
    mine_opt = FusedSGD([torch.nn.Parameter(torch.zeros(1))], lr=1e-3)
    mine = get_linear_schedule_with_warmup(mine_opt, warm, total)
    for step in range(60):
        assert mine.get_last_lr()[0] == pytest.approx(ref.get_last_lr()[0], abs=1e-12)
        assert warmup_decay_factor(step, warm, total) == pytest.approx(lr_lambda(step))
        ref_opt.step(); ref.step(); mine.step()
    sd = mine.state_dict()
    again = get_linear_schedule_with_warmup(FusedSGD([torch.nn.Parameter(torch.zeros(1))], lr=1e-3), warm, total)
    again.load_state_dict(sd)
    assert again.get_last_lr() == mine.get_last_lr()


def test_logger_line_shape_and_rank_gating(capsys):
    log = get_logger_with_rank("t_main", 3, 0)
    log.info("Finished training.", dict(global_step=31, average_loss=1.5))
    out = capsys.readouterr().out.strip()
    pat = (r"^\[\d{4}-\d\d-\d\d \d\d:\d\d:\d\d\.\d{3}[+-]\d{4}\] \[INFO    \] \[3 \^ 0\] \[test_host_utils\] "
           r"\[test_host_utils\.py:\d+\] \[Finished training\.\] \[global_step=31\] \[average_loss=1\.5\]$")
    assert re.match(pat, out), out
    quiet = get_logger_with_rank("t_other", 1, 1)
    assert quiet.level == logging.WARNING and not quiet.propagate
    quiet.info("hidden")
    quiet.warning("shown")
    out = capsys.readouterr().out
    assert "hidden" not in out and "[shown]" in out and "[1 ^ 1]" in out


def test_logger_file_handler_and_warning_redirect(tmp_path, capsys):
    path = tmp_path / "rank{rank}.log"
    log = get_logger_with_rank("t_file", 0, -1, log_file=str(path))
    old = warnings.showwarning
    try:
        redirect_warnings_to_logger(log)
        warnings.warn("careful")
    finally:
        warnings.showwarning = old
    out = capsys.readouterr().out
    assert "[careful]" in out and "[filename=" in out and "[lineno=" in out
    assert "careful" in (tmp_path / "rank0.log").read_text()


def test_cli_reference_flags_and_defaults():
    args = build_parser().parse_args([])
    expect = dict(global_step=0, no_cuda=False, output_dir="outputs", seed=42, gradient_accumulation_steps=1,
                  per_gpu_train_batch_size=32, max_steps=0, logging_steps=100, save_steps=1000, num_train_epochs=10,
                  warmup_steps=100, max_grad_norm=1000.0, local_rank=-1, fp16=False, loss_scale=0, fp16_opt_level="O2")
    for k, v in expect.items():
        assert getattr(args, k) == v, k
    assert build_parser().parse_args(["--local-rank=3"]).local_rank == 3      # torch>=2 launcher spelling (Q7)
    assert build_parser().parse_args(["--local_rank", "2"]).local_rank == 2
    assert args.find_unused_parameters is True and args.model == "foo" and args.backend == "auto"
