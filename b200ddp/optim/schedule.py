"""Linear warmup -> linear decay learning-rate schedule.

Parity: reference ``ddp.py:52-61`` (factor rises 0->1 over ``warmup`` optimizer
steps, then falls linearly to 0 at ``total``).  The reference builds a
``LambdaLR``; here the schedule is a small host-side object whose
value is pushed into the optimizer's param groups *and*, for the fused CUDA
optimizer, into a device scalar so a captured CUDA graph never bakes the lr.
"""
from __future__ import annotations

from typing import List


def warmup_decay_factor(step: int, warmup: int, total: int) -> float:
    if step < warmup:
        return step / float(max(1, warmup))
    remaining = total - step
    return max(0.0, remaining / float(max(1, total - warmup)))


class LinearWarmupDecay:
    """Drop-in for the subset of the ``torch.optim.lr_scheduler`` API the
    training loop uses: ``step()``, ``get_last_lr()``, ``state_dict()``,
    ``load_state_dict()``."""

    def __init__(self, optimizer, num_warmup_steps: int, num_training_steps: int, last_step: int = 0):
        self.optimizer = optimizer
        self.num_warmup_steps = int(num_warmup_steps)
        self.num_training_steps = int(num_training_steps)
        self.base_lrs: List[float] = [g.setdefault("initial_lr", g["lr"]) for g in optimizer.param_groups]
        self.last_step = int(last_step)
        self._apply()

    def factor(self) -> float:
        return warmup_decay_factor(self.last_step, self.num_warmup_steps, self.num_training_steps)

    def _apply(self) -> None:
        f = self.factor()
        self._last_lr = [base * f for base in self.base_lrs]
        for group, lr in zip(self.optimizer.param_groups, self._last_lr):
            group["lr"] = lr
        sync = getattr(self.optimizer, "sync_lr_to_device", None)
        if sync is not None:
            sync()

    def step(self) -> None:
        self.last_step += 1
        self._apply()

    def get_last_lr(self) -> List[float]:
        return list(self._last_lr)

    def state_dict(self) -> dict:
        return {"last_step": self.last_step, "base_lrs": list(self.base_lrs),
                "num_warmup_steps": self.num_warmup_steps, "num_training_steps": self.num_training_steps}

    def load_state_dict(self, state: dict) -> None:
        self.last_step = int(state["last_step"])
        self.base_lrs = list(state.get("base_lrs", self.base_lrs))
        self.num_warmup_steps = int(state.get("num_warmup_steps", self.num_warmup_steps))
        self.num_training_steps = int(state.get("num_training_steps", self.num_training_steps))
        self._apply()


def get_linear_schedule_with_warmup(optimizer, num_warmup_steps: int, num_training_steps: int,
                                    last_epoch: int = -1) -> LinearWarmupDecay:
    """Reference-named constructor (``ddp.py:52``); ``last_epoch=-1`` means a fresh run."""
    return LinearWarmupDecay(optimizer, num_warmup_steps, num_training_steps, last_step=max(0, last_epoch + 1))
