"""Fused SGD with built-in gradient clipping.

Reference behaviour: ``optim.SGD(model.parameters(), lr=1e-3)`` (``ddp.py:183``) preceded every step by
``clip_grad_norm_(model.parameters(), max_grad_norm)`` (``ddp.py:238-239``), with an (intended, broken)
apex O2 mixed-precision variant (``ddp.py:165-181``: fp16 model, fp32 master weights, FusedSGD).

Native design: on CUDA the whole "norm -> clip -> update" sequence is
  [sum-of-squares partials]  (free: written by the fused allreduce epilogue under DDP, otherwise one
                              multi-tensor launch reading the gradients where autograd left them)
  -> clip_coef                (one tiny block: sqrt, clamp - result stays on the device)
  -> multi_sgd                (clip * lr * g, weight decay, momentum, nesterov; fp32 master weights for
                              bf16 parameters; optional grad zeroing in the same pass)
with lr / step count / clip coefficient all device-resident so the step can live inside a CUDA graph.
CPU parameters use plain tensor math (gloo plumbing config).
"""
from __future__ import annotations

from typing import Iterable, Optional

from .fused import FusedMultiTensorOptimizer


class FusedSGD(FusedMultiTensorOptimizer):
    def __init__(self, params: Iterable, lr: float = 1e-3, momentum: float = 0.0, dampening: float = 0.0,
                 weight_decay: float = 0.0, nesterov: bool = False, max_grad_norm: float = 0.0,
                 master_weights: Optional[bool] = None, grad_scale: float = 1.0):
        defaults = dict(lr=lr, momentum=momentum, dampening=dampening, weight_decay=weight_decay, nesterov=nesterov)
        super().__init__(params, defaults, max_grad_norm, master_weights, grad_scale)

    def _validate_groups(self) -> None:
        if len(self.param_groups) != 1:
            raise ValueError("FusedSGD keeps one hyper-parameter group (the reference uses a single group)")

    def _init_native(self, master_weights: Optional[bool]) -> None:
        super()._init_native(master_weights)
        self._momentum_buf = None
        if self.param_groups[0]["momentum"] != 0.0:
            self._momentum_buf = self._flat_buffer()

    def _step_native_update(self, grads_per_group, clip_ptr: int, zero_grad: bool, stream: int) -> None:
        group = self.param_groups[0]
        master = self._master.data_ptr() if self._master is not None else 0
        mom = self._momentum_buf.data_ptr() if self._momentum_buf is not None else 0
        for g, grads in zip(self._groups, grads_per_group):
            g.plan.step(grads, self._lr_ptr(0), clip_ptr, master, mom, self._step_dev.data_ptr(),
                        float(group["momentum"]), float(group["dampening"]), float(group["weight_decay"]),
                        self.grad_scale, bool(group["nesterov"]), bool(zero_grad), stream)
        if self._momentum_buf is not None:
            self._step_dev.add_(1)

    def _step_cpu(self) -> None:
        group = self.param_groups[0]
        params = [p for p in self._params if p.grad is not None]
        if not params:
            return
        coef = self._cpu_grad_coef(params)
        lr, mu, damp, wd, nest = group["lr"], group["momentum"], group["dampening"], group["weight_decay"], group["nesterov"]
        for p in params:
            d = p.grad * coef
            if wd != 0.0:
                d = d.add(p, alpha=wd)
            if mu != 0.0:
                st = self.state[p]
                if "momentum_buffer" not in st:
                    st["momentum_buffer"] = d.clone()
                else:
                    st["momentum_buffer"].mul_(mu).add_(d, alpha=1.0 - damp)
                d = d.add(st["momentum_buffer"], alpha=mu) if nest else st["momentum_buffer"]
            p.add_(d, alpha=-lr)

    # ------------------------------------------------------------------ checkpointing
    def state_dict(self):
        sd = super().state_dict()
        if self._native:
            extra = {"steps": self._steps_host}
            if self._master is not None:
                extra["master"] = self._master.detach().cpu()
            if self._momentum_buf is not None:
                extra["momentum"] = self._momentum_buf.detach().cpu()
            sd["b200_fused"] = extra
        return sd

    def load_state_dict(self, state_dict):
        state_dict = dict(state_dict)
        extra = state_dict.pop("b200_fused", None)
        super().load_state_dict(state_dict)
        if self._native and extra:
            self._steps_host = int(extra.get("steps", 0))
            if self._master is not None and "master" in extra:
                self._master.copy_(extra["master"])
            if self._momentum_buf is not None and "momentum" in extra:
                self._momentum_buf.copy_(extra["momentum"])
                self._step_dev.fill_(self._steps_host)
        if self._native:
            self.sync_lr_to_device()

