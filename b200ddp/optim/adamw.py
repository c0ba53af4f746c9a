"""Fused AdamW (decoupled weight decay) with built-in gradient clipping and fp32 master weights.

The update is ``torch.optim.AdamW``'s, per element in fp32:
  g = g_in * clip_coef * grad_scale
  w = w * (1 - lr * weight_decay)
  m = lerp(m, g, 1 - beta1) ;  v = beta2 * v + (1 - beta2) * g * g
  w -= lr / (1 - beta1^t) * m / (sqrt(v) / sqrt(1 - beta2^t) + eps)
On CUDA it is one ``multi_adamw`` pass per (param group, dtype) after the shared clip (see ``fused.py``): gradients,
masters and both moments are read once and written once, and the gradient can be zeroed in the same pass.  The moments
live in flat fp32 buffers; bf16 parameters get fp32 masters, so updates smaller than bf16's resolution are not lost.

Step count: there is one device counter per optimizer, read by the kernel (so a step replayed from a CUDA graph advances
the bias correction).  ``torch.optim.AdamW`` keeps one per parameter; the two differ only for a parameter that missed
steps (its gradient was ``None``), whose bias correction here follows the optimizer's count.  The CPU path keeps
torch's per-parameter counts.

Checkpoints: ``state_dict()`` writes ``state`` in ``torch.optim.AdamW``'s layout (per parameter ``step``, ``exp_avg``,
``exp_avg_sq``) and the fp32 masters under ``"b200_fused"``, so a ``torch.optim.AdamW`` with the same groups can load it;
``load_state_dict()`` takes either kind of dict.
"""
from __future__ import annotations

import math
from typing import Iterable, List, Optional, Tuple

import torch

from .fused import FusedMultiTensorOptimizer, _physical_flat


class FusedAdamW(FusedMultiTensorOptimizer):
    def __init__(self, params: Iterable, lr: float = 1e-3, betas: Tuple[float, float] = (0.9, 0.999), eps: float = 1e-8,
                 weight_decay: float = 0.0, max_grad_norm: float = 0.0, master_weights: Optional[bool] = None,
                 grad_scale: float = 1.0, amsgrad: bool = False, maximize: bool = False):
        defaults = dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay, amsgrad=amsgrad, maximize=maximize)
        super().__init__(params, defaults, max_grad_norm, master_weights, grad_scale)

    def _validate_groups(self) -> None:
        for group in self.param_groups:
            if group.get("amsgrad", False):
                raise ValueError("FusedAdamW does not implement amsgrad")
            if group.get("maximize", False):
                raise ValueError("FusedAdamW does not implement maximize")
            b1, b2 = group["betas"]
            if not (0.0 <= b1 < 1.0 and 0.0 <= b2 < 1.0):
                raise ValueError(f"FusedAdamW: betas must lie in [0, 1), got {group['betas']}")
            if group["eps"] < 0.0 or group["lr"] < 0.0 or group["weight_decay"] < 0.0:
                raise ValueError("FusedAdamW: lr, eps and weight_decay must be >= 0")

    def _init_native(self, master_weights: Optional[bool]) -> None:
        super()._init_native(master_weights)
        self._exp_avg = self._flat_buffer()
        self._exp_avg_sq = self._flat_buffer()

    def _step_native_update(self, grads_per_group, clip_ptr: int, zero_grad: bool, stream: int) -> None:
        master = self._master.data_ptr() if self._master is not None else 0
        for g, grads in zip(self._groups, grads_per_group):
            group = self.param_groups[g.group_index]
            beta1, beta2 = group["betas"]
            g.plan.adamw(grads, self._lr_ptr(g.group_index), clip_ptr, master, self._exp_avg.data_ptr(),
                         self._exp_avg_sq.data_ptr(), self._step_dev.data_ptr(), float(beta1), float(beta2),
                         float(group["eps"]), float(group["weight_decay"]), self.grad_scale, bool(zero_grad), stream)
        self._step_dev.add_(1)

    def _step_cpu(self) -> None:
        params = [p for p in self._params if p.grad is not None]
        if not params:
            return
        coef = self._cpu_grad_coef(params)
        for group in self.param_groups:
            lr, (beta1, beta2), eps, wd = group["lr"], group["betas"], group["eps"], group["weight_decay"]
            for p in group["params"]:
                if p.grad is None or not p.requires_grad:
                    continue
                st = self.state[p]
                if not st:
                    st["step"] = torch.tensor(0.0, dtype=torch.float32)
                    st["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                g = p.grad * coef
                st["step"] += 1
                t = float(st["step"])
                p.mul_(1.0 - lr * wd)
                st["exp_avg"].lerp_(g, 1.0 - beta1)
                st["exp_avg_sq"].mul_(beta2).addcmul_(g, g, value=1.0 - beta2)
                step_size = lr / (1.0 - beta1 ** t)
                denom = (st["exp_avg_sq"].sqrt() / math.sqrt(1.0 - beta2 ** t)).add_(eps)
                p.addcdiv_(st["exp_avg"], denom, value=-step_size)

    # ------------------------------------------------------------------ checkpointing
    def _indices(self, saved_groups) -> dict:
        """id(parameter) -> its index in a state dict whose ``param_groups`` are ``saved_groups``."""
        index = {}
        for group, saved in zip(self.param_groups, saved_groups):
            for p, i in zip(group["params"], saved["params"]):
                index[id(p)] = i
        return index

    def state_dict(self):
        sd = super().state_dict()
        if not self._native:
            return sd
        steps = int(self._step_dev.item())     # the device count: graph replays never pass through step() on the host
        index = self._indices(sd["param_groups"])
        for g in self._groups:
            for p, off, n in zip(g.params, g.offsets, g.numels):
                sd["state"][index[id(p)]] = {"step": torch.tensor(float(steps), dtype=torch.float32),
                                             "exp_avg": _unflatten(self._exp_avg, p, off, n),
                                             "exp_avg_sq": _unflatten(self._exp_avg_sq, p, off, n)}
        extra = {"steps": steps}
        if self._master is not None:
            extra["master"] = self._master.detach().cpu()
        sd["b200_fused"] = extra
        return sd

    def load_state_dict(self, state_dict):
        state_dict = dict(state_dict)
        extra = state_dict.pop("b200_fused", None) or {}
        if not self._native:
            super().load_state_dict(state_dict)
            return
        state = state_dict.get("state", {})
        # the moments go straight into the flat buffers (torch's loader would cast them to the parameters' dtype)
        super().load_state_dict(dict(state_dict, state={}))
        self._validate_groups()
        index = self._indices(state_dict["param_groups"])
        steps = 0
        for g in self._groups:
            for p, off, n in zip(g.params, g.offsets, g.numels):
                st = state.get(index[id(p)])
                if st is None:
                    self._exp_avg[off:off + n].zero_()
                    self._exp_avg_sq[off:off + n].zero_()
                    continue
                _flatten_into(self._exp_avg, st["exp_avg"], p, off, n)
                _flatten_into(self._exp_avg_sq, st["exp_avg_sq"], p, off, n)
                steps = max(steps, int(float(st["step"])))
        steps = int(extra.get("steps", steps))
        self._steps_host = steps
        self._step_dev.fill_(steps)
        if self._master is not None:
            if "master" in extra:
                self._master.copy_(extra["master"])
            else:
                self._init_master()
        self.sync_lr_to_device()


def _unflatten(buf: torch.Tensor, p: torch.Tensor, off: int, n: int) -> torch.Tensor:
    """Slice ``[off, off + n)`` of a flat buffer (p's storage order) as a tensor shaped and laid out like ``p``."""
    out = torch.empty_like(p, dtype=torch.float32)
    _physical_flat(out).copy_(buf[off:off + n])
    return out


def _flatten_into(buf: torch.Tensor, value: torch.Tensor, p: torch.Tensor, off: int, n: int) -> None:
    tmp = torch.empty_like(p, dtype=torch.float32)
    tmp.copy_(value)
    buf[off:off + n].copy_(_physical_flat(tmp))


def weight_decay_groups(module: torch.nn.Module, weight_decay: float) -> List[dict]:
    """The usual two AdamW groups: matrices and convolution kernels (``ndim >= 2``) decay; biases, LayerNorm / BatchNorm
    affine parameters and the MLM ``decoder_bias`` (all ``ndim < 2``) get ``weight_decay=0``."""
    params = [p for p in module.parameters() if p.requires_grad]
    return [{"params": [p for p in params if p.ndim >= 2], "weight_decay": float(weight_decay)},
            {"params": [p for p in params if p.ndim < 2], "weight_decay": 0.0}]
