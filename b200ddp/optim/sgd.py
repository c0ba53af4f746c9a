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

from typing import Dict, Iterable, List, Optional

import torch

from .. import _ext
from ..utils.precision import is_dense

_DTYPE_CODE = {torch.float32: 0, torch.bfloat16: 1}


class _NativeGroup:
    """All parameters of one dtype: one SgdPlan + slices of the flat state buffers."""

    def __init__(self, C, params: List[torch.nn.Parameter], flat_base: int):
        self.params = params
        self.numels = [p.numel() for p in params]
        self.offsets = []
        off = flat_base
        for n in self.numels:
            self.offsets.append(off)
            off += (n + 7) // 8 * 8
        self.flat_end = off
        code = _DTYPE_CODE[params[0].dtype]
        self.plan = C.SgdPlan([p.data_ptr() for p in params], self.numels, self.offsets, code, code)
        self.block_base = 0


class FusedSGD(torch.optim.Optimizer):
    def __init__(self, params: Iterable, lr: float = 1e-3, momentum: float = 0.0, dampening: float = 0.0,
                 weight_decay: float = 0.0, nesterov: bool = False, max_grad_norm: float = 0.0,
                 master_weights: Optional[bool] = None, grad_scale: float = 1.0):
        defaults = dict(lr=lr, momentum=momentum, dampening=dampening, weight_decay=weight_decay, nesterov=nesterov)
        super().__init__(params, defaults)
        if len(self.param_groups) != 1:
            raise ValueError("FusedSGD keeps one hyper-parameter group (the reference uses a single group)")
        self.max_grad_norm = float(max_grad_norm)
        self.grad_scale = float(grad_scale)
        self._params: List[torch.nn.Parameter] = [p for p in self.param_groups[0]["params"] if p.requires_grad]
        self._native = bool(self._params) and all(p.is_cuda for p in self._params)
        self._steps_host = 0
        self.last_grad_norm: Optional[torch.Tensor] = None
        if self._native:
            self._init_native(master_weights)

    # ------------------------------------------------------------------ native (CUDA) state
    def _init_native(self, master_weights: Optional[bool]) -> None:
        C = self.C = _ext.get()
        dev = self._params[0].device
        by_dtype: Dict[torch.dtype, List[torch.nn.Parameter]] = {}
        for p in self._params:
            if p.dtype not in _DTYPE_CODE:
                raise TypeError(f"FusedSGD supports fp32/bf16 parameters, got {p.dtype}")
            by_dtype.setdefault(p.dtype, []).append(p)
        self._groups: List[_NativeGroup] = []
        base = 0
        for dtype, ps in by_dtype.items():
            # keep parameter storage dense: the kernel walks physical order
            for p in ps:
                if not is_dense(p):
                    p.data = p.data.contiguous()
            g = _NativeGroup(C, ps, base)
            base = g.flat_end
            self._groups.append(g)
        self._flat_elems = base
        blocks = 0
        for g in self._groups:
            g.block_base = blocks
            blocks += g.plan.total_blocks
        self._own_partials = torch.zeros(max(blocks, 1), dtype=torch.float32, device=dev)
        self._lr_dev = torch.full((1,), float(self.param_groups[0]["lr"]), dtype=torch.float32, device=dev)
        self._coef_dev = torch.ones(1, dtype=torch.float32, device=dev)
        self._norm_dev = torch.zeros(1, dtype=torch.float32, device=dev)
        self._step_dev = torch.zeros(1, dtype=torch.int32, device=dev)
        need_master = any(p.dtype == torch.bfloat16 for p in self._params) if master_weights is None else master_weights
        self._master = None
        if need_master:
            self._master = torch.zeros(self._flat_elems, dtype=torch.float32, device=dev)
            for g in self._groups:
                for p, off, n in zip(g.params, g.offsets, g.numels):
                    self._master[off:off + n].copy_(_physical_flat(p.data).float())
        self._momentum_buf = None
        if self.param_groups[0]["momentum"] != 0.0:
            self._momentum_buf = torch.zeros(self._flat_elems, dtype=torch.float32, device=dev)

    def sync_lr_to_device(self) -> None:
        """Called by the scheduler after it changes ``param_groups[0]['lr']``."""
        if self._native:
            # The value travels as a kernel argument, so it is bound at enqueue time: a host that runs several steps
            # ahead of the GPU (prefetcher, graph replay) can never overwrite the lr of a step that has not executed yet
            # (a single pinned staging word + async copy could).
            self._lr_dev.fill_(float(self.param_groups[0]["lr"]))

    # ------------------------------------------------------------------ public API
    def clip_grad_norm_(self, max_norm: float) -> None:
        """API-parity shim: clipping is fused into ``step``; this only sets the threshold."""
        self.max_grad_norm = float(max_norm)

    @torch.no_grad()
    def step(self, closure=None, sq_partials: Optional[torch.Tensor] = None, zero_grad: bool = False):
        """``sq_partials``: per-block sums of squares of the (already reduced) gradients, e.g.
        ``ddp.reducer.grad_sq_partials()``; when given, the gradients are not re-read for the norm."""
        loss = closure() if closure is not None else None
        if not self._params:
            return loss
        if self._native:
            self._step_native(sq_partials, zero_grad)
        else:
            self._step_cpu()
        self._steps_host += 1
        return loss

    def _step_native(self, sq_partials: Optional[torch.Tensor], zero_grad: bool) -> None:
        group = self.param_groups[0]
        stream = torch.cuda.current_stream(self._params[0].device).cuda_stream
        grads_per_group = [[(p.grad.data_ptr() if p.grad is not None else 0) for p in g.params] for g in self._groups]
        clip_ptr = 0
        if self.max_grad_norm > 0.0:
            if sq_partials is None:
                for g, grads in zip(self._groups, grads_per_group):
                    g.plan.sqnorm(grads, self._own_partials.data_ptr() + 4 * g.block_base, stream)
                partials = self._own_partials
            else:
                partials = sq_partials.reshape(-1)
            self.C.clip_coef(partials, partials.numel(), self.max_grad_norm, self.grad_scale, self._coef_dev, self._norm_dev)
            self.last_grad_norm = self._norm_dev
            clip_ptr = self._coef_dev.data_ptr()
        master = self._master.data_ptr() if self._master is not None else 0
        mom = self._momentum_buf.data_ptr() if self._momentum_buf is not None else 0
        for g, grads in zip(self._groups, grads_per_group):
            g.plan.step(grads, self._lr_dev.data_ptr(), clip_ptr, master, mom, self._step_dev.data_ptr(),
                        float(group["momentum"]), float(group["dampening"]), float(group["weight_decay"]),
                        self.grad_scale, bool(group["nesterov"]), bool(zero_grad), stream)
        if self._momentum_buf is not None:
            self._step_dev.add_(1)

    def _step_cpu(self) -> None:
        group = self.param_groups[0]
        params = [p for p in self._params if p.grad is not None]
        if not params:
            return
        coef = self.grad_scale
        if self.max_grad_norm > 0.0:
            total = torch.sqrt(sum((p.grad.float() * self.grad_scale).pow(2).sum() for p in params))
            self.last_grad_norm = total
            coef = coef * float(torch.clamp(self.max_grad_norm / (total + 1e-6), max=1.0))
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

    def grad_norm(self) -> Optional[float]:
        """Host read of the last pre-clip gradient norm (synchronises; for logging only)."""
        return None if self.last_grad_norm is None else float(self.last_grad_norm)

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


def _physical_flat(t: torch.Tensor) -> torch.Tensor:
    """The tensor's elements in storage order (dense tensors only)."""
    if t.is_contiguous():
        return t.reshape(-1)
    return t.as_strided((t.numel(),), (1,))
