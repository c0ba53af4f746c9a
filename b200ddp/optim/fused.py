"""What the fused multi-tensor optimizers (``FusedSGD``, ``FusedAdamW``) share.

On CUDA, parameters are grouped per (param group, dtype); each group gets one native ``OptPlan`` (tables of at most 120
tensors, one kernel launch per table) and a slice of flat fp32 state buffers (masters, moments) whose per-tensor offsets
are rounded up to 8 elements so the kernels can use 32-byte vector accesses.  Gradient clipping runs once over *all*
groups: the sum-of-squares partials come from the DDP allreduce epilogue when given, otherwise from ``multi_sqnorm``,
and ``clip_coef`` turns them into a device scalar.  lr (one device scalar per param group), step count and clip
coefficient stay on the device, so a step captured into a CUDA graph bakes none of them.  CPU parameters use plain
tensor math (gloo plumbing config).
"""
from __future__ import annotations

from typing import Dict, List, Optional

import torch

from .. import _ext
from ..utils.precision import is_dense

_DTYPE_CODE = {torch.float32: 0, torch.bfloat16: 1}


class _NativeGroup:
    """All parameters of one dtype in one param group: one OptPlan + slices of the flat state buffers."""

    def __init__(self, C, params: List[torch.nn.Parameter], flat_base: int, group_index: int):
        self.params = params
        self.group_index = group_index
        self.numels = [p.numel() for p in params]
        self.offsets = []
        off = flat_base
        for n in self.numels:
            self.offsets.append(off)
            off += (n + 7) // 8 * 8
        self.flat_end = off
        code = _DTYPE_CODE[params[0].dtype]
        self.plan = C.OptPlan([p.data_ptr() for p in params], self.numels, self.offsets, code, code)
        self.block_base = 0


class FusedMultiTensorOptimizer(torch.optim.Optimizer):
    """Base of the fused optimizers: grouping, flat state, fused clip, ``step(closure, sq_partials, zero_grad)``.
    Subclasses implement ``_step_native_update`` and ``_step_cpu``."""

    def __init__(self, params, defaults: dict, max_grad_norm: float, master_weights: Optional[bool], grad_scale: float):
        super().__init__(params, defaults)
        self._validate_groups()
        self.max_grad_norm = float(max_grad_norm)
        self.grad_scale = float(grad_scale)
        self._params: List[torch.nn.Parameter] = [p for g in self.param_groups for p in g["params"] if p.requires_grad]
        self._native = bool(self._params) and all(p.is_cuda for p in self._params)
        self._steps_host = 0
        self.last_grad_norm: Optional[torch.Tensor] = None
        if self._native:
            self._init_native(master_weights)

    # ------------------------------------------------------------------ native (CUDA) state
    def _init_native(self, master_weights: Optional[bool]) -> None:
        C = self.C = _ext.get()
        dev = self._params[0].device
        self._groups: List[_NativeGroup] = []
        base = 0
        for gi, group in enumerate(self.param_groups):
            by_dtype: Dict[torch.dtype, List[torch.nn.Parameter]] = {}
            for p in group["params"]:
                if not p.requires_grad:
                    continue
                if p.dtype not in _DTYPE_CODE:
                    raise TypeError(f"{type(self).__name__} supports fp32/bf16 parameters, got {p.dtype}")
                by_dtype.setdefault(p.dtype, []).append(p)
            for dtype, ps in by_dtype.items():
                # keep parameter storage dense: the kernel walks physical order
                for p in ps:
                    if not is_dense(p):
                        p.data = p.data.contiguous()
                g = _NativeGroup(C, ps, base, gi)
                base = g.flat_end
                self._groups.append(g)
        self._flat_elems = base
        blocks = 0
        for g in self._groups:
            g.block_base = blocks
            blocks += g.plan.total_blocks
        self._own_partials = torch.zeros(max(blocks, 1), dtype=torch.float32, device=dev)
        self._lr_dev = torch.tensor([float(g["lr"]) for g in self.param_groups], dtype=torch.float32, device=dev)
        self._coef_dev = torch.ones(1, dtype=torch.float32, device=dev)
        self._norm_dev = torch.zeros(1, dtype=torch.float32, device=dev)
        self._step_dev = torch.zeros(1, dtype=torch.int32, device=dev)
        need_master = any(p.dtype == torch.bfloat16 for p in self._params) if master_weights is None else master_weights
        self._master = None
        if need_master:
            self._master = torch.zeros(self._flat_elems, dtype=torch.float32, device=dev)
            self._init_master()

    def _validate_groups(self) -> None:
        """Raise ValueError for param-group settings the subclass does not support."""

    def _init_master(self) -> None:
        for g in self._groups:
            for p, off, n in zip(g.params, g.offsets, g.numels):
                self._master[off:off + n].copy_(_physical_flat(p.data).float())

    def _flat_buffer(self) -> torch.Tensor:
        return torch.zeros(self._flat_elems, dtype=torch.float32, device=self._params[0].device)

    def _lr_ptr(self, group_index: int) -> int:
        return self._lr_dev.data_ptr() + 4 * group_index

    def sync_lr_to_device(self) -> None:
        """Called by the scheduler after it changes the param groups' ``lr``."""
        if self._native:
            # The value travels as a kernel argument, so it is bound at enqueue time: a host that runs several steps
            # ahead of the GPU (prefetcher, graph replay) can never overwrite the lr of a step that has not executed yet
            # (a single pinned staging word + async copy could).
            for i, group in enumerate(self.param_groups):
                self._lr_dev[i].fill_(float(group["lr"]))

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
        self._step_native_update(grads_per_group, clip_ptr, zero_grad, stream)

    def _step_native_update(self, grads_per_group, clip_ptr: int, zero_grad: bool, stream: int) -> None:
        raise NotImplementedError

    def _step_cpu(self) -> None:
        raise NotImplementedError

    def _cpu_grad_coef(self, params: List[torch.nn.Parameter]) -> float:
        """grad_scale times the clip coefficient of ``torch.nn.utils.clip_grad_norm_`` over ``params``."""
        coef = self.grad_scale
        if self.max_grad_norm > 0.0:
            total = torch.sqrt(sum((p.grad.float() * self.grad_scale).pow(2).sum() for p in params))
            self.last_grad_norm = total
            coef = coef * float(torch.clamp(self.max_grad_norm / (total + 1e-6), max=1.0))
        return coef

    def grad_norm(self) -> Optional[float]:
        """Host read of the last pre-clip gradient norm (synchronises; for logging only)."""
        return None if self.last_grad_norm is None else float(self.last_grad_norm)


def _physical_flat(t: torch.Tensor) -> torch.Tensor:
    """The tensor's elements in storage order (dense tensors only)."""
    if t.is_contiguous():
        return t.reshape(-1)
    return t.as_strided((t.numel(),), (1,))
