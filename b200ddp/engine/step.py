"""One optimizer step as a unit (``TrainStep``) - eager, or captured once into a CUDA graph.

Reference hot loop (``ddp.py:216-243``): forward, loss, backward, two ``loss.item()`` host syncs,
``clip_grad_norm_`` (>=4 launches), ``optimizer.step()``, ``scheduler.step()``, ``model.zero_grad()``.
For the reference's own 165-parameter workload that loop is pure launch/sync latency.

Here the whole step - forward, fused loss fwd+bwd, backward with the DDP reducer's comm kernels forked
onto the comm stream, clip coefficient, fused SGD - is enqueued with no host synchronisation, and with
``use_graph=True`` it is captured once and replayed with a single launch per step.  The learning rate,
step counter and clip coefficient are device scalars, so nothing a scheduler changes is baked into the
graph.  The loss is accumulated on the device; the host reads it only when it logs.
"""
from __future__ import annotations

import contextlib
from typing import Callable, Optional

import torch


class TrainStep:
    def __init__(self, model, criterion, optimizer, device: torch.device, accumulation: int = 1, use_graph: bool = False,
                 input_transform: Optional[Callable] = None, target_transform: Optional[Callable] = None,
                 graph_warmup: int = 3, loss_scale: float = 1.0, paired: bool = False):
        self.model = model
        # paired inputs (CLIP's image-caption pairs, an encoder-decoder's source ids and labels): the model takes both,
        # model(x, y), and the criterion scores its output
        self.paired = bool(paired)
        self.criterion = criterion
        self.optimizer = optimizer
        self.device = torch.device(device)
        self.accumulation = max(1, int(accumulation))
        self.input_transform = input_transform
        self.target_transform = target_transform
        self.use_graph = bool(use_graph) and self.device.type == "cuda"
        self.graph_warmup = graph_warmup
        if self.use_graph and hasattr(model, "set_graph_captured_loop"):
            model.set_graph_captured_loop(True)
        # static loss scaling (the reference's --loss_scale, ddp.py:179/307): the loss is multiplied before backward and the
        # optimizer divides the gradients again inside the fused kernel (grad_scale); bf16 needs none, so the default is 1
        self.loss_scale = float(loss_scale) if loss_scale and loss_scale > 0 else 1.0
        if self.loss_scale != 1.0 and hasattr(optimizer, "grad_scale"):
            optimizer.grad_scale = 1.0 / self.loss_scale
        # accumulation == 1: one graph ("single").  accumulation > 1: a window of micro-steps replays "first" (gradients are
        # written into static buffers), "middle" x (accumulation - 2) (accumulate in place, no communication) and "last"
        # (accumulate, DDP reduction, clip + SGD) - three graphs over the same static gradient buffers and one memory pool.
        self.graph: Optional[torch.cuda.CUDAGraph] = None          # "single" or "last": the graph that holds the optimizer
        self._graphs = {}
        self._window_pos = 0
        self._rebuilt = False
        self._static_x = self._static_y = self._static_loss = None
        self._graph_shapes = None
        self._eager_iters = 0
        self.loss_sum = torch.zeros((), dtype=torch.float32, device=self.device)   # device-side running loss
        self.micro_steps = 0
        self.captured_native_launches = 0

    # ------------------------------------------------------------------------------------------
    def _reducer_partials(self):
        red = getattr(self.model, "reducer", None)
        if red is not None and getattr(self.model, "world_size", 1) > 1 and hasattr(red, "grad_sq_partials"):
            return red.grad_sq_partials()
        return None

    def _sync_ctx(self, boundary: bool):
        if not boundary and hasattr(self.model, "no_sync"):
            return self.model.no_sync()
        return contextlib.nullcontext()

    def _fwd_bwd(self, x, y, boundary: bool) -> torch.Tensor:
        with self._sync_ctx(boundary):
            out = self.model(x, y) if self.paired else self.model(x)
            loss = self.criterion(out, y)
            if self.accumulation > 1:
                loss = loss / self.accumulation
            (loss * self.loss_scale if self.loss_scale != 1.0 else loss).backward()
        return loss.detach()

    def _apply_optimizer(self) -> None:
        opt = self.optimizer
        if hasattr(opt, "_step_native"):
            opt.step(sq_partials=self._reducer_partials())
        else:
            if getattr(opt, "max_grad_norm", 0.0) and not hasattr(opt, "clip_grad_norm_"):
                torch.nn.utils.clip_grad_norm_(self.model.parameters(), opt.max_grad_norm)
            opt.step()

    # ------------------------------------------------------------------------------------------
    def _capture(self, x, y) -> None:
        self._static_x = torch.empty_like(x)
        self._static_y = torch.empty_like(y)
        self._static_x.copy_(x)
        self._static_y.copy_(y)
        self._graph_shapes = (tuple(x.shape), x.dtype, tuple(y.shape), y.dtype)
        side = torch.cuda.Stream(device=self.device)
        side.wait_stream(torch.cuda.current_stream(self.device))
        self.optimizer.zero_grad(set_to_none=True)
        counter = None
        try:
            from .. import _ext
            counter = _ext.get(build_if_missing=False).launch_count
        except Exception:
            pass
        before = counter() if counter else 0
        kinds = ["single"] if self.accumulation == 1 else (["first"] + (["middle"] if self.accumulation > 2 else []) + ["last"])
        pool = None
        self._static_loss = torch.zeros((), dtype=torch.float32, device=self.device)
        with torch.cuda.stream(side):
            for kind in kinds:
                g = torch.cuda.CUDAGraph()
                boundary = kind in ("single", "last")
                # "first" is captured with .grad == None, so autograd leaves freshly written gradients in static (pool)
                # buffers; the later captures find those tensors in .grad and accumulate into them in place
                # thread_local: the loader's helper threads keep gathering batches while this thread captures, and they
                # wait on a pinned slot's copy event before refilling it; in the default global mode that wait, from
                # another thread, invalidates the capture
                with torch.cuda.graph(g, stream=side, pool=pool, capture_error_mode="thread_local"):
                    loss = self._fwd_bwd(self._static_x, self._static_y, boundary)
                    if boundary:
                        self._apply_optimizer()
                    self._static_loss.copy_(loss.float() if loss.dtype != torch.float32 else loss)
                    self.loss_sum.add_(self._static_loss)
                pool = g.pool()
                self._graphs[kind] = g
        torch.cuda.current_stream(self.device).wait_stream(side)
        self.graph = self._graphs[kinds[-1]]
        # native (b200ddp extension) kernel launches recorded while capturing (one of each graph kind)
        self.captured_native_launches = (counter() - before) if counter else 0

    def _replay_kind(self) -> str:
        if self.accumulation == 1:
            return "single"
        if self._window_pos == 0:
            return "first"
        return "last" if self._window_pos == self.accumulation - 1 else "middle"

    def _graph_ok(self, x, y) -> bool:
        return self._graph_shapes == (tuple(x.shape), x.dtype, tuple(y.shape), y.dtype)

    # ------------------------------------------------------------------------------------------
    def __call__(self, x: torch.Tensor, y: torch.Tensor, boundary: bool = True) -> torch.Tensor:
        """Run one micro-step (and the optimizer when ``boundary``).  Returns the (device) loss of this
        micro-step; nothing here blocks the host."""
        if self.input_transform is not None:
            x = self.input_transform(x)
        if self.target_transform is not None:
            y = self.target_transform(y)
        self.micro_steps += 1
        if self.use_graph:
            if self.graph is None and self._eager_iters >= self.graph_warmup * self.accumulation and self._window_pos == 0:
                self._capture(x, y)
                # the capture itself does not execute; fall through to replay for this batch
            if self.graph is not None and self._graph_ok(x, y):
                if x.data_ptr() != self._static_x.data_ptr():
                    self._static_x.copy_(x, non_blocking=True)
                if y.data_ptr() != self._static_y.data_ptr():
                    self._static_y.copy_(y, non_blocking=True)
                kind = self._replay_kind()
                if (kind in ("single", "last")) != bool(boundary):
                    raise RuntimeError("TrainStep: `boundary` must be True exactly on every accumulation-th micro-step under --cuda_graph")
                self._graphs[kind].replay()
                self._window_pos = 0 if boundary else self._window_pos + 1
                return self._static_loss
        # eager path (CPU, graph warm-up, odd-shaped tail batch)
        if self.graph is not None and self._window_pos == 0:
            # grads are graph-owned static buffers: leave them in place, the eager pass accumulates into
            # fresh ones instead
            for p in self.model.parameters():
                if p.grad is not None:
                    p.grad = None
        loss = self._fwd_bwd(x, y, boundary)
        self.loss_sum.add_(loss.float())
        if boundary:
            self._apply_optimizer()
            self.optimizer.zero_grad(set_to_none=True)
            if not self._rebuilt:
                # what stock DDP does once after the first iteration when find_unused_parameters=False: re-plan
                # the buckets by the gradient-ready order just observed - before any graph is captured
                self._rebuilt = True
                if getattr(self.model, "world_size", 1) > 1 and hasattr(self.model, "rebuild_buckets") \
                        and not getattr(self.model, "find_unused_parameters", True):
                    self.model.rebuild_buckets()
        self._window_pos = 0 if boundary else self._window_pos + 1
        self._eager_iters += 1
        return loss

    def static_inputs(self):
        """Graph input buffers (None before capture): writers may fill them directly and skip a copy."""
        return self._static_x, self._static_y

    def read_loss_sum(self) -> float:
        """Host read of the running loss (synchronises)."""
        return float(self.loss_sum)
