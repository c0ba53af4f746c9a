"""DistributedDataParallel - the H100-native replacement for ``torch.nn.parallel.DistributedDataParallel``
as the reference uses it (``ddp.py:194-195``: ``DistributedDataParallel(model, device_ids=[local_rank],
output_device=local_rank, find_unused_parameters=True)``).

Stock behaviour being replaced: parameter verification + rank-0 broadcast at wrap
time, per-parameter autograd hooks that copy ``grad/world`` into flat buckets, one NCCL allreduce per
bucket overlapped with the rest of backward, an extra allreduce of the unused-parameter bitmap,
copy-back into ``.grad``.

Native design:
* hooks are ``register_post_accumulate_grad_hook`` callbacks; they never touch gradient *data* on the
  b200 backend - they hand the gradient's device pointer to the C++ reducer (``csrc/reducer.cpp``),
  which, once a bucket's last gradient is enqueued, records an event on the compute stream and
  launches ONE fused kernel on a high-priority comm stream: gather(flatten) + 1/world scale + cast to
  the wire dtype + allreduce over NVSwitch peer memory (NVLS multimem / one-shot / two-shot) + cast
  back + scatter (+ sum-of-squares partial for clipping).  No NCCL call, no separate elementwise
  kernel on that path.
* the "which parameters were used" bitmap rides in the bucket itself (``BucketSpec.flags_offset``):
  no second collective (stock K5).
* ``no_sync()`` makes gradient accumulation skip communication on non-boundary micro-steps (the
  reference allreduces every micro-step).
* gloo / nccl backends run the same bucket plan through ``torch.distributed`` for CPU tests and for
  baseline comparison.
"""
from __future__ import annotations

import contextlib
import os
from typing import List, Optional

import torch
import torch.distributed as dist
import torch.nn as nn
from torch.autograd import Variable

from .backend import TorchCollectives, pick_backend_name
from .buckets import (BucketSpec, DEFAULT_BUCKET_CAP_BYTES, DEFAULT_FIRST_BUCKET_BYTES, MiB, plan_buckets)


class _PyReducer:
    """Bucket bookkeeping for the torch.distributed transports (gloo / nccl)."""

    def __init__(self, params: List[nn.Parameter], specs: List[BucketSpec], comm: TorchCollectives,
                 gradient_as_bucket_view: bool, find_unused: bool):
        self.params = params
        self.specs = specs
        self.comm = comm
        self.world = comm.world
        self.as_view = gradient_as_bucket_view
        self.find_unused = find_unused
        self.where = {}
        self.flats: List[torch.Tensor] = []
        self.views: List[List[torch.Tensor]] = []
        for spec in specs:
            p0 = params[spec.param_indices[0]]
            flat = torch.zeros(spec.total_elems, dtype=p0.dtype, device=p0.device)
            self.flats.append(flat)
            vs = []
            for k, (pi, off, n) in enumerate(zip(spec.param_indices, spec.offsets, spec.numels)):
                self.where[pi] = (spec.index, k)
                vs.append(flat[off:off + n].view(params[pi].shape))
            self.views.append(vs)
        self.stats = {"buckets_launched": 0, "bytes_reduced": 0, "iterations": 0}
        self.ready_order: List[int] = []
        self.reset()

    def reset(self) -> None:
        self.pending = [len(s.param_indices) for s in self.specs]
        self.fired = [[False] * len(s.param_indices) for s in self.specs]
        self.launched = [False] * len(self.specs)
        self.handles = [None] * len(self.specs)
        self.next_bucket = 0
        self.active = True
        self._order_now: List[int] = []

    def mark_ready(self, pi: int) -> None:
        if not self.active:        # second backward without an intervening forward: start a fresh pass, like Reducer::mark_ready
            self.reset()
        b, k = self.where[pi]
        if self.fired[b][k]:
            raise RuntimeError(
                f"parameter #{pi} produced a gradient twice in one backward pass; wrap shared/re-entrant "
                "use in no_sync() or run one backward per forward")
        p = self.params[pi]
        view = self.views[b][k]
        with torch.no_grad():
            if p.grad.data_ptr() == view.data_ptr():
                if self.world > 1:
                    view.mul_(1.0 / self.world)
            else:
                torch.mul(p.grad, 1.0 / self.world, out=view) if self.world > 1 else view.copy_(p.grad)
        self.fired[b][k] = True
        self._order_now.append(pi)
        self.pending[b] -= 1
        if self.pending[b] == 0:
            self._launch_in_order()

    def _launch_in_order(self) -> None:
        # buckets go out strictly in plan order so every rank issues the same sequence
        while self.next_bucket < len(self.specs) and self.pending[self.next_bucket] == 0:
            self._launch(self.next_bucket)
            self.next_bucket += 1

    def _launch(self, b: int) -> None:
        spec, flat = self.specs[b], self.flats[b]
        with torch.no_grad():
            if spec.total_elems > spec.flags_offset:
                # device-side fills only (no H2D copy): stays legal under CUDA-graph capture
                lo = spec.flags_offset
                flat[lo:lo + len(self.fired[b])].fill_(1.0)
                for k, f in enumerate(self.fired[b]):
                    if not f:
                        flat[lo + k:lo + k + 1].zero_()
        self.handles[b] = self.comm.allreduce_async(flat)
        self.launched[b] = True
        self.stats["buckets_launched"] += 1
        self.stats["bytes_reduced"] += flat.numel() * flat.element_size()

    def finalize(self) -> None:
        if not self.active:
            return
        self.active = False
        missing = [self.specs[b].param_indices[k] for b in range(len(self.specs))
                   for k, f in enumerate(self.fired[b]) if not f]
        if missing and not self.find_unused:
            raise RuntimeError(
                f"{len(missing)} parameter(s) (indices {missing[:8]}...) received no gradient in this backward "
                "pass; construct DistributedDataParallel(find_unused_parameters=True) if that is expected")
        with torch.no_grad():
            for b, spec in enumerate(self.specs):
                if self.launched[b]:
                    continue
                for k, f in enumerate(self.fired[b]):
                    if not f:
                        self.views[b][k].zero_()
                self.pending[b] = 0
            self._launch_in_order()
            for b, spec in enumerate(self.specs):
                if self.handles[b] is not None:
                    self.handles[b].wait()
                flat = self.flats[b]
                nflag = len(spec.param_indices)
                used = flat[spec.flags_offset:spec.flags_offset + nflag].float().cpu().tolist() \
                    if (missing and self.find_unused) else None
                for k, pi in enumerate(spec.param_indices):
                    p = self.params[pi]
                    if used is not None and not self.fired[b][k] and used[k] <= 0.0:
                        continue  # unused on every rank: leave .grad untouched (stock semantics)
                    view = self.views[b][k]
                    if self.as_view:
                        p.grad = view
                    elif p.grad is None:
                        p.grad = view.clone()
                    elif p.grad.data_ptr() != view.data_ptr():
                        p.grad.copy_(view)
        if self.stats["iterations"] == 0:
            self.ready_order = list(self._order_now)
        self.stats["iterations"] += 1


class DistributedDataParallel(nn.Module):
    def __init__(self, module: nn.Module, device_ids=None, output_device=None, process_group=None,
                 bucket_cap_mb: Optional[float] = None, first_bucket_mb: float = 1.0,
                 find_unused_parameters: bool = False, gradient_as_bucket_view: bool = False,
                 broadcast_buffers: bool = True, backend: str = "auto", wire_dtype: Optional[str] = None,
                 bucket_order: str = "backward", init_sync: bool = True, reduce_algo: str = "auto"):
        super().__init__()
        self.module = module
        self.device_ids = device_ids
        self.output_device = output_device
        self.process_group = process_group
        self.find_unused_parameters = find_unused_parameters
        self.gradient_as_bucket_view = gradient_as_bucket_view
        self.broadcast_buffers = broadcast_buffers
        self.require_backward_grad_sync = True
        self.bucket_cap_bytes = int((25.0 if bucket_cap_mb is None else bucket_cap_mb) * MiB)
        self.first_bucket_bytes = int(first_bucket_mb * MiB)
        self.wire_dtype = wire_dtype
        self.bucket_order = bucket_order

        self._params = [p for p in module.parameters() if p.requires_grad]
        if not self._params:
            raise RuntimeError("DistributedDataParallel needs at least one parameter that requires grad")
        self._names = {id(p): n for n, p in module.named_parameters()}
        device = self._params[0].device
        self.backend_name = pick_backend_name(backend, device, process_group)
        alone = not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(process_group) == 1
        if self.backend_name == "b200" and alone:
            self.backend_name = "single"           # nothing to reduce: no arena, no hooks
        if self.backend_name == "b200":
            from .peer import PeerCollectives
            grad_bytes = sum(p.numel() * max(4, p.element_size()) for p in self._params)
            self.comm = PeerCollectives.get(process_group, device, min_bytes=int(grad_bytes * 1.25))
        else:
            self.comm = TorchCollectives(process_group)
        self.world_size = self.comm.world
        self.rank = self.comm.rank

        self._verify_params_across_ranks()
        if init_sync:
            self.sync_module_states(src=0)

        keys = [(str(p.dtype), str(p.device)) for p in self._params]
        self._specs = plan_buckets([p.numel() for p in self._params], [p.element_size() for p in self._params],
                                   keys, self.bucket_cap_bytes, self.first_bucket_bytes, order=bucket_order)
        if self.backend_name == "b200":
            from .peer import NativeReducer
            self.reducer = NativeReducer(self._params, self._specs, self.comm, gradient_as_bucket_view,
                                         find_unused_parameters, wire_dtype=wire_dtype, algo=reduce_algo)
        else:
            self.reducer = _PyReducer(self._params, self._specs, self.comm, gradient_as_bucket_view,
                                      find_unused_parameters)
        self._callback_queued = False
        self._comm_stream = None
        self._buf_pending = None
        self._hook_handles = []
        if self.world_size > 1:   # a single rank has nothing to reduce: no hooks, zero overhead
            for i, p in enumerate(self._params):
                self._hook_handles.append(p.register_post_accumulate_grad_hook(self._make_hook(i)))

    # ---- wrap-time checks / broadcast -------------------------------------------------------
    def _verify_params_across_ranks(self) -> None:
        """Host-side shape/dtype agreement check over the store (stock N3 uses two NCCL collectives)."""
        if self.world_size == 1:
            return
        sig = [(tuple(p.shape), str(p.dtype)) for p in self._params]
        everyone = self.comm.allgather_object(sig)
        for r, other in enumerate(everyone):
            if other != sig:
                raise RuntimeError(f"parameter shapes/dtypes on rank {self.rank} differ from rank {r}")

    def sync_module_states(self, src: int = 0) -> None:
        """Rank ``src`` parameters + buffers reach every rank (stock ``_sync_module_states``, N4/K3)."""
        if self.world_size == 1:
            return
        tensors = [p.data for p in self.module.parameters()] + [b.data for b in self.module.buffers()]
        self.comm.broadcast_tensors(tensors, src=src)

    def _sync_buffers(self) -> None:
        if self.world_size == 1 or not self.broadcast_buffers:
            return
        bufs = [b.data for b in self.module.buffers()]
        if bufs:
            self.comm.broadcast_tensors(bufs, src=0)

    def _sync_buffers_after_forward(self) -> None:
        """Native backend: rank 0's buffers (BatchNorm running statistics) reach every rank on the COMM stream right after
        the forward pass, overlapped with backward, instead of on the compute stream before the forward pass (stock
        ``_sync_buffers``).  Training-mode forward never reads the running statistics, so at every forward
        start each rank still holds "rank 0's buffers as of its previous forward" - the stock contract - but the
        cross-GPU rendezvous of the broadcast kernel is off the critical path.  It is the first kernel on the comm stream
        of this iteration on every rank (bucket launches follow in plan order), and ``Reducer::finalize`` joins that
        stream back into the compute stream."""
        bufs = [b.data for b in self.module.buffers()]
        if not bufs:
            return
        cur = torch.cuda.current_stream(bufs[0].device)
        if self.reducer._c.runs_inline(cur.cuda_stream):
            # captured step: everything stays one linear chain on the compute stream (see ReducerOptions::serial)
            self.comm.broadcast_tensors(bufs, src=0)
            return
        if self._comm_stream is None:
            self._comm_stream = torch.cuda.ExternalStream(self.reducer._c.comm_stream(), device=bufs[0].device)
        fork = torch.cuda.Event()
        fork.record(cur)
        self._comm_stream.wait_event(fork)
        with torch.cuda.stream(self._comm_stream):
            self.comm.broadcast_tensors(bufs, src=0)
            done = torch.cuda.Event()
            done.record(self._comm_stream)
        self.reducer._c.note_comm_stream_used()
        self._buf_pending = done

    # ---- autograd plumbing -------------------------------------------------------------------
    def _make_hook(self, index: int):
        def hook(param):
            if not self.require_backward_grad_sync:
                return
            if not self._callback_queued:
                self._callback_queued = True
                Variable._execution_engine.queue_callback(self._finalize_backward)
            self.reducer.mark_ready(index)
        return hook

    def _finalize_backward(self) -> None:
        self._callback_queued = False
        self.reducer.finalize()
        self._buf_pending = None          # finalize joined the comm stream (buffer broadcast included) into the compute stream

    def forward(self, *inputs, **kwargs):
        sync = self.world_size > 1 and self.require_backward_grad_sync and torch.is_grad_enabled()
        overlap = sync and self.broadcast_buffers and self.backend_name == "b200"
        if sync:
            self.reducer.reset()
            if overlap:
                if self._buf_pending is not None:       # a forward that was never followed by backward: join its broadcast now
                    torch.cuda.current_stream().wait_event(self._buf_pending)
                    self._buf_pending = None
            else:
                self._sync_buffers()
        out = self.module(*inputs, **kwargs)
        if overlap:
            self._sync_buffers_after_forward()
        return out

    @contextlib.contextmanager
    def no_sync(self):
        """Skip gradient communication inside the context (accumulation micro-steps)."""
        previous = self.require_backward_grad_sync
        self.require_backward_grad_sync = False
        try:
            yield
        finally:
            self.require_backward_grad_sync = previous

    def set_graph_captured_loop(self, on: bool = True) -> None:
        """Tell the reducer that the training step will be replayed from a CUDA graph: its few eager warm-up steps then
        launch the communication kernels in line on the compute stream instead of on the comm stream (a third live stream
        slows every later graph replay down, see ``ReducerOptions::serial``); captured launches still fork and overlap."""
        self._graph_loop = bool(on)
        if hasattr(self.reducer, "_c") and hasattr(self.reducer._c, "set_eager_inline"):
            self.reducer._c.set_eager_inline(self._graph_loop)

    # ---- introspection -----------------------------------------------------------------------
    def bucket_sizes_mib(self) -> List[float]:
        return [round(sum(n * self._params[i].element_size() for i, n in zip(s.param_indices, s.numels)) / MiB, 2)
                for s in self._specs]

    def ddp_stats(self) -> dict:
        stats = dict(getattr(self.reducer, "stats", {}))
        stats.update(backend=self.backend_name, world_size=self.world_size, buckets=len(self._specs),
                     bucket_mib=self.bucket_sizes_mib())
        return stats

    def rebuild_buckets(self) -> bool:
        """Re-plan buckets by the gradient-ready order observed in the first iteration (stock Reducer
        does this once when ``find_unused_parameters=False``).  Deterministic across ranks
        because every rank runs the same graph; verified over the store."""
        order = list(getattr(self.reducer, "ready_order", []))
        if len(order) != len(self._params):
            return False
        if self.world_size > 1:
            everyone = self.comm.allgather_object(order)
            order = everyone[0]
        keys = [(str(p.dtype), str(p.device)) for p in self._params]
        self._specs = plan_buckets([p.numel() for p in self._params], [p.element_size() for p in self._params],
                                   keys, self.bucket_cap_bytes, self.first_bucket_bytes, ready_order=order)
        if hasattr(self.reducer, "rebuilt"):
            self._comm_stream = None                     # belongs to the reducer that is about to be destroyed
            self._buf_pending = None
            self.reducer = self.reducer.rebuilt(self._specs)
            if getattr(self, "_graph_loop", False):
                self.set_graph_captured_loop(True)
        else:
            self.reducer = _PyReducer(self._params, self._specs, self.comm, self.gradient_as_bucket_view,
                                      self.find_unused_parameters)
        return True

    def state_dict(self, *args, **kwargs):
        # checkpoints never carry a "module." prefix (reference ddp.py:72 unwraps before saving)
        return self.module.state_dict(*args, **kwargs)

    def load_state_dict(self, state_dict, *args, **kwargs):
        return self.module.load_state_dict(state_dict, *args, **kwargs)
