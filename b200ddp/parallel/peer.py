"""Python face of the NVSwitch peer-memory transport (``csrc/peer_mem.cpp``, ``allreduce.cu``,
``broadcast.cu``, ``reducer.cpp``).

Bootstrap (once per process group): rank 0 draws a job id, every rank creates its VMM arena, binds an
abstract unix socket, [store barrier], swaps POSIX FDs with every peer and maps all arenas into one
VA window; if every GPU reports multicast support the arenas are also bound to one NVLS multicast
object.  ``torch.distributed`` is used for those barriers / tiny object exchanges only - it is the
rendezvous, not the data path.
"""
from __future__ import annotations

import os
from typing import Dict, List, Optional, Sequence

import torch
import torch.distributed as dist

from .. import _ext
from ..utils.precision import is_dense
from .buckets import BucketSpec

MiB = 1 << 20
_DTYPE_CODE = {torch.float32: 0, torch.bfloat16: 1}
_WIRE_NAME = {"fp32": torch.float32, "float32": torch.float32, "bf16": torch.bfloat16, "bfloat16": torch.bfloat16}
_ALGO = {"auto": -1, "one_shot": 0, "two_shot": 1, "nvls": 2, "nvls_one_shot": 3}


class PeerCommError(RuntimeError):
    pass


class PeerCollectives:
    """One symmetric-memory arena + the generic collectives built on it."""

    _instances: Dict[int, "PeerCollectives"] = {}
    name = "b200"

    @classmethod
    def get(cls, group=None, device: Optional[torch.device] = None, min_bytes: int = 0) -> "PeerCollectives":
        key = id(group) if group is not None else 0
        inst = cls._instances.get(key)
        if inst is None:
            inst = cls(group, device, min_bytes)
            cls._instances[key] = inst
        return inst

    @classmethod
    def shutdown_all(cls) -> None:
        for inst in list(cls._instances.values()):
            inst.close()
        cls._instances.clear()

    def __init__(self, group=None, device: Optional[torch.device] = None, min_bytes: int = 0):
        self.C = _ext.get()
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        if device is None:
            device = torch.device("cuda", torch.cuda.current_device())
        self.device = device
        if self.world > 8:
            raise PeerCommError("the b200 backend spans one NVSwitch domain (<= 8 GPUs); use backend='nccl' across nodes")
        self.scratch_bytes = int(os.environ.get("B200DDP_SCRATCH_MB", "64")) * MiB
        arena_mb = int(os.environ.get("B200DDP_ARENA_MB", "0"))
        want = max(arena_mb * MiB, min_bytes + self.scratch_bytes + 16 * MiB)
        uid = [os.urandom(8).hex() + f"-{os.getpid()}"]
        if self.world > 1:
            dist.broadcast_object_list(uid, src=0, group=group)
        index = device.index if device.index is not None else torch.cuda.current_device()
        self.arena = self.C.PeerArena(self.rank, self.world, index, want, uid[0])
        self.arena.bind_socket()
        self._host_barrier()
        self.arena.exchange()
        self._host_barrier()
        self.nvls = False
        if self.world > 1 and os.environ.get("B200DDP_DISABLE_NVLS", "0") != "1":
            self._setup_multicast()
        self.scratch_off = self.arena.alloc(self.scratch_bytes, 4096)
        self.timeout_s = float(os.environ.get("B200DDP_TIMEOUT_S", "30"))
        self.blocks = int(os.environ.get("B200DDP_COMM_BLOCKS", "24"))
        self.tail_blocks = int(os.environ.get("B200DDP_TAIL_BLOCKS", "96"))
        self.closed = False
        if self.world > 1:
            # device-side rendezvous with a generous budget: absorbs first-launch skew between ranks (lazy module
            # loading, allocator warm-up) so the per-operation timeout only ever measures a peer that is really gone
            self.C.peer_barrier(self.arena, 1, 0, 120.0)
            torch.cuda.synchronize(self.device)
            self.check()
            self._host_barrier()

    # ---- bootstrap helpers --------------------------------------------------------------------
    def _host_barrier(self) -> None:
        if self.world > 1:
            self.allgather_object(0)

    def _agree(self, ok: bool) -> bool:
        return all(self.allgather_object(bool(ok)))

    def _setup_multicast(self) -> None:
        if not self._agree(self.arena.multicast_supported()):
            self.arena.disable_multicast()
            return
        ok = True
        for stage in ("multicast_create", "multicast_add_device", "multicast_bind"):
            try:
                if ok:
                    getattr(self.arena, stage)()
            except Exception:
                ok = False
            ok = self._agree(ok)
            if not ok:
                break
        if ok:
            torch.cuda.synchronize(self.device)
            self.nvls = bool(self.arena.has_multicast())
        else:
            self.arena.disable_multicast()
        self._host_barrier()

    # ---- collectives with the TorchCollectives interface ---------------------------------------
    def allgather_object(self, obj):
        if self.world == 1:
            return [obj]
        out = [None] * self.world
        dist.all_gather_object(out, obj, group=self.group)
        return out

    def barrier(self) -> None:
        self._host_barrier()

    def check(self) -> None:
        code = self.arena.check_error()
        if code:
            raise PeerCommError(f"peer-memory barrier timed out (code {code}): a peer rank is not participating")

    def broadcast_tensors(self, tensors: Sequence[torch.Tensor], src: int = 0) -> int:
        """Peer-memory broadcast kernel; tensors are written in place on non-source ranks."""
        tensors = [t for t in tensors if t.numel() > 0]
        if self.world == 1 or not tensors:
            return 0
        dense = []
        fixups = []
        for t in tensors:
            if is_dense(t):
                dense.append(t)
            else:
                c = t.contiguous()
                dense.append(c)
                fixups.append((t, c))
        n = self.C.broadcast_tensors(self.arena, dense, src, self.scratch_off, self.scratch_bytes, self.nvls, self.blocks,
                                     1, self.timeout_s)
        if self.rank != src:
            for t, c in fixups:
                t.copy_(c)
        return n

    def allreduce_(self, tensors: Sequence[torch.Tensor], wire: str = "bf16", algo: str = "auto", scale: float = 1.0,
                   blocks: Optional[int] = None) -> None:
        """In-place fused allreduce (sum * scale) of up to 192 same-dtype tensors as one bucket."""
        if self.world == 1:
            return
        self.C.allreduce_tensors(self.arena, list(tensors), wire, _ALGO[algo], blocks or self.blocks, self.scratch_off,
                                 self.scratch_bytes, scale, 1, self.timeout_s, None)

    # ---- symmetric memory: tensors that live at the same arena offset on every rank ---------------------
    def symmetric_empty(self, numel: int, dtype: torch.dtype = torch.float32) -> torch.Tensor:
        """Allocate a 1-D tensor inside the arena (same call sequence on every rank -> same offset everywhere).
        Collectives on such tensors run in place over peer memory with no staging copy."""
        code = _DTYPE_CODE[dtype]
        nbytes = numel * (2 if dtype == torch.bfloat16 else 4)
        off = self.arena.alloc((nbytes + 15) // 16 * 16, 4096)
        t = self.C.arena_tensor(self.arena, off, numel, code)
        t._b200_arena_off = off
        return t

    def allreduce_symmetric_(self, t: torch.Tensor, algo: str = "auto", scale: float = 1.0, blocks: Optional[int] = None,
                             pad_set: int = 0) -> None:
        if self.world == 1:
            if scale != 1.0:
                t.mul_(scale)
            return
        off = t.data_ptr() - self.arena.local_ptr()          # slices / views of a symmetric tensor are symmetric too
        if off < 0 or off + t.numel() * t.element_size() > self.arena.bytes() or not t.is_contiguous():
            raise ValueError("allreduce_symmetric_ needs a contiguous tensor (or slice) from symmetric_empty()")
        self.C.allreduce_symmetric(self.arena, off, t.numel(), _DTYPE_CODE[t.dtype], _ALGO[algo], blocks or self.tail_blocks,
                                   scale, pad_set, self.timeout_s)

    def close(self) -> None:
        if not self.closed:
            self.closed = True
            try:
                torch.cuda.synchronize(self.device)
            except Exception:
                pass
            self.arena.close()


class NativeReducer:
    """Thin Python shell over ``csrc/reducer.cpp``: forwards hook events, owns the flat result
    buffers, swaps ``.grad`` to bucket views at the end of backward."""

    def __init__(self, params: List[torch.nn.Parameter], specs: List[BucketSpec], comm: PeerCollectives,
                 gradient_as_bucket_view: bool, find_unused: bool, wire_dtype: Optional[str] = None,
                 algo: str = "auto", max_blocks: Optional[int] = None):
        C = self.C = comm.C
        self.params = params
        self.specs = specs
        self.comm = comm
        self.as_view = gradient_as_bucket_view
        self.find_unused = find_unused
        self.world = comm.world
        plans = []
        for spec in specs:
            p0 = params[spec.param_indices[0]]
            if p0.dtype not in _DTYPE_CODE:
                raise TypeError(f"b200 backend reduces fp32/bf16 gradients, got {p0.dtype}")
            wire = _WIRE_NAME[wire_dtype] if wire_dtype else p0.dtype
            plan = C.BucketPlan()
            plan.param_indices = list(spec.param_indices)
            plan.numels = list(spec.numels)
            plan.offsets = list(spec.offsets)
            plan.data_elems = spec.flags_offset
            plan.total_elems = spec.total_elems
            plan.grad_dtype = _DTYPE_CODE[p0.dtype]
            plan.wire_dtype = _DTYPE_CODE[wire]
            plan.tail = bool(getattr(spec, "tail", False))
            plans.append(plan)
        blocks = max_blocks or comm.blocks
        self._arena_mark = comm.arena.used()
        self._ctor = dict(wire_dtype=wire_dtype, algo=algo, max_blocks=max_blocks)
        one_shot_max = int(os.environ.get("B200DDP_ONE_SHOT_MAX_KB", "256")) * 1024
        serial = int(os.environ.get("B200DDP_DDP_SERIAL", "-1"))       # -1: in line under CUDA-graph capture, overlapped otherwise
        wide = int(os.environ.get("B200DDP_WIDE_BLOCKS", "264"))
        self._c = C.Reducer(comm.arena, plans, len(params), _ALGO[algo], blocks, comm.tail_blocks, one_shot_max, gradient_as_bucket_view,
                            find_unused, 1.0, comm.timeout_s, serial, wide,
                            int(float(os.environ.get("B200DDP_TAIL_ONE_SHOT_MAX_MB", "8")) * MiB))
        device = params[0].device
        self.flat_out: List[Optional[torch.Tensor]] = []
        self.views: List[List[torch.Tensor]] = []
        for b, spec in enumerate(specs):
            if gradient_as_bucket_view or find_unused:
                dtype = params[spec.param_indices[0]].dtype
                flat = torch.zeros(spec.total_elems, dtype=dtype, device=device)
                self._c.set_flat_out(b, flat.data_ptr())
                self.flat_out.append(flat)
                self.views.append([flat[o:o + n].as_strided(params[i].size(), params[i].stride())
                                   for i, o, n in zip(spec.param_indices, spec.offsets, spec.numels)])
            else:
                self.flat_out.append(None)
                self.views.append([])
        self.sq_partials = torch.zeros(len(specs), C.MAX_COMM_BLOCKS, dtype=torch.float32, device=device)
        self._c.set_sq_partials(self.sq_partials.data_ptr(), C.MAX_COMM_BLOCKS)
        self._last_fired = set()

    # the DDP wrapper calls these ----------------------------------------------------------------
    def reset(self) -> None:
        self._c.reset()
        self._last_fired = set()

    def mark_ready(self, index: int) -> None:
        p = self.params[index]
        g = p.grad
        if not is_dense(g):
            g = g.contiguous()
            p.grad = g
        self._last_fired.add(index)
        self._c.mark_ready(index, g.data_ptr(), torch.cuda.current_stream(g.device).cuda_stream)

    def finalize(self) -> None:
        stream = torch.cuda.current_stream(self.params[0].device).cuda_stream
        missing = self._c.finalize(stream)
        if self.as_view and not missing:
            for b, spec in enumerate(self.specs):
                for view, i in zip(self.views[b], spec.param_indices):
                    self.params[i].grad = view
        elif missing:
            self._finalize_with_unused()
        code = self._c.error_code()
        if code:
            raise PeerCommError(f"peer-memory barrier timed out (code {code})")

    def _finalize_with_unused(self) -> None:
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError("parameters without gradients were found while capturing a CUDA graph: which parameters "
                               "are used must be static under --cuda_graph (the reduced 'used' flags need a host read)")
        for b, spec in enumerate(self.specs):
            flags = None
            for k, i in enumerate(spec.param_indices):
                p = self.params[i]
                fired = i in self._last_fired
                if fired:
                    if self.as_view:
                        p.grad = self.views[b][k]
                    continue
                if flags is None:
                    flags = self._c.read_used_flags(b)
                if flags[k] > 0.0:   # used on some other rank: take the reduced value from the flat bucket
                    p.grad = self.views[b][k] if self.as_view else self.views[b][k].clone()

    def rebuilt(self, specs: List[BucketSpec]) -> "NativeReducer":
        """New reducer for a new bucket plan; the old staging regions go back to the arena first."""
        self._c.synchronize()
        torch.cuda.synchronize(self.params[0].device)
        self.comm.barrier()
        del self._c
        self.comm.arena.rewind(self._arena_mark)
        return NativeReducer(self.params, specs, self.comm, self.as_view, self.find_unused, **self._ctor)

    @property
    def stats(self) -> dict:
        return {"buckets_launched": int(self._c.launches), "bytes_reduced": int(self._c.bytes_on_wire),
                "iterations": int(self._c.iterations),
                "algos": [int(self._c.bucket_algo(b)) for b in range(len(self.specs))],
                "blocks": [int(self._c.bucket_blocks(b)) for b in range(len(self.specs))]}

    @property
    def ready_order(self) -> List[int]:
        return list(self._c.ready_order)

    def grad_sq_partials(self) -> torch.Tensor:
        """Per-(bucket, block) sum of squares of the *reduced* gradients, written by the allreduce
        epilogue; the fused optimizer turns it into the clip coefficient without re-reading grads."""
        return self.sq_partials

    def synchronize(self) -> None:
        self._c.synchronize()
