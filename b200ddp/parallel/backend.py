"""Communication backends behind the DDP wrapper.

The reference hard-codes ``init_process_group(backend="nccl")`` (``ddp.py:103``) and lets torch's
Reducer issue NCCL calls.  Here the wrapper talks to one of:

* ``b200``  - the product: hand-written sm_90a kernels over NVSwitch peer memory
              (``csrc/peer_mem.cpp`` + ``csrc/allreduce.cu`` + ``csrc/broadcast.cu``); torch's
              process group is used only to bootstrap (handle exchange) and for host-side checks.
* ``nccl``  - stock ``torch.distributed`` collectives on GPU: the *baseline* path, kept for
              comparison runs and as the multi-node fallback.
* ``gloo``  - CPU plumbing (world_size=2 on CPU, no GPU).

This is a transport choice for one hardware target, not a multi-vendor dispatch layer: the b200
path is the only one with native kernels.
"""
from __future__ import annotations

import os
from typing import List, Optional, Sequence

import torch
import torch.distributed as dist


class TorchCollectives:
    """gloo / nccl through ``torch.distributed`` (baseline + CPU tests)."""

    name = "torch"

    def __init__(self, group=None):
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.name = dist.get_backend(group) if dist.is_initialized() else "single"

    def allreduce_async(self, flat: torch.Tensor):
        if self.world == 1:
            return None
        return dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=self.group, async_op=True)

    def broadcast_flat(self, flat: torch.Tensor, src: int = 0) -> None:
        if self.world > 1:
            dist.broadcast(flat, src=src, group=self.group)

    def broadcast_tensors(self, tensors: Sequence[torch.Tensor], src: int = 0,
                          chunk_bytes: int = 250 * 1024 * 1024) -> None:
        """Coalesced broadcast: group by dtype, flatten into <= chunk_bytes pieces, broadcast,
        copy back on non-source ranks (what ``_sync_module_states`` does in the stock stack, N4)."""
        if self.world == 1 or not tensors:
            return
        by_dtype = {}
        for t in tensors:
            by_dtype.setdefault((t.dtype, t.device), []).append(t)
        for (_, _), group in by_dtype.items():
            chunk: List[torch.Tensor] = []
            size = 0
            for t in group + [None]:
                if t is not None:
                    chunk.append(t)
                    size += t.numel() * t.element_size()
                if chunk and (t is None or size >= chunk_bytes):
                    flat = torch.cat([c.detach().reshape(-1) for c in chunk])
                    dist.broadcast(flat, src=src, group=self.group)
                    if self.rank != src:
                        off = 0
                        with torch.no_grad():
                            for c in chunk:
                                n = c.numel()
                                c.copy_(flat[off:off + n].view_as(c))
                                off += n
                    chunk, size = [], 0

    def allgather_object(self, obj):
        if self.world == 1:
            return [obj]
        out = [None] * self.world
        dist.all_gather_object(out, obj, group=self.group)
        return out

    def barrier(self) -> None:
        if self.world > 1:
            dist.barrier(group=self.group)


def spans_one_nvswitch_domain(group=None) -> bool:
    """True when every rank of ``group`` can sit in one peer-memory arena: <= 8 ranks, all on this host
    (torchrun exports LOCAL_WORLD_SIZE; without a launcher there is only one process anyway)."""
    if not (dist.is_available() and dist.is_initialized()):
        return True
    world = dist.get_world_size(group)
    local_world = int(os.environ.get("LOCAL_WORLD_SIZE", world))
    return world <= 8 and local_world >= world


def pick_backend_name(requested: str, device: torch.device, group=None) -> str:
    """Resolve ``auto``: b200 on CUDA when the native extension is usable and the job fits one NVSwitch domain,
    otherwise the process group's own backend (multi-node jobs launched by ``run.sbatch`` reduce over NCCL)."""
    if requested != "auto":
        return requested
    if device.type == "cuda":
        try:
            from .. import _ext
            if _ext.available() and spans_one_nvswitch_domain(group):
                return "b200"
        except Exception:
            pass
        return "nccl"
    return "gloo"
