"""Gradient bucket planning (host logic; pure Python mirror of ``csrc/reducer.cpp``).

What the reference runs (delegated): ``torch.distributed._compute_bucket_assignment_by_size``
called from ``TORCH/nn/parallel/distributed.py:1237-1244`` with limits ``[1 MiB, 25 MiB]``
(because ``ddp.py:195`` passes ``find_unused_parameters=True``), and the result reversed before it
reaches the Reducer.  ``assign_by_size`` reproduces that greedy algorithm exactly so the
layouts stock DDP builds can be asserted on CPU.

The native design differs in two ways: (1) ``plan_buckets`` walks the parameters in *reverse*
registration order (the order gradients become ready in backward) so the small first bucket is the
one that launches first, and (2) each tensor's slot in the flat bucket is padded to ``align``
elements so a 16-byte wire vector never straddles two tensors (the fused kernel's pack/unpack
relies on it).  ``plan_buckets(order="torch")`` gives the stock layout + launch order instead.
"""
from __future__ import annotations

import os

from dataclasses import dataclass, field
from typing import Dict, Hashable, List, Optional, Sequence, Tuple

MiB = 1024 * 1024
DEFAULT_FIRST_BUCKET_BYTES = 1 * MiB
DEFAULT_BUCKET_CAP_BYTES = 25 * MiB
SLOT_ALIGN_ELEMS = 8          # 8 x bf16 = one 16-byte wire vector
MAX_TENSORS_PER_BUCKET = 192  # table rides in kernel parameters (csrc/tensor_table.h)


def assign_by_size(nbytes: Sequence[int], keys: Optional[Sequence[Hashable]] = None,
                   limits: Sequence[int] = (DEFAULT_BUCKET_CAP_BYTES,),
                   max_tensors: Optional[int] = None) -> List[List[int]]:
    """Greedy size-capped grouping.  A group is closed as soon as its byte count reaches the
    current limit for its key; limits advance per key and the last one repeats.  Open groups are
    flushed at the end and the result is ordered by each group's smallest index."""
    if not limits:
        raise ValueError("need at least one size limit")
    if keys is None:
        keys = [0] * len(nbytes)
    open_groups: Dict[Hashable, Tuple[List[int], int]] = {}
    cursor: Dict[Hashable, int] = {}
    closed: List[List[int]] = []
    for idx, (size, key) in enumerate(zip(nbytes, keys)):
        members, total = open_groups.get(key, ([], 0))
        members.append(idx)
        total += int(size)
        pos = cursor.setdefault(key, 0)
        full = total >= limits[pos] or (max_tensors is not None and len(members) >= max_tensors)
        if full:
            closed.append(members)
            open_groups.pop(key, None)
            if total >= limits[pos] and pos + 1 < len(limits):
                cursor[key] = pos + 1
        else:
            open_groups[key] = (members, total)
    for members, _ in open_groups.values():
        if members:
            closed.append(members)
    closed.sort(key=min)
    return closed


@dataclass
class BucketSpec:
    """One flat bucket: which parameters, and where each lives in the flat space."""
    index: int
    param_indices: List[int]
    numels: List[int]
    offsets: List[int] = field(default_factory=list)   # element offset of each tensor's slot
    flags_offset: int = 0                              # start of the per-tensor "used" flags
    total_elems: int = 0                               # padded data + flags, rounded to align
    key: Hashable = 0
    tail: bool = False                                 # completes at the very end of backward: latency is exposed

    @property
    def data_elems(self) -> int:
        return self.flags_offset

    def layout(self, align: int = SLOT_ALIGN_ELEMS, with_flags: bool = True) -> "BucketSpec":
        off = 0
        self.offsets = []
        for n in self.numels:
            self.offsets.append(off)
            off += -(-n // align) * align
        self.flags_offset = off
        if with_flags:
            off += -(-len(self.numels) // align) * align
        self.total_elems = off
        return self


def plan_buckets(numels: Sequence[int], elem_sizes: Sequence[int], keys: Optional[Sequence[Hashable]] = None,
                 bucket_cap_bytes: int = DEFAULT_BUCKET_CAP_BYTES,
                 first_bucket_bytes: int = DEFAULT_FIRST_BUCKET_BYTES,
                 order: str = "backward", align: int = SLOT_ALIGN_ELEMS, with_flags: bool = True,
                 ready_order: Optional[Sequence[int]] = None,
                 max_tensors: int = MAX_TENSORS_PER_BUCKET, tail_window: int = 4,
                 tail_bucket_bytes: int = 4 * MiB) -> List[BucketSpec]:
    """Return buckets in LAUNCH order.

    order="backward": walk params last-to-first (or ``ready_order`` if observed), first bucket small.
    order="torch":    stock layout (forward walk, ``[first, cap]`` limits) then reversed.
    """
    n = len(numels)
    if keys is None:
        keys = [0] * n
    if os.environ.get("B200DDP_TAIL_BUCKET_MB"):            # diagnostics: bound of the bucket that completes last
        tail_bucket_bytes = int(float(os.environ["B200DDP_TAIL_BUCKET_MB"]) * MiB)
    if order == "torch":
        walk = list(range(n))
    elif ready_order is not None:
        seen = set(ready_order)
        walk = list(ready_order) + [i for i in reversed(range(n)) if i not in seen]
    elif order == "backward":
        walk = list(reversed(range(n)))
    else:
        raise ValueError(f"unknown bucket order {order!r}")
    limits = [first_bucket_bytes, bucket_cap_bytes] if first_bucket_bytes > 0 else [bucket_cap_bytes]
    groups = assign_by_size([numels[i] * elem_sizes[i] for i in walk], [keys[i] for i in walk], limits,
                            max_tensors=max_tensors)
    if order == "torch":
        groups = list(reversed(groups))
    else:
        # Bound what is exposed at the end of backward: the group that finishes last (per dtype) is cut so its
        # final piece carries at most `tail_bucket_bytes`; everything before the cut goes out one bucket earlier.
        if tail_bucket_bytes > 0:
            sizes = [numels[i] * elem_sizes[i] for i in walk]
            split = []
            for grp in groups:
                is_last_of_key = not any(keys[walk[g2[0]]] == keys[walk[grp[0]]] and max(g2) > max(grp) for g2 in groups)
                total = sum(sizes[j] for j in grp)
                if is_last_of_key and total > tail_bucket_bytes and len(grp) > 1:
                    acc, cut = 0, len(grp)
                    for pos in range(len(grp) - 1, -1, -1):
                        acc += sizes[grp[pos]]
                        if acc > tail_bucket_bytes:
                            break
                        cut = pos
                    cut = min(max(cut, 1), len(grp) - 1)
                    split += [grp[:cut], grp[cut:]]
                else:
                    split.append(grp)
            groups = split
        # Launch order = completion order.  A bucket is complete when its LAST gradient (largest walk position)
        # is ready; with several dtypes in play (bf16 weights + fp32 BatchNorm) the per-dtype groups interleave,
        # and sorting by first member would park e.g. the all-BatchNorm bucket (finishes at the very end) in
        # front of buckets that finish early - the in-order launch rule would then hold those back until the
        # end of backward and expose all of their communication.
        groups.sort(key=lambda grp: (max(grp), min(grp)))
    specs = []
    last_positions = set(range(max(0, n - tail_window), n))
    for b, grp in enumerate(groups):
        members = [walk[j] for j in grp]
        spec = BucketSpec(index=b, param_indices=members, numels=[numels[i] for i in members], key=keys[members[0]])
        spec.tail = order != "torch" and any(j in last_positions for j in grp)
        specs.append(spec.layout(align=align, with_flags=with_flags))
    if specs:
        specs[-1].tail = True
    return specs


def bucket_sizes_mib(specs: Sequence[BucketSpec], elem_size: int = 4) -> List[float]:
    return [round(sum(s.numels) * elem_size / MiB, 2) for s in specs]
