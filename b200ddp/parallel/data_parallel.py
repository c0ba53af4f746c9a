"""Single-process multi-GPU mode (reference ``ddp.py:189-191``: ``DataParallel(model)`` when launched
without a launcher on a multi-GPU host).  Kept for CLI parity only - the reference README itself says
DDP is the faster choice (``README.md:5``) and this is not a performance target.

Implementation: scatter the batch along dim 0, replicate the module onto every visible GPU, run the
replicas on threads, gather outputs on the first device.  Gradients flow back through the differentiable
replicate/gather primitives and sum on device 0, so the optimizer only ever sees the original module."""
from __future__ import annotations

from typing import List, Optional, Sequence

import torch
import torch.nn as nn
from torch.nn.parallel import gather, parallel_apply, replicate, scatter


class DataParallel(nn.Module):
    def __init__(self, module: nn.Module, device_ids: Optional[Sequence[int]] = None, output_device: Optional[int] = None):
        super().__init__()
        self.module = module
        if device_ids is None:
            device_ids = list(range(torch.cuda.device_count()))
        self.device_ids: List[int] = list(device_ids)
        self.output_device = self.device_ids[0] if output_device is None and self.device_ids else output_device

    def forward(self, *inputs, **kwargs):
        if len(self.device_ids) <= 1:
            return self.module(*inputs, **kwargs)
        chunks = scatter(inputs, self.device_ids, dim=0)
        kw_chunks = scatter(kwargs, self.device_ids, dim=0) if kwargs else [{} for _ in chunks]
        used = self.device_ids[:len(chunks)]
        if len(used) == 1:
            return self.module(*chunks[0], **kw_chunks[0])
        replicas = replicate(self.module, used)
        outputs = parallel_apply(replicas, list(chunks), list(kw_chunks)[:len(chunks)], used)
        return gather(outputs, self.output_device, dim=0)

    def state_dict(self, *args, **kwargs):
        return self.module.state_dict(*args, **kwargs)

    def load_state_dict(self, state_dict, *args, **kwargs):
        return self.module.load_state_dict(state_dict, *args, **kwargs)
