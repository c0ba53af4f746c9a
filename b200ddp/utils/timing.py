"""Device-side timing helpers (the reference has no timers beyond tqdm's it/s).

``StepTimer`` brackets optimizer steps with CUDA events on the launching stream and reports milliseconds per step
and samples/s as the MAX over ranks (a multi-GPU step is as slow as its slowest rank); nothing synchronises until
``summary()`` is called.  ``nvtx_range`` wraps ``torch.cuda.nvtx`` so timelines show per-phase ranges when a
profiler is attached and cost nothing otherwise."""
from __future__ import annotations

import contextlib
from typing import List, Optional

import torch

from .dist import max_over_ranks


class StepTimer:
    def __init__(self, device: torch.device, samples_per_step: int = 0, skip_first: int = 3):
        self.device = torch.device(device)
        self.cuda = self.device.type == "cuda"
        self.samples_per_step = samples_per_step
        self.skip_first = skip_first
        self._events: List["torch.cuda.Event"] = []
        self._host: List[float] = []

    def tick(self) -> None:
        """Call once per optimizer step (at the same point of every step)."""
        if self.cuda:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record(torch.cuda.current_stream(self.device))
            self._events.append(ev)
        else:
            import time
            self._host.append(time.perf_counter())

    def summary(self, reset: bool = True) -> Optional[dict]:
        n = len(self._events) if self.cuda else len(self._host)
        if n - self.skip_first < 2:
            return None
        if self.cuda:
            self._events[-1].synchronize()
            first, last = self._events[self.skip_first], self._events[-1]
            ms = first.elapsed_time(last)
        else:
            ms = (self._host[-1] - self._host[self.skip_first]) * 1e3
        steps = n - self.skip_first - 1
        ms_per_step = max_over_ranks(ms / steps)
        out = {"steps": steps, "ms_per_step": ms_per_step}
        if self.samples_per_step:
            out["samples_per_s"] = self.samples_per_step / (ms_per_step / 1e3)
        if reset:
            self._events, self._host, self.skip_first = [], [], 0
        return out


@contextlib.contextmanager
def nvtx_range(name: str):
    pushed = False
    if torch.cuda.is_available():
        try:
            torch.cuda.nvtx.range_push(name)
            pushed = True
        except Exception:
            pushed = False
    try:
        yield
    finally:
        if pushed:
            torch.cuda.nvtx.range_pop()
