"""Batch loading and host->device staging.

Reference: ``DataLoader(dataset, batch_size, sampler, pin_memory=True)`` with no workers, followed by a
*blocking* ``x.to(device)`` per step (``ddp.py:148-152,220``).

Here:
* ``BatchLoader`` walks a sampler and gathers a whole batch with one ``index_select`` per field straight
  into a rotating set of pinned host buffers (no per-sample ``__getitem__`` + collate + pin copy).
  Falls back to the generic per-sample path for datasets without ``batch()``.
* ``DevicePrefetcher`` issues the H2D copies for batch i+1 on a dedicated copy stream while batch i
  computes; the consumer waits on an event, never on the host.  Device buffers are static (two slots),
  which is also what CUDA-graph replay needs.
"""
from __future__ import annotations

import atexit
import queue
import threading
from typing import Iterator, List, Optional, Sequence, Tuple

import torch


_ACTIVE = []          # (stop event, queue, thread) of running loader helper threads
_ACTIVE_LOCK = threading.Lock()


def _stop_helper(entry) -> None:
    entry.stop()


@atexit.register
def _shutdown_loader_threads() -> None:
    """A helper thread left inside native code at interpreter teardown aborts the process; stop them first."""
    with _ACTIVE_LOCK:
        entries = list(_ACTIVE)
        _ACTIVE.clear()
    for e in entries:
        _stop_helper(e)


class PinnedBatch(tuple):
    """A batch living in one of the loader's pinned slots; ``slot`` lets the prefetcher mark it busy."""
    slot: int = -1


class BatchLoader:
    def __init__(self, dataset, batch_size: int, sampler=None, drop_last: bool = False, pin_memory: bool = True,
                 num_slots: int = 8, background: bool = True, workers: int = 3):
        self.dataset = dataset
        self.batch_size = int(batch_size)
        self.sampler = sampler if sampler is not None else torch.utils.data.SequentialSampler(dataset)
        self.drop_last = drop_last
        self.pin = bool(pin_memory) and torch.cuda.is_available()
        self.num_slots = num_slots
        self._slots: List[Optional[Tuple[torch.Tensor, ...]]] = [None] * num_slots
        self._fast = hasattr(dataset, "batch")
        self._into = hasattr(dataset, "batch_into")
        # gather batches on a helper thread (index_select / memcpy release the GIL) so the training thread only
        # ever launches work; depth is bounded by the number of pinned slots
        self.background = bool(background) and self.pin
        self.workers = max(1, int(workers))
        # set by DevicePrefetcher: event that fires when the async H2D copy out of a pinned slot is done
        self.slot_events: List[Optional["torch.cuda.Event"]] = [None] * num_slots
        self.last_slot = 0

    def __len__(self) -> int:
        n = len(self.sampler)
        return n // self.batch_size if self.drop_last else (n + self.batch_size - 1) // self.batch_size

    def _slot_like(self, slot: int, fields: Sequence[torch.Tensor]) -> Tuple[torch.Tensor, ...]:
        cur = self._slots[slot]
        if cur is None or any(c.shape != f.shape or c.dtype != f.dtype for c, f in zip(cur, fields)):
            cur = tuple(torch.empty(f.shape, dtype=f.dtype, pin_memory=self.pin) for f in fields)
            self._slots[slot] = cur
        return cur

    def _index_batches(self) -> Iterator[List[int]]:
        """Lazily group the sampler's indices into batches (the sampler may be endless, see ``EndlessSampler``)."""
        cur: List[int] = []
        for idx in self.sampler:
            cur.append(idx)
            if len(cur) == self.batch_size:
                yield cur
                cur = []
        if cur and not self.drop_last:
            yield cur

    def __iter__(self) -> Iterator[Tuple[torch.Tensor, ...]]:
        batches = self._index_batches()
        if not self.background:
            for k, idxs in enumerate(batches):
                yield self._make(idxs, k % self.num_slots)
            return
        # `workers` helper threads gather whole batches into the rotating pinned slots (index_select / memcpy release
        # the GIL); batch k always lands in slot k % num_slots and is handed out in order.  A worker may run at most
        # `window` batches ahead of the consumer, so a slot is never refilled before its previous batch was taken
        # (and `_make` additionally waits for that batch's H2D copy to finish).
        window = max(1, self.num_slots - 3)
        cv = threading.Condition()
        state = {"next": 0, "taken": 0, "stop": False, "err": None, "exhausted": False}
        ready = {}

        def work():
            while True:
                with cv:
                    while not state["stop"] and not state["exhausted"] and state["next"] >= state["taken"] + window:
                        cv.wait(0.05)
                    if state["stop"] or state["exhausted"]:
                        return
                    try:
                        idxs = next(batches)          # the index stream is shared: pulled under the lock, in order
                    except StopIteration:
                        state["exhausted"] = True
                        cv.notify_all()
                        return
                    except BaseException as exc:
                        state["err"] = exc
                        cv.notify_all()
                        return
                    k = state["next"]
                    state["next"] += 1
                try:
                    item = self._make(idxs, k % self.num_slots)
                except BaseException as exc:      # surface loader errors in the consumer
                    with cv:
                        state["err"] = exc
                        cv.notify_all()
                    return
                with cv:
                    ready[k] = item
                    cv.notify_all()

        threads = [threading.Thread(target=work, name=f"b200ddp-batch-loader-{i}", daemon=True) for i in range(self.workers)]
        for t in threads:
            t.start()

        class _Entry:
            def stop(self_inner):
                with cv:
                    state["stop"] = True
                    cv.notify_all()
                for t in threads:
                    t.join(timeout=2.0)

        entry = _Entry()
        with _ACTIVE_LOCK:
            _ACTIVE.append(entry)
        try:
            k = 0
            while True:
                with cv:
                    while k not in ready and state["err"] is None and not (state["exhausted"] and k >= state["next"]):
                        cv.wait(0.05)
                    if state["err"] is not None:
                        raise state["err"]
                    if k not in ready:
                        break                          # stream exhausted and every produced batch handed out
                    item = ready.pop(k)
                    state["taken"] = k + 1
                    cv.notify_all()
                yield item
                k += 1
        finally:
            with _ACTIVE_LOCK:
                if entry in _ACTIVE:
                    _ACTIVE.remove(entry)
            entry.stop()

    def _tag(self, fields, slot: int):
        b = PinnedBatch(fields)
        b.slot = slot
        return b

    def _make(self, indices: List[int], slot: int) -> Tuple[torch.Tensor, ...]:
        self.last_slot = slot
        busy = self.slot_events[slot]
        if busy is not None:          # never overwrite pinned memory an in-flight copy still reads
            busy.synchronize()
            self.slot_events[slot] = None
        if self._fast:
            idx = torch.as_tensor(indices, dtype=torch.long)
            if not self.pin:
                return tuple(self.dataset.batch(idx))
            cur = self._slots[slot]
            if self._into and cur is not None and cur[0].shape[0] == len(indices):
                self.dataset.batch_into(idx, cur)          # one pass: gather straight into pinned memory
                return self._tag(cur, slot)
            fields = self.dataset.batch(idx)
            out = self._slot_like(slot, fields)
            for o, f in zip(out, fields):
                o.copy_(f)
            return self._tag(out, slot)
        samples = [self.dataset[i] for i in indices]
        fields = tuple(torch.stack([s[k] for s in samples]) for k in range(len(samples[0])))
        if not self.pin:
            return fields
        out = self._slot_like(slot, fields)
        for o, f in zip(out, fields):
            o.copy_(f)
        return self._tag(out, slot)


class DevicePrefetcher:
    """Wraps an iterator of host (pinned) batches; yields device batches whose H2D copy ran on a side
    stream.  ``h2d_bytes`` counts the bytes actually copied (bench.py reports it per step)."""

    def __init__(self, loader, device: torch.device, slots: int = 2):
        self.loader = loader
        self.device = torch.device(device)
        self.cuda = self.device.type == "cuda"
        self.slots = slots
        self.h2d_bytes = 0
        if self.cuda:
            self.copy_stream = torch.cuda.Stream(device=self.device)
            self._dev: List[Optional[Tuple[torch.Tensor, ...]]] = [None] * slots
            self._ready = [torch.cuda.Event() for _ in range(slots)]
            self._consumed = [torch.cuda.Event() for _ in range(slots)]

    def __len__(self) -> int:
        return len(self.loader)

    def _stage(self, host: Tuple[torch.Tensor, ...], slot: int):
        cur = self._dev[slot]
        consumer = torch.cuda.current_stream(self.device)
        fresh = cur is None or any(c.shape != h.shape or c.dtype != h.dtype for c, h in zip(cur, host))
        if fresh:
            cur = tuple(torch.empty(h.shape, dtype=h.dtype, device=self.device) for h in host)
            self._dev[slot] = cur
        with torch.cuda.stream(self.copy_stream):
            if fresh:
                # The allocator hands out memory freed on the consumer stream at once, though kernels queued there may
                # still use it (an eager step's activations, say): the copy must not write it before they ran.
                self.copy_stream.wait_stream(consumer)
            self.copy_stream.wait_event(self._consumed[slot])      # previous user of this slot is done
            for d, h in zip(cur, host):
                d.copy_(h, non_blocking=True)
                d.record_stream(self.copy_stream)                  # freed with the copy in flight: not reused before it ends
                self.h2d_bytes += h.numel() * h.element_size()
            self._ready[slot].record(self.copy_stream)
        events = getattr(self.loader, "slot_events", None)
        host_slot = getattr(host, "slot", -1)
        if events is not None and host_slot >= 0:
            done = torch.cuda.Event()
            done.record(self.copy_stream)
            events[host_slot] = done
        return cur

    def __iter__(self):
        if not self.cuda:
            for batch in self.loader:
                yield batch
            return
        it = iter(self.loader)
        slot = 0
        try:
            pending = (self._stage(next(it), slot), slot)
        except StopIteration:
            return
        while pending is not None:
            batch, s = pending
            nxt = (s + 1) % self.slots
            try:
                pending = (self._stage(next(it), nxt), nxt)
            except StopIteration:
                pending = None
            torch.cuda.current_stream(self.device).wait_event(self._ready[s])
            yield batch
            # whatever the consumer enqueued on the current stream has been issued by now
            self._consumed[s].record(torch.cuda.current_stream(self.device))
