"""Host -> device input staging that overlaps the copy of step i+1 with the compute of step i.

The reference moves the whole dataset to the device once (`large/main.py:83-85`) or, in the mini-batch driver, copies each
batch synchronously inside the loop (`large/main-batch.py:141-143`: `x_i = x[idx_i].to(device)`).  A full-batch
products-shaped step moves 3 GB of features and int64 edge indices over PCIe, a large share of the step when copied
synchronously; `HostFeeder` hides it behind the previous step with a second CUDA stream and
two persistent device slots (no allocation, no host synchronisation per step).
"""
from __future__ import annotations

from collections import deque
from typing import Callable, Deque, List, Optional, Sequence, Tuple

import torch
from torch import Tensor


class HostFeeder:
    """Double-buffered (or `slots`-deep) staging of a tuple of host tensors.

    `submit(host_tensors)` enqueues the copies on the feeder's stream - followed, when given, by `prepare(*device_tensors)` on the
    same stream (e.g. `model.prepare_graph(edge_index, n)`: the CSR build of the NEXT step's graph then runs beside the current
    step instead of in front of the next one); `get()` makes the caller's current stream wait for the oldest outstanding submit
    and returns its device tensors.  A slot is overwritten only after the step that consumed it: `get()` records an event on the
    caller's stream that marks the end of everything enqueued since the previous `get()`, and the overwriting `submit` waits for
    the event of its slot.  Both loop orders are race-free with `slots=2`:

        feeder.submit(batch0)
        for i in range(steps):
            dev = feeder.get()
            step(*dev)                    # enqueue the step first ...
            feeder.submit(next_batch)     # ... then the copy (+ prepare) of the next batch: the host may block in prepare's
                                          #     device syncs while the GPU is busy with the step

    (or `get(); submit(); step()` when `prepare` does not synchronise).  Host tensors should be pinned (`.pin_memory()`), otherwise
    the copy is synchronous.
    """

    def __init__(self, device: torch.device, slots: int = 2, prepare: Optional[Callable] = None):
        if slots < 2:
            raise ValueError("HostFeeder needs at least two slots")
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("sgformer_b200 has no CPU path: HostFeeder stages onto a CUDA device")
        self.stream = torch.cuda.Stream(self.device)
        self._prepare = prepare
        self._slots: List[List[Tensor]] = [[] for _ in range(slots)]
        self._free: List[Optional[torch.cuda.Event]] = [None] * slots    # slot -> "its last consumer has finished"
        self._held: Optional[int] = None                                  # slot handed out by the last get()
        self._next = 0
        self._prepared = None                                             # what prepare() returned for the slot in use
        self._pending: Deque[Tuple[int, List[Tensor], torch.cuda.Event, object]] = deque()

    def _buffers(self, slot: int, host: Sequence[Tensor]) -> List[Tensor]:
        bufs = self._slots[slot]
        if len(bufs) != len(host) or any(b.shape != t.shape or b.dtype != t.dtype for b, t in zip(bufs, host)):
            bufs = [torch.empty(t.shape, dtype=t.dtype, device=self.device) for t in host]
            self._slots[slot] = bufs
            self._free[slot] = None
        return bufs

    def submit(self, host: Sequence[Tensor]) -> None:
        # one slot always belongs to the consumer (the tensors handed out by the last get())
        if len(self._pending) >= len(self._slots) - 1:
            raise RuntimeError("HostFeeder: all slots are in flight; call get() before submitting more")
        slot = self._next
        self._next = (self._next + 1) % len(self._slots)
        bufs = self._buffers(slot, host)
        free = self._free[slot]
        if free is not None and slot != self._held:
            self.stream.wait_event(free)          # the step that last read this slot has finished
        else:
            # fresh buffers (or no event yet): everything enqueued so far on the consumer's stream goes first
            self.stream.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(self.stream):
            for b, t in zip(bufs, host):
                b.copy_(t, non_blocking=True)
            extra = self._prepare(*bufs) if self._prepare is not None else None
            ev = torch.cuda.Event()
            ev.record(self.stream)
        self._pending.append((slot, bufs, ev, extra))

    def get(self) -> Tuple[Tensor, ...]:
        if not self._pending:
            raise RuntimeError("HostFeeder.get() without a pending submit")
        cur = torch.cuda.current_stream(self.device)
        if self._held is not None:
            done = torch.cuda.Event()
            done.record(cur)                       # everything that read the previously handed-out slot is in front of this
            self._free[self._held] = done
        slot, bufs, ev, self._prepared = self._pending.popleft()
        cur.wait_event(ev)
        self._held = slot
        return tuple(bufs)

    @property
    def bytes_per_submit(self) -> int:
        return sum(b.numel() * b.element_size() for b in self._slots[0])
