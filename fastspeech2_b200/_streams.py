"""Stream ordering of the device state the modules keep between calls.

Every call enqueues its device work on the CUDA stream current at that call.  State a module keeps from one call to the next
(packed weights, position tables, resampler taps, stream() iterators, stream pools) can be made on one stream and read on another,
so it carries a StreamState: the event of the last work that made or wrote it, which a call on another stream waits on first, and
the streams that have used it, on which its tensors are recorded before they are dropped, so that the caching allocator does not
hand their memory out while one of those streams still reads it.  A workspace is only ever used on the stream it was allocated on
(workspace()).
"""
from __future__ import annotations

import torch


def workspace(cached, nbytes: int, device, grow: float = 1.0, slack: int = 0):
    """Scratch memory of at least nbytes for a call on the current stream.  cached: (tensor, stream) of the module's previous call,
    or (None, None).  It is reused when it was allocated on the current stream and is large enough; otherwise it is dropped and
    int(nbytes * grow) + slack bytes are allocated on the current stream.  So a workspace is only used on the stream it was
    allocated on, and dropping it is safe while that stream's queued work still uses it: the caching allocator reuses its memory
    for later allocations on that stream only.  Calls on two streams each get their own.  Returns the new (tensor, stream)."""
    ws, stream = cached
    cur = torch.cuda.current_stream(device)
    if ws is None or stream != cur or ws.numel() < nbytes:
        ws = torch.empty(int(nbytes * grow) + slack, dtype=torch.uint8, device=device)
    return ws, cur


class StreamState:
    """The stream ordering of one piece of state on `device` (a no-op for a non-CUDA device).

    enter() before a call's work that reads or writes the state: the current stream waits for the state's last recorded work unless
    it is already ordered after it.  record() after a call's work that wrote the state (or made it).  release(*tensors) before the
    state drops tensors."""
    __slots__ = ("device", "event", "ordered", "used")

    def __init__(self, device):
        self.device = torch.device(device)
        self.event, self.ordered, self.used = None, set(), set()

    def enter(self):
        if self.device.type != "cuda":
            return None
        cur = torch.cuda.current_stream(self.device)
        if self.event is not None and cur not in self.ordered:
            cur.wait_event(self.event)
            self.ordered.add(cur)
        self.used.add(cur)
        return cur

    def record(self):
        if self.device.type != "cuda":
            return
        cur = torch.cuda.current_stream(self.device)
        if self.event is None:
            self.event = torch.cuda.Event()
        self.event.record(cur)
        self.ordered = {cur}
        self.used.add(cur)

    def release(self, *tensors):
        """Keeps the memory of `tensors` from reuse until every stream that used the state has finished the work queued on it so far
        (nothing to do while a single stream has used it: that stream's later work is ordered after its earlier work)."""
        if len(self.used) < 2:
            return
        for t in tensors:
            if isinstance(t, torch.Tensor) and t.device.type == "cuda":
                for s in self.used:
                    t.record_stream(s)


def made(device) -> StreamState:
    """The StreamState of state just made on the current stream."""
    st = StreamState(device)
    st.record()
    return st
