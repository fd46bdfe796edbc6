"""Stream ordering of the device state the package keeps between calls (packed weights, attention constants, coordinate
tables, NIQE tables, captured graphs).

Such state is written by kernels on whatever stream was current when it was first needed and read later from any
stream.  Every cache keeps each entry as a `Produced`: its tensors plus an event recorded on the producing stream right
after the entry's last producing launch.  `use()` from another stream makes that stream wait on the event (the entry
is complete before any kernel reads it) and marks the tensors as used by that stream (record_stream), so that the
caching allocator does not hand their memory out again before that stream's queued reads have run, however the entry
is dropped later (resolution change, set_precision, an in-place edit, eviction).  No host synchronisation is added.
"""
import copy

import torch


def tensors(v):
    """The tensors of a value: a tensor, or a (nested) tuple / list / dict of them; anything else holds none."""
    if isinstance(v, torch.Tensor):
        yield v
    elif isinstance(v, (tuple, list)):
        for e in v:
            yield from tensors(e)
    elif isinstance(v, dict):
        for e in v.values():
            yield from tensors(e)


class Produced:
    """A cache entry: `value` (tensors, see `tensors`) whose producing launches have all been issued on the current
    stream.  Entries on the CPU or made inside a CUDA-graph capture carry no event."""

    __slots__ = ("value", "stream", "event")

    def __init__(self, value):
        self.value, self.stream, self.event = value, None, None
        if any(t.is_cuda for t in tensors(value)) and not torch.cuda.is_current_stream_capturing():
            self.stream = torch.cuda.current_stream()
            self.event = torch.cuda.Event()
            self.event.record(self.stream)

    def use(self):
        """The value, ordered for the current stream.  Inside a capture nothing is waited on: an event recorded outside
        it cannot be, and the captured graph keeps its own references (GRL._forward_graphed orders its warm-ups)."""
        if self.event is None:
            return self.value
        s = torch.cuda.current_stream()
        if s != self.stream and not torch.cuda.is_current_stream_capturing():
            s.wait_event(self.event)
            for t in tensors(self.value):
                if t.is_cuda:
                    t.record_stream(s)
        return self.value

    def __deepcopy__(self, memo):  # copy.deepcopy of a model: the copies are made on the current stream
        return Produced(copy.deepcopy(self.use(), memo))


def upload(t, device):
    """Host tensor -> `device` without a host synchronisation: staged through pinned memory (the caching host allocator
    keeps the staging block until the copy has run) and copied on the current stream."""
    device = torch.device(device)
    if device.type != "cuda":
        return t.to(device)
    return t.pin_memory().to(device, non_blocking=True)
