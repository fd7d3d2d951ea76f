"""``ReplayStamps``: the ``Comm(s)`` / ``Reduce(s)`` intervals of an epoch replayed from a CUDA graph.

``CommTimer`` and the reducer bracket their intervals with CUDA events that the host records anew in every eager
epoch; a replay records nothing from the host.  So an epoch captured with ``train.GraphedEpoch(timed=True)`` brackets
each interval with two ``ops.stamp_globaltimer`` kernels instead: one thread each, storing the GPU's ``%globaltimer``
in nanoseconds, on the stream that does the work.  Every interval owns a
fixed pair of slots of one preallocated int64 device buffer, assigned in the order the capture opens the intervals, so
every replay rewrites the same addresses.  After the replay has been waited for, ``read`` copies the buffer to the host
once and ``seconds`` sums the intervals of each kind: ``comm`` (the exchange intervals ``CommTimer`` names in an eager
epoch) and ``reduce`` (the gradient all-reduce).  Intervals are differences of one GPU's clock."""
from contextlib import contextmanager

import torch


class ReplayStamps(object):

    def __init__(self, n_intervals: int, device):
        self.slots = torch.zeros(2 * n_intervals, dtype=torch.int64, device=device)
        self.names = {}             # interval name -> (kind, slot pair); slots[2 i] opens pair i, slots[2 i + 1] closes it

    @contextmanager
    def interval(self, name, stream, kind="comm"):
        """Stamp the start and the end of the work enqueued on ``stream`` inside the block (during a capture)."""
        from ... import ops
        if name in self.names:
            raise Exception(name + " already exists")
        i = len(self.names)
        if 2 * i + 2 > self.slots.numel():
            raise RuntimeError(f"ReplayStamps: interval {name!r} is number {i + 1}, the buffer holds "
                               f"{self.slots.numel() // 2}")
        self.names[name] = (kind, i)
        ops.stamp_globaltimer(self.slots[2 * i:2 * i + 1], stream)
        yield
        ops.stamp_globaltimer(self.slots[2 * i + 1:2 * i + 2], stream)

    def read(self) -> torch.Tensor:
        """The stamps of the last replay on the host (call after the replay was waited for)."""
        return self.slots.cpu()

    def seconds(self, values) -> dict:
        """``{"comm": s, "reduce": s}`` from the host copy ``values``: per kind, the sum of its intervals; 0.0 for a
        kind without intervals (one rank exchanges and all-reduces nothing, as in an eager epoch)."""
        out = {"comm": 0.0, "reduce": 0.0}
        for kind, i in self.names.values():
            out[kind] = out.get(kind, 0.0) + int(values[2 * i + 1] - values[2 * i]) * 1e-9
        return out
