"""``Reducer``: the weight-gradient all-reduce (reference: helper/reducer.py:17-55).

Same surface (``init(model)``, ``reduce(param, name, grad, n_train)`` called from the per-parameter autograd
hooks of train.py:239-242/337-338, ``synchronize()`` before ``optimizer.step``), different plumbing: the
reference divides each gradient by ``n_train``, copies it to pinned host memory and issues one gloo all-reduce per
parameter on a thread pool (:28-38).  Here every hook writes ``grad / n_train`` into its slice of ONE flat device
bucket and ``synchronize()`` issues a single NCCL all-reduce of the bucket on a side stream, then points each
``param.grad`` at its slice (no copy back)."""
from __future__ import annotations

import torch

from . import context as ctx


class Reducer(object):

    def __init__(self):
        super(Reducer, self).__init__()
        self._slices = {}
        self._flat = None
        self._stream = None
        self._pending = []
        self._events = None
        self.graph_mode = False
        self.stamps = None          # a timed capture (train.GraphedEpoch): timer.ReplayStamps bracket the all-reduce

    def init(self, model):
        params = [(n, p) for n, p in model.named_parameters()]
        total = sum(p.numel() for _, p in params)
        dev = params[0][1].device if params else torch.device('cpu')
        self._flat = torch.zeros(total, dtype=torch.float32, device=dev)
        off = 0
        for n, p in params:
            self._slices[n] = (off, p.numel())
            off += p.numel()
        if dev.type == 'cuda':
            self._stream = torch.cuda.Stream(device=dev)
        self._comm = ctx.comm()

    def init_arena(self, arena):
        """Fused training step (fused.ParamArena): the arena's gradient buffer IS the all-reduce bucket; the layer
        functions fill it (already divided by n_train: the factor rides on d(logits)), no per-parameter hook runs."""
        self._arena = arena
        self._flat = arena.flat_g
        dev = self._flat.device
        if dev.type == 'cuda':
            self._stream = torch.cuda.Stream(device=dev)
        self._comm = ctx.comm()

    def reduce(self, param, name, data, n_train):
        off, n = self._slices[name]
        torch.div(data, n_train, out=self._flat[off:off + n].view_as(data))      # reducer.py:34 (grad /= n_train)
        self._pending.append((param, name))

    def synchronize(self):
        if not self._pending and getattr(self, "_arena", None) is None:
            return
        c = self._comm
        if c.size > 1:
            if self._stream is not None:
                cur = torch.cuda.current_stream(self._flat.device)
                self._stream.wait_stream(cur)
                with torch.cuda.stream(self._stream):
                    if self.graph_mode and self.stamps is not None:
                        with self.stamps.interval("reduce", self._stream, kind="reduce"):
                            c.all_reduce_sum(self._flat)
                    elif self.graph_mode:
                        c.all_reduce_sum(self._flat)
                    else:
                        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        s.record(self._stream)
                        c.all_reduce_sum(self._flat)                              # reducer.py:37 / :46, one message
                        e.record(self._stream)
                        self._events = (s, e)
                cur.wait_stream(self._stream)
            else:
                c.all_reduce_sum(self._flat)
        for param, name in self._pending:
            off, n = self._slices[name]
            param.grad = self._flat[off:off + n].view_as(param)
        self._pending.clear()

    def last_reduce_seconds(self) -> float:
        if self._events is None:
            return 0.0
        s, e = self._events
        e.synchronize()
        return s.elapsed_time(e) * 1e-3
