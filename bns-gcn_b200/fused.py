"""The fused training step: what train.py:400-413 of the reference does with ~300 small launches per epoch
(autograd nodes, per-parameter hooks and Adam updates, index / softmax / nll kernels, pads and transposes of the
weights) done with one launch per STEP of the algorithm, all in libbnsgcn.so (csrc/fused.cuh):

* ``ParamArena``     every parameter, its gradient and both Adam moments at the same offsets of four flat buffers.  The
                     gradient buffer is the Reducer's all-reduce bucket (helper/reducer.py:28-38 -> one message), the
                     layer functions below write each gradient exactly once, straight into its slot (no per-parameter
                     hook, no ``grad / n_train`` pass -- the factor rides on d(logits)), Adam is one kernel over the
                     arena.  Rows that TMA cannot address (41 classes) are stored padded (44) with the pad kept at zero;
                     W^T and bias sums the layer functions need are cached and refreshed by one kernel after each step.
* ``FusedAdam``      torch.optim.Adam (train.py:362) as ``bns_adam_step_f32`` + ``bns_derive_refresh``.
* ``softmax_xent``   loss + d(logits) of train.py:358-361 / 406-408 as one kernel (``bns_xent_f32``).
* ``PPLinearFn``     layer 0 with precomputed features (module/layer.py:29-30, 82-83): dropout -> GEMM.
* ``SageConvFn``     GraphSAGELayer.forward (module/layer.py:85-92) with a hand-written backward.

The mirrored modules keep their interface (module/layer.py, module/model.py); they take this path when the model was
given an arena by ``train.setup`` (GraphSAGE + LayerNorm/ReLU + --use-pp, the BASELINE configuration); everything else
runs the op-by-op autograd path as before.
"""
from __future__ import annotations

import ctypes
from typing import Dict, List, Optional, Tuple

import torch

from . import ops
from ._lib import DeriveEntry, check, lib
from .graph import PartitionGraph, halo_aggregate
from .module import dense


def _ceil4(n: int) -> int:
    return (n + 3) // 4 * 4


class Transient:
    """Per-step scratch a module may hold (e.g. the padded output that the loss kernel differentiates): never copied,
    never pickled -- ``copy.deepcopy(model)`` (evaluate.py snapshots the model) must not drag autograd graphs along."""

    def __init__(self):
        self.value = None

    def __deepcopy__(self, memo):
        return Transient()

    def __getstate__(self):
        return {"value": None}


class ParamArena:
    """Flat storage for a model's parameters (``flat_p``), gradients (``flat_g``) and Adam moments (``exp_avg``,
    ``exp_avg_sq``).  2-D parameters are stored with their row count padded to a multiple of 4, 1-D ones with their
    length padded to a multiple of 4 (pad = 0 forever: zero gradient, zero moments)."""

    def __init__(self, model: torch.nn.Module):
        params = [(n, p) for n, p in model.named_parameters()]
        if not params:
            raise ValueError("ParamArena: the model has no parameters")
        dev = params[0][1].device
        self.device = dev
        self.slots: Dict[int, Tuple[int, int, Tuple[int, ...]]] = {}        # id(param) -> (offset, numel, padded shape)
        off = 0
        for _, p in params:
            if p.dim() == 2:
                shape = (_ceil4(p.shape[0]), p.shape[1])
                size = _ceil4(shape[0] * shape[1])
            else:
                shape = (_ceil4(p.numel()),)
                size = shape[0]
            self.slots[id(p)] = (off, p.numel(), shape)
            off += size
        self.total = off
        self.flat_p = torch.zeros(off, dtype=torch.float32, device=dev)
        self.flat_g = torch.zeros(off, dtype=torch.float32, device=dev)
        self.exp_avg = torch.zeros(off, dtype=torch.float32, device=dev)
        self.exp_avg_sq = torch.zeros(off, dtype=torch.float32, device=dev)
        self.params = [p for _, p in params]
        self.names = [n for n, _ in params]
        with torch.no_grad():
            for p in self.params:
                o, n, _ = self.slots[id(p)]
                self.flat_p[o:o + n].copy_(p.detach().reshape(-1))
                p.data = self.flat_p[o:o + n].view(p.shape)
                p.grad = self.flat_g[o:o + n].view(p.shape)
        # derived parameters: (kind, ids) -> tensor; the table lives on the device and is rebuilt when an entry is added
        self._derived: Dict[tuple, torch.Tensor] = {}
        self._entries: List[DeriveEntry] = []
        self._table: Optional[torch.Tensor] = None
        self._keep: List[torch.Tensor] = []
        # --dense-dtype bf16: every GEMM of the fused layers rounds its operands to bf16 inside the kernel (f32 sums);
        # per run, never global: ranks that are threads of one process may differ
        self.dense_bf16 = False

    def __deepcopy__(self, memo):
        """A copied model (evaluate.py's snapshots) owns plain parameter tensors and takes the op-by-op path."""
        return None

    # ---- views ----------------------------------------------------------------------------------------------------
    def padded(self, p: torch.nn.Parameter) -> torch.Tensor:
        """The parameter with its padded shape (``[ceil4(rows), cols]`` / ``[ceil4(n)]``), a view of the arena."""
        o, _, shape = self.slots[id(p)]
        n = 1
        for s in shape:
            n *= s
        return self.flat_p[o:o + n].view(shape)

    def grad_padded(self, p: torch.nn.Parameter) -> torch.Tensor:
        o, _, shape = self.slots[id(p)]
        n = 1
        for s in shape:
            n *= s
        return self.flat_g[o:o + n].view(shape)

    def unpadded(self, flat: torch.Tensor, p: torch.nn.Parameter) -> torch.Tensor:
        """``p``'s slot of one of the four flat buffers, with ``p``'s own shape (the pad left out)."""
        o, n, _ = self.slots[id(p)]
        return flat[o:o + n].view(p.shape)

    # ---- derived parameters ------------------------------------------------------------------------------------------
    def _add(self, key, entry: DeriveEntry, out: torch.Tensor) -> torch.Tensor:
        self._derived[key] = out
        self._entries.append(entry)
        raw = b"".join(bytes(e) for e in self._entries)
        self._table = torch.frombuffer(bytearray(raw), dtype=torch.uint8).to(self.device)
        self.refresh(advance=None)
        return out

    def transposed(self, p: torch.nn.Parameter) -> torch.Tensor:
        """``padded(p).t()`` as a contiguous ``[cols, ceil4(rows)]`` matrix, refreshed after every optimizer step (the
        B operand of the input-gradient GEMM dX = dY W; the op-by-op path made this copy in every backward)."""
        key = ("T", id(p))
        hit = self._derived.get(key)
        if hit is not None:
            return hit
        w = self.padded(p)
        out = torch.zeros(w.shape[1], w.shape[0], dtype=torch.float32, device=self.device)
        e = DeriveEntry()
        e.op, e.rows, e.cols, e.ld_a, e.ld_dst = 0, w.shape[0], w.shape[1], w.stride(0), out.stride(0)
        e.a, e.b, e.dst = w.data_ptr(), None, out.data_ptr()
        return self._add(key, e, out)

    def bias_sum(self, b1: torch.nn.Parameter, b2: torch.nn.Parameter) -> torch.Tensor:
        """``padded(b1) + padded(b2)`` (the two biases of ``linear1(h) + linear2(ah)`` as one epilogue vector)."""
        key = ("S", id(b1), id(b2))
        hit = self._derived.get(key)
        if hit is not None:
            return hit
        x, y = self.padded(b1), self.padded(b2)
        out = torch.zeros_like(x)
        e = DeriveEntry()
        e.op, e.rows, e.cols, e.ld_a, e.ld_dst = 1, x.numel(), 1, 1, 1
        e.a, e.b, e.dst = x.data_ptr(), y.data_ptr(), out.data_ptr()
        return self._add(key, e, out)

    def refresh(self, advance: Optional[torch.Tensor]) -> None:
        """Recompute every derived parameter (one launch); ``advance``: the optimizer's step counter to increment."""
        n = len(self._entries)
        if n == 0 and advance is None:
            return
        with torch.cuda.device(self.device):
            check(lib.bns_derive_refresh(None if n == 0 else self._table.data_ptr(), n,
                                         None if advance is None else advance.data_ptr(),
                                         torch.cuda.current_stream(self.device).cuda_stream), "bns_derive_refresh")


class FusedAdam(torch.optim.Optimizer):
    """``torch.optim.Adam(model.parameters(), lr, weight_decay)`` (train.py:362-364) over a ``ParamArena``: one kernel
    for the update, one for the derived parameters and the step counter (which lives on the device: graph-safe)."""

    def __init__(self, arena: ParamArena, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0):
        super().__init__(arena.params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))
        self.arena = arena
        self.step_dev = torch.zeros(1, dtype=torch.int64, device=arena.device)

    def zero_grad(self, set_to_none: bool = True):
        """No-op: every gradient slot of the arena is overwritten (not accumulated) by each backward."""
        return None

    @torch.no_grad()
    def step(self, closure=None):
        g = self.param_groups[0]
        a = self.arena
        with torch.cuda.device(a.device):
            check(lib.bns_adam_step_f32(a.flat_p.data_ptr(), a.flat_g.data_ptr(), a.exp_avg.data_ptr(),
                                        a.exp_avg_sq.data_ptr(), a.total, float(g["lr"]), float(g["betas"][0]),
                                        float(g["betas"][1]), float(g["eps"]), float(g["weight_decay"]),
                                        self.step_dev.data_ptr(), torch.cuda.current_stream(a.device).cuda_stream),
                  "bns_adam_step_f32")
        a.refresh(advance=self.step_dev)
        return None

    _HYPER = ("lr", "betas", "eps", "weight_decay")

    def state_dict(self) -> dict:
        """Adam's state as copies on the device: ``{"step": int64 [1], "state": {parameter name: {"exp_avg",
        "exp_avg_sq"}} (each moment unpadded, in its parameter's shape), "param_groups": [the hyperparameters]}``."""
        a = self.arena
        state = {name: {"exp_avg": a.unpadded(a.exp_avg, p).clone(), "exp_avg_sq": a.unpadded(a.exp_avg_sq, p).clone()}
                 for name, p in zip(a.names, a.params)}
        g = self.param_groups[0]
        return {"step": self.step_dev.clone(), "state": state,
                "param_groups": [{k: g[k] for k in self._HYPER}]}

    @torch.no_grad()
    def load_state_dict(self, state_dict: dict) -> None:
        """The inverse of ``state_dict``: the moments go into their arena slots (the pad stays zero), the step into
        ``step_dev`` in place (a captured graph keeps reading the same counter).  The weights are not part of it: after
        loading them into the model, call ``arena.refresh(advance=None)``."""
        a = self.arena
        got = state_dict["state"]
        if set(got) != set(a.names):
            raise ValueError(f"FusedAdam.load_state_dict: parameters {sorted(set(a.names) - set(got))} missing, "
                             f"{sorted(set(got) - set(a.names))} unexpected")
        for name, p in zip(a.names, a.params):
            for key, flat in (("exp_avg", a.exp_avg), ("exp_avg_sq", a.exp_avg_sq)):
                src = got[name][key]
                if tuple(src.shape) != tuple(p.shape):
                    raise ValueError(f"FusedAdam.load_state_dict: {name}.{key} has shape {tuple(src.shape)}, the "
                                     f"parameter {tuple(p.shape)}")
                a.unpadded(flat, p).copy_(src)
        self.step_dev.copy_(torch.as_tensor(state_dict["step"]).reshape(1))
        for k, v in state_dict["param_groups"][0].items():
            self.param_groups[0][k] = v


# ---- loss ------------------------------------------------------------------------------------------------------------
_XENT_WS: Dict[tuple, torch.Tensor] = {}


def softmax_xent(logits_padded: torch.Tensor, n_class: int, labels: torch.Tensor, mask: Optional[torch.Tensor],
                 grad_scale: float):
    """``(loss, dlogits)``: sum-reduced CrossEntropy (int64 ``labels [n]``) or BCE-with-logits (float ``labels [n, C]``)
    over the rows where ``mask`` is set, and its gradient times ``grad_scale`` with the layout of ``logits_padded``
    (``[n, >= n_class]``; pad columns and unmasked rows get zeros)."""
    x = logits_padded
    if not (x.is_cuda and x.dtype == torch.float32 and x.dim() == 2 and x.stride(1) == 1):
        raise RuntimeError("softmax_xent: logits must be a row-major f32 CUDA matrix")
    n, cp = x.shape
    dev = x.device
    key = (dev, torch.cuda.current_stream(dev).cuda_stream)
    ws = _XENT_WS.get(key)
    if ws is None:
        ws = _XENT_WS[key] = torch.zeros(lib.bns_xent_workspace_bytes(), dtype=torch.uint8, device=dev)
    loss = torch.empty(1, dtype=torch.float32, device=dev)
    dl = torch.empty((n, cp), dtype=torch.float32, device=dev)
    ce = labels.dtype == torch.int64
    if not ce:
        labels = labels.to(torch.float32)
        if labels.stride(1) != 1:
            labels = labels.contiguous()
    m = None
    if mask is not None:
        m = mask if mask.dtype == torch.uint8 else mask.view(torch.uint8) if mask.dtype == torch.bool else mask.to(torch.uint8)
    with torch.cuda.device(dev):
        check(lib.bns_xent_f32(x.data_ptr(), x.stride(0), n, n_class, labels.data_ptr() if ce else None,
                               None if ce else labels.data_ptr(), 0 if ce else labels.stride(0),
                               None if m is None else m.data_ptr(), float(grad_scale), loss.data_ptr(), dl.data_ptr(),
                               dl.stride(0), cp, ws.data_ptr(), ws.numel(), torch.cuda.current_stream(dev).cuda_stream),
              "bns_xent_f32")
    return loss[0], dl


# ---- element-wise ------------------------------------------------------------------------------------------------------
def dropout(x: torch.Tensor, p: float, seed: int) -> torch.Tensor:
    """``dropout_p(x)`` with the Philox stream of ``ops.RNG`` (offset = the epoch; replay-safe through offset_dev)."""
    if p <= 0.0:
        return x
    x = x.contiguous()
    y = torch.empty_like(x)
    off, off_dev = ops.RNG["offset"], ops.RNG["offset_dev"]
    with torch.cuda.device(x.device):
        check(lib.bns_dropout_f32(x.data_ptr(), x.stride(0), x.shape[0], x.shape[1], float(p), seed & (2 ** 64 - 1),
                                  off & (2 ** 64 - 1), ops._ptr(off_dev), y.data_ptr(), y.stride(0),
                                  torch.cuda.current_stream(x.device).cuda_stream), "bns_dropout_f32")
    return y


class DropoutFn(torch.autograd.Function):
    """``dropout_p`` as an autograd node on ``bns_dropout_f32``: the backward regenerates the Philox mask of the forward
    (same seed, same epoch offset) instead of storing it."""

    @staticmethod
    def forward(ctx, x, p: float, seed: int):
        ctx.p, ctx.seed = p, seed
        ctx.rng = (ops.RNG["seed"], ops.RNG["offset"], ops.RNG["offset_dev"])
        return dropout(x, p, seed)

    @staticmethod
    def backward(ctx, dy):
        keep = ops.RNG["seed"], ops.RNG["offset"], ops.RNG["offset_dev"]
        ops.RNG.update(seed=ctx.rng[0], offset=ctx.rng[1], offset_dev=ctx.rng[2])
        dx = dropout(dy, ctx.p, ctx.seed)
        ops.RNG.update(seed=keep[0], offset=keep[1], offset_dev=keep[2])
        return dx, None, None


def gather_friendly(rows: int, width: int, device) -> torch.Tensor:
    """An uninitialised ``[rows, width]`` f32 matrix whose row stride is a multiple of 64 bytes: a narrow row that the
    SpMM gathers (44 padded class scores = 176 bytes) then always spans the minimum number of 128-byte lines (2), where
    a 176-byte stride makes 3 of every 8 rows straddle a third line."""
    ld = (width + 15) // 16 * 16
    return torch.empty(rows, ld, dtype=torch.float32, device=device)[:, :width]


def scale_rows(x: torch.Tensor, rs: Optional[torch.Tensor], out: Optional[torch.Tensor] = None,
               bias: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``x * rs[:, None] + bias`` (``bns_scale_rows_f32``)."""
    if x.stride(1) != 1:
        x = x.contiguous()
    y = torch.empty(x.shape, dtype=torch.float32, device=x.device) if out is None else out
    with torch.cuda.device(x.device):
        check(lib.bns_scale_rows_f32(x.data_ptr(), x.stride(0), x.shape[0], x.shape[1], ops._ptr(rs), ops._ptr(bias),
                                     y.data_ptr(), y.stride(0), torch.cuda.current_stream(x.device).cuda_stream),
              "bns_scale_rows_f32")
    return y


def dropout_supported(x: torch.Tensor) -> bool:
    return x.is_cuda and x.dtype == torch.float32 and x.dim() == 2 and x.shape[1] % 4 == 0 and x.stride(1) == 1


# ---- layer functions ---------------------------------------------------------------------------------------------------
class PPLinearFn(torch.autograd.Function):
    """``dropout(x) @ W^T + b`` for the precomputed layer 0 (module/layer.py:29-30, 82-83 after module/model.py:45/80).
    The parameters are inputs only so that autograd records the node; their gradients are written into the arena."""

    @staticmethod
    def forward(ctx, x, weight, bias, arena: ParamArena, p: float, seed: int):
        xd = dropout(x, p, seed)
        y = dense.tc_mm_tn(xd, arena.padded(weight), None if bias is None else arena.padded(bias), bf16=arena.dense_bf16)
        ctx.save_for_backward(xd)
        ctx.arena, ctx.weight, ctx.bias, ctx.p, ctx.seed = arena, weight, bias, p, seed
        ctx.rng = (ops.RNG["seed"], ops.RNG["offset"], ops.RNG["offset_dev"])
        return y

    @staticmethod
    def backward(ctx, dy):
        (xd,) = ctx.saved_tensors
        a = ctx.arena
        dy = dy.contiguous()
        if ctx.bias is not None:
            dense.colsum(dy, out=a.grad_padded(ctx.bias))
        dense.tc_mm_nt(dy, xd, out=a.grad_padded(ctx.weight), bf16=a.dense_bf16)
        dx = None
        if ctx.needs_input_grad[0]:
            dx = dense.tc_mm_tn(dy, a.transposed(ctx.weight), bf16=a.dense_bf16)
            if ctx.p > 0.0:                     # d dropout: the same mask, regenerated
                keep = ops.RNG["seed"], ops.RNG["offset"], ops.RNG["offset_dev"]
                ops.RNG.update(seed=ctx.rng[0], offset=ctx.rng[1], offset_dev=ctx.rng[2])
                dx = dropout(dx, ctx.p, ctx.seed)
                ops.RNG.update(seed=keep[0], offset=keep[1], offset_dev=keep[2])
        return dx, None, None, None, None, None


def _gather_table(x: torch.Tensor, bf16: bool) -> torch.Tensor:
    """What an aggregation pass gathers: ``x`` itself, or (``--agg-dtype bf16``) its rows rounded to bf16."""
    return ops.cvt_rows_bf16(x) if bf16 else x


def _aggregate(g: PartitionGraph, x_u: torch.Tensor, rs: torch.Tensor, ready, bf16: bool = False,
               halo: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``rs * (A_in x_u[:n_in] + A_out[:, sampled] x_u[n_in:])`` -- the inner pass first (it needs local rows only), the
    halo pass after the exchange's event.  ``bf16``: both passes gather bf16 copies of the rows (f32 sums).  ``halo``:
    the halo rows as they arrived in bf16 (``--comm-dtype bf16``; ``x_u`` is then the inner rows alone), gathered as
    they are."""
    y = ops.spmm_auto(g.a_in, _gather_table(x_u[:g.n_in], bf16), row_scale=rs)
    if ready is not None:
        torch.cuda.current_stream(x_u.device).wait_event(ready)
    if halo is not None:
        if g.a_out is not None and halo.shape[0]:
            halo_aggregate(g, halo, y, rs, None)
    elif g.a_out is not None and x_u.shape[0] > g.n_in:
        halo_aggregate(g, _gather_table(x_u[g.n_in:], bf16), y, rs, None)
    return y


def _halo_rows(h_u: torch.Tensor, n_in: int, halo: Optional[torch.Tensor]) -> torch.Tensor:
    """The f32 halo rows a narrow layer transforms: ``h_u[n_in:]``, or (``--comm-dtype bf16``) the received bf16 rows
    widened into a matrix of their own -- the inner rows stay where they are."""
    return h_u[n_in:] if halo is None else ops.cvt_rows_f32(halo)


def _weight_grad(dt: torch.Tensor, saved, n_in: int, out: torch.Tensor, bf16: bool) -> None:
    """``dt^T h_u`` into ``out``.  ``saved``: ``(h_u,)``, or ``(h_in, h_halo)`` when the halo rows are kept apart
    (``--comm-dtype bf16``): the inner rows' product, then the halo rows' product added (one f32 add per element).
    ``bf16``: the products of ``--dense-dtype bf16``."""
    if len(saved) == 1:
        dense.tc_mm_nt(dt, saved[0], out=out, bf16=bf16)
        return
    h_in, h_halo = saved
    dense.tc_mm_nt(dt[:n_in], h_in, out=out, bf16=bf16)
    if h_halo.shape[0]:
        part = dense.tc_mm_nt(dt[n_in:], h_halo, bf16=bf16)
        rows = torch.arange(out.shape[0], dtype=torch.int64, device=out.device)
        ops.scatter_add_div(out, rows, part, 1.0)                      # x / 1 is x: an exact row-wise add


def _aggregate_t(g: PartitionGraph, dys: torch.Tensor, n_u: int, cs_in=None, cs_halo=None, after_halo=None,
                 bf16: bool = False) -> torch.Tensor:
    """``cs * (A^T dys)`` over the epoch's graph: ``[n_u, F]`` (inner rows, then the sampled halo rows); ``cs``: GCN's
    per-source scale (1/sqrt(out_deg)), applied as the row scale of the transposed products.  The halo rows come first;
    ``after_halo(du)`` is called as soon as they are final (the gradient return trip starts there).  ``bf16``: both
    passes gather one bf16 copy of ``dys``."""
    du = torch.empty(n_u, dys.shape[1], dtype=torch.float32, device=dys.device)
    dys = _gather_table(dys, bf16)
    if n_u > g.n_in:
        tail = du[g.n_in:]
        tail.zero_()
        if g.a_out_t is not None:
            ops.spmm(g.a_out_t, dys, tail, row_scale=cs_halo, row_map=g.slot)
    if after_halo is not None:
        after_halo(du)
    ops.spmm_auto(g.a_in_t, dys, du[:g.n_in], row_scale=cs_in)
    return du


class SageConvFn(torch.autograd.Function):
    """GraphSAGELayer.forward, training branch (module/layer.py:85-92):

        ah = (A h_u) / deg;   out = linear1(h_u[:n_in]) + linear2(ah)

    Wide layers run exactly that; a layer that narrows (256 -> 41 classes) transforms first, ``A (h_u W2^T)``, so that
    the aggregation gathers 44-float rows (same math, see module/layer.py AGGREGATE_AFTER_TRANSFORM).  Output:
    ``[n_in, ceil4(out_features)]`` (pad columns exactly zero).  Backward writes the six parameter gradients into the
    arena and returns d h_u ``[n_u, in_features]``."""

    @staticmethod
    def forward(ctx, h_u, w1, b1, w2, b2, g: PartitionGraph, rs, ready, arena: ParamArena, narrow_first: bool,
                exchange=None, halo=None):
        """``exchange = (Buffer, layer)`` when ``h_u`` came out of ``Buffer.update``: the backward then hands the halo
        rows of its gradient to ``Buffer.begin_backward`` as soon as they are final.  ``halo``: the received halo rows in
        bf16 (``--comm-dtype bf16``); ``h_u`` is then the inner rows alone, and so is the returned gradient."""
        ctx.exchange, ctx.inner_only = exchange, halo is not None
        n_in = g.n_in
        h_u = h_u.contiguous()
        W1, W2 = arena.padded(w1), arena.padded(w2)
        bf = arena.dense_bf16
        h_in = h_u[:n_in]
        if narrow_first:
            # transform, then aggregate; the local rows go first -- their GEMM and the inner-edge pass need nothing from
            # the peers and hide the exchange -- the halo rows after the exchange's event
            n_u = h_u.shape[0] if halo is None else n_in + halo.shape[0]
            t = gather_friendly(n_u, W2.shape[0], h_u.device)                   # [n_u, out_p]
            dense.tc_mm_tn(h_in, W2, out=t[:n_in], bf16=bf)
            out = dense.tc_mm_tn(h_in, W1, arena.bias_sum(b1, b2), bf16=bf)     # linear1(h) + b1 + b2 ...
            ops.spmm_auto(g.a_in, t[:n_in], out, row_scale=rs, accumulate=True)  # ... + (A_in t) / deg
            if ready is not None:
                torch.cuda.current_stream(h_u.device).wait_event(ready)
            h_halo = _halo_rows(h_u, n_in, halo)
            if g.a_out is not None and n_u > n_in:
                dense.tc_mm_tn(h_halo, W2, out=t[n_in:], bf16=bf)
                halo_aggregate(g, t[n_in:], out, rs, None)                      # ... + (A_out t_halo) / deg
            ctx.save_for_backward(*((h_u,) if halo is None else (h_in, h_halo)))
        else:
            ah = _aggregate(g, h_u, rs, ready, g.agg_bf16, halo)                # [n_in, in]
            t = dense.tc_mm_tn(ah, W2, arena.padded(b2), bf16=bf)
            out = dense.tc_mm_tn(h_in, W1, arena.padded(b1), addend=t, bf16=bf)
            ctx.save_for_backward(h_u, ah)
        ctx.n_u = h_u.shape[0] if halo is None else n_in + halo.shape[0]
        ctx.g, ctx.rs, ctx.arena, ctx.narrow = g, rs, arena, narrow_first
        ctx.params = (w1, b1, w2, b2)
        return out

    @staticmethod
    def backward(ctx, dout):
        g, rs, a = ctx.g, ctx.rs, ctx.arena
        w1, b1, w2, b2 = ctx.params
        n_in = g.n_in
        bf = a.dense_bf16
        dout = dout.contiguous()
        dense.colsum(dout, out=a.grad_padded(b1), out2=a.grad_padded(b2))
        begin = None
        if ctx.exchange is not None:
            buf, layer = ctx.exchange
            begin = lambda du_: buf.begin_backward(layer, du_)      # noqa: E731
        if ctx.narrow:
            saved = ctx.saved_tensors
            h_in, n_u = saved[0][:n_in], ctx.n_u
            dys = scale_rows(dout, rs, out=gather_friendly(n_in, dout.shape[1], dout.device))
            dt = _aggregate_t(g, dys, n_u)                                      # [n_u, out_p]
            du = torch.empty(n_u, h_in.shape[1], dtype=torch.float32, device=dout.device)
            if n_u > n_in:                                                      # halo rows first: they travel ...
                dense.tc_mm_tn(dt[n_in:], a.transposed(w2), out=du[n_in:], bf16=bf)
            if begin is not None:
                begin(du)
            dense.tc_mm_tn(dt[:n_in], a.transposed(w2), out=du[:n_in], bf16=bf)  # ... while the local rows are computed
            dense.tc_mm_nt(dout, h_in, out=a.grad_padded(w1), bf16=bf)
            _weight_grad(dt, saved, n_in, a.grad_padded(w2), bf)
        else:
            h_u, ah = ctx.saved_tensors
            dys = dense.tc_mm_tn(dout, a.transposed(w2), row_scale=rs, bf16=bf)  # (dout W2) / deg
            du = _aggregate_t(g, dys, ctx.n_u, after_halo=begin, bf16=g.agg_bf16)
            dense.tc_mm_nt(dout, h_u[:n_in], out=a.grad_padded(w1), bf16=bf)
            dense.tc_mm_nt(dout, ah, out=a.grad_padded(w2), bf16=bf)
        inner = du[:n_in]
        dense.tc_mm_tn(dout, a.transposed(w1), addend=inner, out=inner, bf16=bf)  # += dout W1, in place
        return inner if ctx.inner_only else du, None, None, None, None, None, None, None, None, None, None, None


class GcnConvFn(torch.autograd.Function):
    """GCNLayer.forward, training branch (module/layer.py:32-38):

        out = linear( (A (h_u / out_norm_u)) / in_norm )

    with the same aggregate-after-transform rewrite as ``SageConvFn`` where the layer narrows.  ``rs = 1/in_norm``
    (``[n_in]``), ``cs_u = 1/out_norm`` over the STATIC ``[inner | halo]`` numbering; the halo part rides in the epoch's
    compaction as per-entry weights (``PartitionGraph.halo_col_scale``)."""

    @staticmethod
    def forward(ctx, h_u, w, b, g: PartitionGraph, rs, cs_u, ready, arena: ParamArena, narrow_first: bool,
                exchange=None, halo=None):
        """``exchange`` / ``halo``: as for ``SageConvFn`` (``--comm-dtype bf16``)."""
        ctx.exchange, ctx.inner_only = exchange, halo is not None
        n_in = g.n_in
        h_u = h_u.contiguous()
        W, bp = arena.padded(w), arena.padded(b)
        bf = arena.dense_bf16
        cs_in, cs_halo = cs_u[:n_in], cs_u[n_in:]
        n_u = h_u.shape[0] if halo is None else n_in + halo.shape[0]
        has_halo = g.a_out is not None and n_u > n_in
        if narrow_first:
            t = gather_friendly(n_u, W.shape[0], h_u.device)                                          # [n_u, out_p]
            dense.tc_mm_tn(h_u[:n_in], W, out=t[:n_in], bf16=bf)                                      # local rows first
            ts = scale_rows(t[:n_in], cs_in, out=gather_friendly(n_in, W.shape[0], h_u.device))
            s = ops.spmm_auto(g.a_in, ts)                                                             # raw sums
            if ready is not None:
                torch.cuda.current_stream(h_u.device).wait_event(ready)
            h_halo = _halo_rows(h_u, n_in, halo)
            if has_halo:
                dense.tc_mm_tn(h_halo, W, out=t[n_in:], bf16=bf)
                halo_aggregate(g, t[n_in:], s, None, cs_halo)
            out = scale_rows(s, rs, bias=bp)                                                          # / in_norm + b
            ctx.save_for_backward(*((h_u,) if halo is None else (h_u[:n_in], h_halo)))
        else:
            bf16 = g.agg_bf16
            y = ops.spmm_auto(g.a_in, _gather_table(scale_rows(h_u[:n_in], cs_in), bf16), row_scale=rs)
            if ready is not None:
                torch.cuda.current_stream(h_u.device).wait_event(ready)
            if has_halo:
                halo_aggregate(g, halo if halo is not None else _gather_table(h_u[n_in:], bf16), y, rs, cs_halo)
            out = dense.tc_mm_tn(y, W, bp, bf16=bf)
            ctx.save_for_backward(y)
        ctx.n_u = n_u
        ctx.g, ctx.rs, ctx.cs, ctx.arena, ctx.narrow, ctx.params = g, rs, (cs_in, cs_halo), arena, narrow_first, (w, b)
        return out

    @staticmethod
    def backward(ctx, dout):
        g, rs, a = ctx.g, ctx.rs, ctx.arena
        cs_in, cs_halo = ctx.cs
        w, b = ctx.params
        bf = a.dense_bf16
        dout = dout.contiguous()
        dense.colsum(dout, out=a.grad_padded(b))
        begin = None
        if ctx.exchange is not None:
            buf, layer = ctx.exchange
            begin = lambda du_: buf.begin_backward(layer, du_)      # noqa: E731
        if ctx.narrow:
            dys = scale_rows(dout, rs, out=gather_friendly(g.n_in, dout.shape[1], dout.device))
            dt = _aggregate_t(g, dys, ctx.n_u, cs_in, cs_halo)                  # [n_u, out_p]
            _weight_grad(dt, ctx.saved_tensors, g.n_in, a.grad_padded(w), bf)
            du = dense.tc_mm_tn(dt, a.transposed(w), bf16=bf)                   # [n_u, in]
            if begin is not None:
                begin(du)
        else:
            (y,) = ctx.saved_tensors
            dense.tc_mm_nt(dout, y, out=a.grad_padded(w), bf16=bf)
            dys = dense.tc_mm_tn(dout, a.transposed(w), row_scale=rs, bf16=bf)  # (dout W) / in_norm
            du = _aggregate_t(g, dys, ctx.n_u, cs_in, cs_halo, after_halo=begin, bf16=g.agg_bf16)
        return du[:g.n_in] if ctx.inner_only else du, None, None, None, None, None, None, None, None, None, None


def sage_layer_eligible(layer, feat: torch.Tensor) -> bool:
    """Shapes the wgmma kernels take on every GEMM of the fused layer."""
    lin = layer.linear if layer.use_pp else layer.linear1
    k = lin.in_features
    return (feat.is_cuda and feat.dtype == torch.float32 and feat.dim() == 2 and feat.stride(1) == 1 and k % 4 == 0
            and feat.shape[1] == k and feat.stride(0) % 4 == 0 and feat.data_ptr() % 16 == 0 and lin.bias is not None)
