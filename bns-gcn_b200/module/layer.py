"""``GCNLayer`` / ``GraphSAGELayer`` with the reference's constructor, parameter names, initialisation and
``forward`` signatures (module/layer.py:8-103); the DGL message passing inside is one call into libbnsgcn.so."""
import math

import torch
import torch.nn.functional as F
from torch import nn

from ..graph import FullGraphHandle, PartitionAggregate, PartitionEvalGraph, PartitionGraph
from . import dense
from ..ops import AggregateSum


# Aggregate-after-transform.  The reference computes  linear(A @ h)  (module/layer.py:38, 91-92).  A is linear, so
# (A @ h) @ W^T == A @ (h @ W^T): when the layer narrows (out_feats < in_feats, e.g. 256 -> 41 classes) doing the
# dense transform first shrinks every gathered row of the SpMM -- forward and transpose -- by in/out (6x on the
# last layer of the Reddit config), at the price of transforming the n_U - n_in halo rows too.  Same math, f32
# rounding differs at the 1e-7 level (tests pin it against the oracle at 1e-4).  Set to False for the literal order.
AGGREGATE_AFTER_TRANSFORM = True


def _narrow_first(weight, feat):
    """``feat @ W^T`` with the output padded to a multiple of 4 columns (16-byte SpMM lanes).

    This reads EVERY row of ``feat`` -- including the halo rows an overlapped exchange may still be writing -- so it
    first makes the current stream wait for that exchange (``Buffer.update(..., overlap=True)`` leaves the event on
    the tensor)."""
    ready = getattr(feat, '_bns_ready', None)
    if ready is not None:
        torch.cuda.current_stream(feat.device).wait_event(ready)
    out = weight.shape[0]
    pad = (-out) % 4
    w = F.pad(weight, (0, 0, 0, pad)) if pad else weight
    return dense.linear(feat, w), out


def _aggregate(graph, feat, rs, cs_u=None):
    """``update_all(copy_u, sum)`` with the row / column scalings fused (K1+K2)."""
    if isinstance(graph, PartitionGraph):
        cs_in = cs_halo = None
        if cs_u is not None:
            cs_in, cs_halo = cs_u[:graph.n_in], cs_u[graph.n_in:]
        return PartitionAggregate.apply(feat, graph, rs, cs_in, cs_halo, getattr(feat, '_bns_ready', None))
    if isinstance(graph, FullGraphHandle):
        return AggregateSum.apply(feat, graph.a, rs, cs_u)
    if isinstance(graph, PartitionEvalGraph):
        return graph.aggregate(feat, rs, cs_u)
    raise TypeError(f"unsupported graph handle {type(graph).__name__}")


def _uniform_init(*linears):
    """``reset_parameters`` of the reference's layers (module/layer.py:20-24, 65-77): every weight, then every bias,
    from U(-1/sqrt(fan_in), 1/sqrt(fan_in)) of the FIRST linear -- the draw order fixes the weights under a seed."""
    bound = 1. / math.sqrt(linears[0].weight.size(1))
    for t in [lin.weight for lin in linears] + [lin.bias for lin in linears if lin.bias is not None]:
        t.data.uniform_(-bound, bound)


def _apply(lin, x, addend=None):
    return dense.linear(x, lin.weight, lin.bias, addend=addend)


class GCNLayer(nn.Module):

    def __init__(self, in_feats, out_feats, bias=True, use_pp=False):
        super().__init__()
        self.use_pp = use_pp
        self.linear = nn.Linear(in_feats, out_feats, bias=bias)
        self.reset_parameters()

    def reset_parameters(self):
        _uniform_init(self.linear)

    _lin = staticmethod(_apply)

    def forward(self, graph, feat, in_norm, out_norm, fused=None):
        """``out_norm``: sqrt(out_deg) of every *local* node (inner then halo, static) -- the reference rebuilds a
        U-ordered copy of it every epoch (train.py:245-253), which the slot map makes unnecessary.
        ``fused``: see ``GraphSAGELayer.forward``."""
        if self.training and fused is not None:
            from .. import fused as _f
            arena, p, seed, holder = fused
            if self.use_pp:
                return _f.PPLinearFn.apply(feat, self.linear.weight, self.linear.bias, arena, p, seed)
            out_f, in_f = self.linear.out_features, self.linear.in_features
            narrow = AGGREGATE_AFTER_TRANSFORM and out_f < in_f
            # --comm-dtype bf16 / fp8: the halo rows arrive apart from feat, and their gradient returns through the exchange
            halo = getattr(feat, '_bns_halo', None)
            out = _f.GcnConvFn.apply(feat, self.linear.weight, self.linear.bias, graph, graph.recip(in_norm),
                                     graph.recip(out_norm), getattr(feat, '_bns_ready', None), arena, narrow,
                                     None if halo is None else getattr(feat, '_bns_exchange', None), halo)
            holder.value = out
            return out if out.shape[1] == out_f else out[:, :out_f]
        if self.training:
            if self.use_pp:
                return self._lin(self.linear, feat)                                 # layer.py:29-30
            if AGGREGATE_AFTER_TRANSFORM and self.linear.out_features < self.linear.in_features:
                t, out = _narrow_first(self.linear.weight, feat)
                h = _aggregate(graph, t, graph.recip(in_norm), graph.recip(out_norm))[:, :out]
                return h + self.linear.bias if self.linear.bias is not None else h
            h = _aggregate(graph, feat, graph.recip(in_norm), graph.recip(out_norm))  # :32-38
            return self._lin(self.linear, h)
        if self.use_pp and isinstance(graph, PartitionEvalGraph):
            # D_in^-1/2 A D_out^-1/2 x over the whole graph, restricted to the inner rows, IS the precomputed input
            # this rank holds (train.precompute): nothing to aggregate, nothing to exchange
            return self._lin(self.linear, feat)
        in_n = torch.sqrt(graph.in_degrees().float())                                # :40-45
        out_n = torch.sqrt(graph.out_degrees().float())
        return self._lin(self.linear, _aggregate(graph, feat, 1.0 / in_n, 1.0 / out_n))


class GraphSAGELayer(nn.Module):
    """Parameters ``linear`` (precomputed layer 0: input ``[x | mean_nbr(x)]``) or ``linear1`` (self) + ``linear2``
    (neighbours), named as in the reference."""

    def __init__(self, in_feats, out_feats, bias=True, use_pp=False):
        super().__init__()
        self.use_pp = use_pp
        if use_pp:
            self.linear = nn.Linear(2 * in_feats, out_feats, bias=bias)
        else:
            self.linear1 = nn.Linear(in_feats, out_feats, bias=bias)
            self.linear2 = nn.Linear(in_feats, out_feats, bias=bias)
        self.reset_parameters()

    def reset_parameters(self):
        _uniform_init(*([self.linear] if self.use_pp else [self.linear1, self.linear2]))

    _lin = staticmethod(_apply)

    def forward(self, graph, feat, in_norm, fused=None):
        """``fused = (arena, dropout p of the input, Philox seed, holder)``: the fused training step (fused.py) -- one
        autograd node for the whole layer, parameter gradients written into the arena; ``holder.value`` receives the
        output with its padded width (what the loss kernel reads and differentiates)."""
        if self.training and fused is not None:
            from .. import fused as _f
            arena, p, seed, holder = fused
            if self.use_pp:
                return _f.PPLinearFn.apply(feat, self.linear.weight, self.linear.bias, arena, p, seed)
            out_f, in_f = self.linear2.out_features, self.linear2.in_features
            narrow = AGGREGATE_AFTER_TRANSFORM and out_f < in_f
            out = _f.SageConvFn.apply(feat, self.linear1.weight, self.linear1.bias, self.linear2.weight,
                                      self.linear2.bias, graph, graph.recip(in_norm), getattr(feat, '_bns_ready', None),
                                      arena, narrow, getattr(feat, '_bns_exchange', None), getattr(feat, '_bns_halo', None))
            holder.value = out                  # [n_in, ceil4(out_features)]
            return out if out.shape[1] == out_f else out[:, :out_f]
        if self.training:
            if self.use_pp:
                return self._lin(self.linear, feat)                                 # layer.py:82-83
            num_dst = graph.num_nodes('_V')
            if AGGREGATE_AFTER_TRANSFORM and self.linear2.out_features < self.linear2.in_features:
                t, out = _narrow_first(self.linear2.weight, feat)
                ah = _aggregate(graph, t, graph.recip(in_norm))      # [n_in, out padded to 4]; the "+ ah" rides in
                res = dense.linear(feat[0:num_dst], self.linear1.weight, self.linear1.bias, addend=ah)   # the epilogue
                return res + self.linear2.bias if self.linear2.bias is not None else res
            ah = _aggregate(graph, feat, graph.recip(in_norm))                       # :85-91  (sum / degs)
            return dense.linear(feat[0:num_dst], self.linear1.weight, self.linear1.bias,
                                addend=self._lin(self.linear2, ah))                  # :92, "+" fused into the epilogue
        if self.use_pp and isinstance(graph, PartitionEvalGraph):
            # [x | mean over the whole graph's in-neighbours] of the inner rows IS the precomputed input this rank
            # holds (train.precompute / precompute_streaming): nothing to aggregate, nothing to exchange
            return self._lin(self.linear, feat)
        degs = graph.in_degrees()                                                    # :94-102
        ah = _aggregate(graph, feat, 1.0 / degs.float())
        if self.use_pp:
            return self._lin(self.linear, torch.cat((feat, ah), dim=1))
        return self._lin(self.linear1, feat) + self._lin(self.linear2, ah)
