"""``TransformerConv``: the graph transformer layer (Shi et al., "Masked Label Prediction: Unified Message Passing Model
for Semi-Supervised Classification", IJCAI 2021), with the parameter names and creation order of
``torch_geometric.nn.TransformerConv(in, out, heads, concat=False, root_weight=True, bias=True)`` (``lin_key``,
``lin_query``, ``lin_value``, ``lin_skip``; ``nn.Linear``'s default initialisation) and the forward contract of
``GATv2Conv`` on GAT's layer stack:

    x_src = feat_drop(h_src)   x_dst = feat_drop(h_dst)                                  # two Philox streams
    q = lin_query(x_dst)   k = lin_key(x_src)   v = lin_value(x_src)                     # [*, H, C]
    s_uv = <q_v, k_u> / sqrt(C)     a = attn_drop(edge_softmax(s))
    rst_v = sum_u a_uv v_u + lin_skip(x_dst)_v                                           # [n, H, C]

The stack averages the heads (``.mean(1)``), so the skip term is added to every head: ``mean_h(a_h + s) = mean_h(a_h) +
s``, PyG's ``concat=False``.  The key and value projections run as one GEMM on the stacked weights ``[W_k; W_v]``, so
the attention kernels (``graph.TconvAttention`` in training, ``graph.tconv_infer`` / ``tconv_infer_block`` in
evaluation) read one contiguous ``[k | v]`` row per entry.  A per-head width that is not a multiple of 4 is padded with
zero rows of the q, k and v weights and biases (a pad column adds 0 to every dot product) and sliced off; the scale
stays ``1/sqrt(C)`` with the unpadded ``C``.  The constructor refuses more than 8 heads or 1024 padded columns."""
import math

import torch
import torch.nn.functional as F
from torch import nn

from .. import fused, ops
from ..graph import (FullGraphHandle, PartitionEvalGraph, PartitionGraph, TconvAttention, gat_padded_width,
                     gat_unsupported, tconv_infer, tconv_infer_block)
from . import dense
from .gat import _refuse_zero_in_degree


class TransformerConv(nn.Module):

    def __init__(self, in_feats, out_feats, num_heads, feat_drop=0., attn_drop=0., root_weight=True, bias=True,
                 concat=False, beta=False, edge_dim=None):
        super(TransformerConv, self).__init__()
        if concat or beta or edge_dim is not None:
            raise NotImplementedError("TransformerConv: only TransformerConv(in, out, heads, feat_drop, attn_drop) "
                                      "with averaged heads (concat=False), no beta gating and no edge features")
        why = gat_unsupported(num_heads, out_feats)
        if why is not None:
            raise NotImplementedError(f"TransformerConv: the attention kernels do not take this layer: {why}")
        self._num_heads, self._in_feats, self._out_feats = num_heads, in_feats, out_feats
        self.lin_key = nn.Linear(in_feats, num_heads * out_feats, bias=bias)
        self.lin_query = nn.Linear(in_feats, num_heads * out_feats, bias=bias)
        self.lin_value = nn.Linear(in_feats, num_heads * out_feats, bias=bias)
        self.lin_skip = nn.Linear(in_feats, out_feats, bias=bias) if root_weight else None
        self.feat_drop = nn.Dropout(feat_drop)
        self.attn_drop = nn.Dropout(attn_drop)

    def forward(self, graph, feat):
        if isinstance(graph, FullGraphHandle) and isinstance(feat, torch.Tensor):
            if self.training:
                raise NotImplementedError("TransformerConv: layer(g, h) on the full graph is the evaluation forward "
                                          "only; call .eval() first")
            return self._forward_full_graph(graph, feat)
        if isinstance(graph, PartitionEvalGraph):
            if self.training:
                raise NotImplementedError("TransformerConv: the partition graph with every halo node is for "
                                          "evaluation only; call .eval() first")
            return self._forward_partition(graph, feat)
        if not isinstance(graph, PartitionGraph) or not isinstance(feat, tuple):
            raise NotImplementedError("TransformerConv: the training call layer(g, (h_src, h_dst)) on a partition "
                                      "graph, or layer(g, h) on the full graph in evaluation")
        H, C, Cp, wq, bq, wkv, bkv = self._padded_params()
        ready = getattr(feat[0], '_bns_ready', None)
        if ready is not None:          # every row of h_src is read below: wait for the overlapped exchange
            torch.cuda.current_stream(feat[0].device).wait_event(ready)
        salt = ops.RNG["seed"] + 15485863 * (1 + getattr(self, "_layer_index", 0))
        pf = self.feat_drop.p if self.training else 0.0
        if pf > 0 and fused.dropout_supported(feat[0]) and fused.dropout_supported(feat[1]):
            h_src, h_dst = fused.DropoutFn.apply(feat[0], pf, salt + 1), fused.DropoutFn.apply(feat[1], pf, salt + 2)
        else:
            h_src, h_dst = self.feat_drop(feat[0]), self.feat_drop(feat[1])
        q = dense.linear(h_dst, wq, bq)                             # [n_V, H * Cp]
        kv = dense.linear(h_src, wkv, bkv)                          # [n_U, 2 * H * Cp]: [k | v]
        p = self.attn_drop.p if self.training else 0.0
        rst = TconvAttention.apply(q, kv, graph, H, Cp, 1.0 / math.sqrt(C), p, salt)
        return self._finish(rst, h_dst)

    def _padded_params(self):
        """``H, C, Cp``, then the query weight and bias and the stacked ``[key; value]`` weight and bias, each head's
        rows padded to ``Cp``, a multiple of 4."""
        H, C = self._num_heads, self._out_feats
        Cp = gat_padded_width(C)
        ws = [self.lin_query.weight, self.lin_key.weight, self.lin_value.weight]
        bs = [self.lin_query.bias, self.lin_key.bias, self.lin_value.bias]
        if Cp != C:
            pad = Cp - C
            ws = [F.pad(w.view(H, C, -1), (0, 0, 0, pad)).reshape(H * Cp, -1) for w in ws]
            bs = [F.pad(b.view(H, C), (0, pad)).reshape(-1) if b is not None else None for b in bs]
        bkv = torch.cat(bs[1:]) if bs[1] is not None else None
        return H, C, Cp, ws[0], bs[0], torch.cat(ws[1:]), bkv

    def _finish(self, rst, x_dst):
        """``[n, H, C]``: the attention's heads without their pad columns, plus ``lin_skip(x_dst)`` on every head."""
        H, C = self._num_heads, self._out_feats
        out = rst.view(-1, H, gat_padded_width(C))[..., :C]
        if self.lin_skip is not None:
            out = out + dense.linear(x_dst, self.lin_skip.weight, self.lin_skip.bias).unsqueeze(1)
        return out

    @torch.no_grad()
    def _forward_full_graph(self, graph: FullGraphHandle, feat: torch.Tensor) -> torch.Tensor:
        """The homogeneous branch with ``h_src = h_dst = feat``: the two GEMMs, then the one-pass attention kernel
        (``graph.tconv_infer``), then the skip term."""
        _refuse_zero_in_degree(graph, "TransformerConv")
        H, C, Cp, wq, bq, wkv, bkv = self._padded_params()
        q, kv = dense.linear(feat, wq, bq), dense.linear(feat, wkv, bkv)
        return self._finish(tconv_infer(graph.a, q, kv, H, Cp, 1.0 / math.sqrt(C)), feat)

    @torch.no_grad()
    def _forward_partition(self, graph: PartitionEvalGraph, feat) -> torch.Tensor:
        """``_forward_full_graph`` over this rank's inner rows: the inner block first, then one block per peer, the
        online-softmax state carried between them (``tconv_infer_block``).  ``feat``: the inner rows (each peer's halo
        rows are exchanged and projected one peer at a time), or ``(h_src, h_dst)`` when ``h_src`` already holds
        ``[inner | every halo row]`` (layer 0 of the model, ``evaluate.eval_input``)."""
        _refuse_zero_in_degree(graph, "TransformerConv")
        H, C, Cp, wq, bq, wkv, bkv = self._padded_params()
        scale = 1.0 / math.sqrt(C)
        n_in = graph.n_in
        held = isinstance(feat, tuple)
        src = feat[0] if held else feat
        kv = dense.linear(src, wkv, bkv)                            # [n_in (+ n_halo), 2 * H * Cp]
        q = dense.linear(src[:n_in], wq, bq)
        m = torch.empty(n_in, H, dtype=torch.float32, device=q.device)
        l = torch.empty_like(m)
        acc = torch.empty(n_in, H * Cp, dtype=torch.float32, device=q.device)
        live = [j for j in graph.order if graph.blocks[j].nnz]
        tconv_infer_block(graph.a_in, q, kv[:n_in], H, Cp, scale, m, l, acc, True, not live, acc)
        if held:
            for j in live:
                rows = slice(n_in + graph.halo_begin[j], n_in + graph.halo_begin[j] + graph.halo_count[j])
                tconv_infer_block(graph.blocks[j], q, kv[rows], H, Cp, scale, m, l, acc, False, j == live[-1], acc)
        else:
            for j, blk, xr in graph.peer_rows(src):
                if blk.nnz == 0:
                    continue
                tconv_infer_block(blk, q, dense.linear(xr, wkv, bkv), H, Cp, scale, m, l, acc, False,
                                  j == live[-1], acc)
        return self._finish(acc, src[:n_in])
