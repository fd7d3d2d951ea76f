"""``GATConv``: the layer ``module/model.py:102`` takes from ``dgl.nn.GATConv`` (DGL 0.9, README.md:41; not
vendored with the reference).  Same constructor arguments, parameter names (``fc.weight``, ``attn_l``, ``attn_r``,
``bias``), initialisation (xavier-normal with the ReLU gain, zero bias) and forward contract as DGL's layer for the
call the reference makes -- ``layer(g, (h_src, h_dst))`` on the bipartite ``_U -> _V`` graph in training:

    ft = fc(feat_drop(h))            el = <ft_src, attn_l>      er = <ft_dst, attn_r>
    e_uv = leaky_relu(el_u + er_v)   a = attn_drop(edge_softmax(e))     rst_v = sum_u a_uv ft_u + bias

Everything after ``fc`` runs as kernels of libbnsgcn.so (``graph.GatProjection``, ``graph.GatAttention``; feature
dropout on the Philox kernel).  The kernels read each head's columns as 16-byte lanes, so every forward pads a per-head
width that is not a multiple of 4 (zero rows of ``fc.weight``, zero columns of ``attn_l`` / ``attn_r`` / ``bias`` per
head) and slices the pad off; in training the gradients flow back through the padding to the unpadded parameters.
The kernels take at most 8 heads and 1024 padded columns in all (``graph.gat_unsupported``); the constructor refuses
a layer beyond that.

In evaluation the layer also takes DGL's homogeneous call ``layer(g, h)`` on the full graph (``FullGraphHandle``, what
``GAT.forward`` makes when not training): one ``fc`` GEMM, ``el`` / ``er`` from the same ``ft``, and the attention as
one pass over each row (``graph.gat_infer``: online softmax, nothing stored per entry).  On a partition with every
halo node present (``PartitionEvalGraph``, the partition-parallel evaluation) the same forward runs over the inner rows,
the softmax state carried from the inner block to each peer's block (``graph.gat_infer_block``)."""
import torch
import torch.nn.functional as F
from torch import nn

from .. import fused, ops
from ..graph import (FullGraphHandle, GatAttention, GatProjection, PartitionEvalGraph, PartitionGraph, gat_infer,
                     gat_infer_block, gat_padded_width, gat_unsupported)
from . import dense


class GATConv(nn.Module):

    def __init__(self, in_feats, out_feats, num_heads, feat_drop=0., attn_drop=0., negative_slope=0.2,
                 residual=False, activation=None, allow_zero_in_degree=False, bias=True):
        super(GATConv, self).__init__()
        if residual or activation is not None:
            raise NotImplementedError("the reference constructs GATConv(in, out, heads, dropout, dropout) only")
        why = gat_unsupported(num_heads, out_feats)
        if why is not None:
            raise NotImplementedError(f"GATConv: the attention kernels do not take this layer: {why}")
        self._num_heads, self._in_feats, self._out_feats = num_heads, in_feats, out_feats
        self.fc = nn.Linear(in_feats, out_feats * num_heads, bias=False)
        self.attn_l = nn.Parameter(torch.empty(1, num_heads, out_feats))
        self.attn_r = nn.Parameter(torch.empty(1, num_heads, out_feats))
        self.feat_drop = nn.Dropout(feat_drop)
        self.attn_drop = nn.Dropout(attn_drop)
        self.negative_slope = negative_slope
        self.bias = nn.Parameter(torch.empty(num_heads * out_feats)) if bias else None
        self.reset_parameters()

    def reset_parameters(self):
        gain = nn.init.calculate_gain('relu')
        nn.init.xavier_normal_(self.fc.weight, gain=gain)
        nn.init.xavier_normal_(self.attn_l, gain=gain)
        nn.init.xavier_normal_(self.attn_r, gain=gain)
        if self.bias is not None:
            nn.init.constant_(self.bias, 0)

    def forward(self, graph, feat):
        if isinstance(graph, FullGraphHandle) and isinstance(feat, torch.Tensor):
            if self.training:
                raise NotImplementedError("GATConv: layer(g, h) on the full graph is the evaluation forward only; "
                                          "call .eval() first")
            return self._forward_full_graph(graph, feat)
        if isinstance(graph, PartitionEvalGraph):
            if self.training:
                raise NotImplementedError("GATConv: the partition graph with every halo node is for evaluation only; "
                                          "call .eval() first")
            return self._forward_partition(graph, feat)
        if not isinstance(graph, PartitionGraph) or not isinstance(feat, tuple):
            raise NotImplementedError("GATConv: the training call layer(g, (h_src, h_dst)) on a partition graph, or "
                                      "layer(g, h) on the full graph in evaluation")
        H, Fo, Fp, w, al, ar, b = self._padded_params()
        ready = getattr(feat[0], '_bns_ready', None)
        if ready is not None:          # every row of h_src is read below: wait for the overlapped exchange
            torch.cuda.current_stream(feat[0].device).wait_event(ready)
        salt = ops.RNG["seed"] + 15485863 * (1 + getattr(self, "_layer_index", 0))
        pf = self.feat_drop.p if self.training else 0.0
        if pf > 0 and fused.dropout_supported(feat[0]) and fused.dropout_supported(feat[1]):
            # two independent masks, as DGL draws them (feat_drop is applied to the source and the destination rows)
            h_src, h_dst = fused.DropoutFn.apply(feat[0], pf, salt + 1), fused.DropoutFn.apply(feat[1], pf, salt + 2)
        else:
            h_src, h_dst = self.feat_drop(feat[0]), self.feat_drop(feat[1])
        ft_src = dense.linear(h_src, w)                             # [n_U, H * Fp]
        ft_dst = dense.linear(h_dst, w)
        # el / er, score -> edge softmax -> dropout -> weighted aggregation (and their backward) as kernels
        el, er = GatProjection.apply(ft_src, ft_dst, al, ar, H, Fp)
        p = self.attn_drop.p if self.training else 0.0
        rst = GatAttention.apply(ft_src, el, er, graph, H, Fp, self.negative_slope, p, salt)
        if b is not None:
            rst += b                                                # in place: the attention saved nothing of it
        return rst.view(-1, H, Fp)[..., :Fo]

    @torch.no_grad()
    def _forward_full_graph(self, graph: FullGraphHandle, feat: torch.Tensor) -> torch.Tensor:
        """DGL's homogeneous branch with ``h_src = h_dst = feat`` (``feat_drop`` is the identity in evaluation): one
        ``fc`` GEMM, ``el`` / ``er`` from the same ``ft``, then the one-pass attention kernel (``graph.gat_infer``).
        No gradient flows through it."""
        _refuse_zero_in_degree(graph)
        H, Fo, Fp, w, al, ar, b = self._padded_params()
        ft = dense.linear(feat, w)                                  # [n, H * Fp]
        el, er = GatProjection.apply(ft, ft, al, ar, H, Fp)
        rst = gat_infer(graph.a, ft, el, er, H, Fp, self.negative_slope, b)
        return rst.view(-1, H, Fp)[..., :Fo]

    def _padded_params(self):
        """``H, Fo, Fp`` and the parameters with each head's width padded to ``Fp``, a multiple of 4 (the
        parameters themselves when ``Fo`` is one already)."""
        H, Fo = self._num_heads, self._out_feats
        Fp = gat_padded_width(Fo)
        w, al, ar, b = self.fc.weight, self.attn_l, self.attn_r, self.bias
        if Fp != Fo:
            pad = Fp - Fo
            w = F.pad(w.view(H, Fo, -1), (0, 0, 0, pad)).reshape(H * Fp, -1)
            al, ar = F.pad(al, (0, pad)), F.pad(ar, (0, pad))
            b = F.pad(b.view(H, Fo), (0, pad)).reshape(-1) if b is not None else None
        return H, Fo, Fp, w, al, ar, b

    @torch.no_grad()
    def _forward_partition(self, graph: PartitionEvalGraph, feat) -> torch.Tensor:
        """``_forward_full_graph`` over this rank's inner rows: the attention of the inner block first, then one block
        per peer, the online-softmax state carried between them (``gat_infer_block``).  ``feat``: the inner rows (each
        peer's halo rows are exchanged and transformed one peer at a time), or ``(h_src, h_dst)`` when ``h_src`` already
        holds ``[inner | every halo row]`` (layer 0 of the precomputed model: ``train.precompute``)."""
        _refuse_zero_in_degree(graph)
        H, Fo, Fp, w, al, ar, b = self._padded_params()
        n_in = graph.n_in
        held = isinstance(feat, tuple)
        src = feat[0] if held else feat
        ft = dense.linear(src, w)                                   # [n_in (+ n_halo), H * Fp]
        el, er = GatProjection.apply(ft, ft[:n_in], al, ar, H, Fp)
        m = torch.empty(n_in, H, dtype=torch.float32, device=ft.device)
        l = torch.empty_like(m)
        acc = torch.empty(n_in, H * Fp, dtype=torch.float32, device=ft.device)
        live = [j for j in graph.order if graph.blocks[j].nnz]
        slope = self.negative_slope
        gat_infer_block(graph.a_in, ft[:n_in], el[:n_in], er, H, Fp, slope, m, l, acc, True, not live, b, acc)
        if held:
            for j in live:
                rows = slice(n_in + graph.halo_begin[j], n_in + graph.halo_begin[j] + graph.halo_count[j])
                gat_infer_block(graph.blocks[j], ft[rows], el[rows], er, H, Fp, slope, m, l, acc, False, j == live[-1],
                                b, acc)
        else:
            for j, blk, xr in graph.peer_rows(src):
                if blk.nnz == 0:
                    continue
                ft_j = dense.linear(xr, w)
                el_j, _ = GatProjection.apply(ft_j, ft_j[:0], al, ar, H, Fp)
                gat_infer_block(blk, ft_j, el_j, er, H, Fp, slope, m, l, acc, False, j == live[-1], b, acc)
        return acc.view(-1, H, Fp)[..., :Fo]


def _refuse_zero_in_degree(graph, layer: str = "GATConv") -> None:
    if graph.has_zero_in_degree():
        # dgl.nn.GATConv / GATv2Conv(allow_zero_in_degree=False) refuse such a graph (DGLError)
        raise RuntimeError(f"{layer}: there are 0-in-degree nodes in the graph, their output would be invalid; "
                           "add self-loops")
