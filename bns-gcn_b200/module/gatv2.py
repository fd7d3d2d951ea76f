"""``GATv2Conv``: dynamic attention (Brody, Alon and Yahav, "How Attentive are Graph Attention Networks?", ICLR 2022),
with the constructor, parameter names (``fc_src.weight`` / ``.bias``, ``fc_dst.weight`` / ``.bias``, ``attn``),
initialisation (xavier-normal with the ReLU gain, zero biases, in that order) and forward contract of DGL's
``dgl.nn.GATv2Conv(in, out, heads, feat_drop, attn_drop)`` with ``share_weights=False``, no residual, no activation:

    z_src = fc_src(feat_drop(h_src))        z_dst = fc_dst(feat_drop(h_dst))                  # [*, H, F]
    s_uv  = sum_f attn[h, f] * leaky_relu(z_src[u, h, f] + z_dst[v, h, f])
    rst_v = sum_u attn_drop(edge_softmax(s))_uv * z_src[u]

GAT's score ``leaky_relu(el_u + er_v)`` splits into one scalar per source and one per destination, so every destination
ranks its neighbours in the same order; this score does not.  Everything after the two ``fc`` GEMMs runs as kernels of
libbnsgcn.so (``graph.Gatv2Attention`` in training, ``graph.gatv2_infer`` / ``gatv2_infer_block`` in evaluation).  As in
``GATConv``, a per-head width that is not a multiple of 4 is padded (zero rows of the ``fc`` weights and biases, zero
columns of ``attn``: a pad column adds ``attn * leaky_relu(0) = 0`` to every score) and sliced off, and the constructor
refuses more than 8 heads or 1024 padded columns."""
import torch
import torch.nn.functional as F
from torch import nn

from .. import fused, ops
from ..graph import (FullGraphHandle, Gatv2Attention, PartitionEvalGraph, PartitionGraph, gat_padded_width,
                     gat_unsupported, gatv2_infer, gatv2_infer_block)
from . import dense
from .gat import _refuse_zero_in_degree


class GATv2Conv(nn.Module):

    def __init__(self, in_feats, out_feats, num_heads, feat_drop=0., attn_drop=0., negative_slope=0.2,
                 residual=False, activation=None, allow_zero_in_degree=False, bias=True, share_weights=False):
        super(GATv2Conv, self).__init__()
        if residual or activation is not None or share_weights:
            raise NotImplementedError("GATv2Conv: only GATv2Conv(in, out, heads, feat_drop, attn_drop) with "
                                      "share_weights=False, no residual and no activation")
        why = gat_unsupported(num_heads, out_feats)
        if why is not None:
            raise NotImplementedError(f"GATv2Conv: the attention kernels do not take this layer: {why}")
        self._num_heads, self._in_feats, self._out_feats = num_heads, in_feats, out_feats
        self.fc_src = nn.Linear(in_feats, out_feats * num_heads, bias=bias)
        self.fc_dst = nn.Linear(in_feats, out_feats * num_heads, bias=bias)
        self.attn = nn.Parameter(torch.empty(1, num_heads, out_feats))
        self.feat_drop = nn.Dropout(feat_drop)
        self.attn_drop = nn.Dropout(attn_drop)
        self.negative_slope = negative_slope
        self.reset_parameters()

    def reset_parameters(self):
        gain = nn.init.calculate_gain('relu')
        nn.init.xavier_normal_(self.fc_src.weight, gain=gain)
        if self.fc_src.bias is not None:
            nn.init.constant_(self.fc_src.bias, 0)
        nn.init.xavier_normal_(self.fc_dst.weight, gain=gain)
        if self.fc_dst.bias is not None:
            nn.init.constant_(self.fc_dst.bias, 0)
        nn.init.xavier_normal_(self.attn, gain=gain)

    def forward(self, graph, feat):
        if isinstance(graph, FullGraphHandle) and isinstance(feat, torch.Tensor):
            if self.training:
                raise NotImplementedError("GATv2Conv: layer(g, h) on the full graph is the evaluation forward only; "
                                          "call .eval() first")
            return self._forward_full_graph(graph, feat)
        if isinstance(graph, PartitionEvalGraph):
            if self.training:
                raise NotImplementedError("GATv2Conv: the partition graph with every halo node is for evaluation "
                                          "only; call .eval() first")
            return self._forward_partition(graph, feat)
        if not isinstance(graph, PartitionGraph) or not isinstance(feat, tuple):
            raise NotImplementedError("GATv2Conv: the training call layer(g, (h_src, h_dst)) on a partition graph, "
                                      "or layer(g, h) on the full graph in evaluation")
        H, Fo, Fp, ws, bs, wd, bd, at = self._padded_params()
        ready = getattr(feat[0], '_bns_ready', None)
        if ready is not None:          # every row of h_src is read below: wait for the overlapped exchange
            torch.cuda.current_stream(feat[0].device).wait_event(ready)
        salt = ops.RNG["seed"] + 15485863 * (1 + getattr(self, "_layer_index", 0))
        pf = self.feat_drop.p if self.training else 0.0
        if pf > 0 and fused.dropout_supported(feat[0]) and fused.dropout_supported(feat[1]):
            h_src, h_dst = fused.DropoutFn.apply(feat[0], pf, salt + 1), fused.DropoutFn.apply(feat[1], pf, salt + 2)
        else:
            h_src, h_dst = self.feat_drop(feat[0]), self.feat_drop(feat[1])
        zs = dense.linear(h_src, ws, bs)                            # [n_U, H * Fp]
        zd = dense.linear(h_dst, wd, bd)                            # [n_V, H * Fp]
        p = self.attn_drop.p if self.training else 0.0
        rst = Gatv2Attention.apply(zs, zd, at, graph, H, Fp, self.negative_slope, p, salt)
        return rst.view(-1, H, Fp)[..., :Fo]

    def _padded_params(self):
        """``H, Fo, Fp`` and the parameters with each head's width padded to ``Fp``, a multiple of 4 (the parameters
        themselves when ``Fo`` is one already)."""
        H, Fo = self._num_heads, self._out_feats
        Fp = gat_padded_width(Fo)
        ws, bs, wd, bd, at = self.fc_src.weight, self.fc_src.bias, self.fc_dst.weight, self.fc_dst.bias, self.attn
        if Fp != Fo:
            pad = Fp - Fo
            ws, wd = (F.pad(w.view(H, Fo, -1), (0, 0, 0, pad)).reshape(H * Fp, -1) for w in (ws, wd))
            bs, bd = (F.pad(b.view(H, Fo), (0, pad)).reshape(-1) if b is not None else None for b in (bs, bd))
            at = F.pad(at, (0, pad))
        return H, Fo, Fp, ws, bs, wd, bd, at

    @torch.no_grad()
    def _forward_full_graph(self, graph: FullGraphHandle, feat: torch.Tensor) -> torch.Tensor:
        """DGL's homogeneous branch with ``h_src = h_dst = feat``: the two ``fc`` GEMMs, then the one-pass attention
        kernel (``graph.gatv2_infer``)."""
        _refuse_zero_in_degree(graph, "GATv2Conv")
        H, Fo, Fp, ws, bs, wd, bd, at = self._padded_params()
        zs, zd = dense.linear(feat, ws, bs), dense.linear(feat, wd, bd)
        rst = gatv2_infer(graph.a, zs, zd, at, H, Fp, self.negative_slope)
        return rst.view(-1, H, Fp)[..., :Fo]

    @torch.no_grad()
    def _forward_partition(self, graph: PartitionEvalGraph, feat) -> torch.Tensor:
        """``_forward_full_graph`` over this rank's inner rows: the inner block first, then one block per peer, the
        online-softmax state carried between them (``gatv2_infer_block``).  ``feat``: the inner rows (each peer's halo
        rows are exchanged and transformed one peer at a time), or ``(h_src, h_dst)`` when ``h_src`` already holds
        ``[inner | every halo row]`` (layer 0 of the model, ``evaluate.eval_input``)."""
        _refuse_zero_in_degree(graph, "GATv2Conv")
        H, Fo, Fp, ws, bs, wd, bd, at = self._padded_params()
        n_in = graph.n_in
        held = isinstance(feat, tuple)
        src = feat[0] if held else feat
        zs = dense.linear(src, ws, bs)                              # [n_in (+ n_halo), H * Fp]
        zd = dense.linear(src[:n_in], wd, bd)
        m = torch.empty(n_in, H, dtype=torch.float32, device=zs.device)
        l = torch.empty_like(m)
        acc = torch.empty(n_in, H * Fp, dtype=torch.float32, device=zs.device)
        live = [j for j in graph.order if graph.blocks[j].nnz]
        slope = self.negative_slope
        gatv2_infer_block(graph.a_in, zs[:n_in], zd, at, H, Fp, slope, m, l, acc, True, not live, acc)
        if held:
            for j in live:
                rows = slice(n_in + graph.halo_begin[j], n_in + graph.halo_begin[j] + graph.halo_count[j])
                gatv2_infer_block(graph.blocks[j], zs[rows], zd, at, H, Fp, slope, m, l, acc, False, j == live[-1], acc)
        else:
            for j, blk, xr in graph.peer_rows(src):
                if blk.nnz == 0:
                    continue
                gatv2_infer_block(blk, dense.linear(xr, ws, bs), zd, at, H, Fp, slope, m, l, acc, False,
                                  j == live[-1], acc)
        return acc.view(-1, H, Fp)[..., :Fo]

