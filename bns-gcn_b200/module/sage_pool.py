"""``SAGEPoolConv``: GraphSAGE with the max-pooling aggregator (Hamilton, Ying and Leskovec, "Inductive Representation
Learning on Large Graphs", NeurIPS 2017), the layer ``dgl.nn.SAGEConv(in, out, 'pool', feat_drop)`` computes:

    x     = feat_drop(h_src)                      one mask; the destination rows are x[:n_in]
    z     = relu(fc_pool(x))                      fc_pool: Linear(in, in) with bias
    m_v   = max over the entries u -> v of z_u    per column; 0 for a row without entries
    rst_v = fc_self(x_v) + fc_neigh(m_v) + bias   fc_self, fc_neigh: Linear(in, out, bias=False)

Parameters are created in the order ``fc_pool``, ``fc_self``, ``fc_neigh``, ``bias``; the three weights are then drawn
xavier-uniform with the ReLU gain in that order, ``fc_pool.bias`` keeps ``nn.Linear``'s draw and ``bias`` starts at
zero.  (DGL parity of this layout is not verified: the float64 restatement in tests/ defines the layer.)

The max runs as kernels of libbnsgcn.so (``graph.SageMax`` in training, ``graph.sage_max_infer`` /
``sage_max_infer_block`` in evaluation).  The input width is padded to a multiple of 4 (zero rows of ``fc_pool``, which
give zero ``z`` columns, and zero columns of ``fc_neigh``); the constructor refuses a padded width above 1024.  The layer
returns ``[n, 1, out]``: it sits in ``model.GAT``'s stack as a one-head layer."""
import torch
import torch.nn.functional as F
from torch import nn

from .. import fused, ops
from ..graph import (SAGE_MAX_WIDTH, FullGraphHandle, PartitionEvalGraph, PartitionGraph, SageMax, sage_max_infer,
                     sage_max_infer_block)
from . import dense


def sage_padded_width(n: int) -> int:
    return (n + 3) // 4 * 4


class SAGEPoolConv(nn.Module):

    def __init__(self, in_feats, out_feats, feat_drop=0.):
        super(SAGEPoolConv, self).__init__()
        if sage_padded_width(in_feats) > SAGE_MAX_WIDTH:
            raise NotImplementedError(f"SAGEPoolConv: the max kernels do not take this layer: padded input width "
                                      f"{sage_padded_width(in_feats)} exceeds {SAGE_MAX_WIDTH}")
        self._in_feats, self._out_feats = in_feats, out_feats
        self.fc_pool = nn.Linear(in_feats, in_feats)
        self.fc_self = nn.Linear(in_feats, out_feats, bias=False)
        self.fc_neigh = nn.Linear(in_feats, out_feats, bias=False)
        self.bias = nn.Parameter(torch.zeros(out_feats))
        self.feat_drop = nn.Dropout(feat_drop)
        self.reset_parameters()

    def reset_parameters(self):
        gain = nn.init.calculate_gain('relu')
        nn.init.xavier_uniform_(self.fc_pool.weight, gain=gain)
        nn.init.xavier_uniform_(self.fc_self.weight, gain=gain)
        nn.init.xavier_uniform_(self.fc_neigh.weight, gain=gain)

    def forward(self, graph, feat):
        if isinstance(graph, FullGraphHandle) and isinstance(feat, torch.Tensor):
            if self.training:
                raise NotImplementedError("SAGEPoolConv: layer(g, h) on the full graph is the evaluation forward only; "
                                          "call .eval() first")
            return self._forward_full_graph(graph, feat)
        if isinstance(graph, PartitionEvalGraph):
            if self.training:
                raise NotImplementedError("SAGEPoolConv: the partition graph with every halo node is for evaluation "
                                          "only; call .eval() first")
            return self._forward_partition(graph, feat)
        if not isinstance(graph, PartitionGraph) or not isinstance(feat, tuple):
            raise NotImplementedError("SAGEPoolConv: the training call layer(g, (h_src, h_dst)) on a partition graph, "
                                      "or layer(g, h) on the full graph in evaluation")
        wp, bp, wn = self._padded_params()
        h_src = feat[0]
        ready = getattr(h_src, '_bns_ready', None)
        if ready is not None:          # every row of h_src is read below: wait for the overlapped exchange
            torch.cuda.current_stream(h_src.device).wait_event(ready)
        pf = self.feat_drop.p if self.training else 0.0
        if pf > 0 and fused.dropout_supported(h_src):
            salt = ops.RNG["seed"] + 15485863 * (1 + getattr(self, "_layer_index", 0))
            x = fused.DropoutFn.apply(h_src, pf, salt + 1)
        else:
            x = self.feat_drop(h_src)
        m = SageMax.apply(dense.linear(x, wp, bp), graph)                   # [n_in, Ip]
        return self._combine(x[:graph.n_in], m, wn)

    def _padded_params(self):
        """``fc_pool``'s weight and bias and ``fc_neigh``'s weight with the pooled width padded to a multiple of 4."""
        wp, bp, wn = self.fc_pool.weight, self.fc_pool.bias, self.fc_neigh.weight
        pad = sage_padded_width(self._in_feats) - self._in_feats
        if pad:
            wp, bp, wn = F.pad(wp, (0, 0, 0, pad)), F.pad(bp, (0, pad)), F.pad(wn, (0, pad))
        return wp, bp, wn

    def _combine(self, x_dst, m, wn):
        rst = dense.linear(m, wn, self.bias, addend=dense.linear(x_dst, self.fc_self.weight))
        return rst.unsqueeze(1)

    @torch.no_grad()
    def _forward_full_graph(self, graph: FullGraphHandle, feat: torch.Tensor) -> torch.Tensor:
        """The homogeneous branch with ``h_src = h_dst = feat``: ``fc_pool``, the one-pass max
        (``graph.sage_max_infer``), then the two output GEMMs."""
        wp, bp, wn = self._padded_params()
        z = torch.relu(dense.linear(feat, wp, bp))
        return self._combine(feat, sage_max_infer(graph.a, z), wn)

    @torch.no_grad()
    def _forward_partition(self, graph: PartitionEvalGraph, feat) -> torch.Tensor:
        """``_forward_full_graph`` over this rank's inner rows: the inner block first, then one block per peer, the
        running max carried between them (``sage_max_infer_block``).  ``feat``: the inner rows (each peer's halo rows
        are exchanged and transformed one peer at a time), or ``(h_src, h_dst)`` when ``h_src`` already holds ``[inner |
        every halo row]`` (layer 0 of the model, ``evaluate.eval_input``)."""
        wp, bp, wn = self._padded_params()
        n_in = graph.n_in
        held = isinstance(feat, tuple)
        src = feat[0] if held else feat
        z = torch.relu(dense.linear(src, wp, bp))                           # [n_in (+ n_halo), Ip]
        m = torch.empty(n_in, z.shape[1], dtype=torch.float32, device=z.device)
        seen = torch.empty(n_in, dtype=torch.int32, device=z.device)
        live = [j for j in graph.order if graph.blocks[j].nnz]
        sage_max_infer_block(graph.a_in, z[:n_in], m, seen, True, not live, m)
        if held:
            for j in live:
                rows = slice(n_in + graph.halo_begin[j], n_in + graph.halo_begin[j] + graph.halo_count[j])
                sage_max_infer_block(graph.blocks[j], z[rows], m, seen, False, j == live[-1], m)
        else:
            for j, blk, xr in graph.peer_rows(src):
                if blk.nnz == 0:
                    continue
                sage_max_infer_block(blk, torch.relu(dense.linear(xr, wp, bp)), m, seen, False, j == live[-1], m)
        return self._combine(src[:n_in], m, wn)
