"""The CPU oracle's ``transformer`` kind: ``TransformerConvRef`` restates the graph transformer layer
(``torch_geometric.nn.TransformerConv(in, out, heads, concat=False, root_weight=True)`` with feature dropout on both
inputs) over the oracle's explicit edge lists, the way ``tests/gatv2_oracle.py`` restates ``GATv2Conv``;
``TransformerRef`` is the oracle's ``GATRef`` stack with it.

The oracle's rank (``OracleRank``) runs the model through its ``gat`` paths: layer 0 takes the stored halo rows
(precompute, ``construct_feat``), the later layers exchange their input, the gradients are all-reduced.  Two things
differ: the layer, and the exchange's ratio, which is 1.0 for every peer (a softmax takes the sampled rows unscaled).
``oracle_kind`` hands the rank both, and ``run_parity_case`` (tests/harness.py) compares the product with it."""
import argparse
import contextlib

import torch
from torch import nn

from oracle import bns_oracle as O


class TransformerConvRef(nn.Module):
    """Per entry u -> v and head h, ``s = <lin_query(x_dst)[v, h], lin_key(x_src)[u, h]> / sqrt(C)``, softmax over each
    destination's in-edges, attention dropout, ``rst_v = sum_u a_uv lin_value(x_src)[u] + lin_skip(x_dst)_v`` on every
    head.  Parameters in the order ``lin_key``, ``lin_query``, ``lin_value``, ``lin_skip``, ``nn.Linear``'s
    initialisation."""

    def __init__(self, in_feats, out_feats, num_heads, feat_drop=0.0, attn_drop=0.0):
        super().__init__()
        self.H, self.C = num_heads, out_feats
        self.lin_key = nn.Linear(in_feats, num_heads * out_feats)
        self.lin_query = nn.Linear(in_feats, num_heads * out_feats)
        self.lin_value = nn.Linear(in_feats, num_heads * out_feats)
        self.lin_skip = nn.Linear(in_feats, out_feats)
        self.feat_drop, self.attn_drop = nn.Dropout(feat_drop), nn.Dropout(attn_drop)

    def forward(self, g, feat):
        H, C = self.H, self.C
        h_src, h_dst = (self.feat_drop(feat[0]), self.feat_drop(feat[1])) if isinstance(feat, tuple) \
            else (self.feat_drop(feat),) * 2
        q = self.lin_query(h_dst).view(-1, H, C)
        k = self.lin_key(h_src).view(-1, H, C)
        v = self.lin_value(h_src).view(-1, H, C)
        s = (q[g.v] * k[g.u]).sum(-1) / C ** 0.5                                            # [nnz, H]
        idx = g.v.unsqueeze(1).expand(-1, H)
        m = torch.full((g.n_v, H), float("-inf")).scatter_reduce(0, idx, s.detach(), "amax")
        ex = torch.exp(s - m[g.v])
        den = torch.zeros(g.n_v, H).index_add(0, g.v, ex)
        a = self.attn_drop(ex / den[g.v])                                                    # edge_softmax
        rst = torch.zeros(g.n_v, H, C).index_add(0, g.v, a.unsqueeze(-1) * v[g.u])
        return rst + self.lin_skip(h_dst).unsqueeze(1)


class TransformerRef(O.GATRef):
    """``GAT`` with ``TransformerConv`` layers: ``GATRef``'s construction order with ``TransformerConvRef``, and its
    forward."""

    def __init__(self, layer_size, use_pp, heads, dropout, norm, train_size, n_linear):
        nn.Module.__init__(self)
        self.n_layers, self.n_linear, self.use_pp = len(layer_size) - 1, n_linear, use_pp
        self.layers = nn.ModuleList()
        self.use_norm = norm is not None
        if self.use_norm:
            self.norm = nn.ModuleList()
        self.dropout = nn.Dropout(p=dropout)
        for i in range(self.n_layers):
            if i < self.n_layers - n_linear:
                self.layers.append(TransformerConvRef(layer_size[i], layer_size[i + 1], heads, dropout, dropout))
            else:
                self.layers.append(nn.Linear(layer_size[i], layer_size[i + 1]))
            if i < self.n_layers - 1 and self.use_norm:
                self.norm.append(nn.LayerNorm(layer_size[i + 1], elementwise_affine=True) if norm == "layer"
                                 else O.SyncBNRef(layer_size[i + 1], train_size))
        self.oracle = None


def _build_model(kind, layer_size, use_pp, dropout, norm, train_size, n_linear, heads=1):
    if kind != "gat":
        raise NotImplementedError(kind)
    return TransformerRef(layer_size, True, heads, dropout, norm, train_size, n_linear)     # use_pp=True, as GAT


def _unscaled_send_size(self):
    res, ratio = _REAL_SEND_SIZE(self)
    return res, [0 if i == self.rank else 1.0 for i in range(len(ratio))]


_REAL_SEND_SIZE = O.OracleRank._get_send_size


@contextlib.contextmanager
def oracle_kind(monkeypatch):
    """Inside: ``tests.harness.run_oracle`` runs a ``--model transformer`` configuration as the oracle's ``gat`` rank
    with ``TransformerRef`` as its model and a ratio of 1.0 for every peer."""
    from tests import harness
    real = harness.run_oracle

    def run_oracle(parts, args, *a, **kw):
        if args.model != "transformer":
            raise NotImplementedError(args.model)
        as_gat = argparse.Namespace(**vars(args))
        as_gat.model = "gat"
        return real(parts, as_gat, *a, **kw)
    with monkeypatch.context() as m:
        m.setattr(harness, "run_oracle", run_oracle)
        m.setattr(O, "build_model", _build_model)
        m.setattr(O.OracleRank, "_get_send_size", _unscaled_send_size)
        yield
