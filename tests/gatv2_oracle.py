"""The CPU oracle's ``gatv2`` kind: ``GATv2ConvRef`` restates ``dgl.nn.GATv2Conv(in, out, heads, feat_drop, attn_drop)``
(``share_weights=False``, no residual, no activation) over the oracle's explicit edge lists, the way
``oracle.bns_oracle.GATConvRef`` restates ``GATConv``; ``GATv2Ref`` is the oracle's ``GATRef`` stack with it.

The oracle's rank (``OracleRank``) runs GATv2 through its ``gat`` paths: layer 0 takes the stored halo rows
(precompute, ``construct_feat``), the later layers exchange their input, the gradients are all-reduced.  Only the
attention layer differs, so ``oracle_kind`` hands the rank this stack in place of ``GATRef`` (``build_model``), and
``run_parity_case`` (tests/harness.py) compares the product with it."""
import argparse
import contextlib

import torch
import torch.nn.functional as F
from torch import nn

from oracle import bns_oracle as O


class GATv2ConvRef(nn.Module):
    """Per entry u -> v and head h, ``s = sum_f attn[h, f] * leaky_relu(fc_src(h_src)[u, h, f] + fc_dst(h_dst)[v, h, f])``,
    softmax over each destination's in-edges, attention dropout, ``rst_v = sum_u a_uv fc_src(h_src)[u]``.  Parameters
    and their initialisation order: ``fc_src`` (xavier-normal with the ReLU gain, zero bias), ``fc_dst`` (the same),
    ``attn [1, H, F]`` (xavier-normal with the ReLU gain)."""

    def __init__(self, in_feats, out_feats, num_heads, feat_drop=0.0, attn_drop=0.0, negative_slope=0.2):
        super().__init__()
        self.H, self.Fo = num_heads, out_feats
        self.fc_src = nn.Linear(in_feats, out_feats * num_heads, bias=True)
        self.fc_dst = nn.Linear(in_feats, out_feats * num_heads, bias=True)
        self.attn = nn.Parameter(torch.empty(1, num_heads, out_feats))
        self.feat_drop, self.attn_drop = nn.Dropout(feat_drop), nn.Dropout(attn_drop)
        self.negative_slope = negative_slope
        gain = nn.init.calculate_gain("relu")
        nn.init.xavier_normal_(self.fc_src.weight, gain=gain)
        nn.init.constant_(self.fc_src.bias, 0)
        nn.init.xavier_normal_(self.fc_dst.weight, gain=gain)
        nn.init.constant_(self.fc_dst.bias, 0)
        nn.init.xavier_normal_(self.attn, gain=gain)

    def forward(self, g, feat):
        H, Fo = self.H, self.Fo
        h_src, h_dst = (self.feat_drop(feat[0]), self.feat_drop(feat[1])) if isinstance(feat, tuple) \
            else (self.feat_drop(feat),) * 2
        zs = self.fc_src(h_src).view(-1, H, Fo)
        zd = self.fc_dst(h_dst).view(-1, H, Fo)
        s = (F.leaky_relu(zs[g.u] + zd[g.v], self.negative_slope) * self.attn).sum(-1)     # [nnz, H]
        idx = g.v.unsqueeze(1).expand(-1, H)
        m = torch.full((g.n_v, H), float("-inf")).scatter_reduce(0, idx, s.detach(), "amax")
        ex = torch.exp(s - m[g.v])
        den = torch.zeros(g.n_v, H).index_add(0, g.v, ex)
        a = self.attn_drop(ex / den[g.v])                                                    # edge_softmax
        return torch.zeros(g.n_v, H, Fo).index_add(0, g.v, a.unsqueeze(-1) * zs[g.u])


class GATv2Ref(O.GATRef):
    """``GAT`` with ``GATv2Conv`` layers: ``GATRef``'s construction order with ``GATv2ConvRef``, and its forward."""

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
                self.layers.append(GATv2ConvRef(layer_size[i], layer_size[i + 1], heads, dropout, dropout))
            else:
                self.layers.append(nn.Linear(layer_size[i], layer_size[i + 1]))
            if i < self.n_layers - 1 and self.use_norm:
                self.norm.append(nn.LayerNorm(layer_size[i + 1], elementwise_affine=True) if norm == "layer"
                                 else O.SyncBNRef(layer_size[i + 1], train_size))
        self.oracle = None


def _build_model(kind, layer_size, use_pp, dropout, norm, train_size, n_linear, heads=1):
    if kind != "gat":
        raise NotImplementedError(kind)
    return GATv2Ref(layer_size, True, heads, dropout, norm, train_size, n_linear)             # use_pp=True, as GAT


@contextlib.contextmanager
def oracle_kind(monkeypatch):
    """Inside: ``tests.harness.run_oracle`` runs a ``--model gatv2`` configuration as the oracle's ``gat`` rank with
    ``GATv2Ref`` as its model."""
    from tests import harness
    real = harness.run_oracle

    def run_oracle(parts, args, *a, **kw):
        if args.model != "gatv2":
            raise NotImplementedError(args.model)
        as_gat = argparse.Namespace(**vars(args))
        as_gat.model = "gat"
        return real(parts, as_gat, *a, **kw)
    with monkeypatch.context() as m:
        m.setattr(harness, "run_oracle", run_oracle)
        m.setattr(O, "build_model", _build_model)
        yield
