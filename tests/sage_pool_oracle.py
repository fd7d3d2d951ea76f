"""The CPU oracle's ``graphsage-pool`` kind: ``SAGEPoolConvRef`` restates ``SAGEConv(in, out, 'pool', feat_drop)`` over
the oracle's explicit edge lists (the winner rule of tests/sage_pool_reference.py), and ``SAGEPoolRef`` is the oracle's
``GATRef`` stack with it as a one-head layer.

The oracle's rank (``OracleRank``) runs the model through its ``gat`` paths: layer 0 takes the stored halo rows
(precompute, ``construct_feat``), the later layers exchange their input, the gradients are all-reduced.  Two things
differ: the layer, and the exchange's ratio, which is 1.0 for every peer (a max takes the sampled rows unscaled).
``oracle_kind`` hands the rank both, and ``run_parity_case`` (tests/harness.py) compares the product with it."""
import argparse
import contextlib

import torch
from torch import nn

from oracle import bns_oracle as O
from tests.sage_pool_reference import MaxByWinner


class SAGEPoolConvRef(nn.Module):
    """``x = feat_drop(h_src)``, ``z = relu(fc_pool(x))``, ``m_v = max over u -> v of z_u``, ``rst_v = fc_self(x_v) +
    fc_neigh(m_v) + bias`` with ``x_v = x[:n_v]``; returns ``[n_v, 1, out]``.  Parameters in the order ``fc_pool``,
    ``fc_self``, ``fc_neigh``, ``bias``; the three weights xavier-uniform with the ReLU gain, in that order."""

    def __init__(self, in_feats, out_feats, feat_drop=0.0):
        super().__init__()
        self.fc_pool = nn.Linear(in_feats, in_feats)
        self.fc_self = nn.Linear(in_feats, out_feats, bias=False)
        self.fc_neigh = nn.Linear(in_feats, out_feats, bias=False)
        self.bias = nn.Parameter(torch.zeros(out_feats))
        self.feat_drop = nn.Dropout(feat_drop)
        gain = nn.init.calculate_gain("relu")
        nn.init.xavier_uniform_(self.fc_pool.weight, gain=gain)
        nn.init.xavier_uniform_(self.fc_self.weight, gain=gain)
        nn.init.xavier_uniform_(self.fc_neigh.weight, gain=gain)

    def forward(self, g, feat):
        x = self.feat_drop(feat[0] if isinstance(feat, tuple) else feat)
        m = MaxByWinner.apply(torch.relu(self.fc_pool(x)), g.u, g.v, g.n_v)
        return (self.fc_self(x[:g.n_v]) + self.fc_neigh(m) + self.bias).unsqueeze(1)


class SAGEPoolRef(O.GATRef):
    """``GAT``'s stack with ``SAGEPoolConvRef`` layers: ``GATRef``'s construction order and forward."""

    def __init__(self, layer_size, use_pp, dropout, norm, train_size, n_linear):
        nn.Module.__init__(self)
        self.n_layers, self.n_linear, self.use_pp = len(layer_size) - 1, n_linear, use_pp
        self.layers = nn.ModuleList()
        self.use_norm = norm is not None
        if self.use_norm:
            self.norm = nn.ModuleList()
        self.dropout = nn.Dropout(p=dropout)
        for i in range(self.n_layers):
            if i < self.n_layers - n_linear:
                self.layers.append(SAGEPoolConvRef(layer_size[i], layer_size[i + 1], dropout))
            else:
                self.layers.append(nn.Linear(layer_size[i], layer_size[i + 1]))
            if i < self.n_layers - 1 and self.use_norm:
                self.norm.append(nn.LayerNorm(layer_size[i + 1], elementwise_affine=True) if norm == "layer"
                                 else O.SyncBNRef(layer_size[i + 1], train_size))
        self.oracle = None


def _build_model(kind, layer_size, use_pp, dropout, norm, train_size, n_linear, heads=1):
    if kind != "gat":
        raise NotImplementedError(kind)
    return SAGEPoolRef(layer_size, True, dropout, norm, train_size, n_linear)              # use_pp=True, as GAT


def _unscaled_send_size(self):
    res, ratio = _REAL_SEND_SIZE(self)
    return res, [0 if i == self.rank else 1.0 for i in range(len(ratio))]


_REAL_SEND_SIZE = O.OracleRank._get_send_size


@contextlib.contextmanager
def oracle_kind(monkeypatch):
    """Inside: ``tests.harness.run_oracle`` runs a ``--model graphsage-pool`` configuration as the oracle's ``gat`` rank
    with ``SAGEPoolRef`` as its model and a ratio of 1.0 for every peer."""
    from tests import harness
    real = harness.run_oracle

    def run_oracle(parts, args, *a, **kw):
        if args.model != "graphsage-pool":
            raise NotImplementedError(args.model)
        as_gat = argparse.Namespace(**vars(args))
        as_gat.model = "gat"
        return real(parts, as_gat, *a, **kw)
    with monkeypatch.context() as m:
        m.setattr(harness, "run_oracle", run_oracle)
        m.setattr(O, "build_model", _build_model)
        m.setattr(O.OracleRank, "_get_send_size", _unscaled_send_size)
        yield
