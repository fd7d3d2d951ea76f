"""Mint tests/golden/ref_gat_eval_p2.pt: the reference's GAT (2 heads, closing width 5) trained for two epochs by its
own ``train.run`` under make_golden.py's DGL stand-in, then its evaluation forward (train.py:44-49:
``model.eval(); model(g, feat)``) on the whole graph.

In evaluation the reference's GAT calls ``dgl.nn.GATConv`` homogeneously, ``layer(g, h)`` (module/model.py:123), and
DGL then uses ``h_src = h_dst = feat_drop(h)``.  make_golden.py's ``GATConvStandIn`` only takes the bipartite training
call ``layer(g, (h_src, h_dst))``, so this script wraps its forward to accept both and otherwise runs make_golden.py's
worker unchanged.

    python tests/golden/make_golden_gat_eval.py         # writes tests/golden/ref_gat_eval_p2.pt
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402

NAME = "gat_eval"
CONFIG = dict(shape="tiny", n_parts=2, model="gat", n_layers=3, n_hidden=16, rate=0.5, epochs=2, heads=2,
              eval_logits=True, slim=True)
PORT = 29611

_bipartite_forward = mg.GATConvStandIn.forward


def _forward(self, graph, feat):
    if not isinstance(feat, tuple):                  # DGL's homogeneous branch: the same rows are sources and destinations
        feat = (feat, feat)
    return _bipartite_forward(self, graph, feat)


mg.GATConvStandIn.forward = _forward                 # at import: the spawned workers import this module too


def worker(rank, world, cfg, port, out_dir):
    mg.worker(rank, world, cfg, port, out_dir)


def main():
    import tempfile
    import torch.multiprocessing as mp
    cfg = CONFIG
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(worker, args=(cfg["n_parts"], cfg, PORT, d), nprocs=cfg["n_parts"], join=True)
        ranks = [torch.load(os.path.join(d, f"rank{r}.pt")) for r in range(cfg["n_parts"])]
    # "slim", as make_golden.py: every rank's index sets, rank 0's tensors
    keep0 = ("selected", "boundary", "param_names", "logits", "layer_out", "params", "grads", "eval_logits")
    ranks = [{k: ([v[-1]] if k in ("logits", "layer_out") else v) for k, v in rk.items()
              if k in (keep0 if r == 0 else ("selected", "boundary", "param_names"))} for r, rk in enumerate(ranks)]
    out = os.path.join(HERE, f"ref_{NAME}_p{cfg['n_parts']}.pt")
    torch.save({"config": cfg, "ranks": ranks}, out)
    print("wrote", out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main()
