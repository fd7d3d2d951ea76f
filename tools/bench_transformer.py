"""GAT, GATv2 and the graph transformer layer (``--model gat`` / ``gatv2`` / ``transformer``) at P = 1, in one process,
the three models alternating case by case: eager epoch time and ``--cuda-graph`` epochs/s (``train.GraphedEpoch``), the
attention kernels' time in one eager epoch per C entry point from CUDA events, the bytes each score / aggregation pass
gathers (from shapes), peak device memory, and the evaluation forward on the whole graph and partition-parallel at
P = 1 (``tools/bench_gatv2.one_case``).  One JSON line per (shape, heads, model); with ``--out DIR`` also appended to
``DIR/bench_transformer.jsonl``.

  python tools/bench_transformer.py --shape yelp --layers 2 --hidden 256 --heads 1
  python tools/bench_transformer.py --shape reddit --layers 3 --hidden 256 --heads 1 4
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bns_gcn_b200  # noqa: E402,F401
from bns_gcn_b200.data import make_graph, partition_graph  # noqa: E402
from tools import bench_gatv2  # noqa: E402
from tools.bench_gat_eval import gpu_info  # noqa: E402

MODELS = ("gat", "gatv2", "transformer")


def gather_bytes(nnz, heads, hidden, model):
    """Bytes one layer of width ``hidden`` gathers per pass, from the shapes: GAT's score reads el (H floats per
    entry), GATv2's the F-wide z_src row, the transformer's the F-wide key row (its softmax backward reads it again);
    every aggregation reads the F-wide source (value) row once per entry; the transformer's evaluation reads the key
    and the value row of every entry."""
    F = heads * hidden
    score = {"gat": heads, "gatv2": F, "transformer": F}[model]
    return {"score_gather_bytes_per_layer": nnz * 4 * score, "agg_gather_bytes_per_layer": nnz * 4 * F,
            "eval_gather_bytes_per_layer": nnz * 4 * (F + score)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shape", default="yelp")
    ap.add_argument("--layers", type=int, default=2)
    ap.add_argument("--hidden", type=int, default=256)
    ap.add_argument("--heads", type=int, nargs="+", default=[1])
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_transformer: needs a CUDA device")
    bench_gatv2._KERNEL_CALLS += ("bns_tconv_",)
    dev = torch.device("cuda:0")
    name, power = gpu_info()
    fg = make_graph(a.shape, seed=0)
    part = partition_graph(fg, 1, "random", seed=0)[0]
    nnz = int(part.graph.num_edges())
    for heads in a.heads:
        for model in MODELS:
            r = bench_gatv2.one_case(fg, part, a.shape, a.layers, a.hidden, heads, model, a.warmup, a.iters, dev)
            r.update(gather_bytes(nnz, heads, a.hidden, model))
            line = dict(gpu=name, power_limit=power, shape=a.shape, layers=a.layers, hidden=a.hidden, heads=heads,
                        model=model, P=1, **r)
            print(json.dumps(line), flush=True)
            if a.out:
                os.makedirs(a.out, exist_ok=True)
                with open(os.path.join(a.out, "bench_transformer.jsonl"), "a") as f:
                    f.write(json.dumps(line) + "\n")
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
