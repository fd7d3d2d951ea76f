"""Per-part aggregation time under ``--partition-balance nodes`` and ``edges``: a proxy for the slowest rank.

For the Reddit shape at each P, with the ``metis`` stand-in and ``multilevel`` (objective ``vol``), under each balance,
every part is built as ``train.setup`` builds it (``get_in_out_graph`` -> ``PartitionGraph``) and, one part at a time on
one GPU, its two F = 256 aggregation passes are timed: the inner pass (``spmm_auto`` on ``a_in``) and its transposed
pass (``a_in_t``), with CUDA events around ``--iters`` launches after ``--warmup`` launches.  Printed per run: each
part's ms (the two passes together) and in-edges (the nnz of its ``a_in`` plus ``a_out`` rows), max / mean ms, max /
mean in-edges, and the partition's ``vol``; the card's name and power limit come from the same run.  The epoch rate of
a multi-GPU run is not measured here: the slowest part's time only stands in for the rank that sets it.

  python tools/bench_partition_balance.py [--parts 2,4,8] [--methods metis,multilevel] [--out results.json]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402


def part_ms(p, dev, F, warmup, iters):
    """The two aggregation passes of one part: (ms per pair of passes, in-edges)."""
    from bns_gcn_b200 import ops
    from bns_gcn_b200.graph import PartitionGraph
    from bns_gcn_b200.train import get_in_out_graph
    in_graph, out_graph = get_in_out_graph(p.graph, p.node_dict, dev)
    g = PartitionGraph(p.graph.n_in, p.graph.n_halo, in_graph, out_graph, dev)
    n_in = p.graph.n_in
    gen = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(n_in, F, device=dev, generator=gen)
    dy = torch.randn(n_in, F, device=dev, generator=gen)
    y, dx = torch.empty_like(x), torch.empty_like(dy)

    def step():
        ops.spmm_auto(g.a_in, x, y)
        ops.spmm_auto(g.a_in_t, dy, dx)

    for _ in range(warmup):
        step()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize(dev)
    s.record()
    for _ in range(iters):
        step()
    e.record()
    torch.cuda.synchronize(dev)
    ms = s.elapsed_time(e) / iters
    del g, in_graph, out_graph, x, dy, y, dx
    torch.cuda.empty_cache()
    return ms, p.graph.num_edges()


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--shape", default="reddit")
    ap.add_argument("--parts", default="2,4,8")
    ap.add_argument("--methods", default="metis,multilevel")
    ap.add_argument("--F", type=int, default=256)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default="")
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_partition_balance.py measures on a GPU and there is none; it does not fall back to the "
                         "CPU")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    import bns_gcn_b200  # noqa: F401
    from bench_partition import card
    from bns_gcn_b200.data import make_graph, partition_quality
    from bns_gcn_b200.data.partition import assign_parts, extract_partition, relabel
    info = card()
    print(json.dumps({"card": info}), flush=True)
    fg = make_graph(a.shape, seed=0)
    rows = []
    for P in (int(p) for p in a.parts.split(",")):
        for method in a.methods.split(","):
            for balance in ("nodes", "edges"):
                part = assign_parts(fg, P, method, 0, "vol", dev, balance)
                vol = partition_quality(fg, part, P, dev)["vol"]
                g, ranges = relabel(fg, part, P, dev)            # as partition_graph cuts the parts, one at a time
                ind, outd = g.in_degrees(), g.out_degrees()
                ms, edges = [], []
                for r in range(P):
                    t, e = part_ms(extract_partition(g, ranges, r, False, ind, outd), dev, a.F, a.warmup, a.iters)
                    ms.append(round(t, 3))
                    edges.append(e)
                row = {"shape": a.shape, "P": P, "method": method, "balance": balance, "vol": vol, "part_ms": ms,
                       "part_in_edges": edges, "max_over_mean_ms": round(max(ms) * P / sum(ms), 3),
                       "max_over_mean_in_edges": round(max(edges) * P / sum(edges), 3)}
                rows.append(row)
                print(json.dumps(row), flush=True)
    print(f"\n{info}; F = {a.F}; ms = the inner pass plus its transposed pass, per part")
    print("| P | method | balance | vol | max / mean ms | max / mean in-edges | per-part ms | per-part in-edges (M) |")
    print("|---|---|---|---|---|---|---|---|")
    for r in rows:
        print(f"| {r['P']} | {r['method']} | {r['balance']} | {r['vol']:,} | {r['max_over_mean_ms']} | "
              f"{r['max_over_mean_in_edges']} | {' / '.join(str(x) for x in r['part_ms'])} | "
              f"{' / '.join(f'{x / 1e6:.1f}' for x in r['part_in_edges'])} |")
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"card": info, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
