"""Partitioner benchmark: ``random``, the ``metis`` stand-in (on the same GPU) and ``multilevel`` on the Reddit,
ogbn-products and Yelp shapes and on a Reddit-sized degree-corrected block model (40 communities, power-law degrees,
average about 50, 20 % of the edge ends leaving their community), for P in {2, 4, 8} and both objectives.

Reports per run: wall time (host clock around synchronised work, after a warm-up run on a small graph), peak device
memory, the exact cut and vol (``partition_quality``), the smallest and largest part, the most in-edges a part owns
over the mean ``E / P`` (a rank's aggregation work), and the boundary rows each epoch moves at sampling rate 0.1 (each
of the ``vol`` halo rows is sampled with probability 0.1: ``vol * 0.1``).  ``--balance nodes,edges`` runs every
configuration under each ``--partition-balance``.  The card's name and power limit are printed in the same run.  One
JSON line per run, then a markdown table.

  python tools/bench_partition.py [--shapes reddit,blocks,yelp,ogbn-products] [--parts 2,4,8] [--balance nodes,edges]
                                  [--budget-s 1500]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def card() -> str:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else torch.cuda.get_device_name(0)
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0) + " (power limit not read)"


def graph(name: str):
    from bns_gcn_b200.data import make_graph
    if name == "blocks":
        from tests.partition_reference import degree_corrected_blocks
        return degree_corrected_blocks(232_965, 40, 50, 0.2, seed=0)[0]
    return make_graph(name, seed=0)


def run(fg, P, method, objective, dev, balance="nodes"):
    from bns_gcn_b200.data import assign_parts, partition_quality
    torch.cuda.synchronize(dev)
    torch.cuda.reset_peak_memory_stats(dev)
    base = torch.cuda.memory_allocated(dev)
    t0 = time.perf_counter()
    part = assign_parts(fg, P, method, 0, objective, dev, balance)
    torch.cuda.synchronize(dev)
    dt = time.perf_counter() - t0
    peak = torch.cuda.max_memory_allocated(dev) - base
    q = partition_quality(fg, part, P, dev)
    return {"method": method, "P": P, "obj": objective, "time_s": round(dt, 3), "peak_mem_gb": round(peak / 2 ** 30, 3),
            "cut": q["cut"], "vol": q["vol"], "min_size": q["min_size"], "max_size": q["max_size"],
            "balance": balance, "max_over_mean_in_edges": round(q["max_in_edges"] * P / fg.n_edges, 4),
            "rows_per_epoch_p0.1": round(0.1 * q["vol"], 1)}


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="reddit,blocks,yelp,ogbn-products")
    ap.add_argument("--parts", default="2,4,8")
    ap.add_argument("--methods", default="random,metis,multilevel")
    ap.add_argument("--balance", default="nodes", help="comma-separated --partition-balance values: nodes, edges")
    ap.add_argument("--budget-s", type=float, default=1e9, help="skip (and list as not measured) what starts later")
    ap.add_argument("--out", default="")
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_partition.py measures on a GPU and there is none; it does not fall back to the CPU")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    import bns_gcn_b200  # noqa: F401
    from bns_gcn_b200.data import assign_parts, make_graph
    print(json.dumps({"card": card()}), flush=True)
    warm = make_graph("small", seed=0)
    for m in a.methods.split(","):
        assign_parts(warm, 4, m, 0, "vol", dev)
    start, rows, skipped = time.perf_counter(), [], []
    for shape in a.shapes.split(","):
        fg = None
        for P in (int(p) for p in a.parts.split(",")):
            for objective in ("vol", "cut"):
                for m in a.methods.split(","):
                    if m == "random" and objective == "cut":
                        continue                        # random ignores the objective
                    for balance in a.balance.split(","):
                        if time.perf_counter() - start > a.budget_s:
                            skipped.append(f"{shape} P={P} {objective} {m} {balance}")
                            continue
                        if fg is None:
                            fg = graph(shape)
                        r = dict(shape=shape, n=fg.n_nodes, edges=fg.n_edges, **run(fg, P, m, objective, dev, balance))
                        rows.append(r)
                        print(json.dumps(r), flush=True)
    print("\n| shape | P | obj | method | balance | time (s) | peak mem (GB) | cut | vol | min / max part | "
          "max / mean in-edges | rows / epoch at p=0.1 |")
    print("|---|---|---|---|---|---|---|---|---|---|---|---|")
    for r in rows:
        print(f"| {r['shape']} | {r['P']} | {r['obj']} | {r['method']} | {r['balance']} | {r['time_s']} | "
              f"{r['peak_mem_gb']} | {r['cut']:,} | {r['vol']:,} | {r['min_size']:,} / {r['max_size']:,} | "
              f"{r['max_over_mean_in_edges']} | {r['rows_per_epoch_p0.1']:,} |")
    for s in skipped:
        print("not measured:", s)
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"card": card(), "rows": rows, "not_measured": skipped}, f, indent=1)


if __name__ == "__main__":
    main()
