"""GAT against GATv2 (``--model gat`` / ``--model gatv2``) at P = 1, in one process, the two models alternating case by
case: eager epoch time and ``--cuda-graph`` epochs/s (``train.GraphedEpoch``), the attention kernels' time in one eager
epoch per C entry point from CUDA events, the bytes each score / aggregation pass gathers (from shapes), peak device
memory, and the evaluation forward on the whole graph and partition-parallel at P = 1.  One JSON line per (shape, heads, model); with ``--out DIR`` also appended to
``DIR/bench_gatv2.jsonl``.

  python tools/bench_gatv2.py --shape yelp --layers 2 --hidden 256 --heads 1
  python tools/bench_gatv2.py --shape reddit --layers 3 --hidden 256 --heads 1 4
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bns_gcn_b200  # noqa: E402,F401
from bns_gcn_b200 import train  # noqa: E402
from bns_gcn_b200.data import make_graph, partition_graph  # noqa: E402
from bns_gcn_b200.graph import FullGraphHandle  # noqa: E402
from bns_gcn_b200.helper.comm import run_threads  # noqa: E402
from tests.harness import make_args  # noqa: E402
from tools.bench_gat_eval import gpu_info, timed  # noqa: E402


# the C entry points of the attention layers (GAT's and GATv2's kernels and the SpMM / SDDMM passes they share)
_KERNEL_CALLS = ("bns_gat_", "bns_gatv2_", "bns_spmm_weighted_f32", "bns_spmm_compact_f32", "bns_sddmm_dot_f32")


def _kernel_ms(step):
    """One eager ``step()`` with a pair of CUDA events around every call of the C entry points above (on the stream
    the call is given, the current one): ms per entry point, summed over the step's calls."""
    from bns_gcn_b200 import _lib
    lib, saved, evs = _lib.lib, {}, {}
    names = [n for n in _lib.SIGNATURES if n.startswith(_KERNEL_CALLS) and not n.endswith("_bytes")]
    for n in names:
        fn = saved[n] = getattr(lib, n)

        def wrapped(*args, _fn=fn, _n=n):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            rc = _fn(*args)
            e1.record()
            evs.setdefault(_n, []).append((e0, e1))
            return rc
        setattr(lib, n, wrapped)
    try:
        step()
        torch.cuda.synchronize()
    finally:
        for n, fn in saved.items():
            setattr(lib, n, fn)
    return {n: round(sum(e0.elapsed_time(e1) for e0, e1 in v), 3) for n, v in sorted(evs.items())}


def one_case(fg, part, shape, layers, hidden, heads, model, warmup, iters, dev):
    args = make_args(dataset=shape, model=model, n_layers=layers, n_hidden=hidden, heads=heads, dropout=0.5,
                     sampling_rate=1.0, n_partitions=1, n_train=part.meta["n_train"])
    args.n_feat, args.n_class = part.meta["n_feat"], part.meta["n_class"]
    res = {}
    comm = None

    def body():
        torch.cuda.reset_peak_memory_stats(dev)
        st = train.setup(part.graph, part.node_dict, part.gpb, args, dev)
        ep = [0]

        def step():
            train.train_epoch(st, ep[0])
            ep[0] += 1
        res["epoch_ms"], res["epoch_ms_min"] = timed(step, warmup, iters)
        res["peak_mem_gb"] = round(torch.cuda.max_memory_allocated(dev) / 2 ** 30, 3)
        res["kernels_ms"] = _kernel_ms(step)
        graphed = train.GraphedEpoch(st, warmup)
        graphed()
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(iters):
            graphed()
        e.record()
        torch.cuda.synchronize()
        res["graph_epochs_per_s"] = round(1e3 * iters / s.elapsed_time(e), 3)
        # the whole-graph evaluation forward (layer(g, h) on the one-pass inference kernel)
        from bns_gcn_b200 import ops
        a = ops.DeviceGraph.from_csr(fg.indptr.to(dev), fg.src.int().to(dev), fg.n_nodes)
        h = FullGraphHandle(a, fg.in_degrees().to(dev), fg.out_degrees().to(dev))
        feat = fg.feat.to(dev)
        st.model.eval()
        with torch.no_grad():
            res["eval_whole_ms"], _ = timed(lambda: st.model(h, feat), 1, max(2, iters // 2))
        # the partition-parallel evaluation forward (--parallel-eval) of this one partition
        from bns_gcn_b200.evaluate import ParallelEvaluator, build_partition_eval_graph
        eg = build_partition_eval_graph(st.part, part.node_dict, st.boundary, comm)
        ev = ParallelEvaluator(args, eg, st.feat, st.labels, part.node_dict["val_mask"].to(dev),
                               part.node_dict["test_mask"].to(dev), comm)
        res["eval_parallel_p1_ms"], _ = timed(lambda: ev.logits(st.model), 1, max(2, iters // 2))
        st.model.train()

    def fn(comm_, r):
        nonlocal comm
        comm = comm_
        with torch.cuda.stream(torch.cuda.Stream(dev)):    # GraphedEpoch captures on a non-default stream
            body()
    run_threads(1, fn, device=str(dev))
    # bytes one score pass and one aggregation pass gather per layer of width hidden: GAT's score reads el (H floats per
    # entry), GATv2's reads the F-wide z_src row; both aggregations read the F-wide row once per entry
    nnz = int(part.graph.num_edges())
    res["score_gather_bytes_per_layer"] = nnz * 4 * (heads if model == "gat" else heads * hidden)
    res["agg_gather_bytes_per_layer"] = nnz * 4 * heads * hidden
    return res


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
        raise SystemExit("bench_gatv2: needs a CUDA device")
    dev = torch.device("cuda:0")
    name, power = gpu_info()
    fg = make_graph(a.shape, seed=0)
    part = partition_graph(fg, 1, "random", seed=0)[0]
    for heads in a.heads:
        for model in ("gat", "gatv2"):
            r = one_case(fg, part, a.shape, a.layers, a.hidden, heads, model, a.warmup, a.iters, dev)
            line = dict(gpu=name, power_limit=power, shape=a.shape, layers=a.layers, hidden=a.hidden, heads=heads,
                        model=model, P=1, **r)
            print(json.dumps(line), flush=True)
            if a.out:
                os.makedirs(a.out, exist_ok=True)
                with open(os.path.join(a.out, "bench_gatv2.jsonl"), "a") as f:
                    f.write(json.dumps(line) + "\n")
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
