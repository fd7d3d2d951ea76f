"""GraphSAGE with the mean aggregator against the max-pooling one (``--model graphsage`` / ``--model graphsage-pool``)
at P = 1, in one process, the two models alternating round by round: eager epoch time and ``--cuda-graph`` epochs/s
(``train.GraphedEpoch``), peak device memory, the time of every max and SpMM call of one eager epoch from CUDA events
(in call order: the max forward per layer, then the backward per layer), the bytes each pass gathers (from shapes), and
the evaluation forward on the whole graph and partition-parallel at P = 1.  One JSON line per (round, model); with
``--out DIR`` also appended to ``DIR/bench_sage_pool.jsonl``.

  python tools/bench_sage_pool.py --shape reddit --layers 3 --hidden 256 --rounds 2
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

# the max kernels and the SpMM passes (GraphSAGE's mean aggregation and its transpose)
_KERNEL_CALLS = ("bns_sage_max_", "bns_spmm")


def _kernel_ms(step):
    """One eager ``step()`` with a pair of CUDA events around every call of the C entry points above: per entry point,
    the ms of each call in call order."""
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
    return {n: [round(e0.elapsed_time(e1), 3) for e0, e1 in v] for n, v in sorted(evs.items())}


def one_case(fg, part, shape, layers, hidden, model, warmup, iters, dev):
    args = make_args(dataset=shape, model=model, n_layers=layers, n_hidden=hidden, dropout=0.5, sampling_rate=1.0,
                     n_partitions=1, n_train=part.meta["n_train"])
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
        res["peak_mem_gb"] = round(torch.cuda.max_memory_allocated(dev) / 2 ** 30, 3)
        from bns_gcn_b200 import ops
        a = ops.DeviceGraph.from_csr(fg.indptr.to(dev), fg.src.int().to(dev), fg.n_nodes)
        h = FullGraphHandle(a, fg.in_degrees().to(dev), fg.out_degrees().to(dev))
        feat = fg.feat.to(dev)
        st.model.eval()
        with torch.no_grad():
            res["eval_whole_ms"], _ = timed(lambda: st.model(h, feat), 1, max(2, iters // 2))
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
    # bytes gathered per pass: one source row per entry; the max gathers the pooled width (layer 0: the padded input
    # width, 604 on Reddit), its backward one int32 winner row per entry (plus d m where the entry won), GraphSAGE's
    # SpMM passes the hidden width (its layer 0 is precomputed)
    nnz = int(part.graph.num_edges())
    n_feat = part.meta["n_feat"]
    widths = [(n_feat + 3) // 4 * 4] + [hidden] * (layers - 1)
    if model == "graphsage-pool":
        res["max_fwd_gather_bytes"] = [nnz * 4 * w for w in widths]
        res["max_bwd_win_gather_bytes"] = [nnz * 4 * w for w in widths]
    else:
        res["spmm_gather_bytes"] = [nnz * 4 * hidden] * (layers - 1)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shape", default="reddit")
    ap.add_argument("--layers", type=int, default=3)
    ap.add_argument("--hidden", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sage_pool: needs a CUDA device")
    dev = torch.device("cuda:0")
    name, power = gpu_info()
    fg = make_graph(a.shape, seed=0)
    part = partition_graph(fg, 1, "random", seed=0)[0]
    for rnd in range(a.rounds):
        for model in ("graphsage", "graphsage-pool"):
            r = one_case(fg, part, a.shape, a.layers, a.hidden, model, a.warmup, a.iters, dev)
            line = dict(gpu=name, power_limit=power, shape=a.shape, layers=a.layers, hidden=a.hidden, model=model,
                        round=rnd, P=1, **r)
            print(json.dumps(line), flush=True)
            if a.out:
                os.makedirs(a.out, exist_ok=True)
                with open(os.path.join(a.out, "bench_sage_pool.jsonl"), "a") as f:
                    f.write(json.dumps(line) + "\n")
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
