"""``train.run``'s epoch loop, eager against ``--cuda-graph``, and the cost and resolution of the replay stamps.  Prints
one JSON line (rank 0) with the card name and power limit read in the same run.

  python tools/bench_cli_graph.py                                       # P = 1, Reddit shape, no evaluation
  torchrun --nproc-per-node 4 tools/bench_cli_graph.py --backend p2p    # P = 4: also Comm(s) / Reduce(s) of both modes

* ``run``: ``train.run`` on the generated shape (random partition, 3-layer GraphSAGE, hidden 256, --use-pp, sampling
  rate 0.1, dropout 0.5, no evaluation), once eagerly and once with ``--cuda-graph``, ``--epochs`` epochs each: the
  mean ``Time(s)`` over the timed epochs (the first 5 excluded, as the log line does), epochs/s, and the mean
  ``Comm(s)`` / ``Reduce(s)``.  Every rank's numbers are maxed over the ranks.
* ``stamp_cost``: two ``GraphedEpoch`` s of one fresh training state, ``timed=True`` and ``timed=False``, replayed in
  ``--rounds`` alternating rounds of ``--replays`` replays; the per-epoch difference of their medians.  At P = 1 no
  interval exists (one rank exchanges and all-reduces nothing), so both graphs are the same graph.
* ``stamp_kernel``: one graph of 1024 back-to-back stamps on one stream -- the time per stamp, and the distinct steps
  between consecutive stamps (the resolution ``%globaltimer`` shows on this card).
"""
import argparse
import contextlib
import io
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bns_gcn_b200  # noqa: E402,F401
from bns_gcn_b200 import ops, train  # noqa: E402
from bns_gcn_b200.data import make_graph, partition_graph  # noqa: E402
from bns_gcn_b200.helper import context as ctx  # noqa: E402

from bench_gat_eval import gpu_info  # noqa: E402


def make_args(a, P, **kw):
    return argparse.Namespace(dataset=a.shape, model="graphsage", n_layers=3, n_hidden=a.hidden, sampling_rate=0.1,
                              use_pp=True, dropout=0.5, norm="layer", lr=1e-2, weight_decay=0.0, seed=0, n_linear=0,
                              backend=a.backend, sampler_seed=0, n_epochs=a.epochs, log_every=10 ** 9, heads=1,
                              n_partitions=P, inductive=False, partition_method="random", eval=False, chunk_nnz=0, **kw)


def with_meta(args, part):
    a = argparse.Namespace(**vars(args))
    a.n_feat, a.n_class, a.n_train = part.meta["n_feat"], part.meta["n_class"], part.meta["n_train"]
    return a


def max_over_ranks(x, world, dev):
    if world == 1:
        return x
    import torch.distributed as dist
    t = torch.tensor([x], dtype=torch.float64, device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def one_run(a, part, P, dev, cuda_graph):
    """``train.run`` (log line silenced); mean Time(s), Comm(s), Reduce(s) over its timed epochs."""
    ctx.reset()
    with contextlib.redirect_stdout(io.StringIO()):
        _, res = train.run(part.graph, part.node_dict, part.gpb, with_meta(make_args(a, P, cuda_graph=cuda_graph), part),
                           dev)
    ctx.reset()
    return {k: statistics.fmean(res[k]) for k in ("time", "comm", "reduce")}


def stamp_cost(a, part, P, dev):
    ctx.reset()
    ms = {True: [], False: []}
    with torch.cuda.stream(torch.cuda.Stream(dev)), torch.autograd.set_multithreading_enabled(False):
        with contextlib.redirect_stdout(io.StringIO()):
            st = train.setup(part.graph, part.node_dict, part.gpb, with_meta(make_args(a, P), part), dev)
        graphs = {True: train.GraphedEpoch(st, warmup=3, timed=True),
                  False: train.GraphedEpoch(st, warmup=0, timed=False)}
        n_stamps = 2 * len(graphs[True].stamps.names)
        for g in graphs.values():                       # warm both
            g()
        cur = torch.cuda.current_stream(dev)
        for r in range(a.rounds):
            for timed in ((True, False) if r % 2 == 0 else (False, True)):
                torch.cuda.synchronize(dev)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(cur)
                for _ in range(a.replays):
                    graphs[timed]()
                e1.record(cur)
                torch.cuda.synchronize(dev)
                ms[timed].append(e0.elapsed_time(e1) / a.replays)
    ctx.reset()
    on, off = statistics.median(ms[True]), statistics.median(ms[False])
    return {"stamps_per_epoch": n_stamps, "timed_ms": on, "untimed_ms": off, "diff_ms": on - off,
            "spread_timed_ms": [min(ms[True]), max(ms[True])], "spread_untimed_ms": [min(ms[False]), max(ms[False])]}


def stamp_kernel(dev, n=1024):
    s = torch.cuda.Stream(dev)
    with torch.cuda.stream(s):
        slots = torch.zeros(n, dtype=torch.int64, device=dev)
        ops.stamp_globaltimer(slots[0:1])
        torch.cuda.synchronize(dev)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            for i in range(n):
                ops.stamp_globaltimer(slots[i:i + 1])
        g.replay()
        torch.cuda.synchronize(dev)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(s)
        for _ in range(10):
            g.replay()
        e1.record(s)
        torch.cuda.synchronize(dev)
        v = slots.cpu().tolist()
    steps = [b - a for a, b in zip(v, v[1:])]
    nonzero = sorted(d for d in steps if d > 0)
    hist = {}
    for d in steps:
        hist[d] = hist.get(d, 0) + 1
    return {"us_per_stamp": e0.elapsed_time(e1) * 1e3 / (10 * n), "zero_steps": steps.count(0),
            "min_nonzero_step_ns": nonzero[0] if nonzero else None,
            "most_common_steps_ns": sorted(hist.items(), key=lambda kv: -kv[1])[:6],
            "span_ns": v[-1] - v[0], "n": n}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shape", default="reddit")
    ap.add_argument("--hidden", type=int, default=256)
    ap.add_argument("--backend", default="p2p")
    ap.add_argument("--epochs", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--replays", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_cli_graph.py measures on the GPU; there is no CPU path")
    world, rank = int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=dev)
    part = partition_graph(make_graph(a.shape, seed=0), world, "random", seed=0)[rank]
    out = {"shape": a.shape, "P": world, "backend": a.backend, "epochs": a.epochs, "timed_epochs": a.epochs - 5}
    for name, flag in (("eager", False), ("cuda_graph", True)):
        r = one_run(a, part, world, dev, flag)
        r = {k: max_over_ranks(v, world, dev) for k, v in r.items()}
        out[name] = {"time_s": r["time"], "epochs_per_s": 1.0 / r["time"], "comm_s": r["comm"], "reduce_s": r["reduce"]}
    out["stamp_cost"] = stamp_cost(a, part, world, dev)
    out["stamp_cost"]["diff_ms"] = max_over_ranks(out["stamp_cost"]["diff_ms"], world, dev)
    out["stamp_kernel"] = stamp_kernel(dev)
    name, power = gpu_info()
    out.update(gpu=name, power_limit=power)
    if rank == 0:
        print(json.dumps(out))
    if world > 1:
        import torch.distributed as dist
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
