"""One evaluation forward, whole-graph (rank 0 alone, ``evaluate.Evaluator``'s path) or partition-parallel (every rank
on its own partition, ``evaluate.ParallelEvaluator``'s path, ``--parallel-eval``): time with CUDA events after a
warm-up (median of ``--iters``), and peak device memory per rank -- what the whole run holds at the evaluation's peak,
and what the forward adds on top of what was resident before it.  Prints one JSON line (rank 0) with the card name and
power limit read in the same run.

  python tools/bench_eval.py --mode whole --shape reddit --model graphsage
  python tools/bench_eval.py --mode parallel --shape reddit --model gat --heads 4                 # P = 1
  torchrun --nproc-per-node 8 tools/bench_eval.py --mode parallel --shape reddit --model gcn        # P = 8
  torchrun --nproc-per-node 8 tools/bench_eval.py --mode parallel --shape papers100m --scale 0.1    # generated per rank
  python tools/bench_eval.py --inductive --mode whole --shape reddit --model gcn    # val_g and test_g, one forward each
  python tools/bench_eval.py --inductive --mode parallel --shape reddit --model gcn # their partitions (+ set-up ms)

The papers100M shape is never built as one graph: every rank generates its piece (``data.make_local_partition``), so
only ``--mode parallel`` takes it.  The other shapes are generated whole on every rank and cut by ``partition_graph``
(random partition).  The model has its seeded initial weights (``train.setup``): the forward's cost does not depend
on their values.

``--check`` (torchrun): rank 0 also runs the same partitions as in-process ranks (threads on its GPU, ``ThreadComm``)
and compares every rank's logits and the summed accuracy counts with the ``DistComm`` run; exit code 1 on mismatch.
"""
import argparse
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bns_gcn_b200  # noqa: E402,F401
from bns_gcn_b200 import train  # noqa: E402
from bns_gcn_b200.data import make_graph, make_local_partition, partition_graph  # noqa: E402
from bns_gcn_b200.helper import context as ctx  # noqa: E402
from bns_gcn_b200.helper.utils import get_layer_size  # noqa: E402

from bench_gat_eval import gpu_info, timed  # noqa: E402


def make_args(a, P):
    return argparse.Namespace(dataset=a.shape, model=a.model, n_layers=a.layers, n_hidden=a.hidden, sampling_rate=0.1,
                              use_pp=True, dropout=0.5, norm="layer", lr=1e-2, weight_decay=0.0, seed=0, n_linear=0,
                              backend="nccl", sampler_seed=0, n_epochs=0, log_every=10 ** 9, heads=a.heads,
                              n_partitions=P, inductive=False, partition_method="random", eval=True,
                              parallel_eval=True, chunk_nnz=0)


def parallel_rank(part, args, dev, comm, warmup=0, iters=0):
    """setup + the partition-parallel evaluation of one rank.  Returns logits, val / test counts and, when timed, the
    median / min forward time and the memory figures."""
    from bns_gcn_b200.evaluate import ParallelEvaluator, acc_counts, build_partition_eval_graph
    a = argparse.Namespace(**vars(args))
    a.n_feat, a.n_class, a.n_train = part.meta["n_feat"], part.meta["n_class"], part.meta["n_train"]
    st = train.setup(part.graph, part.node_dict, part.gpb, a, dev)
    eg = build_partition_eval_graph(st.part, part.node_dict, st.boundary, comm)
    ev = ParallelEvaluator(a, eg, st.feat, st.labels, part.node_dict["val_mask"].to(dev),
                           part.node_dict["test_mask"].to(dev), comm)
    logits = ev.logits(st.model)                     # also builds the peer blocks
    torch.cuda.synchronize(dev)
    out = {"logits": logits.cpu(), "val": acc_counts(logits[ev.val_mask], ev.labels[ev.val_mask]).cpu(),
           "test": acc_counts(logits[ev.test_mask], ev.labels[ev.test_mask]).cpu()}
    if iters:
        del logits
        base = torch.cuda.memory_allocated(dev)
        torch.cuda.reset_peak_memory_stats(dev)

        def fwd():
            comm.barrier()                           # every rank starts the collective forward together
            ev.logits(st.model)
        out["ms"] = timed(fwd, warmup, iters)
        torch.cuda.synchronize(dev)
        peak = torch.cuda.max_memory_allocated(dev)
        out["peak_GB"], out["extra_GB"] = peak / 2 ** 30, (peak - base) / 2 ** 30
    return out


def whole(a, dev):
    from bns_gcn_b200.evaluate import build_eval_graph
    fg = make_graph(a.shape, seed=0, device=dev)
    g = build_eval_graph(fg, dev)
    args = make_args(a, 1)
    args.n_feat, args.n_class, args.n_train = fg.n_feat, fg.n_class, int(fg.train_mask.sum())
    torch.manual_seed(args.seed)
    net = train.create_model(get_layer_size(fg.n_feat, a.hidden, fg.n_class, a.layers), args).to(dev).eval()
    feat = g.ndata["feat"]
    del fg
    torch.cuda.synchronize(dev)
    base = torch.cuda.memory_allocated(dev)
    torch.cuda.reset_peak_memory_stats(dev)
    with torch.no_grad():
        med, mn = timed(lambda: net(g.handle, feat), a.warmup, a.iters)
    peak = torch.cuda.max_memory_allocated(dev)
    return {"P": 1, "ms_median": round(med, 3), "ms_min": round(mn, 3), "peak_GB": [round(peak / 2 ** 30, 3)],
            "extra_GB": [round((peak - base) / 2 ** 30, 3)]}


def max_sm_clock():
    """The card's max SM clock (read-only query), reported beside the times."""
    import subprocess
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:                       # noqa: BLE001 - the times stand without it
        return "unknown"


def _model(a, args, fg, dev):
    args.n_feat, args.n_class, args.n_train = fg.n_feat, fg.n_class, int(fg.train_mask.sum())
    torch.manual_seed(args.seed)
    return train.create_model(get_layer_size(fg.n_feat, a.hidden, fg.n_class, a.layers), args).to(dev).eval()


def _ms(t0):
    torch.cuda.synchronize()
    return round((time.perf_counter() - t0) * 1e3, 3)


def inductive_whole(a, dev):
    """``--inductive --mode whole``: rank 0's ``Evaluator``, which holds the train | val subgraph (``val_g``) and the
    full graph (``test_g``) for the whole run; one forward on each."""
    from bns_gcn_b200.evaluate import eval_graphs
    fg = make_graph(a.shape, seed=0, device=dev)
    args = make_args(a, 1)
    args.inductive = True
    net = _model(a, args, fg, dev)
    torch.cuda.synchronize(dev)
    base = torch.cuda.memory_allocated(dev)
    torch.cuda.reset_peak_memory_stats(dev)
    val_g, test_g = eval_graphs(fg, True, dev)
    del fg
    rec = {"P": 1}
    with torch.no_grad():
        for w, g in (("val", val_g), ("test", test_g)):
            med, mn = timed(lambda: net(g.handle, g.ndata["feat"]), a.warmup, a.iters)
            rec[w + "_ms_median"], rec[w + "_ms_min"] = round(med, 3), round(mn, 3)
    peak = torch.cuda.max_memory_allocated(dev)
    rec.update(peak_GB=[round(peak / 2 ** 30, 3)], extra_GB=[round((peak - base) / 2 ** 30, 3)])
    return rec


def inductive_parallel(a, rank, world, dev, comm):
    """``--inductive --mode parallel``: this rank's parts of the two evaluation graphs (``data.eval_partitions``, what
    the store holds), each turned into the ``evaluate.EvalPart`` ``ParallelEvaluator`` evaluates (set-up: degrees,
    boundary, the layer-0 precompute) when it is needed -- the val graph first, the test graph in its place."""
    from bns_gcn_b200.data import eval_partitions
    from bns_gcn_b200.evaluate import build_eval_part
    fg = make_graph(a.shape, seed=0, device=dev)
    args = make_args(a, world)
    args.inductive = True
    net = _model(a, args, fg, dev)
    parts = {w: eval_partitions(fg, w, args, dev)[rank] for w in ("val", "test")}
    del fg
    torch.cuda.synchronize(dev)
    base = torch.cuda.memory_allocated(dev)
    torch.cuda.reset_peak_memory_stats(dev)
    rec, ep = {}, None
    for w in ("val", "test"):
        ep = None                                    # the val graph goes before the test graph is built
        comm.barrier()
        t0 = time.perf_counter()
        ep = build_eval_part(args, (parts[w].graph, parts[w].node_dict, parts[w].gpb), w, dev, comm)
        with torch.no_grad():
            net(ep.graph, ep.feat)                   # the first forward also cuts the peer blocks
        rec[w + "_setup_ms"] = _ms(t0)

        def fwd():
            comm.barrier()
            with torch.no_grad():
                net(ep.graph, ep.feat)
        rec[w + "_ms"] = timed(fwd, a.warmup, a.iters)
    peak = torch.cuda.max_memory_allocated(dev)
    rec.update(peak_GB=peak / 2 ** 30, extra_GB=(peak - base) / 2 ** 30)
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", choices=["whole", "parallel"], default="parallel")
    ap.add_argument("--shape", default="reddit")
    ap.add_argument("--scale", type=float, default=1.0, help="papers100m only: node and edge counts times this")
    ap.add_argument("--model", default="graphsage", choices=["graphsage", "gcn", "gat"])
    ap.add_argument("--heads", type=int, default=1)
    ap.add_argument("--layers", type=int, default=3)
    ap.add_argument("--hidden", type=int, default=256)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--check", action="store_true", help="compare the torchrun run with in-process ranks")
    ap.add_argument("--comm", default="torch", choices=["torch", "abi"],
                    help="abi: collectives through libbnsgcn.so's own communicator")
    ap.add_argument("--out", default=None, help="directory to append the JSON line to (eval.jsonl)")
    ap.add_argument("--inductive", action="store_true",
                    help="evaluate as an inductive run does: one forward on the train | val subgraph and one on the "
                         "full graph (parallel: on partitions of each, with the set-up time of each)")
    a = ap.parse_args()
    os.environ["BNS_COMM"] = a.comm
    dist_run = "WORLD_SIZE" in os.environ
    rank, world, local = (int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])) \
        if dist_run else (0, 1, 0)
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if a.inductive and (a.shape == "papers100m" or a.check):
        raise SystemExit("--inductive: not with the papers100m shape (never built whole) or --check")
    if a.mode == "whole":
        if dist_run or a.shape == "papers100m":
            raise SystemExit("--mode whole: one process on one GPU, and not the papers100m shape (never built whole)")
        rec = inductive_whole(a, dev) if a.inductive else whole(a, dev)
    elif a.inductive:
        from bns_gcn_b200.helper.comm import DistComm, SoloComm
        if dist_run:
            import torch.distributed as dist
            dist.init_process_group("nccl", device_id=dev)
            comm = DistComm()
        else:
            comm = SoloComm()
        ctx.set_comm(comm)
        torch.cuda.set_stream(torch.cuda.Stream(dev))
        mine = inductive_parallel(a, rank, world, dev, comm)
        import pickle
        every = [pickle.loads(b) for b in comm.all_gather_bytes(pickle.dumps(mine))]
        rec = {"P": world}
        for w in ("val", "test"):
            rec[w + "_ms_median"] = round(max(e[w + "_ms"][0] for e in every), 3)
            rec[w + "_ms_min"] = round(max(e[w + "_ms"][1] for e in every), 3)
            rec[w + "_setup_ms"] = round(max(e[w + "_setup_ms"] for e in every), 3)
        rec.update(peak_GB=[round(e["peak_GB"], 3) for e in every], extra_GB=[round(e["extra_GB"], 3) for e in every])
    else:
        from bns_gcn_b200.helper.comm import DistComm, SoloComm
        if dist_run:
            import torch.distributed as dist
            dist.init_process_group("nccl", device_id=dev)
            comm = DistComm()
        else:
            comm = SoloComm()
        ctx.set_comm(comm)
        torch.cuda.set_stream(torch.cuda.Stream(dev))
        if a.shape == "papers100m":
            parts = None
            part = make_local_partition(a.shape, rank, world, seed=0, device=dev, scale=a.scale)
        else:
            parts = partition_graph(make_graph(a.shape, seed=0, device=dev), world, "random", seed=0, device=dev)
            part = parts[rank]
        out = parallel_rank(part, make_args(a, world), dev, comm, a.warmup, a.iters)
        mine = {k: out[k] for k in ("ms", "peak_GB", "extra_GB")}
        import pickle
        every = [pickle.loads(b) for b in comm.all_gather_bytes(pickle.dumps(mine))]
        rec = {"P": world, "ms_median": round(max(e["ms"][0] for e in every), 3),
               "ms_min": round(max(e["ms"][1] for e in every), 3),
               "ms_median_per_rank": [round(e["ms"][0], 3) for e in every],
               "peak_GB": [round(e["peak_GB"], 3) for e in every], "extra_GB": [round(e["extra_GB"], 3) for e in every]}
        if a.check:
            if parts is None:
                raise SystemExit("--check: not for the per-rank generated papers100m shape")
            got = [pickle.loads(b) for b in comm.all_gather_bytes(pickle.dumps(
                {k: out[k] for k in ("logits", "val", "test")}))]
            ok = True
            if rank == 0:
                from bns_gcn_b200.helper.comm import run_threads
                ctx.reset()
                ref = run_threads(world, lambda c, r: parallel_rank(parts[r], make_args(a, world), dev, c),
                                  device=str(dev))
                ctx.set_comm(comm)
                errs = [((x["logits"] - y["logits"]).norm() / y["logits"].norm().clamp(min=1e-30)).item()
                        for x, y in zip(got, ref)]
                counts_equal = all(torch.equal(x[k], y[k]) for x, y in zip(got, ref) for k in ("val", "test"))
                ok = max(errs) < 1e-6 and counts_equal
                rec.update(check_max_rel_err_vs_inprocess=max(errs), check_counts_equal=counts_equal, ok=bool(ok))
            comm.barrier()
    if rank == 0:
        name, power = gpu_info()
        if a.inductive:
            rec["max_sm_clock"] = max_sm_clock()
        rec = {"mode": a.mode, "shape": a.shape, "scale": a.scale, "model": a.model, "heads": a.heads,
               "layers": a.layers, "hidden": a.hidden, "comm": a.comm, "inductive": a.inductive, **rec, "gpu": name,
               "power_limit": power}
        line = json.dumps(rec)
        print(line)
        if a.out:
            os.makedirs(a.out, exist_ok=True)
            with open(os.path.join(a.out, "eval.jsonl"), "a") as f:
                f.write(line + "\n")
    if a.mode == "parallel" and dist_run:
        import torch.distributed as dist
        dist.destroy_process_group()
    sys.exit(0 if rec.get("ok", True) else 1)


if __name__ == "__main__":
    main()
