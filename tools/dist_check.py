"""Multi-process / multi-GPU check of the exchange transports (run under torchrun, one rank per GPU):

  python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29511 \
      tools/dist_check.py [--shape small] [--rate 0.3] [--graph] [--dropout 0.5] [--comm-dtype bf16|fp8]

Every rank trains a few epochs of the same seeded configuration with backend=nccl and backend=p2p (real NCCL
send/recv, real cudaIpc peer mappings over NVLink) and rank 0 compares the result -- loss, all-reduced weight
gradients, updated weights -- with the in-process (threads on one GPU) run of the same configuration, which
tests/test_parity_gpu.py pins to the CPU oracle.  Prints one JSON line; exit code 1 on mismatch.
"""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bns_gcn_b200  # noqa: E402,F401
from bns_gcn_b200 import train  # noqa: E402
from bns_gcn_b200.data import make_graph, partition_graph  # noqa: E402
from bns_gcn_b200.helper import context as ctx  # noqa: E402
from bns_gcn_b200.helper.comm import run_threads  # noqa: E402
from bns_gcn_b200.helper.timer.timer import comm_timer  # noqa: E402


def mk_args(shape, rate, backend, hidden, P, dropout=0.0, comm_dtype="f32"):
    return argparse.Namespace(dataset=shape, model="graphsage", n_layers=3, n_hidden=hidden, sampling_rate=rate,
                              use_pp=True, dropout=dropout, norm="layer", lr=1e-2, weight_decay=0.0, seed=0, n_linear=0,
                              backend=backend, sampler_seed=0, n_epochs=0, log_every=10 ** 9, heads=1, n_partitions=P,
                              inductive=False, partition_method="random", eval=False, chunk_nnz=0, comm_dtype=comm_dtype)


def train_rank(part, args, dev, n_epochs, graph=False):
    a = argparse.Namespace(**vars(args))
    a.n_feat, a.n_class, a.n_train = part.meta["n_feat"], part.meta["n_class"], part.meta["n_train"]
    st = train.setup(part.graph, part.node_dict, part.gpb, a, dev)
    losses = []
    if graph:        # 1 eager epoch (GraphedEpoch's warm-up) + replays: must equal n_epochs eager epochs
        torch.autograd.set_multithreading_enabled(False)
        ge = train.GraphedEpoch(st, warmup=1)
        losses.append(float("nan"))
        for e in range(1, n_epochs):
            losses.append(ge().item())
    for e in range(0 if not graph else n_epochs, n_epochs):
        losses.append(train.train_epoch(st, e).item())
    torch.cuda.synchronize(dev)
    comm_s = comm_timer.tot_time()
    return {"loss": losses, "grads": [p.grad.detach().cpu().clone() for p in st.model.parameters()],
            "params": [p.detach().cpu().clone() for p in st.model.parameters()], "comm_s": comm_s}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shape", default="small")
    ap.add_argument("--rate", type=float, default=0.3)
    ap.add_argument("--hidden", type=int, default=64)
    ap.add_argument("--epochs", type=int, default=3)
    ap.add_argument("--graph", action="store_true", help="run the distributed side from a captured CUDA graph")
    ap.add_argument("--dropout", type=float, default=0.0,
                    help="dropout rate of the model (the replayed masks must equal the eager ones)")
    ap.add_argument("--comm", default="torch", choices=["torch", "abi"],
                    help="abi: all-reduce / all-to-all through libbnsgcn.so's own communicator (bns_ctx_create ...)")
    ap.add_argument("--comm-dtype", default="f32", choices=["f32", "bf16", "fp8"],
                    help="element type of the exchanged boundary rows, on both sides of the comparison")
    a = ap.parse_args()
    os.environ["BNS_COMM"] = a.comm
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    torch.cuda.set_stream(torch.cuda.Stream(dev))       # one non-default stream for setup, eager epochs and capture
    fg = make_graph(a.shape, seed=0, device=dev)
    parts = partition_graph(fg, world, "random", seed=0, device=dev)
    res = {}
    # replayed from a CUDA graph the staged transport is only supported at 2 ranks (train.GraphedEpoch refuses otherwise)
    backends = ("p2p",) if (a.graph and world > 2) else ("nccl", "p2p")
    for backend in backends:
        ctx.reset()
        out = train_rank(parts[rank], mk_args(a.shape, a.rate, backend, a.hidden, world, a.dropout, a.comm_dtype), dev,
                         a.epochs, a.graph)
        tot = torch.tensor(out["loss"], dtype=torch.float64, device=dev)
        dist.all_reduce(tot)
        out["loss_sum"] = tot.tolist()
        res[backend] = out
        dist.barrier()
    ok, report = True, {}
    if rank == 0:
        ctx.reset()
        ref = run_threads(world, lambda c, r: train_rank(parts[r], mk_args(a.shape, a.rate, "nccl", a.hidden, world, a.dropout,
                                                                           a.comm_dtype), dev, a.epochs), device=str(dev))
        # bf16 / fp8 rows: a last-bit difference of an f32 quotient (the all-reduce sums in NCCL's order, not the
        # in-process one) can move a row element across a rounding boundary, a 2^-8 (bf16) or 2^-4 (fp8) step of it
        tol = 1e-5 if a.comm_dtype == "f32" else 1e-4
        ref_loss = [sum(ref[r]["loss"][e] for r in range(world)) for e in range(a.epochs)]
        for backend in backends:
            errs = [((x - y).norm() / y.norm().clamp(min=1e-30)).item()
                    for x, y in zip(res[backend]["grads"] + res[backend]["params"], ref[0]["grads"] + ref[0]["params"])]
            lerr = max(abs(x - y) / abs(y) for x, y in zip(res[backend]["loss_sum"], ref_loss) if x == x)
            report[backend] = {"max_rel_err_vs_inprocess": max(errs), "loss_rel_err": lerr,
                               "comm_s_last_epoch": res[backend]["comm_s"]}
            ok &= max(errs) < tol and lerr < tol
        print(json.dumps({"world": world, "shape": a.shape, "graph": a.graph, "comm": a.comm, "comm_dtype": a.comm_dtype,
                          "ok": bool(ok), **report}))
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
