"""``--comm-dtype f32`` against ``bf16`` and ``fp8``: what the boundary exchange moves and what it costs.

* ``bytes``: exact counts from shapes (no GPU): per epoch and rank, the feature bytes sent and received forward and
  backward per communicating layer, and the peer-mapped slab (``feature_buffer.slab_layout``), for the Reddit shape at
  P = 2 / 4 / 8 and the papers100M per-rank shape, at the benchmark's sampling rate 0.1 and hidden width 256.  Reddit:
  232,965 nodes in random partitions, where every inner node is on every peer's boundary, so each rank sends
  int(0.1 n_in) rows to each peer; papers100M: 13.9 M inner nodes and 9.7 M sampled halo rows per rank (sent as many).
* ``kernels`` (one GPU): CUDA-event time per launch of the all-peer put and the gradient scatter in each mode, at
  the Reddit shape's per-rank sizes at P = 4.  The peers are slabs of this process on the same GPU, so a put's stores
  go to this GPU's HBM: these times say nothing about NVLink.
* ``epochs``: eager epochs/s of the benchmark's model on the Reddit shape with 4 in-process ranks (threads of this
  process on one GPU, peer-mapped transport), both modes.  In-process ranks share one GPU's HBM and run one after the
  other's kernels, and cannot be captured into CUDA graphs (each waits on events of the others' streams): this is not a
  multi-GPU number.
* ``convergence``: the ``small`` shape, 4 in-process partitions, 200 epochs, both modes: final training loss (summed
  over ranks) and validation accuracy of a dropout-free forward of the trained model on each rank's inner nodes.

    python tools/bench_comm_dtype.py [--only bytes] > result.json
"""
import argparse
import contextlib
import ctypes
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

REDDIT_NODES = 232_965
RATE, WIDTH, N_COMM = 0.1, 256, 2          # the benchmark's model: 3 layers, the inputs of layers 1 and 2 exchanged
MODES = ("f32", "bf16", "fp8")


def byte_counts() -> dict:
    from bns_gcn_b200.helper.feature_buffer import slab_layout, wire_bytes
    shapes = {}
    for P in (2, 4, 8):
        n_in = -(-REDDIT_NODES // P)
        send = recv = (P - 1) * int(RATE * n_in)
        shapes[f"reddit_P{P}"] = (n_in, send, recv)
    shapes["papers100m_per_rank_P8"] = (111_059_956 // 8, 9_700_000, 9_700_000)
    out = {}
    for name, (n_in, send, recv) in shapes.items():
        row = {"n_in": n_in, "send_rows": send, "recv_rows": recv}
        for m in MODES:
            w = wire_bytes(send, recv, WIDTH, m)
            lay = slab_layout(n_in, recv, send, WIDTH, N_COMM, m)
            row[m] = {"per_layer": w, "per_epoch_sent": N_COMM * (w["fwd_send"] + w["bwd_send"]),
                      "per_epoch_received": N_COMM * (w["fwd_recv"] + w["bwd_recv"]),
                      "slab_bytes": lay["slab_bytes"],
                      "slab_halo_region": lay["halo_bytes"] + lay.get("halo_scale_bytes", 0),
                      "slab_backward_region": lay["bwd_bytes"] + lay.get("bwd_scale_bytes", 0)}
        row["sent_ratio_bf16_over_f32"] = row["bf16"]["per_epoch_sent"] / row["f32"]["per_epoch_sent"]
        row["sent_ratio_fp8_over_bf16"] = row["fp8"]["per_epoch_sent"] / row["bf16"]["per_epoch_sent"]
        out[name] = row
    return out


def card() -> dict:
    import subprocess
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    f = [s.strip() for s in q.stdout.splitlines()[0].split(",")] if q.returncode == 0 and q.stdout else []
    return {"name": f[0] if f else torch.cuda.get_device_name(0), "power_limit": f[1] if len(f) > 1 else "not read",
            "sm_max_clock": f[2] if len(f) > 2 else "not read"}


def kernel_times(iters: int = 200) -> dict:
    """Rank 0 of P = 4 on the Reddit shape: 3 peers, int(0.1 n_in) rows each, F = 256."""
    import torch
    from bns_gcn_b200 import ops
    from bns_gcn_b200._lib import PutAll, check, lib
    dev = torch.device("cuda", 0)
    P, n_in = 4, -(-REDDIT_NODES // 4)
    k = int(RATE * n_in)
    slab = 2 * 3 * k * WIDTH * 4 + (1 << 20)
    hs = []
    for r in range(P):
        h = ctypes.c_void_p()
        check(lib.bns_p2p_create(ctypes.byref(h), r, P, slab, 8), "bns_p2p_create")
        hs.append(h)
    info = []
    for h in hs:
        s, f, n = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_size_t()
        check(lib.bns_p2p_local(h, ctypes.byref(s), ctypes.byref(f), ctypes.byref(n)), "bns_p2p_local")
        info.append((s.value, f.value, n.value))
    for r in range(1, P):
        check(lib.bns_p2p_set_peer(hs[0], r, *info[r]), "bns_p2p_set_peer")
    g = torch.Generator(device=dev).manual_seed(0)
    H = torch.randn(n_in, WIDTH, device=dev, generator=g)
    idx = torch.randperm(n_in, device=dev, generator=g)[:3 * k].contiguous()
    st = torch.cuda.current_stream().cuda_stream
    res = {"rows_per_peer": k, "peers": P - 1, "F": WIDTH, "iters": iters}

    def segs(esz):
        s = PutAll()
        s.n_seg = P - 1
        for i in range(P - 1):
            s.row_begin[i], s.peer[i], s.remote_off[i], s.div[i] = i * k, i + 1, 0, 0.1
        s.row_begin[P - 1] = (P - 1) * k
        return s

    def timed(fn):
        for _ in range(10):
            fn()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        b.synchronize()
        return a.elapsed_time(b) / iters
    s32, s16, s8 = segs(4), segs(2), segs(1)
    scale_off = (ctypes.c_uint64 * (P - 1))(*[k * WIDTH] * (P - 1))          # the codes at 0, their scales after them
    put = {"f32": lambda: check(lib.bns_p2p_put_all_f32(hs[0], ctypes.byref(s32), WIDTH, H.data_ptr(), WIDTH, WIDTH,
                                                        idx.data_ptr(), 1, P, 1, None, st), "put f32"),
           "bf16": lambda: check(lib.bns_p2p_put_all_bf16(hs[0], ctypes.byref(s16), WIDTH, H.data_ptr(), WIDTH, WIDTH,
                                                          idx.data_ptr(), 1, P, 1, None, st), "put bf16"),
           "fp8": lambda: check(lib.bns_p2p_put_all_fp8(hs[0], ctypes.byref(s8), scale_off, WIDTH, H.data_ptr(), WIDTH,
                                                        WIDTH, idx.data_ptr(), 1, P, 1, None, st), "put fp8")}
    invs = []
    for i in range(P - 1):
        m = torch.full((n_in,), -1, dtype=torch.int32, device=dev)
        m[idx[i * k:(i + 1) * k]] = torch.arange(k, dtype=torch.int32, device=dev)
        invs.append(m)
    recv32 = [torch.randn(k, WIDTH, device=dev, generator=g) for _ in range(P - 1)]
    recv16 = [r.to(torch.bfloat16) for r in recv32]
    recv8 = [ops.cvt_rows_fp8(r) for r in recv32]
    G = torch.zeros(n_in, WIDTH, device=dev)
    inv = (ctypes.c_void_p * (P - 1))(*[m.data_ptr() for m in invs])
    div = (ctypes.c_float * (P - 1))(*[0.1] * (P - 1))
    r32 = (ctypes.c_void_p * (P - 1))(*[r.data_ptr() for r in recv32])
    r16 = (ctypes.c_void_p * (P - 1))(*[r.data_ptr() for r in recv16])
    r8 = (ctypes.c_void_p * (P - 1))(*[r.codes.data_ptr() for r in recv8])
    sc8 = (ctypes.c_void_p * (P - 1))(*[r.scale.data_ptr() for r in recv8])
    scat = {"f32": lambda: check(lib.bns_scatter_rows_all_f32(G.data_ptr(), WIDTH, n_in, WIDTH, P - 1, inv, r32, WIDTH,
                                                              div, st), "scatter f32"),
            "bf16": lambda: check(lib.bns_scatter_rows_all_bf16(G.data_ptr(), WIDTH, n_in, WIDTH, P - 1, inv, r16, WIDTH,
                                                                div, st), "scatter bf16"),
            "fp8": lambda: check(lib.bns_scatter_rows_all_fp8(G.data_ptr(), WIDTH, n_in, WIDTH, P - 1, inv, r8, sc8, WIDTH,
                                                              div, st), "scatter fp8")}
    for rnd in range(3):                        # alternate the modes: other work on the host shares the GPU
        for m in MODES:
            res.setdefault(f"put_ms_{m}", []).append(round(timed(put[m]), 5))
            res.setdefault(f"scatter_ms_{m}", []).append(round(timed(scat[m]), 5))
    torch.cuda.synchronize()
    for h in hs:
        lib.bns_p2p_destroy(h)
    return res


def _train(shape: str, P: int, comm_dtype: str, epochs: int, warmup: int, accuracy: bool) -> dict:
    import torch
    import bench
    from bns_gcn_b200 import train
    from bns_gcn_b200.data import make_graph, partition_graph
    from bns_gcn_b200.helper.comm import run_threads
    dev = torch.device("cuda", 0)
    parts = partition_graph(make_graph(shape, seed=0, device=dev), P, "random", seed=0, device=dev)

    def fn(comm, r):
        p = parts[r]
        args = bench.make_args(P, "p2p", {"n_feat": p.meta["n_feat"], "n_class": p.meta["n_class"],
                                          "n_train": p.meta["n_train"], "dataset": shape, "comm_dtype": comm_dtype})
        st = train.setup(p.graph, p.node_dict, p.gpb, args, dev)
        losses = [float(train.train_epoch(st, e).item()) for e in range(warmup)]
        torch.cuda.synchronize()
        comm.barrier()
        t0 = time.perf_counter()
        losses += [train.train_epoch(st, e) for e in range(warmup, warmup + epochs)]
        torch.cuda.synchronize()
        comm.barrier()
        dt = time.perf_counter() - t0
        out = {"seconds": dt, "loss": [float(x) for x in losses]}
        if accuracy:
            keep, st.model.dropout.p = st.model.dropout.p, 0.0
            with torch.no_grad():
                logits = train._forward_logits(st, warmup + epochs)
            st.model.dropout.p = keep
            n_in = p.graph.n_in
            m = p.node_dict["val_mask"][:n_in].to(dev).bool()
            lab = p.node_dict["label"][:n_in].to(dev)
            out["val_correct"] = int((logits[:n_in].argmax(1)[m] == lab[m]).sum().item())
            out["val_total"] = int(m.sum().item())
        return out

    with contextlib.redirect_stdout(sys.stderr):
        res = run_threads(P, fn, device=str(dev))
    rep = {"epochs_per_s": round(epochs / max(r["seconds"] for r in res), 3),
           "final_train_loss_sum_over_ranks": sum(r["loss"][-1] for r in res)}
    if accuracy:
        rep["val_accuracy"] = sum(r["val_correct"] for r in res) / max(sum(r["val_total"] for r in res), 1)
    return rep


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", choices=["bytes", "kernels", "epochs", "convergence"], default=None)
    ap.add_argument("--epochs", type=int, default=10)
    a = ap.parse_args()
    out = {}
    if a.only in (None, "bytes"):
        out["bytes"] = byte_counts()
    if a.only is None or a.only != "bytes":
        import torch
        if not torch.cuda.is_available():
            raise SystemExit("the timed parts need a GPU")
        out["card"] = card()
    if a.only in (None, "kernels"):
        out["kernels"] = kernel_times()
        out["kernels"]["note"] = ("in-process peers share one GPU's HBM: these times say nothing about NVLink")
    if a.only in (None, "epochs"):
        out["epochs_reddit_P4_inprocess_eager"] = {m: _train("reddit", 4, m, a.epochs, 2, False) for m in MODES}
        out["epochs_reddit_P4_inprocess_eager"]["note"] = (
            "4 ranks as threads of one process on one GPU (shared HBM, eager: in-process ranks cannot be graph-captured)")
    if a.only in (None, "convergence"):
        out["convergence_small_P4_200_epochs"] = {m: _train("small", 4, m, 198, 2, True) for m in MODES}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
