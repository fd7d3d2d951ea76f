"""``--dense-dtype f32`` / ``bf16`` / ``fp8`` on the benchmark's workload (BASELINE.json configs[1]: Reddit-shape graph,
3-layer GraphSAGE, hidden 256, --use-pp) at ONE partition, all modes in one process:

* the mean time of every dense GEMM call of the epoch (``dense.PROFILE`` CUDA events, eager epochs, modes alternating),
  by call site in launch order with its shape, and the dense milliseconds per epoch; under fp8 the quantization passes
  (``ops.cvt_rows_fp8_any`` and layer 0's ``fused.dropout_fp8``, which also does the dropout) are timed on their own;
* epochs/s of ``train.GraphedEpoch`` replays in alternating rounds, in four pairings: f32 against ``--dense-dtype bf16``,
  ``--agg-dtype bf16`` alone against ``--agg-dtype bf16 --dense-dtype bf16``, ``--dense-dtype bf16`` against ``fp8``, and
  ``--agg-dtype fp8`` with ``--dense-dtype bf16`` against it with ``fp8``.  One arena serves every mode, so once the
  fp8 weights exist every mode's optimizer step also refreshes them (one launch either way);
* the relative difference of the dropout-free forward loss at the initial weights (``train.probe_loss``) and of the
  same forward's logits (norm of the difference over the norm);
* the card's name, power limit and maximum SM clock, read in the same run.

    python tools/bench_dense_dtype.py [--rounds 5] [--steps 20] [--shape reddit] > result.json
"""
import argparse
import contextlib
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    f = [s.strip() for s in q.stdout.splitlines()[0].split(",")] if q.returncode == 0 and q.stdout else []
    return {"name": f[0] if f else torch.cuda.get_device_name(0), "power_limit": f[1] if len(f) > 1 else "not read",
            "sm_max_clock": f[2] if len(f) > 2 else "not read"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shape", default="reddit")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20, help="replays per mode and round")
    ap.add_argument("--profile-epochs", type=int, default=3)
    a = ap.parse_args()
    import bench
    from bns_gcn_b200 import train
    from bns_gcn_b200.module import dense

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    torch.cuda.set_stream(torch.cuda.Stream(dev))
    torch.autograd.set_multithreading_enabled(False)
    part, gstats = bench.build_partition(a.shape, 1, 0, dev)
    args = bench.make_args(1, "nccl", {"n_feat": part.meta["n_feat"], "n_class": part.meta["n_class"],
                                       "n_train": part.meta["n_train"], "dataset": a.shape, "dense_dtype": "bf16",
                                       "agg_dtype": "bf16"})
    with contextlib.redirect_stdout(sys.stderr):
        st = train.setup(part.graph, part.node_dict, part.gpb, args, dev)
    assert st.arena is not None

    from bns_gcn_b200 import fused, ops
    modes = ("f32", "bf16", "fp8")

    def set_mode(dense_mode: str, agg_mode: str = "f32"):
        st.arena.dense_bf16, st.arena.dense_fp8 = dense_mode == "bf16", dense_mode == "fp8"
        st.part.agg_bf16, st.part.agg_fp8 = agg_mode == "bf16", agg_mode == "fp8"

    # ---- forward loss at the initial weights, dropout off ----
    loss, logits = {}, {}
    for m in modes:
        set_mode(m)
        loss[m] = float(train.probe_loss(st, 0).item())
        keep, st.model.dropout.p = st.model.dropout.p, 0.0
        with torch.no_grad():
            logits[m] = train._forward_logits(st, 0).double()
        st.model.dropout.p = keep
        st.epoch_dev.sub_(1)
    logits_rel = {m: float((logits[m] - logits["f32"]).norm() / logits["f32"].norm()) for m in modes[1:]}
    del logits

    # ---- per-GEMM times (eager epochs), call sites in launch order ----
    sites, quant = [], []
    plain = dense.tc_mm_tn, dense.tc_mm_nt, dense.tc_mm_tn_fp8
    plain_q = ops.cvt_rows_fp8_any, fused.dropout_fp8

    def tn(a_, b_, *args_, **kw):
        sites.append(f"TN M={a_.shape[0]} K={a_.shape[1]} N={b_.shape[0]}")
        return plain[0](a_, b_, *args_, **kw)

    def nt(a_, b_, *args_, **kw):
        sites.append(f"NT R={a_.shape[0]} N1={a_.shape[1]} N2={b_.shape[1]}")
        return plain[1](a_, b_, *args_, **kw)

    def tn_fp8(a_, b_, *args_, **kw):
        sites.append(f"TN M={a_.shape[0]} K={a_.shape[1]} N={b_.shape[0]}")
        return plain[2](a_, b_, *args_, **kw)

    def timed(name, fn):
        def run(x, *args_, **kw):
            if dense.PROFILE is None:
                return fn(x, *args_, **kw)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out_ = fn(x, *args_, **kw)
            e1.record()
            quant.append((f"{name} {x.shape[0]} x {x.shape[1]}", e0, e1))
            return out_
        return run
    dense.tc_mm_tn, dense.tc_mm_nt, dense.tc_mm_tn_fp8 = tn, nt, tn_fp8
    ops.cvt_rows_fp8_any = timed("cvt_rows_fp8_any", plain_q[0])
    fused.dropout_fp8 = timed("dropout_fp8", plain_q[1])
    epoch = 0
    gemm, qpass = {}, {}
    try:
        for m in modes + modes:
            set_mode(m)
            train.train_epoch(st, epoch)                             # warm the mode's shapes
            epoch += 1
            torch.cuda.synchronize()
            dense.PROFILE, sites[:], quant[:] = [], [], []
            for _ in range(a.profile_epochs):
                train.train_epoch(st, epoch)
                epoch += 1
            torch.cuda.synchronize()
            prof, dense.PROFILE = dense.PROFILE, None
            ms = [e0.elapsed_time(e1) for (e0, e1, _, _) in prof]
            n = len(ms) // a.profile_epochs
            d = gemm.setdefault(m, {"ms": [], "sites": sites[:n], "flops": [p[2] for p in prof[:n]]})
            d["ms"].append([statistics.mean(ms[i::n]) for i in range(n)])
            if m == "fp8":
                nq = len(quant) // a.profile_epochs
                q = qpass.setdefault("sites", [s_ for s_, _, _ in quant[:nq]])
                qpass.setdefault("ms", []).append(
                    [statistics.mean(e0.elapsed_time(e1) for _, e0, e1 in quant[i::nq]) for i in range(len(q))])
    finally:
        dense.tc_mm_tn, dense.tc_mm_nt, dense.tc_mm_tn_fp8 = plain
        ops.cvt_rows_fp8_any, fused.dropout_fp8 = plain_q
    per_call = {m: [statistics.mean(x) for x in zip(*d["ms"])] for m, d in gemm.items()}
    calls = [{"site": s, "gflop": f / 1e9, "f32_ms": x, "bf16_ms": y, "fp8_ms": z, "bf16_over_fp8": y / z}
             for s, f, x, y, z in zip(gemm["f32"]["sites"], gemm["f32"]["flops"], per_call["f32"], per_call["bf16"],
                                      per_call["fp8"])]
    assert all(gemm[m]["sites"] == gemm["f32"]["sites"] for m in modes), "the modes' GEMM call sites differ"
    quant_ms = [statistics.mean(x) for x in zip(*qpass["ms"])]
    quant_calls = [{"site": s, "ms": t} for s, t in zip(qpass["sites"], quant_ms)]

    # ---- epochs/s of graph replays, modes alternating, one pairing at a time ----
    def pairing(modes):
        graphs = {}
        for name, (dm, am) in modes.items():
            set_mode(dm, am)
            graphs[name] = train.GraphedEpoch(st, warmup=1)
            for _ in range(2):
                graphs[name]()
        torch.cuda.synchronize()
        rates = {name: [] for name in modes}
        for _ in range(a.rounds):
            for name in modes:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                e0.record()
                for _ in range(a.steps):
                    graphs[name]()
                e1.record()
                torch.cuda.synchronize()
                rates[name].append(1000.0 * a.steps / e0.elapsed_time(e1))
        del graphs
        torch.cuda.empty_cache()
        names = list(modes)
        return {"epochs_per_s": {k: {"median": statistics.median(v), "all": v} for k, v in rates.items()},
                "speedup": statistics.median(rates[names[1]]) / statistics.median(rates[names[0]])}

    out = {
        "workload": f"{a.shape}: {gstats['n_nodes']} nodes, {gstats['n_edges']} edges, 3-layer GraphSAGE, hidden 256, "
                    "--use-pp, 1 partition",
        "card": card(),
        "gemm_calls": calls,
        "fp8_quantization_passes": quant_calls,
        "dense_ms_per_epoch": {m: sum(v) for m, v in per_call.items()},
        "dense_ms_per_epoch_fp8_with_quantization": sum(per_call["fp8"]) + sum(quant_ms),
        "graphed_f32_vs_dense_bf16": pairing({"f32": ("f32", "f32"), "dense_bf16": ("bf16", "f32")}),
        "graphed_agg_bf16_vs_agg_dense_bf16": pairing({"agg_bf16": ("f32", "bf16"), "agg_dense_bf16": ("bf16", "bf16")}),
        "graphed_dense_bf16_vs_dense_fp8": pairing({"dense_bf16": ("bf16", "f32"), "dense_fp8": ("fp8", "f32")}),
        "graphed_agg_fp8_dense_bf16_vs_dense_fp8": pairing({"agg_fp8_dense_bf16": ("bf16", "fp8"),
                                                             "agg_fp8_dense_fp8": ("fp8", "fp8")}),
        "probe_loss": loss,
        "probe_loss_rel_diff": {m: abs(loss[m] - loss["f32"]) / abs(loss["f32"]) for m in modes[1:]},
        "probe_logits_rel_diff_norm": logits_rel,
    }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
