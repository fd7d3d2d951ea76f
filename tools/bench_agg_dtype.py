"""``--agg-dtype f32``, ``bf16`` and ``fp8`` on the benchmark's workload (BASELINE.json configs[1]: Reddit-shape graph,
3-layer GraphSAGE, hidden 256, --use-pp) at ONE partition, all modes in one process:

* epochs/s of ``train.GraphedEpoch`` replays, the modes' graphs replayed in alternating rounds;
* the mean per-launch time of every F = 256 aggregation pass (``ops.PROFILE``, eager epochs, modes alternating), by pass;
* the rounding cost: the time of the bf16 / fp8 conversion kernels per epoch (CUDA events around each call);
* the relative difference of the dropout-free forward loss at the initial weights (``train.probe_loss``, an f32 sum:
  differences under its last bit read as 0) and of the same forward's logits (norm of the difference over the norm);
* the card's name, power limit and maximum SM clock, read in the same run.

    python tools/bench_agg_dtype.py [--rounds 5] [--steps 20] [--profile-rounds 2] [--shape reddit] > result.json
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
    ap.add_argument("--profile-rounds", type=int, default=2, help="eager rounds per mode, modes alternating")
    a = ap.parse_args()
    import bench
    from bns_gcn_b200 import fused, ops, train

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    torch.cuda.set_stream(torch.cuda.Stream(dev))
    torch.autograd.set_multithreading_enabled(False)
    part, gstats = bench.build_partition(a.shape, 1, 0, dev)
    args = bench.make_args(1, "nccl", {"n_feat": part.meta["n_feat"], "n_class": part.meta["n_class"],
                                       "n_train": part.meta["n_train"], "dataset": a.shape, "agg_dtype": "fp8"})
    with contextlib.redirect_stdout(sys.stderr):
        st = train.setup(part.graph, part.node_dict, part.gpb, args, dev)
    g = st.part

    modes = ("f32", "bf16", "fp8")

    def set_mode(m: str):
        g.agg_bf16, g.agg_fp8 = m == "bf16", m == "fp8"

    # ---- forward loss at the initial weights, dropout off ----
    loss, logits = {}, {}
    for m in modes:
        set_mode(m)
        loss[m] = float(train.probe_loss(st, 0).item())
        keep, st.model.dropout.p = st.model.dropout.p, 0.0          # the same forward, its logits kept
        with torch.no_grad():
            logits[m] = train._forward_logits(st, 0).double()
        st.model.dropout.p = keep
        st.epoch_dev.sub_(1)
    logits_rel = {m: float((logits[m] - logits["f32"]).norm() / logits["f32"].norm()) for m in modes[1:]}
    del logits

    # ---- per-pass times (eager epochs) and the conversion kernels' time ----
    cvt_events = []
    plain_cvt = {n: getattr(ops, n) for n in ("cvt_rows_bf16", "cvt_rows_fp8")}

    def timed(fn):
        def call(src, out=None):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            r = fn(src, out)
            e1.record()
            cvt_events.append((e0, e1))
            return r
        return call
    for n, fn in plain_cvt.items():
        setattr(ops, n, timed(fn))
    epoch = 0
    passes = {}
    try:
        for m in modes * a.profile_rounds:
            set_mode(m)
            train.train_epoch(st, epoch)                             # warm the mode's shapes
            epoch += 1
            torch.cuda.synchronize()
            ops.PROFILE, cvt_events[:] = [], []
            for _ in range(a.profile_epochs):
                train.train_epoch(st, epoch)
                epoch += 1
            torch.cuda.synchronize()
            prof, ops.PROFILE = ops.PROFILE, None
            wide = [e0.elapsed_time(e1) for (e0, e1, _, nnz, F, _) in prof if F == 256]
            per_epoch = len(wide) // a.profile_epochs
            # launch order within an epoch: forward a_in (layer 1), backward a_in_t (layer 1)
            by_pass = [statistics.mean(wide[i::per_epoch]) for i in range(per_epoch)] if per_epoch else []
            d = passes.setdefault(m, {"pass_ms": [], "cvt_ms_per_epoch": []})
            d["pass_ms"].append(by_pass)
            d["cvt_ms_per_epoch"].append(sum(e0.elapsed_time(e1) for e0, e1 in cvt_events) / a.profile_epochs)
    finally:
        for n, fn in plain_cvt.items():
            setattr(ops, n, fn)

    # ---- epochs/s of graph replays, modes alternating ----
    graphs = {}
    for m in modes:
        set_mode(m)
        graphs[m] = train.GraphedEpoch(st, warmup=1)
        for _ in range(2):
            graphs[m]()
    torch.cuda.synchronize()
    rates = {m: [] for m in modes}
    for _ in range(a.rounds):
        for m in modes:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(a.steps):
                graphs[m]()
            e1.record()
            torch.cuda.synchronize()
            rates[m].append(1000.0 * a.steps / e0.elapsed_time(e1))

    pass_ms = {m: [statistics.mean(x) for x in zip(*d["pass_ms"])] for m, d in passes.items()}
    out = {
        "workload": f"{a.shape}: {gstats['n_nodes']} nodes, {gstats['n_edges']} edges, 3-layer GraphSAGE, hidden 256, "
                    "--use-pp, 1 partition",
        "card": card(),
        "epochs_per_s": {m: {"median": statistics.median(v), "all": v} for m, v in rates.items()},
        "speedup_epochs_per_s": {m: statistics.median(rates[m]) / statistics.median(rates["f32"]) for m in modes[1:]},
        "speedup_epochs_per_s_fp8_vs_bf16": statistics.median(rates["fp8"]) / statistics.median(rates["bf16"]),
        "f256_pass_ms": pass_ms,
        "f256_pass_ms_all_rounds": {m: d["pass_ms"] for m, d in passes.items()},
        "f256_pass_order": ["forward A_in h (layer 1)", "backward A_in^T dys (layer 1)"],
        "f256_pass_speedup_fp8_vs_bf16": [b / f for b, f in zip(pass_ms["bf16"], pass_ms["fp8"])],
        "cvt_ms_per_epoch": {m: statistics.mean(d["cvt_ms_per_epoch"]) for m, d in passes.items()},
        "probe_loss": loss,
        "probe_loss_rel_diff": {m: abs(loss[m] - loss["f32"]) / abs(loss["f32"]) for m in modes[1:]},
        "probe_logits_rel_diff_norm": logits_rel,
    }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
