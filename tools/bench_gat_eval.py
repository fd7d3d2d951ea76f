"""GAT evaluation forward on the whole graph (the homogeneous call of GATConv on bns_gat_infer_f32): time of the
model's forward, of the attention kernel of each layer alone and of that kernel on the graph's longest row alone (the
tail: one warp walks one row), with CUDA events after a warm-up, and the peak
device memory the forward adds on top of the graph, features and weights.  Prints one JSON line per case.

  python tools/bench_gat_eval.py --shape yelp --layers 2 --hidden 256 --heads 1
  python tools/bench_gat_eval.py --shape reddit --layers 3 --hidden 256 --heads 4 [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bns_gcn_b200  # noqa: E402,F401
from bns_gcn_b200 import ops  # noqa: E402
from bns_gcn_b200.data import make_graph  # noqa: E402
from bns_gcn_b200.graph import FullGraphHandle, GatProjection, gat_infer, gat_padded_width  # noqa: E402
from bns_gcn_b200.module import dense  # noqa: E402
from bns_gcn_b200.module.model import GAT  # noqa: E402


def timed(fn, warmup, iters):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    ts.sort()
    return ts[len(ts) // 2], ts[0]


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = (s.strip() for s in out.split(","))
    except Exception:                       # noqa: BLE001 - the device name from the library is still reported
        name, power = ops.device_info()["name"], "unknown"
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shape", default="yelp")
    ap.add_argument("--layers", type=int, default=2)
    ap.add_argument("--hidden", type=int, default=256)
    ap.add_argument("--heads", type=int, default=1)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--out", default=None, help="directory to append the JSON line to (gat_eval.jsonl)")
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    fg = make_graph(a.shape, seed=0, device=dev)
    g = FullGraphHandle(ops.DeviceGraph.from_csr(fg.indptr.to(dev), fg.src.to(torch.int32).to(dev), fg.n_nodes),
                        fg.in_degrees().to(dev), fg.out_degrees().to(dev))
    feat = fg.feat.to(dev)
    deg = (fg.indptr[1:] - fg.indptr[:-1]).cpu()
    r_max = int(deg.argmax())
    layer_size = [fg.n_feat] + [a.hidden] * (a.layers - 1) + [fg.n_class]
    torch.manual_seed(0)
    net = GAT(layer_size, F.relu, use_pp=True, heads=a.heads, dropout=0.5, norm="layer").to(dev).eval()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated(dev)
    torch.cuda.reset_peak_memory_stats(dev)
    with torch.no_grad():
        logits = net(g, feat)
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated(dev)
        fwd_med, fwd_min = timed(lambda: net(g, feat), a.warmup, a.iters)
        # the attention kernel of every layer on its own (inputs of the right widths, random values)
        kern = []
        for i, layer in enumerate(net.layers):
            H, Fo = layer._num_heads, layer._out_feats
            Fp = gat_padded_width(Fo)
            ft = torch.randn(fg.n_nodes, H * Fp, device=dev)
            el, er = GatProjection.apply(ft, ft, torch.randn(1, H, Fp, device=dev), torch.randn(1, H, Fp, device=dev), H, Fp)
            med, mn = timed(lambda: gat_infer(g.a, ft, el, er, H, Fp, 0.2), a.warmup, a.iters)
            # the tail: one warp walks a row, so no launch is shorter than the longest row alone
            one = ops.DeviceGraph.from_csr(torch.tensor([0, int(deg[r_max])], dtype=torch.int64, device=dev),
                                           fg.src[int(fg.indptr[r_max]):int(fg.indptr[r_max + 1])].to(torch.int32).to(dev),
                                           fg.n_nodes)
            er1 = er[r_max:r_max + 1].contiguous()
            med1, _ = timed(lambda: gat_infer(one, ft, el, er1, H, Fp, 0.2), a.warmup, a.iters)
            kern.append({"layer": i, "heads": H, "out_feats": Fo, "padded_width": Fp, "ms_median": round(med, 3),
                         "ms_min": round(mn, 3),
                         "gathered_GB_per_s": round(4.0 * g.a.nnz * H * Fp / (med * 1e-3) / 1e9, 1),
                         "longest_row_alone_ms": round(med1, 3)})
            del ft, el, er, one
    name, power = gpu_info()
    rec = {"shape": a.shape, "n_nodes": fg.n_nodes, "nnz": g.a.nnz, "max_in_degree": int(deg.max()),
           "mean_in_degree": round(float(deg.double().mean()), 1), "layers": a.layers, "hidden": a.hidden,
           "heads": a.heads, "forward_ms_median": round(fwd_med, 3), "forward_ms_min": round(fwd_min, 3),
           "peak_mem_GB": round(peak / 2 ** 30, 3), "forward_extra_mem_GB": round((peak - base) / 2 ** 30, 3),
           "resident_mem_GB": round(base / 2 ** 30, 3), "attention_kernel": kern,
           "logits_finite": bool(torch.isfinite(logits).all()), "gpu": name, "power_limit": power,
           "dense_mode": dense.MODE}
    line = json.dumps(rec)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "gat_eval.jsonl"), "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
