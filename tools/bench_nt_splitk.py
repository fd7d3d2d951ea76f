"""Time the weight-gradient GEMM ``bns_dense_nt_3xtf32`` (dW = dY^T X, split-K over the rows, slices summed by
``splitk_reduce_kernel``) at the Reddit and papers100M per-rank shapes, and split its time between the GEMM and the
reduce with torch.profiler.

  python tools/bench_nt_splitk.py [--lib PATH] [--save DIR] [--against DIR] [--iters N]

``--lib`` times another build of libbnsgcn.so (e.g. of an earlier commit); run the builds alternately, one process each
(two builds do not share a process).  ``--save`` writes each shape's dW (same seeded operands every run), ``--against``
compares this run's dW bit for bit with one saved before.  Prints one JSON line per shape with the GPU's name and power
limit."""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPES = [  # (label, R, N1, N2)
    ("reddit layer-0 dW", 232_965, 256, 1204),
    ("reddit hidden dW", 232_965, 256, 256),
    ("reddit class dW", 232_965, 44, 256),
    ("reddit/8 layer-0 dW", 29_121, 256, 1204),
    ("papers100m/8 hidden dW", 111_059_956 // 8, 256, 256),
    ("papers100m/8 class dW", 111_059_956 // 8, 44, 256),
]


def load(path):
    lib = ctypes.CDLL(path)
    lib.bns_dense_nt_workspace_bytes.restype = ctypes.c_size_t
    lib.bns_dense_nt_workspace_bytes.argtypes = [ctypes.c_int64] * 3
    lib.bns_last_error.restype = ctypes.c_char_p
    lib.bns_dense_nt_3xtf32.restype = ctypes.c_int
    lib.bns_dense_nt_3xtf32.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p,
                                        ctypes.c_int64, ctypes.c_int64, ctypes.c_int64, ctypes.c_int64, ctypes.c_void_p,
                                        ctypes.c_size_t, ctypes.c_void_p]
    return lib


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = torch.cuda.get_device_name(0)
    return out


def run(lib, a, b, out, ws):
    R, N1 = a.shape
    N2 = b.shape[1]
    need = lib.bns_dense_nt_workspace_bytes(R, N1, N2)
    rc = lib.bns_dense_nt_3xtf32(a.data_ptr(), a.stride(0), b.data_ptr(), b.stride(0), out.data_ptr(), out.stride(0),
                                 R, N1, N2, ws.data_ptr() if need else None, need, torch.cuda.current_stream().cuda_stream)
    if rc != 0:
        raise RuntimeError(f"bns_dense_nt_3xtf32 failed ({rc}): {lib.bns_last_error().decode()}")


def time_ms(lib, a, b, out, ws, iters):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(iters):
        run(lib, a, b, out, ws)
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / iters


def split_ms(lib, a, b, out, ws, iters):
    """(gemm, reduce) device ms per call from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            run(lib, a, b, out, ws)
        torch.cuda.synchronize()
    gemm = red = 0.0
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if "gemm3x_kernel" in e.key:
            gemm += t
        elif "splitk_reduce_kernel" in e.key:
            red += t
    return gemm / iters / 1e3, red / iters / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=os.path.join(ROOT, "bns-gcn_b200", "csrc", "libbnsgcn.so"))
    ap.add_argument("--save", default=None)
    ap.add_argument("--against", default=None)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a GPU")
    lib = load(args.lib)
    gpu = gpu_info()
    g = torch.Generator(device="cuda").manual_seed(0)
    if args.save:
        os.makedirs(args.save, exist_ok=True)
    for label, R, N1, N2 in SHAPES:
        a = torch.rand(R, N1, generator=g, device="cuda")
        b = torch.rand(R, N2, generator=g, device="cuda")
        need = lib.bns_dense_nt_workspace_bytes(R, N1, N2)
        ws = torch.empty(max(need, 16), dtype=torch.uint8, device="cuda")
        out = torch.empty(N1, N2, device="cuda")
        run(lib, a, b, out, ws)                                           # warm-up; the result compared below
        torch.cuda.synchronize()
        first = out.clone()
        ms = [time_ms(lib, a, b, out, ws, args.iters) for _ in range(args.rounds)]
        gemm, red = split_ms(lib, a, b, out, ws, args.iters)
        rec = {"shape": label, "R": R, "N1": N1, "N2": N2, "lib": args.lib, "slices": max(1, need // (4 * N1 * N2)),
               "workspace_mb": round(need / 2 ** 20, 1), "ms_per_call": [round(x, 4) for x in ms],
               "gemm_ms": round(gemm, 4), "reduce_ms": round(red, 4), "gpu": gpu}
        name = f"{R}_{N1}_{N2}.pt"
        if args.save:
            torch.save(first.cpu(), os.path.join(args.save, name))
        if args.against:
            rec["bit_identical_to_saved"] = bool(torch.equal(first.cpu().view(torch.int32),
                                                             torch.load(os.path.join(args.against, name)).view(torch.int32)))
        print(json.dumps(rec), flush=True)
        del a, b, ws, out, first
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
