"""Bring-up / diagnosis of the wgmma dense kernels (csrc/dense_tc.cuh).

  python tools/check_dense_tc.py tn     structured + random checks of bns_dense_tn_3xtf32
  python tools/check_dense_tc.py nt     structured + random checks of bns_dense_nt_3xtf32
  python tools/check_dense_tc.py perf   timings on the Reddit-shape layer GEMMs vs cuBLAS fp32 / tf32

Structured inputs (one-hot A, integer-coded B) make a wrong shared-memory descriptor readable: every output
value names the B element it was computed from.
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bns_gcn_b200  # noqa: F401,E402
from bns_gcn_b200.module import dense  # noqa: E402

dev = torch.device("cuda:0")


WORST = [0.0]


def report(name, got, ref, tol=2e-5):
    got, ref = got.double().cpu(), ref.double().cpu()
    err = (got - ref).abs()
    scale = ref.abs().max().item() + 1e-30
    rel = err.max().item() / scale
    if not (rel == rel):
        rel = float("inf")
    WORST[0] = max(WORST[0], rel / tol)
    bad = ~(err <= tol * scale)
    print(f"[{name}] max|err|/max|ref| = {rel:.3e}   bad elements {int(bad.sum())}/{bad.numel()}", flush=True)
    if bad.any():
        rows = bad.any(1).nonzero().flatten()
        cols = bad.any(0).nonzero().flatten()
        print(f"    bad rows {len(rows)} (first {rows[:12].tolist()}), bad cols {len(cols)} (first {cols[:12].tolist()})")
        blk = torch.zeros((got.shape[0] + 31) // 32, (got.shape[1] + 31) // 32)
        for i in range(blk.shape[0]):
            for j in range(blk.shape[1]):
                blk[i, j] = err[32 * i:32 * i + 32, 32 * j:32 * j + 32].max() / scale
        print("    max rel err per 32x32 block (first 8x8 blocks):")
        for i in range(min(8, blk.shape[0])):
            print("     ", " ".join(f"{v:8.1e}" for v in blk[i, :8].tolist()))
    return rel


def structured_tn(M, N, K):
    a = torch.zeros(M, K, device=dev)
    a[torch.arange(M), torch.arange(M) % K] = 1.0
    b = (torch.arange(N, device=dev, dtype=torch.float32)[:, None] * 1000 + torch.arange(K, device=dev, dtype=torch.float32)[None, :])
    got = dense.tc_mm_tn(a, b)
    torch.cuda.synchronize()
    ref = a.double() @ b.double().t()
    rel = report(f"tn structured M={M} N={N} K={K}", got, ref, 1e-6)
    if rel > 1e-6:
        g = got.cpu()
        for (m, n) in [(0, 0), (1, 0), (0, 1), (5, 3), (8, 0), (9, 2), (33, 40), (64, 64), (127, 127)]:
            if m < M and n < N:
                v = g[m, n].item()
                print(f"    C[{m},{n}] = {v:.1f} -> B[n'={int(v) // 1000}, k'={int(v) % 1000}]   expected B[{n},{m % K}]")


def structured_nt(R, N1, N2):
    a = torch.zeros(R, N1, device=dev)
    a[torch.arange(N1) % R, torch.arange(N1)] = 1.0          # column m picks row m % R
    b = (torch.arange(R, device=dev, dtype=torch.float32)[:, None] * 1000 + torch.arange(N2, device=dev, dtype=torch.float32)[None, :])
    got = dense.tc_mm_nt(a, b)
    torch.cuda.synchronize()
    ref = a.double().t() @ b.double()
    rel = report(f"nt structured R={R} N1={N1} N2={N2}", got, ref, 1e-6)
    if rel > 1e-6:
        g = got.cpu()
        for (m, n) in [(0, 0), (1, 0), (0, 1), (5, 3), (8, 0), (9, 2), (33, 40), (64, 64), (127, 127)]:
            if m < N1 and n < N2:
                v = g[m, n].item()
                print(f"    C[{m},{n}] = {v:.1f} -> B[r'={int(v) // 1000}, n'={int(v) % 1000}]   expected B[{m % R},{n}]")


def random_tn(M, N, K, bias=True):
    g = torch.Generator(device="cpu").manual_seed(M * 7 + N * 3 + K)
    a = torch.randn(M, K, generator=g).to(dev)
    b = torch.randn(N, K, generator=g).to(dev)
    bi = torch.randn(N, generator=g).to(dev) if bias else None
    got = dense.tc_mm_tn(a, b, bi)
    torch.cuda.synchronize()
    ref = a.double() @ b.double().t() + (bi.double() if bias else 0)
    r3 = report(f"tn random M={M} N={N} K={K} bias={bias}", got, ref)
    f32 = (a @ b.t() + (bi if bias else 0))
    print(f"    (cuBLAS fp32 on the same inputs: {((f32.double() - ref).abs().max() / ref.abs().max()).item():.3e})")
    return r3


def random_nt(R, N1, N2):
    g = torch.Generator(device="cpu").manual_seed(R * 7 + N1 * 3 + N2)
    a = torch.randn(R, N1, generator=g).to(dev)
    b = torch.randn(R, N2, generator=g).to(dev)
    got = dense.tc_mm_nt(a, b)
    torch.cuda.synchronize()
    ref = a.double().t() @ b.double()
    r3 = report(f"nt random R={R} N1={N1} N2={N2}", got, ref)
    f32 = a.t() @ b
    print(f"    (cuBLAS fp32 on the same inputs: {((f32.double() - ref).abs().max() / ref.abs().max()).item():.3e})")
    return r3


def timeit(fn, it=10):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(it):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / it


def perf():
    M = 232965
    for (K, N) in [(1204, 256), (256, 256), (512, 256)]:
        x = torch.randn(M, K, device=dev)
        w = torch.randn(N, K, device=dev)
        dy = torch.randn(M, N, device=dev)
        wt = w.t().contiguous()
        gf = 2 * M * K * N / 1e9
        rows = []
        rows.append(("fwd  tc 3xtf32", timeit(lambda: dense.tc_mm_tn(x, w))))
        rows.append(("fwd  cuBLAS fp32", timeit(lambda: torch.mm(x, w.t()))))
        rows.append(("dX   tc 3xtf32", timeit(lambda: dense.tc_mm_tn(dy, wt))))
        rows.append(("dX   cuBLAS fp32", timeit(lambda: torch.mm(dy, w))))
        rows.append(("dW   tc 3xtf32", timeit(lambda: dense.tc_mm_nt(dy, x))))
        rows.append(("dW   cuBLAS fp32", timeit(lambda: torch.mm(dy.t(), x))))
        torch.backends.cuda.matmul.allow_tf32 = True
        rows.append(("fwd  cuBLAS 1xtf32", timeit(lambda: torch.mm(x, w.t()))))
        rows.append(("dW   cuBLAS 1xtf32", timeit(lambda: torch.mm(dy.t(), x))))
        torch.backends.cuda.matmul.allow_tf32 = False
        print(f"M={M} K={K} N={N}: {gf:.0f} GFLOP per GEMM")
        for k, v in rows:
            print(f"   {k:22s} {v:8.3f} ms   {gf / v:8.1f} TFLOP/s (f32-equivalent)", flush=True)
        del x, w, dy, wt


if __name__ == "__main__":
    what = sys.argv[1] if len(sys.argv) > 1 else "tn"
    print(torch.cuda.get_device_name(0), flush=True)
    if what == "tn":
        structured_tn(128, 128, 32)
        structured_tn(128, 128, 128)
        structured_tn(256, 256, 64)
        random_tn(128, 128, 32, bias=False)
        random_tn(128, 128, 320, bias=True)
        random_tn(300, 136, 100, bias=True)
        random_tn(1000, 256, 1204, bias=True)
        random_tn(4099, 44, 256, bias=False)
        random_tn(232965, 256, 1204, bias=True)
    elif what == "nt":
        structured_nt(32, 128, 128)
        structured_nt(128, 128, 128)
        structured_nt(512, 256, 256)
        random_nt(32, 128, 128)
        random_nt(1000, 136, 100)
        random_nt(5000, 256, 1204)
        random_nt(232965, 256, 256)
        random_nt(232965, 256, 1204)
    elif what == "perf":
        perf()
    print("worst error / tolerance:", WORST[0], flush=True)
    sys.exit(0 if WORST[0] <= 1.0 else 1)
