"""Independent L2 / HBM bandwidth probes (csrc/microbench.cu -> libbnsmicro.so): the ceilings the SpMM's gather rate is
compared with.  No code shared with spmm_kernel.

    python tools/l2_microbench.py [--out FILE.md]
"""
import argparse
import ctypes
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "bns-gcn_b200", "csrc", "libbnsmicro.so")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    lib = ctypes.CDLL(LIB)
    lib.bnsm_stream_read.restype = ctypes.c_double
    lib.bnsm_stream_read.argtypes = [ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_int]
    lib.bnsm_row_gather.restype = ctypes.c_double
    lib.bnsm_row_gather.argtypes = [ctypes.c_int64, ctypes.c_int, ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_int]
    import torch
    gpu = torch.cuda.get_device_name(0)
    lines = [f"# L2 / HBM microbenchmarks ({gpu}, CUDA events, best of 5 launches after 2 warm-up launches)", "",
             "## Streaming 16-byte reads (`ld.global.nc.L1::no_allocate.v4`), whole grid, 8 loads in flight per thread", "",
             "| buffer | passes per launch | CTAs/SM | GB/s |", "|---:|---:|---:|---:|"]
    for mb, reps in ((16, 64), (32, 32), (64, 16), (96, 12), (119, 8), (256, 4), (1024, 2), (4096, 1)):
        for bps in (4, 8):
            v = lib.bnsm_stream_read(mb << 20, reps, bps, 5)
            lines.append(f"| {mb} MB | {reps} | {bps} | {v:,.0f} |")
    lines += ["", "## Random whole-row gathers (one coalesced 512-byte request per warp instruction; ids from an in-register LCG)", "",
              "| table | row bytes | loads in flight / lane | CTAs/SM | GB/s of gathered rows | rows/s (G) |",
              "|---:|---:|---:|---:|---:|---:|"]
    for n_rows, rb in ((50_000, 1024), (100_000, 512), (232_965, 512), (232_965, 1024), (116_000, 1024),
                       (2_449_029, 512)):
        for unroll in ((4, 8) if rb == 512 else (2, 4)):
            for bps in (4, 6):
                v = lib.bnsm_row_gather(n_rows, rb, 40_000_000 if rb == 512 else 20_000_000, bps, unroll, 5)
                lines.append(f"| {n_rows * rb / 2**20:,.0f} MB ({n_rows:,} rows) | {rb} | {unroll * (rb // 512)} | {bps} | {v:,.0f} | "
                             f"{v / rb:,.2f} |")
    text = "\n".join(lines) + "\n"
    print(text)
    if a.out:
        with open(os.path.join(ROOT, a.out) if not os.path.isabs(a.out) else a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    sys.exit(main())
