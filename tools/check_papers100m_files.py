"""Measure the ogbn-papers100M partition step (``store.papers100m_partition``) and a training run on its store.

1. Writes the generated papers100M shape (``make_local_partition`` at ``--scale``, generated in ``--gen-parts`` pieces
   on the GPU) in OGB's raw layout, streaming: ``data.npz`` (``edge_index`` [2, E], ``node_feat`` [N, 128],
   ``num_nodes_list``), ``node-label.npz`` (NaN outside the three splits) and ``split/time/*.csv.gz``.  No array
   that grows with E or N x F is held whole.
2. Runs the partition step at every ``--parts``, reporting for each: wall time per phase (node tables, edge pass,
   parts, features), bytes read, peak host RSS (sampled every 20 ms) and peak device memory.
3. Trains ``main.py`` at P = 1 on the P = 1 store (of a ``--train-scale`` layout if given) with ``--parallel-eval
   --cuda-graph`` for ``--epochs`` epochs and reports the ``Time(s)`` of the last logged line (the mean over the epochs
   after the fifth).

    python tools/check_papers100m_files.py --scale 0.1 --parts 1,2,4,8 --train-scale 0.05 --out results/papers100m

Needs a GPU.  Every file goes to a temporary directory (``--tmp``), removed at the end.  One JSON line per
measurement is printed, and with ``--out`` appended to ``<out>/papers100m_files.jsonl``.
"""
from __future__ import annotations

import argparse
import gzip
import json
import os
import shutil
import subprocess
import sys
import tempfile
import threading
import time
import zipfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _npy_member(z: zipfile.ZipFile, key: str, dtype, shape, pieces) -> None:
    """One stored ``.npy`` member written from ``pieces`` (arrays in C order), header first."""
    with z.open(key + ".npy", "w", force_zip64=True) as f:
        np.lib.format.write_array_header_1_0(f, {"descr": np.lib.format.dtype_to_descr(np.dtype(dtype)),
                                                 "fortran_order": False, "shape": tuple(shape)})
        for a in pieces:
            f.write(np.ascontiguousarray(a, dtype=dtype).tobytes())


def write_generated_layout(root: str, scale: float, gen_parts: int, device, seed: int = 0) -> dict:
    """The generated papers100M shape in OGB's raw layout under ``root``; returns its counts."""
    from bns_gcn_b200.data import make_local_partition

    def pieces():
        for r in range(gen_parts):
            yield make_local_partition("papers100m", r, gen_parts, seed=seed, device=device, scale=scale)

    n_edges, n = 0, None
    for p in pieces():                                         # the edge count goes in the header, before the edges
        n_edges += p.graph.num_edges()
        n = int(p.gpb.ranges[-1])
    raw = os.path.join(root, "ogbn_papers100M", "raw")
    split = os.path.join(root, "ogbn_papers100M", "split", "time")
    os.makedirs(raw, exist_ok=True)
    os.makedirs(split, exist_ok=True)

    def ends(which):
        for p in pieces():
            g, gid = p.graph, p.node_dict["_ID"]
            if which == 0:
                yield gid[g.indices].cpu().numpy()
            else:
                start = int(p.gpb.ranges[p.rank])
                rows = torch.arange(start, start + g.n_in, dtype=torch.int64, device=g.indptr.device)
                yield torch.repeat_interleave(rows, g.indptr[1:] - g.indptr[:-1]).cpu().numpy()

    labels, masks = [], {"train": [], "valid": [], "test": []}
    with zipfile.ZipFile(os.path.join(raw, "data.npz"), "w") as z:
        _npy_member(z, "edge_index", np.int64, (2, n_edges), (a for w in (0, 1) for a in ends(w)))

        def feat_pieces():
            for p in pieces():
                nd = p.node_dict
                start = int(p.gpb.ranges[p.rank])
                lab = nd["label"].float().cpu().numpy()
                some = (nd["train_mask"] | nd["val_mask"] | nd["test_mask"]).cpu().numpy()
                lab[~some] = np.nan
                labels.append(lab)
                for k, m in (("train", "train_mask"), ("valid", "val_mask"), ("test", "test_mask")):
                    masks[k].append(start + np.nonzero(nd[m].cpu().numpy())[0])
                yield nd["feat"].cpu().numpy()
        _npy_member(z, "node_feat", np.float32, (n, 128), feat_pieces())
        _npy_member(z, "num_nodes_list", np.int64, (1,), [np.array([n])])
    np.savez(os.path.join(raw, "node-label.npz"), node_label=np.concatenate(labels).reshape(-1, 1))
    for k, ids in masks.items():
        with gzip.open(os.path.join(split, f"{k}.csv.gz"), "wt", compresslevel=1) as f:
            for a in ids:
                f.write("".join(f"{int(i)}\n" for i in a))
    return {"n": n, "e": n_edges}


class _RssSampler:
    """Peak resident set size of this process, sampled from ``/proc/self/statm``."""

    def __init__(self, every: float = 0.02):
        self.every, self.peak, self._stop = every, 0, threading.Event()
        self._page = os.sysconf("SC_PAGE_SIZE")
        self._t = threading.Thread(target=self._run, daemon=True)

    def _rss(self) -> int:
        with open("/proc/self/statm") as f:
            return int(f.read().split()[1]) * self._page

    def _run(self):
        while not self._stop.is_set():
            self.peak = max(self.peak, self._rss())
            self._stop.wait(self.every)

    def __enter__(self):
        self.peak = self._rss()
        self._t.start()
        return self

    def __exit__(self, *exc):
        self._stop.set()
        self._t.join()
        self.peak = max(self.peak, self._rss())


def measure_partition(data_path: str, part_path: str, n_parts: int, device, chunk: int) -> dict:
    """Run the streaming step once, timing its phases through wrappers around the module's own functions."""
    from bns_gcn_b200.data import store
    phase = {"edge_pass": 0.0, "parts": 0.0, "features": 0.0}

    def timed(name, fn):
        def wrapper(*a, **k):
            torch.cuda.synchronize(device)
            t = time.perf_counter()
            out = fn(*a, **k)
            torch.cuda.synchronize(device)
            phase[name] += time.perf_counter() - t
            return out
        return wrapper
    saved = store._spill_edges, store._streamed_part, store._stream_features
    store._spill_edges = timed("edge_pass", saved[0])
    store._streamed_part = timed("parts", saved[1])
    store._stream_features = timed("features", saved[2])
    args = argparse.Namespace(dataset="ogbn-papers100m", data_source="files", data_path=data_path, part_path=part_path,
                              graph_name="", n_partitions=n_parts, partition_method="random", inductive=False,
                              eval=False, graph_seed=0)
    try:
        torch.cuda.reset_peak_memory_stats(device)
        with _RssSampler() as rss:
            t = time.perf_counter()
            store.papers100m_partition(args, device, chunk=chunk)
            total = time.perf_counter() - t
    finally:
        store._spill_edges, store._streamed_part, store._stream_features = saved
    read = sum(os.path.getsize(os.path.join(d, f)) for d, _, fs in os.walk(os.path.join(data_path, "ogbn_papers100M"))
               for f in fs)
    phase = {k: round(v, 2) for k, v in phase.items()}
    phase["node_tables"] = round(total - sum(phase.values()), 2)
    return {"what": "partition", "P": n_parts, "total_s": round(total, 2), "phase_s": phase, "bytes_read": read,
            "peak_rss_gb": round(rss.peak / 2 ** 30, 2),
            "peak_device_gb": round(torch.cuda.max_memory_allocated(device) / 2 ** 30, 2),
            "graph_name": args.graph_name}


def measure_training(data_path: str, part_path: str, epochs: int, hidden: int, cwd: str) -> dict:
    argv = [sys.executable, "-m", "bns_gcn_b200.main", "--dataset", "ogbn-papers100m", "--data-source", "files",
            "--data-path", data_path, "--part-path", part_path, "--n-partitions", "1", "--partition-method", "random",
            "--model", "graphsage", "--n-layers", "3", "--n-hidden", str(hidden), "--sampling-rate", "0.1", "--use-pp",
            "--parallel-eval", "--cuda-graph", "--n-epochs", str(epochs), "--log-every", str(epochs), "--fix-seed",
            "--skip-partition"]
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    t = time.perf_counter()
    p = subprocess.run(argv, cwd=cwd, env=env, capture_output=True, text=True)
    wall = time.perf_counter() - t
    lines = [ln for ln in p.stdout.splitlines() if "| Time(s)" in ln]
    if p.returncode != 0 or not lines:                      # a rank that fails does not fail the launcher
        return {"what": "train", "P": 1, "failed": p.returncode, "stdout": p.stdout[-3000:], "stderr": p.stderr[-3000:]}
    return {"what": "train", "P": 1, "epochs": epochs, "n_hidden": hidden, "log_line": lines[-1],
            "time_s": float(lines[-1].split("Time(s) ")[1].split()[0]),
            "result_lines": [ln for ln in p.stdout.splitlines() if "Accuracy" in ln], "wall_s": round(wall, 1)}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--scale", type=float, default=0.1)
    ap.add_argument("--parts", default="1,2,4,8")
    ap.add_argument("--gen-parts", type=int, default=8, help="pieces the layout is generated in")
    ap.add_argument("--chunk", type=int, default=None, help="edges / feature rows per step (default: the module's)")
    ap.add_argument("--epochs", type=int, default=10, help="Time(s) averages the epochs after the fifth")
    ap.add_argument("--hidden", type=int, default=128, help="GraphSAGE hidden width of the training run")
    ap.add_argument("--train-scale", type=float, default=None,
                    help="train on a layout of this scale instead of --scale's (at --scale 0.1, P = 1 does not fit "
                         "one 80 GB GPU)")
    ap.add_argument("--tmp", default=None, help="directory for the layout and the stores (default: the system's)")
    ap.add_argument("--out", default=None, help="directory to append the JSON lines to (papers100m_files.jsonl)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU: the partition step's device side and the training run are what is measured")
    import bns_gcn_b200  # noqa: F401
    from bns_gcn_b200.data import store
    dev = torch.device("cuda:0")
    if a.out:
        os.makedirs(a.out, exist_ok=True)

    def emit(rec):
        print(json.dumps(rec), flush=True)
        if a.out:
            with open(os.path.join(a.out, "papers100m_files.jsonl"), "a") as f:
                f.write(json.dumps(rec) + "\n")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    emit({"what": "machine", "gpu": q.stdout.strip(), "cpus": os.cpu_count(),
          "host_mem_gb": round(os.sysconf("SC_PAGE_SIZE") * os.sysconf("SC_PHYS_PAGES") / 2 ** 30, 1)})
    tmp = tempfile.mkdtemp(prefix="papers100m-", dir=a.tmp)
    try:
        emit({"what": "disk", "free_gb": round(shutil.disk_usage(tmp).free / 2 ** 30, 1)})
        data = os.path.join(tmp, "data")
        t = time.perf_counter()
        counts = write_generated_layout(data, a.scale, a.gen_parts, dev)
        emit({"what": "layout", "scale": a.scale, **counts, "write_s": round(time.perf_counter() - t, 1),
              "bytes": sum(os.path.getsize(os.path.join(d, f)) for d, _, fs in os.walk(data) for f in fs)})
        chunk = a.chunk or store.PAPERS_CHUNK
        for p in [int(x) for x in a.parts.split(",") if x]:
            part_path = os.path.join(tmp, f"part{p}")
            rec = measure_partition(data, part_path, p, dev, chunk)
            emit({**rec, "chunk": chunk})
            if p == 1 and a.train_scale is None:
                emit(measure_training(data, part_path, a.epochs, a.hidden, tmp))
            shutil.rmtree(part_path)
        if a.train_scale is not None:                      # a layout of its own, small enough for one GPU at P = 1
            shutil.rmtree(data)
            counts = write_generated_layout(data, a.train_scale, a.gen_parts, dev)
            emit({"what": "layout", "scale": a.train_scale, **counts})
            part_path = os.path.join(tmp, "part1")
            emit({**measure_partition(data, part_path, 1, dev, chunk), "chunk": chunk})
            emit({**measure_training(data, part_path, a.epochs, a.hidden, tmp), "scale": a.train_scale})
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
