"""At-scale check of ``--data-source files``: write the Reddit, ogbn-products and Yelp shapes in their published layouts
(``tools/dataset_files.py``), read each back with ``load_files`` in a fresh process and compare it bit for bit with
the generator; report the write and load wall times, the loading process's peak host memory and the bytes on disk.
Then 5 epochs of ``main.py`` on the Reddit files and on the generated Reddit shape, whose losses must agree.

    python tools/check_dataset_files.py [--out RESULT.json] [--dir WORKDIR] [--epochs 5]

Needs a GPU (the edges are sorted on it) and about 3 GB of free disk under ``--dir`` (default: a temporary directory,
removed at the end).  Prints one line per layout, then the whole result as one JSON line, which ``--out`` also
writes to a file.
"""
import argparse
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

CASES = [("reddit", "reddit"), ("ogbn-products", "ogbn-products"), ("yelp", "yelp")]


def _rss_mb():
    """This process's resident set now, from ``/proc/self/statm`` (None where it cannot be read)."""
    try:
        with open("/proc/self/statm") as f:
            return int(f.read().split()[1]) * os.sysconf("SC_PAGE_SIZE") / 2 ** 20
    except (OSError, ValueError, IndexError):
        return None


class _PeakRss:
    """The largest resident set seen while the block runs, sampled every 5 ms.  (``ru_maxrss`` would not do: it
    carries the parent's peak across the fork and exec that started this process.)"""

    def __enter__(self):
        import threading
        self.peak, self._stop = _rss_mb(), threading.Event()

        def sample():
            while not self._stop.wait(0.005):
                now = _rss_mb()
                if now is not None and self.peak is not None:
                    self.peak = max(self.peak, now)
        self._t = threading.Thread(target=sample, daemon=True)
        self._t.start()
        return self

    def __exit__(self, *exc):
        self._stop.set()
        self._t.join()
        now = _rss_mb()
        if now is not None and self.peak is not None:
            self.peak = max(self.peak, now)


def _load(layout: str, root: str, shape: str) -> dict:
    """In its own process: time ``load_files`` and read its peak RSS, then compare with the generator."""
    import torch
    import bns_gcn_b200  # noqa: F401
    from bns_gcn_b200.data import load_files, make_graph
    torch.zeros(1, device="cuda")                                  # CUDA context outside the timed window
    base = _rss_mb()
    with _PeakRss() as rss:
        t0 = time.time()
        g = load_files(layout, root)
        torch.cuda.synchronize()
        load_s = time.time() - t0
    peak = rss.peak
    fg = make_graph(shape, seed=0)
    if layout == "yelp":
        from tools.dataset_files import standard_scaled
        fg = standard_scaled(fg)
    same = {k: bool(getattr(g, k).dtype == getattr(fg, k).dtype and torch.equal(getattr(g, k), getattr(fg, k)))
            for k in ("indptr", "src", "feat", "label", "train_mask", "val_mask", "test_mask")}
    same["n_class"] = g.n_class == fg.n_class
    mb = lambda x: None if x is None else round(x)      # noqa: E731
    return {"load_s": round(load_s, 2), "rss_before_load_mb": mb(base), "peak_rss_mb": mb(peak),
            "n_nodes": g.n_nodes, "n_edges": g.n_edges, "n_feat": g.n_feat, "bit_identical": all(same.values()),
            "fields": same}


def _du(path: str) -> int:
    return sum(os.path.getsize(os.path.join(d, f)) for d, _, fs in os.walk(path) for f in fs)


def _main_losses(cwd: str, extra, epochs: int):
    flags = ["--n-partitions", "1", "--partition-method", "random", "--model", "graphsage", "--n-layers", "3",
             "--n-hidden", "256", "--sampling-rate", "0.1", "--use-pp", "--n-epochs", str(epochs), "--log-every", "1",
             "--fix-seed", "--seed", "1", "--no-eval", "--part-path", os.path.join(cwd, "partition")]
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    t0 = time.time()
    p = subprocess.run([sys.executable, "-m", "bns_gcn_b200.main"] + flags + extra, cwd=cwd, env=env,
                       capture_output=True, text=True)
    if p.returncode != 0:
        raise RuntimeError(f"main.py {extra} failed:\n{p.stdout[-3000:]}\n{p.stderr[-3000:]}")
    return re.findall(r"Epoch (\d+) \|.*\| Loss (\S+)", p.stdout), round(time.time() - t0, 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the result, as indented JSON, to this file")
    ap.add_argument("--dir", default=None)
    ap.add_argument("--epochs", type=int, default=5)
    ap.add_argument("--load", nargs=3, metavar=("LAYOUT", "ROOT", "SHAPE"), help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.load:
        print(json.dumps(_load(*a.load)))
        return
    import torch
    import bns_gcn_b200  # noqa: F401
    from bns_gcn_b200.data import make_graph
    from tools.dataset_files import WRITERS
    assert torch.cuda.is_available(), "needs a GPU"
    work = a.dir or tempfile.mkdtemp(prefix="bns_files_")
    res = {"gpu": torch.cuda.get_device_name(0), "cpus": os.cpu_count(), "cases": {}}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True)
        res["power_limit_max_sm_clock"] = q.stdout.strip()
    except OSError:
        pass
    try:
        for shape, layout in CASES:
            root = os.path.join(work, layout)
            fg = make_graph(shape, seed=0)
            t0 = time.time()
            WRITERS[layout](fg, root)
            write_s = time.time() - t0
            del fg
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--load", layout, root, shape],
                               capture_output=True, text=True)
            if p.returncode != 0:
                raise RuntimeError(f"loading {layout} failed:\n{p.stdout[-3000:]}\n{p.stderr[-3000:]}")
            r = json.loads(p.stdout.strip().splitlines()[-1])
            r.update(write_s=round(write_s, 1), bytes_on_disk=_du(root))
            res["cases"][layout] = r
            print(layout, json.dumps(r), flush=True)
            if layout != "reddit":
                shutil.rmtree(root)
        runs = {}
        for name, extra in (("files", ["--dataset", "reddit", "--data-source", "files", "--data-path",
                                       os.path.join(work, "reddit")]),
                            ("synthetic", ["--dataset", "reddit"])):
            cwd = os.path.join(work, "run_" + name)
            os.makedirs(cwd)
            runs[name] = _main_losses(cwd, extra, a.epochs)
        res["main"] = {k: {"losses": v[0], "wall_s": v[1]} for k, v in runs.items()}
        res["main"]["same_losses"] = (runs["files"][0] == runs["synthetic"][0]
                                      and len(runs["files"][0]) == a.epochs)
    finally:
        if a.dir is None:
            shutil.rmtree(work, ignore_errors=True)
    res["ok"] = all(c["bit_identical"] for c in res["cases"].values()) and res["main"]["same_losses"]
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))
    sys.exit(0 if res["ok"] else 1)


if __name__ == "__main__":
    main()
