"""Partition-parallel evaluation with one PROCESS per GPU (``DistComm``, the path ``main.py`` and torchrun runs take):
the boundary exchange of every layer through NCCL send / recv (or libbnsgcn.so's own communicator, ``BNS_COMM=abi``)
and the float64 accuracy counts through ``all_reduce``.  ``tools/bench_eval.py --check`` compares every rank's logits
and counts with the in-process run of the same partitions (threads on one GPU, which
tests/test_parallel_eval_gpu.py pins to the whole-graph evaluation).

Skipped unless the machine has at least ``world`` GPUs.
"""
import json
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("world,comm", [(2, "torch"), (4, "torch"), (2, "abi")])
@pytest.mark.parametrize("model,heads", [("graphsage", 1), ("gcn", 1), ("gat", 2)])
def test_parallel_eval_one_process_per_gpu_matches_in_process_run(built, tmp_path, world, comm, model, heads):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs, this box has {torch.cuda.device_count()}")
    port = 29800 + 10 * world + (5 if comm == "abi" else 0) + {"graphsage": 0, "gcn": 1, "gat": 2}[model]
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tools", "bench_eval.py"),
           "--mode", "parallel", "--shape", "small", "--model", model, "--heads", str(heads), "--hidden", "64",
           "--warmup", "1", "--iters", "1", "--check", "--comm", comm]
    env = dict(os.environ)
    env.pop("CUDA_VISIBLE_DEVICES", None)
    p = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    with open(os.path.join(tmp_path, "bench_eval.log"), "w") as f:
        f.write(p.stdout[-20000:] + "\n---- stderr ----\n" + p.stderr[-20000:])
    line = next((json.loads(ln) for ln in p.stdout.splitlines() if ln.startswith("{") and '"P"' in ln), None)
    assert p.returncode == 0 and line is not None, (p.stdout[-3000:], p.stderr[-3000:])
    assert line["ok"] and line["P"] == world and line["check_counts_equal"], line
    assert line["check_max_rel_err_vs_inprocess"] < 1e-6, line
