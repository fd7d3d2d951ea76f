"""One PROCESS per GPU (the deployment shape): torchrun-launched correctness of both exchange transports, eager and
replayed from one CUDA graph, at world 2 / 4 / 8.  Every other `-m gpu` parity test runs its ranks as threads of one
process on one GPU, where the p2p producer hands the consumer a CUDA event (helper/feature_buffer.py); here the
release/acquire flags in peer memory are the only signal, the slabs are cudaIpc mappings over NVLink, and NCCL does the
id exchange and the all-reduce.  tools/dist_check.py compares loss, all-reduced gradients and updated weights of every
configuration with the in-process run of the same seeded inputs (which tests/test_parity_gpu.py pins to the oracle).

Skipped unless the machine has at least `world` GPUs.
"""
import json
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _launch(world: int, extra, port: int, log_dir, timeout: int = 600):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tools", "dist_check.py")] + extra
    env = dict(os.environ)
    env.pop("CUDA_VISIBLE_DEVICES", None)
    p = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=timeout)
    tag = (f"w{world}_{'graph' if '--graph' in extra else 'eager'}{'_abi' if 'abi' in extra else ''}"
           f"{'_dropout' if '--dropout' in extra else ''}")
    with open(os.path.join(log_dir, f"dist_check_{tag}.log"), "w") as f:      # kept for the post-mortem of a failure
        f.write(p.stdout[-20000:] + "\n---- stderr ----\n" + p.stderr[-20000:])
    line = None
    for ln in p.stdout.splitlines():
        if ln.startswith("{") and '"world"' in ln:
            line = json.loads(ln)
    return p, line


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "cuda-graph"])
@pytest.mark.parametrize("world", [2, 4, 8])
def test_one_process_per_gpu_matches_in_process_run(built, tmp_path, world, graph):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs, this box has {torch.cuda.device_count()}")
    extra = ["--shape", "small", "--rate", "0.3", "--hidden", "64", "--epochs", "4"] + (["--graph"] if graph else [])
    p, line = _launch(world, extra, 29600 + world + (50 if graph else 0), tmp_path)
    assert p.returncode == 0 and line is not None, (p.stdout[-3000:], p.stderr[-3000:])
    assert line["ok"] and line["world"] == world, line
    for backend in (("p2p",) if (graph and world > 2) else ("nccl", "p2p")):
        assert line[backend]["max_rel_err_vs_inprocess"] < 1e-5, line
        assert line[backend]["loss_rel_err"] < 1e-5, line
    print("[multiprocess]", json.dumps(line))


def test_replayed_epochs_with_dropout_match_in_process_run(built, tmp_path):
    """World 2 replayed from a CUDA graph at dropout 0.5: every replay's masks take the epoch from the device counter
    (offset 2**64 - 1 + epoch_dev) and must equal those of the eager in-process run."""
    if torch.cuda.device_count() < 2:
        pytest.skip(f"needs 2 GPUs, this box has {torch.cuda.device_count()}")
    extra = ["--shape", "small", "--rate", "0.3", "--hidden", "64", "--epochs", "4", "--graph", "--dropout", "0.5"]
    p, line = _launch(2, extra, 29680, tmp_path)
    assert p.returncode == 0 and line is not None, (p.stdout[-3000:], p.stderr[-3000:])
    assert line["ok"] and line["world"] == 2, line
    for backend in ("nccl", "p2p"):
        assert line[backend]["max_rel_err_vs_inprocess"] < 1e-5, line
        assert line[backend]["loss_rel_err"] < 1e-5, line


@pytest.mark.parametrize("world", [2, 8])
def test_collectives_behind_the_c_abi(built, tmp_path, world):
    """BNS_COMM=abi: the gradient all-reduce, the id exchange and the staged feature exchange go through libbnsgcn.so's
    own NCCL communicator (bns_comm_unique_id / bns_ctx_create / bns_allreduce_sum_f32 / bns_alltoallv_bytes) instead
    of torch.distributed, which then only hands out the unique id.  Same comparison as above."""
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs, this box has {torch.cuda.device_count()}")
    extra = ["--shape", "small", "--rate", "0.3", "--hidden", "64", "--epochs", "3", "--comm", "abi"]
    p, line = _launch(world, extra, 29700 + world, tmp_path)
    assert p.returncode == 0 and line is not None, (p.stdout[-3000:], p.stderr[-3000:])
    assert line["ok"] and line["comm"] == "abi", line
