"""``--comm-dtype fp8`` with one PROCESS per GPU, launched by torchrun: both transports eager, and the epoch replayed
from one CUDA graph (p2p at any world, the staged transport at 2, as in f32), at world 2 / 4.  tools/dist_check.py
compares loss, all-reduced gradients and updated weights with the in-process run of the same seeded inputs in the same
mode.  Skipped unless the machine has at least ``world`` GPUs."""
import json

import pytest
import torch

from tests.test_multiprocess_gpu import _launch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "cuda-graph"])
@pytest.mark.parametrize("world", [2, 4])
def test_fp8_exchange_one_process_per_gpu_matches_in_process_run(built, tmp_path, world, graph):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs, this box has {torch.cuda.device_count()}")
    extra = (["--shape", "small", "--rate", "0.3", "--hidden", "64", "--epochs", "4", "--comm-dtype", "fp8"]
             + (["--graph"] if graph else []))
    p, line = _launch(world, extra, 29900 + world + (50 if graph else 0), tmp_path)
    assert p.returncode == 0 and line is not None, (p.stdout[-3000:], p.stderr[-3000:])
    assert line["ok"] and line["world"] == world and line["comm_dtype"] == "fp8", line
    for backend in (("p2p",) if (graph and world > 2) else ("nccl", "p2p")):
        assert line[backend]["max_rel_err_vs_inprocess"] < 1e-4, line
        assert line[backend]["loss_rel_err"] < 1e-4, line
    print("[multiprocess fp8]", json.dumps(line))
