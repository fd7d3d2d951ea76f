"""``--save-state-every`` / ``--resume`` with one PROCESS per GPU, launched through ``main.py`` under torchrun at world
2 over the peer-memory transport: a run of 3 epochs resumed to 6 ends in the same state, bit for bit, as 6 uninterrupted
epochs, and a launch without ``--fix-seed`` (which draws a new seed) continues with the saved seed.  Skipped unless the
machine has at least 2 GPUs."""
import os
import re
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FLAGS = ["--dataset", "small", "--n-partitions", "2", "--partition-method", "random", "--model", "graphsage",
         "--n-layers", "3", "--n-hidden", "64", "--sampling-rate", "0.3", "--dropout", "0.5", "--use-pp",
         "--backend", "p2p", "--no-eval", "--log-every", "1"]


def _main(cwd, extra, port: int) -> str:
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr",
           "127.0.0.1", "--master-port", str(port), "-m", "bns_gcn_b200.main"] + FLAGS + extra
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    env.pop("CUDA_VISIBLE_DEVICES", None)
    p = subprocess.run(cmd, cwd=cwd, env=env, capture_output=True, text=True, timeout=900)
    with open(os.path.join(cwd, f"main_{port}.log"), "w") as f:          # kept for the post-mortem of a failure
        f.write(p.stdout[-20000:] + "\n---- stderr ----\n" + p.stderr[-20000:])
    assert p.returncode == 0, (p.stdout[-3000:], p.stderr[-3000:])
    return p.stdout


def _state(cwd):
    root = os.path.join(cwd, "checkpoint", "small-2-random-vol-trans_state")
    with open(os.path.join(root, "CURRENT")) as f:
        return torch.load(os.path.join(root, f.read().strip(), "shared.pt"), map_location="cpu")


def _losses(out: str):
    return {(int(m[0]), int(m[1])): m[2] for m in re.findall(r"Process (\d+) \| Epoch (\d+) \|.*\| Loss (\S+)", out)}


@pytest.fixture(scope="module")
def runs(built, tmp_path_factory):
    if torch.cuda.device_count() < 2:
        pytest.skip(f"needs 2 GPUs, this box has {torch.cuda.device_count()}")
    split, whole = tmp_path_factory.mktemp("split"), tmp_path_factory.mktemp("whole")
    first = _main(split, ["--n-epochs", "3", "--save-state-every", "3"], 29910)
    seed = _state(split)["seed"]
    second = _main(split, ["--n-epochs", "6", "--save-state-every", "3", "--resume", "--skip-partition"], 29911)
    uninterrupted = _main(whole, ["--n-epochs", "6", "--save-state-every", "6", "--fix-seed", "--seed", str(seed)],
                          29912)
    return dict(seed=seed, first=first, second=second, whole=uninterrupted, split_state=_state(split),
                whole_state=_state(whole))


def test_resumed_eager_run_is_bit_identical(runs):
    a, b = runs["split_state"], runs["whole_state"]
    assert a["epochs"] == b["epochs"] == 6
    for k, v in b["model"].items():
        assert torch.equal(a["model"][k], v), k
    assert torch.equal(a["optimizer"]["step"], b["optimizer"]["step"]) and int(a["optimizer"]["step"]) == 6
    for name, mom in b["optimizer"]["state"].items():
        for key in ("exp_avg", "exp_avg_sq"):
            assert torch.equal(a["optimizer"]["state"][name][key], mom[key]), (name, key)
    lw, ls = _losses(runs["whole"]), _losses(runs["second"])
    for key in [(r, e) for r in range(2) for e in range(3, 6)]:
        assert ls[key] == lw[key], key


def test_resume_without_fix_seed_adopts_the_saved_seed(runs):
    drawn = [int(s) for s in re.findall(r"Namespace\(.*?\bseed=(\d+)", runs["second"])]
    assert drawn and all(s != runs["seed"] for s in drawn)         # the launch drew its own ...
    assert runs["split_state"]["seed"] == runs["seed"]             # ... and continued with the saved one
    assert "resumes after 3 epochs" in runs["second"]
