"""Parity AT THE BENCH SHAPE (BASELINE.json configs[1]): the Reddit-shape graph (232,965 nodes, ~114.6 M edges, 602
features, 41 classes), 3-layer GraphSAGE, hidden 256, --use-pp, sampling rate 0.1 -- the exact tensors bench.py times,
with dropout 0 so that the CPU oracle can follow.  One epoch: the oracle needs 10-25 s for it on the GPU box's host
cores (plus the one-time layer-0 precompute).

What this covers that the small cases cannot: the SpMM instantiation the heuristic picks for a 238 MB source matrix
(F = 256 cut into two 128-float column slabs, `spmm_kernel<4,32,1>` with n_tiles = 2), the K = 1204 wgmma GEMM inside
the model, the ~17 K rows longer than one chunk (partial sums + fix-up), and at 4 partitions the per-rank shapes of the
headline configuration (58 K inner nodes, ~5.8 K sampled rows per peer).
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

TOL = 1e-4


def _free_gb() -> float:
    free, _ = torch.cuda.mem_get_info(0)
    return free / 2 ** 30


@pytest.mark.parametrize("n_parts", [1, 4])
def test_bench_shape_one_epoch_matches_oracle(built, n_parts):
    from tests.harness import run_parity_case
    if _free_gb() < 40:
        pytest.skip("needs ~40 GB of free device memory (full-size graph + P in-process ranks)")
    res = run_parity_case(shape="reddit", n_parts=n_parts, model="graphsage", sampling_rate=0.1, n_epochs=1,
                          n_layers=3, n_hidden=256, device="cuda:0", backend="p2p" if n_parts > 1 else "nccl")
    bad = {k: v for k, v in res["detail"].items() if v >= TOL}
    assert not bad, (bad, res["kink"])
    assert res["index_sets_equal"]
    for a, b in zip(res["loss"], res["loss_oracle"]):
        assert abs(a - b) <= 1e-4 * abs(b), (a, b)
    print(f"[bench-shape parity] P={n_parts} max rel err {res['max_rel_err']:.3e} loss {res['loss']} kink {res['kink']}")


def test_dump_outputs_are_float32_and_reproducible(built, tmp_path):
    """`bench.py --dump-outputs DIR` writes the last timed step's loss, logits and parameters as float32 .npy files
    (at most 64 MB); two runs with the same arguments write the same arrays, and --steps sets the timed steps."""
    dirs = []
    for i in range(2):
        d = tmp_path / f"run{i}"
        p = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--shape", "tiny", "--steps", "3", "--warmup", "1",
                            "--no-cpu-baseline", "--dump-outputs", str(d)], cwd=ROOT, capture_output=True, text=True,
                           timeout=600)
        assert p.returncode == 0, p.stderr[-3000:]
        assert json.loads(p.stdout)["steps"] == 3
        dirs.append(d)
    names = sorted(os.listdir(dirs[0]))
    assert {"loss.npy", "logits.npy"} <= set(names) and any(n.startswith("param.") for n in names), names
    assert names == sorted(os.listdir(dirs[1]))
    total = 0
    for n in names:
        a, b = np.load(dirs[0] / n), np.load(dirs[1] / n)
        assert a.dtype == np.float32 and np.isfinite(a).all(), n
        np.testing.assert_allclose(a, b, rtol=1e-5, atol=1e-6, err_msg=n)
        total += a.nbytes
    assert total <= 64 << 20
