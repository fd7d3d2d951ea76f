"""ogbn-papers100M's streamed store on the GPU: the partition step on the CUDA device writes the bytes the CPU writes;
training on the streamed store at 2 in-process ranks with ``--eval --parallel-eval`` is bit-identical to training on
``partition_graph`` of the whole fixture graph (every epoch's loss, the final weights, the evaluation lines); and
``main.py --dataset ogbn-papers100m --data-source files`` trains from the fixture, with and without
``--skip-partition``."""
import argparse
import os
import re
import subprocess
import sys

import pytest
import torch

from tests.test_dataset_files_gpu import _Recorder, _args, _compare
from tests.test_papers100m_files_cpu import (assert_same_store, fixture_graph, papers_args, whole_graph,
                                             write_whole_store)

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA = torch.device("cuda:0")
CPU = torch.device("cpu")


@pytest.fixture(scope="module")
def small_layout(tmp_path_factory):
    from tools.dataset_files import write_papers100m
    raw = fixture_graph("small")
    root = tmp_path_factory.mktemp("papers")
    write_papers100m(raw, str(root), compressed=True)
    return root, whole_graph(raw)


@pytest.mark.parametrize("n_parts", [1, 3, 8])
def test_the_step_on_the_device_writes_the_cpu_bytes(built, small_layout, tmp_path, n_parts):
    from bns_gcn_b200.data import store
    root, fg = small_layout
    a, b = papers_args(root, tmp_path / "gpu", n_parts), papers_args(root, tmp_path / "cpu", n_parts)
    store.papers100m_partition(a, CUDA, chunk=50_000)
    store.papers100m_partition(b, CPU, chunk=50_000)
    assert_same_store(tmp_path / "gpu" / a.graph_name, tmp_path / "cpu" / b.graph_name)
    assert_same_store(tmp_path / "gpu" / a.graph_name, write_whole_store(fg, papers_args(root, tmp_path / "w",
                                                                                         n_parts)))


def test_training_on_the_streamed_store_is_bit_identical(built, small_layout, tmp_path, monkeypatch):
    from bns_gcn_b200.data import load_as_partition, partition_graph, store
    root, fg = small_layout
    rec = _Recorder(monkeypatch)
    common = dict(n_partitions=2, parallel_eval=True, dataset="ogbn-papers100m", graph_seed=3)
    (tmp_path / "whole").mkdir()
    monkeypatch.chdir(tmp_path / "whole")
    want = rec.run(partition_graph(fg, 2, "random", seed=3), _args(graph_name="papers", **common))
    (tmp_path / "stream").mkdir()
    monkeypatch.chdir(tmp_path / "stream")
    args = _args(data_source="files", data_path=str(root), part_path=str(tmp_path / "part"), graph_name="papers",
                 **common)
    store.graph_partition(args, device=CUDA)
    parts = [load_as_partition(argparse.Namespace(**vars(args)), r) for r in range(2)]
    got = rec.run(parts, args)
    _compare(got, want, 4, 2)
    assert all("Validation Accuracy" in ln for ln in got[2])


def _main(cwd, argv):
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    p = subprocess.run([sys.executable, "-m", "bns_gcn_b200.main"] + argv, cwd=cwd, env=env, capture_output=True,
                       text=True, timeout=600)
    assert p.returncode == 0, (p.stdout[-3000:], p.stderr[-3000:])
    return p.stdout


def test_command_line_trains_from_the_files(built, small_layout, tmp_path):
    root, _ = small_layout
    flags = ["--dataset", "ogbn-papers100m", "--data-source", "files", "--data-path", str(root), "--n-partitions", "1",
             "--partition-method", "random", "--parallel-eval", "--n-epochs", "4", "--log-every", "2", "--use-pp",
             "--fix-seed", "--seed", "5"]
    outs = [_main(tmp_path, flags), _main(tmp_path, flags + ["--skip-partition"])]
    name = "ogbn-papers100m-files-1-random-vol-trans"
    assert (tmp_path / "partition" / name / f"{name}.json").exists()
    for out in outs:
        assert len(re.findall(r"Epoch \d+ \| Validation Accuracy \S+ \| Test Accuracy", out)) == 2, out[-2000:]
        assert len(re.findall(r"Test Result \| Accuracy", out)) == 1, out[-2000:]
    loss = [re.findall(r"Epoch (\d+) \|.*\| Loss (\S+)", o) for o in outs]
    assert len(loss[0]) == 2 and loss[0] == loss[1], loss
