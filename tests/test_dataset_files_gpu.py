"""``--data-source files`` on the GPU: the edges sorted on the device give the graph the CPU gives, and training on a
generated shape written in a published layout and read back is bit-identical to training on the generated graph --
every epoch's loss, the final weights and the result-file lines -- in process at 1 and 2 ranks (reddit and yelp
layouts), through the partition store at 2 ranks (ogbn-products layout, ``--partition-method metis``), and through
``main.py``."""
import argparse
import os
import re
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA = torch.device("cuda:0")
CPU = torch.device("cpu")


def _same_graph(a, b):
    assert (a.n_nodes, a.n_class) == (b.n_nodes, b.n_class)
    for k in ("indptr", "src", "feat", "label", "train_mask", "val_mask", "test_mask"):
        x, y = getattr(a, k), getattr(b, k)
        assert x.device.type == "cpu" and x.dtype == y.dtype and torch.equal(x, y), k


@pytest.mark.parametrize("shape,layout", [("small", "reddit"), ("small", "ogbn-products"), ("tiny-ml", "yelp")])
def test_device_built_graph_equals_the_cpu_built_one_and_the_generator(built, tmp_path, shape, layout):
    from bns_gcn_b200.data import load_files, make_graph
    from tools.dataset_files import WRITERS, standard_scaled
    fg = make_graph(shape, seed=0, device=CUDA)
    _same_graph(fg, make_graph(shape, seed=0, device=CPU))
    WRITERS[layout](fg, str(tmp_path))
    on_gpu = load_files(layout, str(tmp_path), CUDA)
    _same_graph(on_gpu, load_files(layout, str(tmp_path), CPU))
    _same_graph(on_gpu, standard_scaled(fg) if layout == "yelp" else fg)


class _Recorder:
    """Wraps ``train.train_epoch``: the loss of every epoch, per rank thread."""

    def __init__(self, monkeypatch):
        import threading
        from bns_gcn_b200 import train
        self.losses, self._local, inner = {}, threading.local(), train.train_epoch

        def train_epoch(st, epoch):
            loss = inner(st, epoch)
            self.losses.setdefault(self._local.rank, []).append(loss.item())
            return loss
        monkeypatch.setattr(train, "train_epoch", train_epoch)

    def run(self, parts, args, full_graph=None):
        """``train.run`` on in-process ranks, cwd the current directory.  Returns (losses per rank, rank 0's final
        weights, the result file's lines)."""
        from bns_gcn_b200 import train
        from bns_gcn_b200.evaluate import result_file_name
        from bns_gcn_b200.helper.comm import run_threads
        self.losses = {}

        def fn(comm, r):
            self._local.rank = r
            p = parts[r]
            a = argparse.Namespace(**vars(args))
            a.n_feat, a.n_class, a.n_train = p.meta["n_feat"], p.meta["n_class"], p.meta["n_train"]
            st, _ = train.run(p.graph, p.node_dict, p.gpb, a, CUDA, full_graph=full_graph)
            return {k: v.detach().cpu().clone() for k, v in st.model.state_dict().items()}
        weights = run_threads(len(parts), fn, device="cuda:0")
        for w in weights[1:]:
            assert all(torch.equal(w[k], weights[0][k]) for k in w)      # replicated
        with open(result_file_name(args)) as f:
            lines = f.read().splitlines()
        return self.losses, weights[0], lines


def _compare(a, b, n_epochs, n_ranks):
    (la, wa, ra), (lb, wb, rb) = a, b
    assert sorted(la) == sorted(lb) == list(range(n_ranks))
    for r in la:
        assert len(la[r]) == n_epochs and la[r] == lb[r], (r, la[r], lb[r])          # bit for bit
    assert list(wa) == list(wb) and all(torch.equal(wa[k], wb[k]) for k in wa)
    assert len(ra) == n_epochs // 2 and ra == rb, (ra, rb)


def _args(**kw):
    from tests.harness import make_args
    d = dict(model="graphsage", n_layers=3, n_hidden=32, sampling_rate=0.5, dropout=0.3, n_epochs=4, log_every=2,
             eval=True, partition_method="random")
    d.update(kw)
    return make_args(**d)


@pytest.mark.parametrize("n_ranks", [1, 2])
@pytest.mark.parametrize("shape,layout", [("small", "reddit"), ("tiny-ml", "yelp")])
def test_training_on_files_is_bit_identical_to_the_generated_graph(built, tmp_path, monkeypatch, shape, layout,
                                                                   n_ranks):
    from bns_gcn_b200.data import load_files, make_graph, partition_graph
    from tools.dataset_files import WRITERS, standard_scaled
    fg = make_graph(shape, seed=0)
    WRITERS[layout](fg, str(tmp_path / "data"))
    rec = _Recorder(monkeypatch)
    common = dict(n_partitions=n_ranks)
    # the generated graph; yelp is compared with its standardised features and the yelp loss (BCE)
    (tmp_path / "gen").mkdir()
    monkeypatch.chdir(tmp_path / "gen")
    if layout == "yelp":
        want_g = standard_scaled(fg)
        want = rec.run(partition_graph(want_g, n_ranks, "random", seed=0),
                       _args(dataset="yelp", graph_name="gen", **common), full_graph=want_g)
    else:
        want = rec.run(partition_graph(fg, n_ranks, "random", seed=0), _args(dataset=shape, graph_name="gen", **common))
    # the files: rank 0's evaluator reads them again (train.run -> load_graph)
    (tmp_path / "files").mkdir()
    monkeypatch.chdir(tmp_path / "files")
    g = load_files(layout, str(tmp_path / "data"), CUDA)
    got = rec.run(partition_graph(g, n_ranks, "random", seed=0),
                  _args(dataset=layout, data_source="files", data_path=str(tmp_path / "data"), graph_name="files",
                        **common))
    _compare(got, want, 4, n_ranks)
    assert os.path.exists(tmp_path / "files" / "checkpoint" / "files_final.pth.tar")


def test_products_layout_through_the_store_is_bit_identical(built, tmp_path, monkeypatch):
    """``graph_partition`` -> ``load_partition`` at 2 ranks with the metis stand-in, from the ogbn-products files and
    from the generator."""
    from bns_gcn_b200.data import graph_partition, load_as_partition, make_graph
    from tools.dataset_files import write_products
    write_products(make_graph("small", seed=0), str(tmp_path / "data"))
    rec = _Recorder(monkeypatch)
    out = []
    for name, kw in (("gen", dict(dataset="small")),
                     ("files", dict(dataset="ogbn-products", data_source="files", data_path=str(tmp_path / "data")))):
        (tmp_path / name).mkdir()
        monkeypatch.chdir(tmp_path / name)
        args = _args(n_partitions=2, partition_method="metis", partition_obj="vol", part_path=str(tmp_path / "part"),
                     graph_name="", graph_seed=0, **kw)
        graph_partition(args, device=CUDA)
        parts = [load_as_partition(argparse.Namespace(**vars(args)), r) for r in range(2)]
        out.append(rec.run(parts, args))
    assert sorted(os.listdir(tmp_path / "part")) == ["ogbn-products-files-2-metis-vol-trans", "small-2-metis-vol-trans"]
    _compare(out[1], out[0], 4, 2)


def _main(cwd, argv):
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    p = subprocess.run([sys.executable, "-m", "bns_gcn_b200.main"] + argv, cwd=cwd, env=env, capture_output=True,
                       text=True, timeout=600)
    assert p.returncode == 0, (p.stdout[-3000:], p.stderr[-3000:])
    return p.stdout


def test_command_line_run_on_files(built, tmp_path):
    """``main.py --data-source files`` at one partition leaves the results file and the final checkpoint, with the
    losses and weights of the same command on the generated shape."""
    from bns_gcn_b200.data import make_graph
    from tools.dataset_files import write_reddit
    write_reddit(make_graph("small", seed=0), str(tmp_path / "data"))
    flags = ["--n-partitions", "1", "--partition-method", "random", "--model", "graphsage", "--n-layers", "2",
             "--n-hidden", "16", "--sampling-rate", "1", "--use-pp", "--n-epochs", "4", "--log-every", "2",
             "--fix-seed", "--seed", "3", "--eval"]
    outs, ckpts = [], []
    for name, extra in (("files", ["--dataset", "reddit", "--data-source", "files", "--data-path",
                                   str(tmp_path / "data")]),
                        ("gen", ["--dataset", "small"])):
        cwd = tmp_path / name
        cwd.mkdir()
        outs.append(_main(cwd, flags + extra))
        dataset = extra[1]
        graph_name = f"{dataset}{'-files' if name == 'files' else ''}-1-random-vol-trans"
        assert (cwd / "partition" / graph_name / f"{graph_name}.json").exists()
        with open(cwd / "results" / f"{dataset}_n1_p1.00.txt") as f:
            lines = f.read().splitlines()
        assert len(lines) == 2 and all("Validation Accuracy" in ln for ln in lines), lines
        outs.append(lines)
        ckpts.append(torch.load(cwd / "checkpoint" / f"{graph_name}_final.pth.tar", map_location="cpu"))
    loss = [re.findall(r"Epoch (\d+) \|.*\| Loss (\S+)", o) for o in outs[0::2]]
    assert len(loss[0]) == 2 and loss[0] == loss[1], loss
    assert outs[1] == outs[3]
    assert list(ckpts[0]) == list(ckpts[1]) and all(torch.equal(ckpts[0][k], ckpts[1][k]) for k in ckpts[0])
