"""Host side of the inductive partition-parallel evaluation (``--eval --parallel-eval --inductive``): the two
evaluation partition sets of the store (``val/``: the train | val subgraph, ``test/``: the full graph), their round
trip, the untouched training set, the write-once rule and the refusals."""
import argparse
import json
import os

import pytest
import torch

CPU = torch.device("cpu")
KEEP = {"_ID", "part_id", "inner_node", "feat", "label", "in_deg", "out_deg"}


def _args(tmp_path, flags=True, **kw):
    d = dict(dataset="tiny", n_partitions=2, partition_method="random", partition_obj="vol", inductive=True,
             part_path=str(tmp_path / "part"), graph_name="", graph_seed=0, partition_balance="nodes",
             eval=flags, parallel_eval=flags)
    d.update(kw)
    return argparse.Namespace(**d)


def _files(root, skip_dirs=()):
    """{relative path: bytes} of every file under ``root``, sub-directories in ``skip_dirs`` left out."""
    out = {}
    for d, dirs, names in os.walk(root):
        if d == root:
            dirs[:] = [x for x in dirs if x not in skip_dirs]
        for n in names:
            p = os.path.join(d, n)
            with open(p, "rb") as f:
                out[os.path.relpath(p, root)] = f.read()
    return out


def _mtimes(root):
    return {os.path.join(d, n): os.stat(os.path.join(d, n)).st_mtime_ns for d, _, ns in os.walk(root) for n in ns}


@pytest.fixture(scope="module")
def graphs():
    from bns_gcn_b200.data import make_graph
    return {s: make_graph(s, seed=0) for s in ("tiny", "small")}


@pytest.mark.parametrize("P", [1, 2, 3])
@pytest.mark.parametrize("method", ["random", "metis"])
@pytest.mark.parametrize("shape", ["tiny", "small"])
def test_eval_sets_round_trip_and_equal_the_in_memory_partitions(tmp_path, graphs, shape, method, P):
    """Each set read back == ``partition_graph`` of its graph (indices, node data, gpb), the node data restricted to
    what the evaluation reads plus the mask it is scored on; the degrees are those of that graph."""
    from bns_gcn_b200.data import graph_partition, induced_subgraph, load_eval_partition, partition_graph
    fg = graphs[shape]
    a = _args(tmp_path, dataset=shape, n_partitions=P, partition_method=method)
    graph_partition(a, fg=fg, device=CPU)
    for which, g in (("val", induced_subgraph(fg, fg.train_mask | fg.val_mask)), ("test", fg)):
        want = partition_graph(g, P, method, seed=0, device=CPU, objective="vol", balance="nodes")
        with open(os.path.join(a.part_path, a.graph_name, which, a.graph_name + ".json")) as f:
            cfg = json.load(f)
        assert cfg["eval_graph"] == which and cfg["num_parts"] == P and cfg["part_method"] == method
        assert cfg["balance"] == "nodes" and cfg["data_source"] == "synthetic" and cfg["num_nodes"] == g.n_nodes
        in_sum = 0
        for r in range(P):
            subg, nd, gpb = load_eval_partition(_args(tmp_path, dataset=shape, n_partitions=P,
                                                      partition_method=method, graph_name=a.graph_name), which, r)
            w = want[r]
            assert (subg.n_in, subg.n_halo) == (w.graph.n_in, w.graph.n_halo)
            assert torch.equal(subg.indptr, w.graph.indptr) and torch.equal(subg.indices, w.graph.indices)
            assert torch.equal(gpb.ranges, w.gpb.ranges)
            assert set(nd) == KEEP | {which + "_mask"}
            for k, v in nd.items():
                assert v.dtype == w.node_dict[k].dtype and torch.equal(v, w.node_dict[k]), (which, r, k)
            # every in-edge of an inner node is in the part: its row length is the in-degree in THAT graph
            assert torch.equal(nd["in_deg"], subg.indptr[1:] - subg.indptr[:-1])
            in_sum += int(nd["in_deg"].sum())
        assert in_sum == g.n_edges
    assert induced_subgraph(fg, fg.train_mask | fg.val_mask).n_edges < fg.n_edges


def test_training_set_is_byte_identical_with_and_without_the_flags(tmp_path, graphs):
    from bns_gcn_b200.data import graph_partition
    fg = graphs["small"]
    with_flags = _args(tmp_path / "a", dataset="small", n_partitions=3, partition_method="metis")
    without = _args(tmp_path / "b", flags=False, dataset="small", n_partitions=3, partition_method="metis")
    graph_partition(with_flags, fg=fg, device=CPU)
    graph_partition(without, fg=fg, device=CPU)
    assert with_flags.graph_name == without.graph_name
    d_with = os.path.join(with_flags.part_path, with_flags.graph_name)
    d_without = os.path.join(without.part_path, without.graph_name)
    assert os.path.isdir(os.path.join(d_with, "val")) and os.path.isdir(os.path.join(d_with, "test"))
    assert sorted(os.listdir(d_without)) == sorted(x for x in os.listdir(d_with) if x not in ("val", "test"))
    a, b = _files(d_with, skip_dirs=("val", "test")), _files(d_without)
    assert a.keys() == b.keys() and a == b


@pytest.mark.parametrize("drop", ["eval", "parallel_eval", "inductive"])
def test_no_eval_sets_without_all_three_flags(tmp_path, graphs, drop):
    from bns_gcn_b200.data import graph_partition
    a = _args(tmp_path, **{drop: False})
    graph_partition(a, fg=graphs["tiny"], device=CPU)
    assert not {"val", "test"} & set(os.listdir(os.path.join(a.part_path, a.graph_name)))


def test_a_second_call_rewrites_nothing_and_a_later_call_adds_the_sets(tmp_path, graphs):
    """A store built without the flags gains the two sets on the next run with them, its training files untouched;
    a third call writes no part file again (meta.json is rewritten as always, with the same bytes)."""
    from bns_gcn_b200.data import graph_partition, load_eval_partition
    fg = graphs["tiny"]
    plain = _args(tmp_path, flags=False)
    graph_partition(plain, fg=fg, device=CPU)
    root = os.path.join(plain.part_path, plain.graph_name)
    before, before_bytes = _mtimes(root), _files(root)
    a = _args(tmp_path, graph_name=plain.graph_name)
    graph_partition(a, fg=fg, device=CPU)
    meta = os.path.join(root, "meta.json")
    after = _mtimes(root)
    assert {k: v for k, v in after.items() if k in before and k != meta} == \
        {k: v for k, v in before.items() if k != meta}
    assert {k: v for k, v in _files(root, skip_dirs=("val", "test")).items()} == before_bytes
    for which in ("val", "test"):
        load_eval_partition(a, which, 1)
    graph_partition(_args(tmp_path, graph_name=plain.graph_name), fg=fg, device=CPU)
    again = _mtimes(root)
    assert {k: v for k, v in again.items() if k != meta} == {k: v for k, v in after.items() if k != meta}
    assert not any(n.endswith(".tmp") for n in _files(root))


def _edit_config(path, **kw):
    with open(path) as f:
        cfg = json.load(f)
    cfg.update(kw)
    with open(path, "w") as f:
        json.dump(cfg, f, indent=1)


@pytest.mark.parametrize("which", ["val", "test"])
@pytest.mark.parametrize("field,value,flag", [("balance", "edges", "--partition-balance"),
                                              ("data_source", "files", "--data-source"),
                                              ("num_parts", 3, "--n-partitions"),
                                              ("part_method", "metis", "--partition-method"),
                                              ("eval_graph", "other", "eval_graph")])
def test_a_set_of_another_balance_source_part_count_or_graph_is_refused(tmp_path, graphs, which, field, value, flag):
    """Both the loader and the next ``graph_partition`` refuse it, naming the config and the field."""
    from bns_gcn_b200.data import graph_partition, load_eval_partition
    a = _args(tmp_path)
    graph_partition(a, fg=graphs["tiny"], device=CPU)
    path = os.path.join(a.part_path, a.graph_name, which, a.graph_name + ".json")
    _edit_config(path, **{field: value})
    with pytest.raises(RuntimeError, match=flag) as e:
        load_eval_partition(_args(tmp_path, graph_name=a.graph_name), which, 0)
    assert path in str(e.value)
    with pytest.raises(RuntimeError, match=flag):
        graph_partition(_args(tmp_path, graph_name=a.graph_name), fg=graphs["tiny"], device=CPU)


def test_a_run_with_another_part_count_is_refused(tmp_path, graphs):
    from bns_gcn_b200.data import graph_partition, load_eval_partition
    a = _args(tmp_path)
    graph_partition(a, fg=graphs["tiny"], device=CPU)
    with pytest.raises(RuntimeError, match="--n-partitions"):
        load_eval_partition(_args(tmp_path, graph_name=a.graph_name, n_partitions=3), "val", 0)
    with pytest.raises(IndexError):
        load_eval_partition(_args(tmp_path, graph_name=a.graph_name), "test", 2)
    with pytest.raises(ValueError, match="train"):
        load_eval_partition(_args(tmp_path, graph_name=a.graph_name), "train", 0)


@pytest.mark.parametrize("which", ["val", "test"])
def test_a_missing_set_raises_naming_its_path(tmp_path, graphs, which):
    """A store built without the flags, then read as ``--skip-partition`` does (no ``graph_partition``): the error
    names the missing config and the flags that build it."""
    from bns_gcn_b200.data import graph_partition, load_eval_partition, load_partition
    plain = _args(tmp_path, flags=False)
    graph_partition(plain, fg=graphs["tiny"], device=CPU)
    a = _args(tmp_path, graph_name=plain.graph_name, skip_partition=True)
    load_partition(a, 0)                                   # the training set is there
    path = os.path.join(a.part_path, a.graph_name, which, a.graph_name + ".json")
    with pytest.raises(FileNotFoundError, match="--parallel-eval --inductive") as e:
        load_eval_partition(a, which, 0)
    assert path in str(e.value)
