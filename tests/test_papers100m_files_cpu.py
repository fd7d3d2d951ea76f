"""ogbn-papers100M through the partition store without the whole graph (``store.papers100m_partition``): the streamed
store equals, byte for byte, the store the whole-graph path writes from the same graph (``partition_graph(fg, P,
'random')`` + ``_write_parts``) at every part count, chunk size and archive compression; its parts load back equal;
every malformed input is refused naming its file and leaves nothing behind; the launch-time refusals; the generated
shape through the same store; and the traced host memory of the step.  CPU only."""
import argparse
import gzip
import os
import shutil
import tracemalloc

import numpy as np
import pytest
import torch

import bns_gcn_b200  # noqa: F401
from bns_gcn_b200.data import DataFileError, make_graph, make_local_partition, partition_graph, store
from bns_gcn_b200.data.files import csr_by_destination
from bns_gcn_b200.data.synthetic import FullGraph
from tools.dataset_files import write_papers100m

CPU = torch.device("cpu")
ALL = 1 << 40


def fixture_graph(shape: str) -> FullGraph:
    """The generated ``shape`` as stored in the files: a third of the nodes unlabelled and in no split, 20 extra
    stored self-loops and 50 duplicated edges, in CSR order (self-loops included)."""
    fg = make_graph(shape, seed=0, device=CPU)
    n = fg.n_nodes
    r = torch.randperm(n, generator=torch.Generator().manual_seed(5))
    k = n // 3
    label = fg.label.clone()
    label[r[:k]] = -1
    masks = [torch.zeros(n, dtype=torch.bool) for _ in range(3)]
    rest = r[k:]
    a, b = rest.numel() * 6 // 10, rest.numel() * 6 // 10 + rest.numel() // 5
    masks[0][rest[:a]], masks[1][rest[a:b]], masks[2][rest[b:]] = True, True, True
    src, dst = torch.cat([fg.src, r[:20], fg.src[:50]]), torch.cat([fg.dst(), r[:20], fg.dst()[:50]])
    o = torch.argsort(dst * n + src)
    src, dst = src[o], dst[o]
    indptr = torch.zeros(n + 1, dtype=torch.int64)
    indptr[1:] = torch.cumsum(torch.bincount(dst, minlength=n), 0)
    return FullGraph(n, indptr, src, fg.feat, label, *masks, fg.n_class)


def whole_graph(raw: FullGraph) -> FullGraph:
    """The graph the reference's rules make of the stored edges, built whole."""
    indptr, src = csr_by_destination(raw.n_nodes, raw.src, raw.dst(), CPU)
    return FullGraph(raw.n_nodes, indptr, src, raw.feat, raw.label, raw.train_mask, raw.val_mask, raw.test_mask,
                     int(raw.label.max()) + 1)


def papers_args(data_path, part_path, n_parts, **kw):
    d = dict(dataset="ogbn-papers100m", data_source="files", data_path=str(data_path), part_path=str(part_path),
             graph_name="", n_partitions=n_parts, partition_method="random", inductive=False, eval=False,
             graph_seed=3)
    d.update(kw)
    return argparse.Namespace(**d)


def write_whole_store(fg: FullGraph, args) -> str:
    """What ``graph_partition`` writes for ``fg`` with ``--partition-method random``."""
    graph_dir, part_config = store._dirs(args)
    parts = partition_graph(fg, args.n_partitions, "random", seed=args.graph_seed)
    store._write_parts(parts, graph_dir, part_config, store._config_head(args, parts))
    store._write_meta(graph_dir, fg.n_feat, fg.n_class, int(fg.train_mask.sum()))
    return graph_dir


def tree(d):
    return sorted(os.path.relpath(os.path.join(p, f), d) for p, _, fs in os.walk(d) for f in fs)


def assert_same_store(a, b):
    assert tree(a) == tree(b)
    for f in tree(a):
        with open(os.path.join(a, f), "rb") as x, open(os.path.join(b, f), "rb") as y:
            assert x.read() == y.read(), f


@pytest.fixture(scope="module")
def layouts(tmp_path_factory):
    """``{(shape, compressed): (data path, whole graph)}``."""
    out = {}
    for shape in ("tiny", "small"):
        raw = fixture_graph(shape)
        for compressed in (False, True):
            root = tmp_path_factory.mktemp(f"{shape}-{int(compressed)}")
            write_papers100m(raw, str(root), compressed=compressed)
            out[shape, compressed] = (root, whole_graph(raw))
    return out


CASES = ([("tiny", p, c) for p in (1, 2, 3, 8) for c in (1, 7, 4096, ALL)]
         + [("small", p, c) for p in (1, 2, 3, 8) for c in (4096, ALL)])


@pytest.mark.parametrize("compressed", [False, True], ids=["stored", "deflated"])
@pytest.mark.parametrize("shape,n_parts,chunk", CASES)
def test_streamed_store_equals_the_whole_graph_store(layouts, tmp_path, shape, n_parts, chunk, compressed):
    root, fg = layouts[shape, compressed]
    got = papers_args(root, tmp_path / "stream", n_parts)
    config = store.papers100m_partition(got, CPU, chunk=chunk)
    assert got.graph_name == f"ogbn-papers100m-files-{n_parts}-random-vol-trans"
    assert os.path.exists(config)
    want = write_whole_store(fg, papers_args(root, tmp_path / "whole", n_parts))
    assert_same_store(os.path.dirname(config), want)
    assert not [f for f in os.listdir(os.path.dirname(config)) if f.startswith(".spill")]


def test_graph_partition_streams_and_parts_load_back_equal(layouts, tmp_path):
    root, fg = layouts["small", True]
    a = papers_args(root, tmp_path / "stream", 3)
    store.graph_partition(a, device=CPU)
    b = papers_args(root, tmp_path / "whole", 3)
    write_whole_store(fg, b)
    for r in range(3):
        (ga, na, pa), (gb, nb, pb) = store.load_partition(a, r), store.load_partition(b, r)
        assert (ga.n_in, ga.n_halo) == (gb.n_in, gb.n_halo)
        assert torch.equal(ga.indptr, gb.indptr) and torch.equal(ga.indices, gb.indices)
        assert list(na) == list(nb) and all(na[k].dtype == nb[k].dtype and torch.equal(na[k], nb[k]) for k in na)
        assert torch.equal(pa.ranges, pb.ranges)
    assert (a.n_feat, a.n_class, a.n_train) == (b.n_feat, b.n_class, b.n_train) == \
        (fg.n_feat, fg.n_class, int(fg.train_mask.sum()))
    # a second call keeps the store as it is
    before = {f: os.path.getmtime(os.path.join(tmp_path / "stream", a.graph_name, f))
              for f in tree(tmp_path / "stream" / a.graph_name)}
    store.graph_partition(a, device=CPU)
    assert before == {f: os.path.getmtime(os.path.join(tmp_path / "stream", a.graph_name, f)) for f in before}


def test_unlabelled_nodes_are_stored_as_minus_one(layouts, tmp_path):
    root, fg = layouts["tiny", False]
    a = papers_args(root, tmp_path, 1)
    store.papers100m_partition(a, CPU)
    _, nd, _ = store.load_partition(a, 0)
    unl = ~(nd["train_mask"] | nd["val_mask"] | nd["test_mask"])
    assert int(unl.sum()) == fg.n_nodes // 3 and bool((nd["label"][unl] == -1).all())
    assert bool((nd["label"][~unl] >= 0).all()) and a.n_class == int(fg.label.max()) + 1


# ---- malformed input ----------------------------------------------------------------------------------------------

def _npz(path, compressed=False, **arrays):
    (np.savez_compressed if compressed else np.savez)(path, **arrays)


def _malform(root, case):
    raw = os.path.join(root, "ogbn_papers100M", "raw")
    data, label = os.path.join(raw, "data.npz"), os.path.join(raw, "node-label.npz")
    split = os.path.join(root, "ogbn_papers100M", "split", "time")
    with np.load(data) as z:
        d = {k: z[k] for k in z.files}
    with np.load(label) as z:
        lab = z["node_label"]
    n = int(d["num_nodes_list"][0])
    train = np.loadtxt(gzip.open(os.path.join(split, "train.csv.gz"), "rt"), dtype=np.int64)
    if case == "no data.npz":
        os.remove(data)
        return data
    if case == "no node-label.npz":
        os.remove(label)
        return label
    if case == "no test split":
        os.remove(os.path.join(split, "test.csv.gz"))
        return os.path.join(split, "test.csv.gz")
    if case in ("no edge_index", "no node_feat", "no num_nodes_list"):
        del d[case[3:]]
    elif case == "two node counts":
        d["num_nodes_list"] = np.array([n, n])
    elif case == "edge_index [3, E]":
        d["edge_index"] = np.concatenate([d["edge_index"], d["edge_index"][:1]])
    elif case == "feature rows":
        d["node_feat"] = d["node_feat"][:-1]
    elif case == "integer features":
        d["node_feat"] = d["node_feat"].astype(np.int32)
    elif case == "fortran features":
        d["node_feat"] = np.asfortranarray(d["node_feat"])
    elif case == "edge id N":
        d["edge_index"] = d["edge_index"].copy()
        d["edge_index"][1, -1] = n
    elif case == "edge id -1":
        d["edge_index"] = d["edge_index"].copy()
        d["edge_index"][0, 3] = -1
    elif case == "no key in node-label.npz":
        _npz(label, labels=lab)
        return label
    elif case == "label rows":
        _npz(label, node_label=lab[:-1])
        return label
    elif case in ("NaN train label", "fractional train label", "negative train label"):
        lab = lab.copy()
        lab.reshape(-1)[train[0]] = {"NaN train label": np.nan, "fractional train label": 1.5,
                                     "negative train label": -2.0}[case]
        _npz(label, node_label=lab)
        return label
    elif case == "split id N":
        with gzip.open(os.path.join(split, "valid.csv.gz"), "wt") as f:
            f.write(f"0\n{n}\n")
        return os.path.join(split, "valid.csv.gz")
    elif case == "truncated":
        with open(data, "r+b") as f:
            f.truncate(os.path.getsize(data) // 2)
        return data
    else:
        raise AssertionError(case)
    _npz(data, **d)
    return data


MALFORMED = ["no data.npz", "no node-label.npz", "no test split", "no edge_index", "no node_feat", "no num_nodes_list",
             "two node counts", "edge_index [3, E]", "feature rows", "integer features", "fortran features",
             "edge id N", "edge id -1", "no key in node-label.npz", "label rows", "NaN train label",
             "fractional train label", "negative train label", "split id N", "truncated"]


@pytest.mark.parametrize("case", MALFORMED)
def test_malformed_input_is_refused_naming_the_file_and_leaves_nothing(layouts, tmp_path, case):
    src, _ = layouts["tiny", False]
    root = tmp_path / "data"
    shutil.copytree(src, root)
    path = _malform(str(root), case)
    a = papers_args(root, tmp_path / "part", 2)
    with pytest.raises(DataFileError) as e:
        store.papers100m_partition(a, CPU, chunk=97)
    assert e.value.path == path and str(e.value).startswith(path)
    assert not (tmp_path / "part" / a.graph_name).exists()


def test_an_existing_store_directory_keeps_no_part_after_a_failure(layouts, tmp_path):
    src, _ = layouts["tiny", False]
    root = tmp_path / "data"
    shutil.copytree(src, root)
    _malform(str(root), "edge id N")
    a = papers_args(root, tmp_path / "part", 2, graph_name="g")
    (tmp_path / "part" / "g").mkdir(parents=True)
    with pytest.raises(DataFileError):
        store.papers100m_partition(a, CPU, chunk=97)
    assert os.listdir(tmp_path / "part" / "g") == []


# ---- refusals -----------------------------------------------------------------------------------------------------

REASONS = {"partition_method": ("metis", "--partition-method metis"),
           "partition_balance": ("edges", "--partition-balance edges"),
           "inductive": (True, "--inductive"),
           "eval": (True, "--eval without --parallel-eval")}


@pytest.mark.parametrize("source", ["files", "synthetic"])
def test_every_refusal_is_named_in_one_message_before_any_file_is_read(tmp_path, source):
    missing = tmp_path / "nothing-here"                    # any read of --data-path would raise DataFileError
    a = papers_args(missing, tmp_path / "part", 2, data_source=source,
                    **{k: v for k, (v, _) in REASONS.items()})
    for call in (lambda: store.graph_partition(a, device=CPU), lambda: store.papers100m_partition(a, CPU),
                 lambda: store.check_papers100m(a)):
        with pytest.raises(ValueError) as e:
            call()
        assert not isinstance(e.value, DataFileError)
        assert all(why in str(e.value) for _, why in REASONS.values()), str(e.value)
    assert not (tmp_path / "part").exists()
    for k, (v, why) in REASONS.items():                     # each on its own
        b = papers_args(missing, tmp_path / "part", 2, data_source=source, **{k: v})
        with pytest.raises(ValueError, match=why.split()[0]):
            store.check_papers100m(b)
    for ok in (dict(eval=True, parallel_eval=True), dict(eval=False)):
        store.check_papers100m(papers_args(missing, tmp_path / "part", 2, **ok))
    store.check_papers100m(papers_args(missing, tmp_path, 2, dataset="reddit", partition_method="metis", eval=True))


def test_main_refuses_before_writing(tmp_path, monkeypatch):
    from bns_gcn_b200 import main
    monkeypatch.chdir(tmp_path)
    for argv, why in ((["--partition-method", "multilevel", "--inductive"], ["--partition-method multilevel",
                                                                             "--inductive", "--eval without"]),
                      (["--partition-method", "random", "--partition_balance", "edges", "--no-eval"],
                       ["--partition-balance edges"])):
        with pytest.raises(ValueError) as e:
            main.main(["--dataset", "papers100m", "--data-source", "files", "--data-path", "nowhere"] + argv)
        assert all(w in str(e.value) for w in why), str(e.value)
        assert "--eval without" in str(e.value) or "--no-eval" in argv
    assert os.listdir(tmp_path) == []


def test_default_store_names():
    from bns_gcn_b200.data import default_graph_name
    a = papers_args("d", "p", 8)
    assert default_graph_name(a) == "ogbn-papers100m-files-8-random-vol-trans"
    a.data_source = "synthetic"
    assert default_graph_name(a) == "ogbn-papers100m-8-random-vol-trans"


# ---- the generated shape ------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n_parts", [1, 2, 4])
def test_generated_shape_through_the_store_equals_make_local_partition(tmp_path, n_parts):
    a = papers_args(tmp_path / "unused", tmp_path / "part", n_parts, data_source="synthetic", graph_seed=2,
                    graph_scale=1e-4)
    store.graph_partition(a, device=CPU)
    assert a.graph_name == f"ogbn-papers100m-{n_parts}-random-vol-trans"
    for r in range(n_parts):
        p = make_local_partition("papers100m", r, n_parts, seed=2, device=CPU, scale=1e-4)
        g, nd, gpb = store.load_partition(a, r)
        assert (g.n_in, g.n_halo) == (p.graph.n_in, p.graph.n_halo)
        assert torch.equal(g.indptr, p.graph.indptr) and torch.equal(g.indices, p.graph.indices)
        assert list(nd) == list(p.node_dict)
        assert all(nd[k].dtype == p.node_dict[k].dtype and torch.equal(nd[k], p.node_dict[k]) for k in nd)
        assert torch.equal(gpb.ranges, p.gpb.ranges)
        assert (a.n_feat, a.n_class, a.n_train) == (p.meta["n_feat"], p.meta["n_class"], p.meta["n_train"])


# ---- memory -------------------------------------------------------------------------------------------------------

def test_traced_host_memory_stays_within_node_tables_one_part_and_the_chunks(layouts, tmp_path):
    """numpy reports its buffers to ``tracemalloc`` (the edge and feature chunks, the spill of a part, the node
    tables); torch's host tensors are not traced, so this bounds the numpy side of the step."""
    root, fg = layouts["small", True]
    n_parts, chunk = 4, 1024
    edge_bytes = 2 * 8 * (fg.n_edges - fg.n_nodes + 70)    # the stored edge_index
    budget = chunk * max(16, 4 * fg.n_feat)
    assert edge_bytes >= 20 * budget
    node_tables = 6 * 8 * fg.n_nodes                        # label, owners, ids, degrees, masks: int64 or narrower
    a = papers_args(root, tmp_path, n_parts)
    tracemalloc.start()
    try:
        store.papers100m_partition(a, CPU, chunk=chunk)
        peak = tracemalloc.get_traced_memory()[1]
    finally:
        tracemalloc.stop()
    largest = max(os.path.getsize(os.path.join(tmp_path, a.graph_name, f"part{r}", f))
                  for r in range(n_parts) for f in ("indices.npy", "node_feat.npy")) * 4   # a part's (dst, src) pairs
    assert peak < node_tables + largest + 4 * budget, (peak, node_tables, largest, budget)
    assert peak < edge_bytes / 2
