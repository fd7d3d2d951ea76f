"""``--data-source files``: the Reddit, Yelp and ogbn-products readers (``data/files.py``) against hand-built fixtures
and hand-written expected graphs, the round trip through the layout writers (``tools/dataset_files.py``) at the
generated shapes, every refusal of malformed input, the flag, and the partition store's record of the source.  CPU
only."""
import argparse
import gzip
import json
import os

import numpy as np
import pytest
import torch

import bns_gcn_b200  # noqa: F401
from bns_gcn_b200.data import DataFileError, load_files

CPU = torch.device("cpu")

# One edge list for the reddit and yelp fixtures, (src, dst): 0 -> 1 has no inverse; 1 -> 2 is stored twice; 0 -> 0
# (twice) and 3 -> 3 are stored self-loops; node 4 has no edge at all.
EDGES = [(0, 1), (0, 0), (0, 0), (1, 2), (1, 2), (2, 1), (2, 0), (3, 3), (3, 0)]
# after removing the stored self-loops and adding one per node, CSR by destination with sorted sources
WANT_INDPTR = [0, 3, 6, 9, 10, 11]
WANT_SRC = [0, 2, 3, 0, 1, 2, 1, 1, 2, 3, 4]
WANT_OUT_DEG = [2, 3, 3, 2, 1]
FEAT = np.array([[0.5, -1.25, 7.0], [1.5, 2.0, 7.0], [-3.0, 0.125, 1.0], [2.5, 4.0, 7.0], [0.0, -2.0, -5.0]],
                dtype=np.float32)


def _edges_csr():
    """``EDGES`` as a CSR matrix built from its arrays, so the duplicate entries stay stored."""
    import scipy.sparse as sp
    rows = [[d for s, d in EDGES if s == r] for r in range(5)]
    indptr = np.cumsum([0] + [len(r) for r in rows])
    return sp.csr_matrix((np.ones(len(EDGES), np.float32), np.array(sum(rows, []), np.int32), indptr), shape=(5, 5))


def _edges_coo():
    import scipy.sparse as sp
    s, d = zip(*EDGES)
    return sp.coo_matrix((np.ones(len(EDGES), np.float32), (np.array(s), np.array(d))), shape=(5, 5))


def _reddit(root):
    import scipy.sparse as sp
    d = os.path.join(root, "reddit")
    os.makedirs(d, exist_ok=True)
    np.savez(os.path.join(d, "reddit_data.npz"), feature=FEAT, label=np.array([0, 2, 1, 2, 0]),
             node_types=np.array([1, 2, 3, 1, 3]))
    sp.save_npz(os.path.join(d, "reddit_graph.npz"), _edges_csr())
    return d


def _yelp(root):
    import scipy.sparse as sp
    d = os.path.join(root, "yelp")
    os.makedirs(d, exist_ok=True)
    sp.save_npz(os.path.join(d, "adj_full.npz"), _edges_coo())
    np.save(os.path.join(d, "feats.npy"), FEAT)
    with open(os.path.join(d, "class_map.json"), "w") as f:
        json.dump({"0": [1, 0, 1, 0], "1": [0, 0, 0, 0], "2": [1, 1, 1, 1], "3": [0, 1, 0, 0], "4": [0, 0, 0, 1]}, f)
    with open(os.path.join(d, "role.json"), "w") as f:
        json.dump({"tr": [3, 0, 1], "va": [4], "te": [2]}, f)     # column 2 is 7.0 on every training row
    return d


def _gz(path, text):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with gzip.open(path, "wt") as f:
        f.write(text)


# raw products edges (src, dst): 0 -> 1, 1 -> 2 twice, the self-loop 3 -> 3, 2 -> 0; the reader adds every inverse
PRODUCTS_EDGES = "0,1\n1,2\n1,2\n3,3\n2,0\n"
PRODUCTS_INDPTR = [0, 3, 7, 11, 12, 13]
PRODUCTS_SRC = [0, 1, 2, 0, 1, 2, 2, 0, 1, 1, 2, 3, 4]
PRODUCTS_FEAT = "0.5,-1.25,7\n1.5,2,7\n-3,0.125,1\n2.5,4,7\n0,-2,-5\n"


def _products(root):
    raw = os.path.join(root, "ogbn_products", "raw")
    split = os.path.join(root, "ogbn_products", "split", "sales_ranking")
    _gz(os.path.join(raw, "edge.csv.gz"), PRODUCTS_EDGES)
    _gz(os.path.join(raw, "node-feat.csv.gz"), PRODUCTS_FEAT)
    _gz(os.path.join(raw, "node-label.csv.gz"), "0\n2\n1\n2\n0\n")
    _gz(os.path.join(raw, "num-node-list.csv.gz"), "5\n")
    _gz(os.path.join(split, "train.csv.gz"), "3\n0\n")          # unsorted
    _gz(os.path.join(split, "valid.csv.gz"), "1\n")
    _gz(os.path.join(split, "test.csv.gz"), "4\n2\n")
    return os.path.join(root, "ogbn_products")


def _mask(ids):
    m = torch.zeros(5, dtype=torch.bool)
    m[list(ids)] = True
    return m


def _assert_graph(g, indptr, src, feat, label, train, val, test, n_class):
    assert g.n_nodes == 5 and g.n_class == n_class
    assert g.indptr.dtype == torch.int64 and g.indptr.tolist() == indptr
    assert g.src.dtype == torch.int64 and g.src.tolist() == src
    assert g.feat.dtype == torch.float32 and torch.equal(g.feat, torch.as_tensor(feat))
    assert g.label.dtype == label.dtype and torch.equal(g.label, label)
    for m, want in ((g.train_mask, train), (g.val_mask, val), (g.test_mask, test)):
        assert m.dtype == torch.bool and torch.equal(m, _mask(want))


def test_reddit_fixture(tmp_path):
    _reddit(tmp_path)
    g = load_files("reddit", str(tmp_path), CPU)
    _assert_graph(g, WANT_INDPTR, WANT_SRC, FEAT, torch.tensor([0, 2, 1, 2, 0]), [0, 3], [1], [2, 4], 3)
    assert g.in_degrees().tolist() == [3, 3, 3, 1, 1]                # 1 -> 2 counts twice into node 2
    assert g.out_degrees().tolist() == WANT_OUT_DEG                  # and twice out of node 1
    assert g.src[g.indptr[4]:g.indptr[5]].tolist() == [4]            # the isolated node keeps its one self-loop


def test_yelp_fixture(tmp_path):
    _yelp(tmp_path)
    g = load_files("yelp", str(tmp_path), CPU)
    label = torch.tensor([[1, 0, 1, 0], [0, 0, 0, 0], [1, 1, 1, 1], [0, 1, 0, 0], [0, 0, 0, 1]], dtype=torch.float32)
    assert g.indptr.tolist() == WANT_INDPTR and g.src.tolist() == WANT_SRC
    assert g.out_degrees().tolist() == WANT_OUT_DEG
    assert g.label.dtype == torch.float32 and torch.equal(g.label, label) and g.n_class == 4
    assert torch.equal(g.train_mask, _mask([0, 1, 3])) and torch.equal(g.val_mask, _mask([4]))
    assert torch.equal(g.test_mask, _mask([2]))
    # the standard scaling restated in float64: mean and population variance over the training rows, scale 1 where
    # the variance is 0 (column 2: only centred)
    x = torch.from_numpy(FEAT).double()
    tr = x[[0, 1, 3]]
    mean, var = tr.mean(0), tr.var(0, unbiased=False)
    scale = torch.where(var == 0, torch.ones_like(var), var.sqrt())
    want = ((x - mean) / scale).float()
    ulp = (torch.nextafter(want.abs(), torch.tensor(float("inf"))) - want.abs())
    assert ((g.feat - want).abs() <= ulp).all(), (g.feat, want)
    assert torch.equal(g.feat[:, 2], torch.from_numpy(FEAT[:, 2] - 7.0))
    assert g.feat.dtype == torch.float32


def test_products_fixture(tmp_path):
    _products(tmp_path)
    g = load_files("ogbn-products", str(tmp_path), CPU)
    _assert_graph(g, PRODUCTS_INDPTR, PRODUCTS_SRC, FEAT, torch.tensor([0, 2, 1, 2, 0]), [0, 3], [1], [2, 4], 3)
    assert g.in_degrees().tolist() == [3, 4, 4, 1, 1]                # the stored self-loop 3 -> 3 became one loop
    assert g.out_degrees().tolist() == [3, 4, 4, 1, 1]               # every raw edge and its inverse


def _same(a, b):
    assert (a.n_nodes, a.n_class) == (b.n_nodes, b.n_class)
    for k in ("indptr", "src", "feat", "label", "train_mask", "val_mask", "test_mask"):
        x, y = getattr(a, k), getattr(b, k)
        assert x.dtype == y.dtype and x.shape == y.shape and torch.equal(x, y), k


@pytest.mark.parametrize("shape,layout", [("tiny", "reddit"), ("tiny", "ogbn-products"), ("tiny-ml", "yelp"),
                                          ("small", "reddit"), ("small", "ogbn-products")])
def test_round_trip_is_bit_identical(tmp_path, shape, layout):
    from bns_gcn_b200.data import make_graph
    from tools.dataset_files import WRITERS, standard_scaled
    fg = make_graph(shape, seed=0, device=CPU)
    WRITERS[layout](fg, str(tmp_path))
    g = load_files(layout, str(tmp_path), CPU)
    _same(g, standard_scaled(fg) if layout == "yelp" else fg)


# ---- refusals ----------------------------------------------------------------------------------------------------

def _rewrite_npz(path, **change):
    with np.load(path) as z:
        d = {k: z[k] for k in z.files}
    for k, v in change.items():
        if v is None:
            d.pop(k)
        else:
            d[k] = v
    np.savez(path, **d)


def _save_sparse(path, m):
    import scipy.sparse as sp
    sp.save_npz(path, m)


def _json(path, fn):
    with open(path) as f:
        obj = json.load(f)
    fn(obj)
    with open(path, "w") as f:
        json.dump(obj, f)


def _bad_feat(v):
    f = FEAT.copy()
    f[2, 1] = v
    return f


BAD = {
    # reddit
    "reddit-no-graph": ("reddit", "reddit/reddit_graph.npz", "no such file",
                        lambda d: os.remove(os.path.join(d, "reddit/reddit_graph.npz"))),
    "reddit-no-key": ("reddit", "reddit/reddit_data.npz", "no key 'label'",
                      lambda d: _rewrite_npz(os.path.join(d, "reddit/reddit_data.npz"), label=None)),
    "reddit-feature-rows": ("reddit", "reddit/reddit_data.npz", "4 feature rows for 5 nodes",
                            lambda d: _rewrite_npz(os.path.join(d, "reddit/reddit_data.npz"), feature=FEAT[:4])),
    "reddit-label-count": ("reddit", "reddit/reddit_data.npz", "6 labels for 5 nodes",
                           lambda d: _rewrite_npz(os.path.join(d, "reddit/reddit_data.npz"),
                                                  label=np.zeros(6, np.int64))),
    "reddit-node-types": ("reddit", "reddit/reddit_data.npz", "4 node types for 5 nodes",
                          lambda d: _rewrite_npz(os.path.join(d, "reddit/reddit_data.npz"),
                                                 node_types=np.ones(4, np.int64))),
    "reddit-negative-label": ("reddit", "reddit/reddit_data.npz", "negative label -1 at node 3",
                              lambda d: _rewrite_npz(os.path.join(d, "reddit/reddit_data.npz"),
                                                     label=np.array([0, 2, 1, -1, 0]))),
    "reddit-nan-feature": ("reddit", "reddit/reddit_data.npz", "non-finite feature nan at node 2, column 1",
                           lambda d: _rewrite_npz(os.path.join(d, "reddit/reddit_data.npz"),
                                                  feature=_bad_feat(np.nan))),
    "reddit-not-square": ("reddit", "reddit/reddit_graph.npz", "5 x 6, not square",
                          lambda d: _save_sparse(os.path.join(d, "reddit/reddit_graph.npz"),
                                                 _edges_csr()[:, [0, 1, 2, 3, 4, 4]])),
    # yelp
    "yelp-no-feats": ("yelp", "yelp/feats.npy", "no such file", lambda d: os.remove(os.path.join(d, "yelp/feats.npy"))),
    "yelp-feat-rows": ("yelp", "yelp/feats.npy", "6 feature rows for 5 nodes",
                       lambda d: np.save(os.path.join(d, "yelp/feats.npy"), np.zeros((6, 3), np.float32))),
    "yelp-inf-feature": ("yelp", "yelp/feats.npy", "non-finite feature inf at node 2, column 1",
                         lambda d: np.save(os.path.join(d, "yelp/feats.npy"), _bad_feat(np.inf))),
    "yelp-class-map-count": ("yelp", "yelp/class_map.json", "4 entries for 5 nodes",
                             lambda d: _json(os.path.join(d, "yelp/class_map.json"), lambda o: o.pop("2"))),
    "yelp-not-multi-hot": ("yelp", "yelp/class_map.json", "not rows of 0 / 1",
                           lambda d: _json(os.path.join(d, "yelp/class_map.json"),
                                           lambda o: o.__setitem__("1", [0, 2, 0, 0]))),
    "yelp-role-range": ("yelp", "yelp/role.json", "node id 5 outside [0, 5)",
                        lambda d: _json(os.path.join(d, "yelp/role.json"), lambda o: o["te"].append(5))),
    "yelp-role-key": ("yelp", "yelp/role.json", "no key 'va'",
                      lambda d: _json(os.path.join(d, "yelp/role.json"), lambda o: o.pop("va"))),
    "yelp-not-square": ("yelp", "yelp/adj_full.npz", "6 x 5, not square",
                        lambda d: _save_sparse(os.path.join(d, "yelp/adj_full.npz"), _edges_csr()[[0, 1, 2, 3, 4, 4]])),
    # ogbn-products
    "products-no-node-count": ("ogbn-products", "ogbn_products/raw/num-node-list.csv.gz", "no such file",
                               lambda d: os.remove(os.path.join(d, "ogbn_products/raw/num-node-list.csv.gz"))),
    "products-edge-range": ("ogbn-products", "ogbn_products/raw/edge.csv.gz", "node id 5 outside [0, 5)",
                            lambda d: _gz(os.path.join(d, "ogbn_products/raw/edge.csv.gz"), PRODUCTS_EDGES + "4,5\n")),
    "products-split-range": ("ogbn-products", "ogbn_products/split/sales_ranking/valid.csv.gz",
                             "node id -1 outside [0, 5)",
                             lambda d: _gz(os.path.join(d, "ogbn_products/split/sales_ranking/valid.csv.gz"),
                                           "1\n-1\n")),
    "products-feature-rows": ("ogbn-products", "ogbn_products/raw/node-feat.csv.gz", "6 feature rows for 5 nodes",
                              lambda d: _gz(os.path.join(d, "ogbn_products/raw/node-feat.csv.gz"),
                                            PRODUCTS_FEAT + "1,1,1\n")),
    "products-inf-feature": ("ogbn-products", "ogbn_products/raw/node-feat.csv.gz", "non-finite feature inf",
                             lambda d: _gz(os.path.join(d, "ogbn_products/raw/node-feat.csv.gz"),
                                           PRODUCTS_FEAT.replace("0.125", "inf"))),
    "products-label-count": ("ogbn-products", "ogbn_products/raw/node-label.csv.gz", "4 labels for 5 nodes",
                             lambda d: _gz(os.path.join(d, "ogbn_products/raw/node-label.csv.gz"), "0\n1\n2\n0\n")),
    "products-negative-label": ("ogbn-products", "ogbn_products/raw/node-label.csv.gz", "negative label -2 at node 1",
                                lambda d: _gz(os.path.join(d, "ogbn_products/raw/node-label.csv.gz"),
                                              "0\n-2\n1\n2\n0\n")),
    "products-ragged-edges": ("ogbn-products", "ogbn_products/raw/edge.csv.gz", "malformed edge list",
                              lambda d: _gz(os.path.join(d, "ogbn_products/raw/edge.csv.gz"), "0,1\n2\n")),
}
FIXTURES = {"reddit": _reddit, "yelp": _yelp, "ogbn-products": _products}


def _store_args(tmp_path, dataset, **kw):
    d = dict(dataset=dataset, data_source="files", data_path=str(tmp_path / "data"), n_partitions=2,
             partition_method="random", partition_obj="vol", inductive=False, part_path=str(tmp_path / "part"),
             graph_name="", graph_seed=0)
    d.update(kw)
    return argparse.Namespace(**d)


@pytest.mark.parametrize("case", sorted(BAD))
def test_malformed_input_is_refused_before_the_store_is_written(tmp_path, case):
    from bns_gcn_b200.data import graph_partition
    dataset, rel, what, spoil = BAD[case]
    root = tmp_path / "data"
    FIXTURES[dataset](str(root))
    load_files(dataset, str(root), CPU)                              # the unspoilt fixture loads
    spoil(str(root))
    with pytest.raises(DataFileError) as e:
        graph_partition(_store_args(tmp_path, dataset), device=CPU)
    msg = str(e.value)
    assert msg.startswith(os.path.join(str(root), rel) + ":"), msg
    assert what in msg, msg
    assert not (tmp_path / "part").exists()


# ---- the flag and the names ----------------------------------------------------------------------------------------

def test_flag_defaults_to_the_generator_and_takes_both_spellings():
    from bns_gcn_b200.helper.parser import create_parser
    assert create_parser([]).data_source == "synthetic"
    assert create_parser(["--data-source", "files"]).data_source == "files"
    assert create_parser(["--data_source", "files"]).data_source == "files"
    assert create_parser(["--data-source", "synthetic"]).data_source == "synthetic"
    with pytest.raises(SystemExit):
        create_parser(["--data-source", "download"])


@pytest.mark.parametrize("name", ["ogbn-papers100m", "papers100m"])
def test_papers100m_from_files_is_refused(tmp_path, name):
    with pytest.raises(ValueError, match="111 M nodes and 57 GB of features"):
        load_files(name, str(tmp_path), CPU)


@pytest.mark.parametrize("name", ["tiny", "synthetic-10k", "ogbn-arxiv", "Reddit"])
def test_other_names_are_refused(tmp_path, name):
    with pytest.raises(ValueError, match="no published layout is read for it"):
        load_files(name, str(tmp_path), CPU)


def test_load_graph_chooses_by_the_source(tmp_path):
    from bns_gcn_b200.data import load_graph, make_graph
    _reddit(str(tmp_path / "data"))
    _same(load_graph(_store_args(tmp_path, "reddit"), CPU), load_files("reddit", str(tmp_path / "data"), CPU))
    a = _store_args(tmp_path, "tiny", data_source="synthetic", graph_seed=3)
    _same(load_graph(a, CPU), make_graph("tiny", seed=3, device=CPU))
    del a.data_source                                                # a namespace from before the flag: the generator
    _same(load_graph(a, CPU), make_graph("tiny", seed=3, device=CPU))
    with pytest.raises(ValueError, match="--data-source 'web'"):
        load_graph(_store_args(tmp_path, "reddit", data_source="web"), CPU)


def test_files_and_synthetic_stores_get_different_names():
    from bns_gcn_b200.data import default_graph_name
    kw = dict(dataset="reddit", n_partitions=2, partition_method="metis", partition_obj="vol", inductive=True)
    assert default_graph_name(argparse.Namespace(data_source="files", **kw)) == "reddit-files-2-metis-vol-induc"
    assert default_graph_name(argparse.Namespace(data_source="synthetic", **kw)) == "reddit-2-metis-vol-induc"
    assert default_graph_name(argparse.Namespace(**kw)) == "reddit-2-metis-vol-induc"


def test_store_records_its_source_and_refuses_the_other(tmp_path):
    from bns_gcn_b200.data import graph_partition, load_partition
    _reddit(str(tmp_path / "data"))
    files = _store_args(tmp_path, "reddit")
    cfg_path = graph_partition(files, device=CPU)
    assert os.path.basename(cfg_path) == "reddit-files-2-random-vol-trans.json"
    with open(cfg_path) as f:
        assert json.load(f)["data_source"] == "files"
    g, nd, _ = load_partition(_store_args(tmp_path, "reddit", graph_name=files.graph_name), 0)
    assert g.n_in + load_partition(_store_args(tmp_path, "reddit", graph_name=files.graph_name), 1)[0].n_in == 5
    synth = _store_args(tmp_path, "reddit", data_source="synthetic", graph_name=files.graph_name)
    with pytest.raises(RuntimeError, match="partitioned from --data-source files, this run reads --data-source synthetic"):
        load_partition(synth, 0)
    with pytest.raises(RuntimeError, match="--data-source files"):
        graph_partition(synth, device=CPU)                           # refused before the graph is built


def test_store_without_a_recorded_source_is_synthetic(tmp_path):
    from bns_gcn_b200.data import graph_partition, load_partition, make_graph
    a = _store_args(tmp_path, "tiny", data_source="synthetic")
    cfg_path = graph_partition(a, fg=make_graph("tiny", seed=0, device=CPU), device=CPU)
    assert os.path.basename(cfg_path) == "tiny-2-random-vol-trans.json"
    with open(cfg_path) as f:
        cfg = json.load(f)
    assert cfg.pop("data_source") == "synthetic"
    with open(cfg_path, "w") as f:                                   # a store written before the key existed
        json.dump(cfg, f)
    load_partition(_store_args(tmp_path, "tiny", data_source="synthetic", graph_name=a.graph_name), 0)
    load_partition(argparse.Namespace(**{k: v for k, v in vars(a).items() if k != "data_source"}), 0)
    with pytest.raises(RuntimeError, match="partitioned from --data-source synthetic"):
        load_partition(_store_args(tmp_path, "tiny", graph_name=a.graph_name), 0)
