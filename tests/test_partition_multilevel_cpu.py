"""The host side of ``--partition-method multilevel``: the flag, the store name, the refusals and the host initial
partition of the coarsest graph."""
import argparse

import numpy as np
import pytest
import torch


def test_parser_accepts_multilevel_and_keeps_metis_the_default():
    from bns_gcn_b200.helper.parser import create_parser
    assert create_parser(["--partition-method", "multilevel"]).partition_method == "multilevel"
    assert create_parser(["--partition_method", "multilevel"]).partition_method == "multilevel"
    assert create_parser([]).partition_method == "metis"
    with pytest.raises(SystemExit):
        create_parser(["--partition-method", "kahip"])


def test_store_name():
    from bns_gcn_b200.data.store import default_graph_name
    a = argparse.Namespace(dataset="reddit", n_partitions=4, partition_method="multilevel", partition_obj="vol",
                           inductive=False, data_source="files")
    assert default_graph_name(a) == "reddit-files-4-multilevel-vol-trans"
    a.data_source, a.inductive, a.partition_obj = "synthetic", True, "cut"
    assert default_graph_name(a) == "reddit-4-multilevel-cut-induc"


def test_cpu_device_is_refused_with_the_cpu_choices():
    from bns_gcn_b200.data import make_graph, partition_graph
    fg = make_graph("tiny", seed=0, device=torch.device("cpu"))
    with pytest.raises(ValueError, match=r"CUDA device.*metis.*random"):
        partition_graph(fg, 2, "multilevel", device=torch.device("cpu"))
    from bns_gcn_b200.data.multilevel import check_parts
    for n, P, msg in ((100, 65, "<= 64"), (100, 0, "2 <= n_partitions"), (5, 6, "node count")):
        with pytest.raises(ValueError, match=msg):
            check_parts(n, P)


def _weighted_graph(n, m, seed):
    rng = np.random.default_rng(seed)
    a, b = rng.integers(0, n, m), rng.integers(0, n, m)
    keep = a != b
    a, b = a[keep], b[keep]
    w = rng.integers(1, 6, a.size)
    rows, cols, ws = np.concatenate([a, b]), np.concatenate([b, a]), np.concatenate([w, w])
    o = np.lexsort((cols, rows))
    rows, cols, ws = rows[o], cols[o], ws[o]
    indptr = np.zeros(n + 1, dtype=np.int64)
    indptr[1:] = np.cumsum(np.bincount(rows, minlength=n))
    nw = rng.integers(1, 4, n)
    return indptr, cols, ws, nw


@pytest.mark.parametrize("n,m,P", [(60, 200, 2), (300, 1500, 4), (500, 1200, 8), (40, 100, 40)])
def test_initial_partition_is_balanced_and_deterministic(n, m, P):
    from bns_gcn_b200.data.multilevel import initial_partition
    indptr, idx, w, nw = _weighted_graph(n, m, seed=n + P)
    if P == n:
        nw = np.ones(n, dtype=np.int64)
    total = int(nw.sum())
    lo, hi = max(int(0.97 * total / P), 1), int(1.03 * total / P) + 1
    hi_w = hi + int(nw.max())           # weighted nodes: a part may overshoot its share by less than one node
    a = initial_partition(indptr, idx, w, nw, P, lo, hi, seed=1)
    b = initial_partition(indptr, idx, w, nw, P, lo, hi, seed=1)
    assert np.array_equal(a, b) and a.dtype == np.int64 and a.shape == (n,)
    sizes = np.bincount(a, weights=nw, minlength=P)
    assert sizes.size == P and (sizes > 0).all() and sizes.max() <= hi_w, sizes
    assert sizes.min() >= lo - int(nw.max()), sizes
    # better than a random assignment of the same sizes
    rng = np.random.default_rng(0)
    rnd = rng.permutation(a)
    rows = np.repeat(np.arange(n), np.diff(indptr))
    assert w[a[rows] != a[idx]].sum() <= w[rnd[rows] != rnd[idx]].sum()


def test_block_partition_is_balanced():
    from bns_gcn_b200.data.multilevel import block_partition
    indptr, idx, w, nw = _weighted_graph(400, 3000, seed=9)
    a = block_partition(indptr, idx, nw, 6)
    assert np.array_equal(a, block_partition(indptr, idx, nw, 6))
    sizes = np.bincount(a, weights=nw, minlength=6)
    assert (sizes > 0).all() and sizes.max() - sizes.min() <= 2 * nw.max(), sizes
