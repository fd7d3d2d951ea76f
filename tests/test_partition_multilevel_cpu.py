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


def _admit_case(seed, n_parts=6, n=400):
    """Unique movers with weights 1..4, gains from a small range (many ties) and sizes around [lo, hi]."""
    g = torch.Generator().manual_seed(seed)
    nodes = torch.randperm(4 * n, generator=g)[:n]
    frm = torch.randint(0, n_parts, (n,), generator=g)
    to = (frm + torch.randint(1, n_parts, (n,), generator=g)) % n_parts
    gain = torch.randint(-2, 3, (n,), generator=g)
    wt = torch.randint(1, 5, (n,), generator=g)
    sizes = torch.randint(90, 131, (n_parts,), generator=g)
    return nodes, to, gain, wt, frm, sizes


_ADMIT_MODES = {
    "cap": lambda s: dict(hi=125),
    "cap-floor": lambda s: dict(hi=125, lo=95),
    "need-in": lambda s: dict(hi=125, lo=95, need_in=(110 - s).clamp(min=0)),
    "need-out": lambda s: dict(hi=125, need_out=(s - 110).clamp(min=0)),
}


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("mode", sorted(_ADMIT_MODES))
def test_admit_is_the_running_sum_prefix(mode, seed):
    """admit against its move-by-move restatement: per target in (gain desc, id) order, the running weight of every
    earlier candidate (admitted or not) counts; then per source over the survivors."""
    from bns_gcn_b200.data.multilevel import admit
    from tests import partition_reference as R
    nodes, to, gain, wt, frm, sizes = _admit_case(seed)
    kw = _ADMIT_MODES[mode](sizes)
    got_n, got_t = admit(nodes, to, gain, wt, frm, sizes, **kw)
    got = sorted(zip(got_n.tolist(), got_t.tolist()))
    assert got == R.admit(nodes, to, gain, wt, frm, sizes, **kw)
    assert 0 < len(got) < nodes.numel()                 # the case is neither trivial nor empty


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("mode", sorted(_ADMIT_MODES))
def test_admitted_moves_keep_the_bounds_in_any_subset(mode, seed):
    """"The bounds hold whatever subset is applied": every part that started at or below ``hi`` stays there, and with a
    floor, every part that started inside [lo, hi] stays inside, for the whole admitted set, its halves and random
    subsets."""
    from bns_gcn_b200.data.multilevel import admit
    nodes, to, gain, wt, frm, sizes = _admit_case(seed)
    kw = _ADMIT_MODES[mode](sizes)
    hi, lo = kw["hi"], kw.get("lo")
    got_n, got_t = admit(nodes, to, gain, wt, frm, sizes, **kw)
    where = {int(v): i for i, v in enumerate(nodes.tolist())}
    idx = torch.tensor([where[int(v)] for v in got_n.tolist()], dtype=torch.int64)
    assert torch.equal(to[idx], got_t)
    g = torch.Generator().manual_seed(100 + seed)
    k = idx.numel()
    subsets = [torch.ones(k, dtype=torch.bool), torch.arange(k) < k // 2, torch.arange(k) >= k // 2]
    subsets += [torch.rand(k, generator=g) < p for p in (0.1, 0.5, 0.9) for _ in range(20)]
    for sel in subsets:
        i = idx[sel]
        after = sizes.clone()
        after.index_add_(0, to[i], wt[i])
        after.index_add_(0, frm[i], -wt[i])
        assert torch.all(after[sizes <= hi] <= hi), (sizes, after)
        if lo is not None:
            inside = (sizes >= lo) & (sizes <= hi)
            assert torch.all(after[inside] >= lo), (sizes, after)


@pytest.mark.parametrize("P", [5, 33, 64])
def test_gain_restatements_are_the_single_move_delta(P):
    """The host gain restatements the GPU tests compare the kernels with (partition_reference.cut_gains / vol_gains)
    against brute force: the directed objective before and after moving one node."""
    from tests import partition_reference as R
    fg = R.random_graph(60, 500, seed=P)
    n = fg.n_nodes
    part = torch.randint(0, P, (n,), generator=torch.Generator().manual_seed(P)).int()
    src, dst = fg.src, fg.dst()
    g2 = R.edges(fg.indptr, fg.src, None, n, 2, True)
    out_g, in_g = R.edges(fg.indptr, fg.src, None, n, 1, True), R.edges(fg.indptr, fg.src, None, n, 0, True)
    nodes = list(range(n))
    tables = {"cut": R.cut_gains(*g2, part, P, nodes), "vol": R.vol_gains(out_g, in_g, part, P, nodes)}
    hp = part.long()
    for k, objective in enumerate(("cut", "vol")):
        base = R.directed_objective(src, dst, hp, P)[k]
        for v in range(0, n, 3):
            for b in range(P):
                trial = hp.clone()
                trial[v] = b
                assert int(tables[objective][v, b]) == base - R.directed_objective(src, dst, trial, P)[k], (v, b)


def test_best_target_restatement_with_masks():
    from tests import partition_reference as R
    g = torch.tensor([[0, 3, 3, -1], [5, 0, 1, 1], [2, 2, 0, 7]])
    part = torch.tensor([0, 1, 2])
    t, b = R.best_target(g, part)
    assert t.tolist() == [1, 0, 3] and b.tolist() == [3, 5, 7]
    t, b = R.best_target(g, part, 0b1100)
    assert t.tolist() == [2, 2, 3] and b.tolist() == [3, 1, 7]
    t, b = R.best_target(g, part, 0b0100)
    assert t.tolist() == [2, 2, -1] and b.tolist() == [3, 1, 0]
    t, b = R.best_target(g, part, 1 << 63)
    assert t.tolist() == [-1, -1, -1] and b.tolist() == [0, 0, 0]
