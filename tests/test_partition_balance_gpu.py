"""``--partition-balance edges`` on the GPU: the two-cap clustering kernel and the int64 weight sums against host
restatements, the multilevel partitioner under both bounds, and a training run on edge-balanced parts from the store."""
import argparse

import numpy as np
import pytest
import torch

from tests import partition_reference as R

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _cluster_step_edges(rating, label, nw, cw, cap, ew, ce, ecap, seed):
    """bns_part_cluster_edges, node by node: R.cluster_step with the second cap."""
    ip, cid, wt = (t.cpu().long() for t in rating)
    label, cw, ew, ce = label.cpu().long(), cw.cpu().long(), ew.cpu().long(), ce.cpu().long()
    n = label.numel()
    nwl = nw.cpu().long() if nw is not None else torch.ones(n, dtype=torch.int64)
    tgt, gain = torch.full((n,), -1, dtype=torch.int32), torch.zeros(n, dtype=torch.int64)
    for v in range(n):
        if not R.part_hash(seed ^ ((v * 0x9E3779B97F4A7C15) & R.M64)) & 1:
            continue
        cur, best = 0, None
        for k in range(int(ip[v]), int(ip[v + 1])):
            c, w = int(cid[k]), int(wt[k])
            if c == int(label[v]):
                cur = w
                continue
            if int(cw[c]) + int(nwl[v]) > cap or int(ce[c]) + int(ew[v]) > ecap:
                continue
            key = (-w, R.part_hash(seed + c), c)
            if best is None or key < best:
                best = key
        if best is not None and -best[0] > cur:
            tgt[v], gain[v] = best[2], -best[0] - cur
    return tgt, gain


def _active(v, seed):
    return R.part_hash(seed ^ ((v * 0x9E3779B97F4A7C15) & R.M64)) & 1


def test_two_cap_cluster_kernel_on_crafted_rows(built):
    """Rows whose candidate clusters sit exactly at either cap, one above, ties in weight (broken by the seeded hash
    and by id), a hub whose in-edges alone exceed the cap, and an empty row."""
    from bns_gcn_b200 import ops
    seed = 12345
    n_pool, cap, ecap = 8, 10, 100
    # pool clusters 0 .. 7: (node weight, in-edge weight)
    cw = [4, 6, 7, 3, 9, 2, 5, 5]
    ce = [40, 60, 90, 99, 10, 101, 50, 50]
    movers = [v for v in range(n_pool, n_pool + 4000) if _active(v, seed)][:6]
    n = movers[-1] + 1
    label = torch.arange(n)                                   # every node alone in its own cluster
    nw = torch.ones(n, dtype=torch.int32)
    ew = torch.ones(n, dtype=torch.int64)
    cwt = torch.zeros(n, dtype=torch.int64)
    cet = torch.zeros(n, dtype=torch.int64)
    cwt[:n_pool], cet[:n_pool] = torch.tensor(cw), torch.tensor(ce)
    rows = {v: [] for v in range(n)}
    # mover 0 (nw 1, ew 10): cluster 2 ends at 100 in-edges exactly (ok), cluster 3 at 109 (no), cluster 1 at 7 nodes
    v = movers[0]
    ew[v] = 10
    rows[v] = [(1, 2), (2, 5), (3, 9)]
    # mover 1 (nw 6): cluster 0 reaches the node cap exactly (4 + 6 = 10), cluster 4 passes it
    v = movers[1]
    nw[v] = 6
    rows[v] = [(0, 3), (4, 8)]
    # mover 2: three clusters tied at weight 4 with room (0, 6, 7): the seeded hash picks, then the id
    rows[movers[2]] = [(0, 4), (6, 4), (7, 4)]
    # mover 3: a hub whose in-edges exceed the cap alone: no cluster takes it
    v = movers[3]
    ew[v] = 150
    rows[v] = [(0, 9), (4, 2)]
    # mover 4: cluster 5 is already above the in-edge cap, cluster 3 at 99 takes one in-edge exactly
    rows[movers[4]] = [(3, 1), (5, 7)]
    # mover 5: empty row
    ip = [0]
    cid, wt = [], []
    for u in range(n):
        for c, w in sorted(rows[u]):
            cid.append(c)
            wt.append(w)
        ip.append(len(cid))
    rating = (torch.tensor(ip, dtype=torch.int64).to(DEV), torch.tensor(cid, dtype=torch.int32).to(DEV),
              torch.tensor(wt, dtype=torch.int32).to(DEV))
    args = (label.to(DEV, torch.int32), nw.to(DEV), cwt.to(DEV), cap)
    t, g = ops.part_cluster(rating, *args, seed, ew=ew.to(DEV), ce=cet.to(DEV), ecap=ecap)
    th, gh = _cluster_step_edges(rating, args[0], nw, cwt, cap, ew, cet, ecap, seed)
    assert torch.equal(t.cpu(), th) and torch.equal(g.cpu(), gh)
    t = t.cpu()
    assert int(t[movers[0]]) == 2 and int(t[movers[1]]) == 0 and int(t[movers[3]]) == -1
    assert int(t[movers[4]]) == 3 and int(t[movers[5]]) == -1
    assert int(t[movers[2]]) in (0, 6, 7)
    # with the in-edge cap out of reach it is the one-cap kernel, proposal for proposal
    t1, g1 = ops.part_cluster(rating, *args, seed)
    t2, g2 = ops.part_cluster(rating, *args, seed, ew=ew.to(DEV), ce=cet.to(DEV), ecap=1 << 60)
    assert torch.equal(t1, t2) and torch.equal(g1, g2)


@pytest.mark.parametrize("name", ["tiny", "small"])
def test_two_cap_cluster_step_on_graphs(built, name):
    from bns_gcn_b200 import ops
    from bns_gcn_b200.data import make_graph
    from bns_gcn_b200.data import multilevel as ml
    fg = make_graph(name, seed=0)
    n = fg.n_nodes
    ip, ix = fg.indptr.to(DEV), fg.src.to(DEV, torch.int32)
    g0 = ml.Csr(*ops.part_edges(ip, ix, None, n, 2, True))
    ew = (ip[1:] - ip[:-1]).contiguous()
    for layout in ("pairs", "blocks"):
        label = (torch.arange(n) // (2 if layout == "pairs" else 7)).to(DEV, torch.int32)
        rating = ops.part_edges(g0.indptr, g0.idx, g0.w, n, 0, False, col_map=label)
        cw = ops.part_weights(label, None, n)
        ce = ops.part_weights(label, ew, n)
        for ecap in (int(ce.max()), int(ce.float().mean()) + 1, 1):
            t, g = ops.part_cluster(rating, label, None, cw, 9, 7, ew=ew, ce=ce, ecap=ecap)
            th, gh = _cluster_step_edges(rating, label, None, cw, 9, ew, ce, ecap, 7)
            assert torch.equal(t.cpu(), th) and torch.equal(g.cpu(), gh), (layout, ecap)
    # clustering under both caps keeps every cluster within both
    lab = ml.cluster(g0, None, 6, seed=3, ew=ew, ecap=200)
    hl = lab.cpu().long()
    assert int(torch.bincount(hl, minlength=n).max()) <= 6
    ce = torch.zeros(n, dtype=torch.int64).index_add_(0, hl, ew.cpu())
    alone = torch.bincount(hl, minlength=n) == 1
    assert bool((ce[~alone] <= 200).all())                  # a node above the cap stays alone
    cmap, nc = ml.compact(lab)
    cg, cnw, cew = ml.contract(g0, None, cmap, nc, ew)
    assert cew.dtype == torch.int64 and int(cew.sum()) == fg.n_edges
    assert torch.equal(cew.cpu(), torch.zeros(nc, dtype=torch.int64).index_add_(0, cmap.cpu().long(), ew.cpu()))


def test_int64_weight_sums_are_exact_past_2_to_the_31(built):
    from bns_gcn_b200 import ops
    g = torch.Generator().manual_seed(0)
    n, L = 300_000, 37
    label = torch.randint(0, L, (n,), generator=g)
    w = torch.randint(0, 1 << 40, (n,), generator=g)
    w[:5] = (1 << 62) // 8                                   # five into label[0..4]: sums up to 2^61 and more
    out = ops.part_weights(label.to(DEV, torch.int32), w.to(DEV), L).cpu()
    want = torch.zeros(L, dtype=torch.int64).index_add_(0, label, w)
    assert torch.equal(out, want) and int(want.max()) > 2 ** 31
    one = ops.part_weights(torch.zeros(3_000_000, dtype=torch.int32, device=DEV),
                           torch.full((3_000_000,), 1000, dtype=torch.int64, device=DEV), 1)
    assert int(one[0]) == 3_000_000_000


_GRAPHS = {}


def _graph(name):
    if name not in _GRAPHS:
        from bns_gcn_b200.data import make_graph
        if name == "blocks":
            _GRAPHS[name] = R.degree_corrected_blocks(232_965, 40, 50, 0.2, seed=0)[0]
        elif name == "grid":
            _GRAPHS[name] = R.grid_graph(512)
        else:
            _GRAPHS[name] = make_graph(name, seed=0)
    return _GRAPHS[name]


def _check(fg, part, P):
    from bns_gcn_b200.data.partition import in_edge_bound
    n = fg.n_nodes
    lo, hi = max(int(0.97 * n / P), 1), int(1.03 * n / P) + 1
    ehi = in_edge_bound(fg.in_degrees(), P)
    sizes = torch.bincount(part, minlength=P)
    esizes = torch.zeros(P, dtype=torch.int64).index_add_(0, part, fg.in_degrees())
    assert int(sizes.min()) >= lo and int(sizes.max()) <= hi, (sizes.tolist(), lo, hi)
    assert int(esizes.max()) <= ehi, (esizes.max(), ehi)
    return esizes


@pytest.mark.parametrize("P", [2, 4, 8, 33, 64])
@pytest.mark.parametrize("name", ["tiny", "small", "yelp", "blocks", "grid"])
def test_multilevel_edges_within_both_bounds_and_deterministic(built, name, P):
    from bns_gcn_b200.data.multilevel import multilevel_partition
    fg = _graph(name)
    a, info = multilevel_partition(fg, P, "vol", 0, balance="edges")
    esizes = _check(fg, a, P)
    assert (info["min_in_edges"], info["max_in_edges"]) == (int(esizes.min()), int(esizes.max()))
    b, _ = multilevel_partition(fg, P, "vol", 0, balance="edges")
    assert torch.equal(a, b)


def test_multilevel_edges_on_reddit(built):
    from bns_gcn_b200.data.multilevel import multilevel_partition
    fg = _graph("reddit")
    a, _ = multilevel_partition(fg, 8, "vol", 0, balance="edges")
    _check(fg, a, 8)
    assert torch.equal(a, multilevel_partition(fg, 8, "vol", 0, balance="edges")[0])


@pytest.mark.parametrize("name,P", [("reddit", 8), ("yelp", 4)])
def test_multilevel_edges_no_worse_than_the_stand_in_on_chung_lu(built, name, P):
    from bns_gcn_b200.data import assign_parts, partition_quality
    fg = _graph(name)
    ml_part = assign_parts(fg, P, "multilevel", 0, "vol", DEV, balance="edges")
    si_part = assign_parts(fg, P, "metis", 0, "vol", DEV, balance="edges")
    _check(fg, ml_part, P)
    assert partition_quality(fg, ml_part, P, DEV)["vol"] <= partition_quality(fg, si_part, P, DEV)["vol"]


def test_nodes_is_the_call_without_the_keyword(built):
    from bns_gcn_b200.data.multilevel import multilevel_partition
    fg = _graph("small")
    for P in (2, 8):
        a, _ = multilevel_partition(fg, P, "vol", 0)
        b, _ = multilevel_partition(fg, P, "vol", 0, balance="nodes")
        assert torch.equal(a, b)


def test_training_on_edge_balanced_parts_from_the_store(built, tmp_path, monkeypatch):
    """graph_partition -> load_partition -> the training step at 4 in-process ranks on ``small``: every loaded part's
    a_in + a_out nnz is within the in-edge bound and the losses are finite."""
    from bns_gcn_b200.data import graph_partition, load_as_partition, make_graph
    from bns_gcn_b200.data.partition import in_edge_bound
    from tests.harness import make_args, run_product
    monkeypatch.chdir(tmp_path)
    fg = make_graph("small", seed=0)
    ehi = in_edge_bound(fg.in_degrees(), 4)
    for method in ("multilevel", "metis"):
        args = make_args(dataset="small", n_partitions=4, partition_method=method, partition_obj="vol",
                         part_path=str(tmp_path / "part"), graph_name="", graph_seed=0, partition_balance="edges",
                         n_hidden=16, n_layers=2, sampling_rate=0.5)
        graph_partition(args, device=DEV)
        assert args.graph_name == f"small-4-{method}-vol-edges-trans"
        parts = [load_as_partition(argparse.Namespace(**vars(args)), r) for r in range(4)]
        assert sum(p.graph.num_edges() for p in parts) == fg.n_edges
        for p in parts:
            assert p.graph.num_edges() <= ehi
        out = run_product(parts, args, DEV, 3, capture=False)
        for r in range(4):
            assert np.isfinite(out[r]["loss"]).all()
