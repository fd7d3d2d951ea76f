"""The multilevel GPU partitioner (``--partition-method multilevel``): every kernel against its host restatement
(tests/partition_reference.py) and single-move brute force, the partition contract and size bounds, quality where the
answer is known, determinism, refusals, and training on its partitions."""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import pytest
import torch

from tests import partition_reference as R

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = torch.device("cuda:0")


def _graphs():
    return {
        "directed-multi": R.random_graph(80, 400, seed=1, isolated=5),
        "symmetric": R.random_graph(70, 300, seed=2, symmetric=True, multi=False),
        "star-components": R.star_plus_components(),
        "directed-dense": R.random_graph(40, 900, seed=3),
    }


def _csr(fg):
    return fg.indptr.to(DEV), fg.src.to(DEV, torch.int32)


def _same(dev_csr, host_csr):
    for a, b in zip(dev_csr, host_csr):
        assert torch.equal(a.cpu().long(), b.long())


@pytest.mark.parametrize("name", sorted(_graphs()))
def test_edges_match_the_host(built, name):
    from bns_gcn_b200 import ops
    fg = _graphs()[name]
    ip, ix = _csr(fg)
    n = fg.n_nodes
    for mode in (0, 1, 2):
        for drop in (False, True):
            _same(ops.part_edges(ip, ix, None, n, mode, drop), R.edges(ip, ix, None, n, mode, drop))
    g = torch.Generator().manual_seed(4)
    cmap = torch.randint(0, 9, (n,), generator=g).to(DEV, torch.int32)
    w = torch.randint(1, 5, (ix.numel(),), generator=g).to(DEV, torch.int32)
    _same(ops.part_edges(ip, ix, w, 9, 0, True, row_map=cmap, col_map=cmap),
          R.edges(ip, ix, w, 9, 0, True, cmap, cmap))
    _same(ops.part_edges(ip, ix, w, n, 0, False, col_map=cmap), R.edges(ip, ix, w, n, 0, False, None, cmap))


@pytest.mark.parametrize("name", sorted(_graphs()))
def test_clustering_respects_the_cap_and_contraction_is_exact(built, name):
    from bns_gcn_b200 import ops
    from bns_gcn_b200.data import multilevel as ml
    fg = _graphs()[name]
    n = fg.n_nodes
    ip, ix = _csr(fg)
    g0 = ml.Csr(*ops.part_edges(ip, ix, None, n, 2, True))
    # one step of the kernel equals its host restatement
    label = (torch.arange(n) // 2).to(DEV, torch.int32)
    rating = ops.part_edges(g0.indptr, g0.idx, g0.w, n, 0, False, col_map=label)
    cw = ops.part_weights(label, None, n)
    assert torch.equal(cw.cpu(), torch.bincount(label.cpu().long(), minlength=n))
    for seed in (1, 99):
        t, gn = ops.part_cluster(rating, label, None, cw, 3, seed)
        th, gh = R.cluster_step(rating, label, None, cw, 3, seed)
        assert torch.equal(t.cpu(), th) and torch.equal(gn.cpu(), gh)
    for cap in (1, 3, 7):
        lab = ml.cluster(g0, None, cap, seed=5)
        assert int(lab.min()) >= 0 and int(lab.max()) < n                      # every node is in a cluster
        assert int(torch.bincount(lab.cpu().long(), minlength=n).max()) <= cap
        cmap, nc = ml.compact(lab)
        cg, cnw = ml.contract(g0, None, cmap, nc)
        assert int(cnw.sum()) == n and int(cnw.max()) <= cap
        _same(cg, R.edges(g0.indptr, g0.idx, g0.w, nc, 0, True, cmap, cmap))
        # the coarse edge weights are the fine cross-cluster weights
        hc = cmap.cpu().long()
        rows = torch.repeat_interleave(torch.arange(n), (g0.indptr[1:] - g0.indptr[:-1]).cpu())
        cross = hc[rows] != hc[g0.idx.cpu().long()]
        assert int(cg.w.sum()) == int(g0.w.cpu()[cross].sum())
        # weighted nodes: a second level keeps the cap
        lab2 = ml.cluster(cg, cnw, 2 * cap, seed=6)
        assert int(torch.zeros(nc, dtype=torch.int64).index_add_(0, lab2.cpu().long(), cnw.cpu().long()).max()) <= 2 * cap


@pytest.mark.parametrize("name", sorted(_graphs()))
@pytest.mark.parametrize("P", [2, 3, 5, 31, 32, 33, 63, 64])
def test_conn_and_quality_are_exact(built, name, P):
    from bns_gcn_b200 import ops
    from bns_gcn_b200.data import partition_quality
    fg = _graphs()[name]
    n = fg.n_nodes
    ip, ix = _csr(fg)
    part = torch.randint(0, P, (n,), generator=torch.Generator().manual_seed(P)).to(DEV, torch.int32)
    for mode in (1, 2):
        g = ops.part_edges(ip, ix, None, n, mode, True)
        conn, occ, q = ops.part_conn(*g, part, P, occ=True, quality=True)
        ch, oh, qh = R.conn(*g, part, P)
        assert torch.equal(conn.cpu(), ch) and torch.equal(occ.cpu(), oh) and tuple(q.cpu().tolist()) == qh
    out = ops.part_edges(ip, ix, None, n, 1, True)
    _, _, q = ops.part_conn(*out, part, P, table=False, quality=True)
    pq = partition_quality(fg, part.cpu().long(), P)
    assert tuple(q.cpu().tolist()) == (pq["cut"], pq["vol"])


@pytest.mark.parametrize("name", sorted(_graphs()))
@pytest.mark.parametrize("objective", ["cut", "vol"])
@pytest.mark.parametrize("P", [4, 31, 32, 33, 63, 64])
def test_every_gain_is_the_single_move_delta(built, P, name, objective):
    """gain(v, b) == objective(before) - objective(after) of moving v alone to b, for every node and every target."""
    from bns_gcn_b200 import ops
    fg = _graphs()[name]
    n = fg.n_nodes
    ip, ix = _csr(fg)
    part = torch.randint(0, P, (n,), generator=torch.Generator().manual_seed(7)).to(DEV, torch.int32)
    if objective == "cut":
        conn, occ, _ = ops.part_conn(*ops.part_edges(ip, ix, None, n, 2, True), part, P)
        in_g = None
    else:
        conn, occ, _ = ops.part_conn(*ops.part_edges(ip, ix, None, n, 1, True), part, P, occ=True)
        in_g = ops.part_edges(ip, ix, None, n, 0, True)
    table = torch.zeros(n, P, dtype=torch.int64)
    for b in range(P):
        t, g = ops.part_gains(objective, part, conn, P, 1 << b, in_graph=in_g, occ=occ)
        t, g = t.cpu(), g.cpu()
        own = part.cpu() == b
        assert torch.all(t[own] == -1) and torch.all(t[~own] == b)
        table[:, b] = g
    src, dst = fg.src, fg.dst()
    hp = part.cpu().long()
    k = 0 if objective == "cut" else 1
    base = R.directed_objective(src, dst, hp, P)[k]
    for v in range(n):
        for b in range(P):
            if b == int(hp[v]):
                continue
            trial = hp.clone()
            trial[v] = b
            assert int(table[v, b]) == base - R.directed_objective(src, dst, trial, P)[k], (v, b)
    # the best target over all parts: largest gain, ties to the lowest part
    t, g = ops.part_gains(objective, part, conn, P, (1 << P) - 1, in_graph=in_g, occ=occ)
    th, gh = R.best_target(table, part)
    assert torch.equal(t.cpu(), th) and torch.equal(g.cpu(), gh)


def _check_contract(fg, parts, P):
    ranges = parts[0].gpb.ranges
    assert int(ranges[-1]) == fg.n_nodes and torch.all(ranges[1:] - ranges[:-1] > 0)
    n_edges = 0
    for r, p in enumerate(parts):
        nd, g = p.node_dict, p.graph
        assert g.n_in == int(ranges[r + 1] - ranges[r])
        assert torch.equal(nd["_ID"][:g.n_in], torch.arange(int(ranges[r]), int(ranges[r + 1])))
        assert nd["inner_node"][:g.n_in].all() and not nd["inner_node"][g.n_in:].any()
        assert torch.all(nd["part_id"][:g.n_in] == r) and torch.all(nd["part_id"][g.n_in:] != r)
        assert torch.equal(g.indptr[1:] - g.indptr[:-1], nd["in_deg"])
        if g.n_halo:
            assert g.indices.max() < g.n_in + g.n_halo and g.indices[g.indices >= g.n_in].unique().numel() == g.n_halo
        n_edges += g.num_edges()
        assert p.meta["n_train"] == int(fg.train_mask.sum())
    assert n_edges == fg.n_edges


def _bounds_hold(sizes, n, P):
    from bns_gcn_b200.data.multilevel import size_bounds
    lo, hi = size_bounds(n, P)
    assert int(0.97 * n / P) <= lo and hi == int(1.03 * n / P) + 1
    assert int(sizes.min()) >= lo and int(sizes.max()) <= hi and int(sizes.min()) > 0, (sizes.tolist(), lo, hi)


@pytest.mark.parametrize("inductive", [False, True])
@pytest.mark.parametrize("objective", ["cut", "vol"])
@pytest.mark.parametrize("P", [2, 3, 4, 8])
@pytest.mark.parametrize("shape", ["tiny", "small"])
def test_partition_contract(built, shape, P, objective, inductive):
    from bns_gcn_b200.data import induced_subgraph, make_graph, partition_graph
    fg = make_graph(shape, seed=1)
    parts = partition_graph(fg, P, "multilevel", seed=1, inductive=inductive, objective=objective)
    g = induced_subgraph(fg, fg.train_mask) if inductive else fg
    _check_contract(g, parts, P)
    _bounds_hold(parts[0].gpb.ranges[1:] - parts[0].gpb.ranges[:-1], g.n_nodes, P)


@pytest.mark.parametrize("case", ["small-64", "n-equals-p", "star-components", "directed-multi"])
def test_size_bounds_at_the_limits(built, case):
    from bns_gcn_b200.data import make_graph
    from bns_gcn_b200.data.multilevel import multilevel_partition
    if case == "small-64":
        fg, P = make_graph("small", seed=2), 64
    elif case == "n-equals-p":
        fg = R.random_graph(48, 200, seed=5)
        P = fg.n_nodes
    else:
        fg, P = _graphs()[case], 7
    for objective in ("cut", "vol"):
        part, info = multilevel_partition(fg, P, objective, seed=3)
        sizes = torch.bincount(part, minlength=P)
        assert sizes.numel() == P
        _bounds_hold(sizes, fg.n_nodes, P)
        assert (info["min_size"], info["max_size"]) == (int(sizes.min()), int(sizes.max()))


_CACHE = {}


def _reddit_blocks():
    if "reddit" not in _CACHE:
        _CACHE["reddit"] = R.degree_corrected_blocks(232_965, 40, 50, 0.2, seed=0)
    return _CACHE["reddit"]


def _compare(fg, planted, P, objective, factor):
    from bns_gcn_b200.data import assign_parts, partition_quality
    from bns_gcn_b200.data.multilevel import multilevel_partition
    part, info = multilevel_partition(fg, P, objective, seed=0)
    q = partition_quality(fg, part, P, DEV)
    assert (q["cut"], q["vol"]) == (info["cut"], info["vol"])
    standin = partition_quality(fg, assign_parts(fg, P, "metis", 0, objective, DEV), P, DEV)
    _bounds_hold(torch.bincount(part, minlength=P), fg.n_nodes, P)
    if planted is not None:
        assert q[objective] <= factor * planted[objective], (q, planted)
    assert q[objective] <= standin[objective], (q, standin)
    return q


@pytest.mark.parametrize("objective", ["cut", "vol"])
def test_finds_the_planted_blocks(built, objective):
    from bns_gcn_b200.data import partition_quality
    from tests.test_host_cpu import _planted_partition_graph
    for n, P in ((8000, 4), (65536, 8)):
        fg, blk = _planted_partition_graph(n, P, 16, 2)
        _compare(fg, partition_quality(fg, blk, P), P, objective, 1.05)


def test_grid_beats_the_strips(built):
    """The 512 x 512 four-neighbour grid at P = 4 with ``cut``: below the three-strip cut (3 x 512 undirected edges =
    3,072 directed ones) and no worse than the stand-in."""
    fg = R.grid_graph(512)
    q = _compare(fg, None, 4, "cut", None)
    assert q["cut"] < 3 * 512 * 2, q


@pytest.mark.parametrize("P", [4, 8])
def test_reddit_sized_block_model(built, P):
    from bns_gcn_b200.data import partition_quality
    fg, blk = _reddit_blocks()
    _compare(fg, partition_quality(fg, blk % P, P, DEV), P, "vol", 1.1)


def _reddit():
    if "reddit-shape" not in _CACHE:
        from bns_gcn_b200.data import make_graph
        _CACHE["reddit-shape"] = make_graph("reddit", seed=0)
    return _CACHE["reddit-shape"]


@pytest.mark.parametrize("objective", ["cut", "vol"])
@pytest.mark.parametrize("P", [2, 8])
def test_reddit_shape_is_no_worse_than_the_standin(built, P, objective):
    """The Reddit shape (Chung-Lu: no community structure, rows of ~19 k entries, 114.6 M edges): coarsening stalls
    there, and the result must still be no worse than the stand-in on the requested objective."""
    _compare(_reddit(), None, P, objective, None)


def test_deterministic(built):
    from bns_gcn_b200.data import make_graph
    from bns_gcn_b200.data.multilevel import multilevel_partition
    for fg, P in ((make_graph("small", seed=0), 4), (_reddit(), 8), (_reddit_blocks()[0], 8)):
        for objective in ("cut", "vol"):
            a, ia = multilevel_partition(fg, P, objective, seed=0)
            b, ib = multilevel_partition(fg, P, objective, seed=0)
            ia.pop("seconds"), ib.pop("seconds")               # the report's stage timings are the only difference
            assert torch.equal(a, b) and ia == ib


def test_device_cache_is_released(built):
    """main.py partitions in its parent process before the ranks start: the call must not leave its workspace reserved
    on the device the ranks train on."""
    from bns_gcn_b200.data import make_graph
    from bns_gcn_b200.data.multilevel import multilevel_partition
    fg = make_graph("small", seed=0)
    torch.cuda.synchronize()
    before = torch.cuda.memory_reserved(DEV)
    multilevel_partition(fg, 4, "vol", seed=0)
    assert torch.cuda.memory_reserved(DEV) <= before


def test_refusals(built):
    from bns_gcn_b200 import _lib
    from bns_gcn_b200.data import make_graph
    from bns_gcn_b200.data.multilevel import multilevel_partition
    fg = make_graph("tiny", seed=0)
    for P, msg in ((0, "2 <= n_partitions <= 64"), (65, "2 <= n_partitions <= 64"), (-3, "2 <= n_partitions")):
        with pytest.raises(ValueError, match=msg):
            multilevel_partition(fg, P)
    small = R.random_graph(10, 20, seed=0)
    with pytest.raises(ValueError, match="node count"):
        multilevel_partition(small, 11)
    with pytest.raises(ValueError, match="metis.*random"):
        multilevel_partition(fg, 2, device=torch.device("cpu"))
    assert torch.equal(multilevel_partition(fg, 1)[0], torch.zeros(fg.n_nodes, dtype=torch.int64))
    L = _lib.lib
    ip, ix = _csr(small)
    d = torch.zeros(64, dtype=torch.int64, device=DEV)
    out = ctypes.c_int64()
    ws = int(L.bns_part_edges_workspace_bytes(ix.numel()))
    bad = [
        L.bns_part_edges(small.n_nodes, ix.numel(), ip.data_ptr(), ix.data_ptr(), None, None, None, 3, 1, small.n_nodes,
                         d.data_ptr(), d.data_ptr(), d.data_ptr(), ctypes.byref(out), d.data_ptr(), ws, None),
        L.bns_part_edges(small.n_nodes, ix.numel(), None, ix.data_ptr(), None, None, None, 0, 1, small.n_nodes,
                         d.data_ptr(), d.data_ptr(), d.data_ptr(), ctypes.byref(out), d.data_ptr(), ws, None),
        L.bns_part_edges(small.n_nodes, ix.numel(), ip.data_ptr(), ix.data_ptr(), None, None, None, 0, 1, small.n_nodes,
                         d.data_ptr(), d.data_ptr(), d.data_ptr(), None, d.data_ptr(), ws, None),
        L.bns_part_edges(small.n_nodes, ix.numel(), ip.data_ptr(), ix.data_ptr(), None, None, None, 2, 1,
                         small.n_nodes - 1, d.data_ptr(), d.data_ptr(), d.data_ptr(), ctypes.byref(out), d.data_ptr(),
                         2 * ws, None),
        L.bns_part_conn(small.n_nodes, ip.data_ptr(), ix.data_ptr(), None, d.data_ptr(), 65, d.data_ptr(), None, None,
                        None),
        L.bns_part_conn(small.n_nodes, ip.data_ptr(), ix.data_ptr(), None, d.data_ptr(), 4, None, None, None, None),
        L.bns_part_conn(-1, ip.data_ptr(), ix.data_ptr(), None, d.data_ptr(), 4, d.data_ptr(), None, None, None),
        L.bns_part_gains(2, small.n_nodes, 4, None, None, None, d.data_ptr(), d.data_ptr(), None, 15, d.data_ptr(),
                         d.data_ptr(), None),
        L.bns_part_gains(0, small.n_nodes, 1, None, None, None, d.data_ptr(), d.data_ptr(), None, 15, d.data_ptr(),
                         d.data_ptr(), None),
        L.bns_part_gains(1, small.n_nodes, 4, None, None, None, d.data_ptr(), d.data_ptr(), None, 15, d.data_ptr(),
                         d.data_ptr(), None),
        L.bns_part_cluster(small.n_nodes, ip.data_ptr(), ix.data_ptr(), d.data_ptr(), d.data_ptr(), None, d.data_ptr(), 0,
                           0, d.data_ptr(), d.data_ptr(), None),
        L.bns_part_cluster(small.n_nodes, ip.data_ptr(), ix.data_ptr(), None, d.data_ptr(), None, d.data_ptr(), 4, 0,
                           d.data_ptr(), d.data_ptr(), None),
        L.bns_part_weights(small.n_nodes, d.data_ptr(), None, 0, d.data_ptr(), None),
        L.bns_part_weights(small.n_nodes, None, None, 4, d.data_ptr(), None),
    ]
    assert bad == [-1] * len(bad), bad
    assert L.bns_part_edges(small.n_nodes, ix.numel(), ip.data_ptr(), ix.data_ptr(), None, None, None, 0, 1,
                            small.n_nodes, d.data_ptr(), d.data_ptr(), d.data_ptr(), ctypes.byref(out), d.data_ptr(),
                            ws - 1, None) == -3
    assert L.bns_part_edges_workspace_bytes(-1) == 0


def test_training_parity_on_a_multilevel_partition(built):
    from tests.test_parity_gpu import _run
    _run(shape="tiny", n_parts=3, model="graphsage", sampling_rate=0.5, n_epochs=2, partition_method="multilevel")


@pytest.mark.parametrize("n_parts", [2, 3])
@pytest.mark.parametrize("case", ["graphsage", "gcn"])
def test_parallel_eval_logits_equal_the_whole_graph_evaluation(built, case, n_parts):
    from tests.test_parallel_eval_gpu import test_partition_logits_equal_the_whole_graph_evaluation as check
    check(built, case, n_parts, "multilevel")


def test_store_build_and_two_ranks_train(built, tmp_path):
    """The store ``graph_partition`` writes for ``main.py`` (name, ``part_method``), then 2 epochs at 2 in-process ranks
    from it."""
    from bns_gcn_b200.data import graph_partition, load_as_partition, make_graph
    from tests.harness import make_args, run_product
    a = argparse.Namespace(dataset="tiny", n_partitions=2, partition_method="multilevel", partition_obj="vol",
                           inductive=False, part_path=str(tmp_path / "partition"), graph_name="")
    cfg_path = graph_partition(a, fg=make_graph("tiny", seed=0))
    assert a.graph_name == "tiny-2-multilevel-vol-trans"
    with open(cfg_path) as f:
        assert json.load(f)["part_method"] == "multilevel"
    parts = [load_as_partition(a, r) for r in range(2)]
    out = run_product(parts, make_args(model="graphsage", sampling_rate=0.5, n_hidden=16, n_partitions=2), "cuda:0", 2,
                      capture=False)
    assert all(torch.isfinite(torch.tensor(o["loss"])).all() for o in out)


def test_main_two_ranks(built, tmp_path):
    """``main.py --partition-method multilevel`` builds the store and trains 2 epochs at 2 ranks, one per GPU."""
    if torch.cuda.device_count() < 2:
        pytest.skip(f"needs 2 GPUs, this box has {torch.cuda.device_count()}")
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    p = subprocess.run([sys.executable, "-m", "bns_gcn_b200.main", "--dataset", "tiny", "--n-partitions", "2",
                        "--partition-method", "multilevel", "--n-epochs", "2", "--log-every", "1", "--fix-seed",
                        "--no-eval"], cwd=tmp_path, env=env, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, (p.stdout[-3000:], p.stderr[-3000:])
    assert (tmp_path / "partition" / "tiny-2-multilevel-vol-trans" / "tiny-2-multilevel-vol-trans.json").exists()
