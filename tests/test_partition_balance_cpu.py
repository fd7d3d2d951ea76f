"""``--partition-balance edges`` on the host: the flag, the store, the ``metis`` stand-in and ``random`` under both
bounds, and the multilevel partitioner's host stages (initial partition, block partition, ``admit``) with in-edge
weights."""
import argparse
import json
import os

import numpy as np
import pytest
import torch

from tests import partition_reference as R

CPU = torch.device("cpu")


def _bounds(fg, P):
    from bns_gcn_b200.data.partition import in_edge_bound
    n = fg.n_nodes
    return max(int(0.97 * n / P), 1), int(1.03 * n / P) + 1, in_edge_bound(fg.in_degrees(), P)


def _assert_within(fg, part, P):
    lo, hi, ehi = _bounds(fg, P)
    deg = fg.in_degrees()
    assert ehi == int(1.03 * fg.n_edges / P) + int(deg.max())
    sizes = torch.bincount(part, minlength=P)
    esizes = torch.zeros(P, dtype=torch.int64).index_add_(0, part, deg)
    assert int(sizes.min()) >= lo and int(sizes.max()) <= hi and int(sizes.min()) > 0, (sizes.tolist(), lo, hi)
    assert int(esizes.max()) <= ehi, (esizes.tolist(), ehi)


def test_parser_spellings_default_and_choices():
    from bns_gcn_b200.helper.parser import create_parser
    assert create_parser([]).partition_balance == "nodes"
    assert create_parser(["--partition-balance", "edges"]).partition_balance == "edges"
    assert create_parser(["--partition_balance", "edges"]).partition_balance == "edges"
    assert create_parser(["--partition-balance", "nodes"]).partition_balance == "nodes"
    with pytest.raises(SystemExit):
        create_parser(["--partition-balance", "train"])
    from bns_gcn_b200.helper.parser import build_parser
    flag = [a for a in build_parser()._actions if a.dest == "partition_balance"][0]
    assert flag.help.startswith("NEW:")


def test_store_name_token():
    from bns_gcn_b200.data.store import default_graph_name
    a = argparse.Namespace(dataset="reddit", n_partitions=4, partition_method="metis", partition_obj="vol",
                           inductive=True)
    assert default_graph_name(a) == "reddit-4-metis-vol-induc"            # no field: nodes, the name of old
    a.partition_balance = "nodes"
    assert default_graph_name(a) == "reddit-4-metis-vol-induc"
    a.partition_balance = "edges"
    assert default_graph_name(a) == "reddit-4-metis-vol-edges-induc"
    a.data_source, a.inductive, a.partition_method = "files", False, "multilevel"
    assert default_graph_name(a) == "reddit-files-4-multilevel-vol-edges-trans"


def _store_args(tmp_path, **kw):
    d = dict(dataset="small", n_partitions=4, partition_method="metis", partition_obj="vol", inductive=False,
             part_path=str(tmp_path / "part"), graph_name="", graph_seed=0, partition_balance="edges")
    d.update(kw)
    return argparse.Namespace(**d)


def test_store_records_the_balance_and_refuses_the_other(tmp_path):
    from bns_gcn_b200.data import graph_partition, load_partition, make_graph
    from bns_gcn_b200.data.partition import in_edge_bound
    fg = make_graph("small", seed=0, device=CPU)
    a = _store_args(tmp_path)
    cfg_path = graph_partition(a, fg=fg, device=CPU)
    assert os.path.basename(cfg_path) == "small-4-metis-vol-edges-trans.json"
    with open(cfg_path) as f:
        assert json.load(f)["balance"] == "edges"
    ehi = in_edge_bound(fg.in_degrees(), 4)
    for r in range(4):
        g, _, _ = load_partition(_store_args(tmp_path, graph_name=a.graph_name), r)
        assert g.num_edges() <= ehi                                    # a_in + a_out nnz of the part
    other = _store_args(tmp_path, graph_name=a.graph_name, partition_balance="nodes")
    with pytest.raises(RuntimeError, match="--partition-balance edges, this run asks for --partition-balance nodes"):
        load_partition(other, 0)
    with pytest.raises(RuntimeError, match="--partition-balance edges.*--partition-balance nodes"):
        graph_partition(other, fg=fg, device=CPU)
    # a store written under nodes records it, and one written before the key existed reads as nodes
    b = _store_args(tmp_path, partition_balance="nodes", partition_method="random")
    cfg_path = graph_partition(b, fg=fg, device=CPU)
    assert os.path.basename(cfg_path) == "small-4-random-vol-trans.json"
    with open(cfg_path) as f:
        cfg = json.load(f)
    assert cfg.pop("balance") == "nodes"
    with open(cfg_path, "w") as f:
        json.dump(cfg, f)
    plain = argparse.Namespace(**{k: v for k, v in vars(b).items() if k != "partition_balance"})
    load_partition(plain, 0)
    with pytest.raises(RuntimeError, match="--partition-balance nodes, this run asks for --partition-balance edges"):
        load_partition(_store_args(tmp_path, graph_name=b.graph_name, partition_method="random"), 0)


def test_inductive_store_bounds_the_train_subgraph(tmp_path):
    from bns_gcn_b200.data import graph_partition, induced_subgraph, load_partition, make_graph
    from bns_gcn_b200.data.partition import in_edge_bound
    fg = make_graph("small", seed=0, device=CPU)
    a = _store_args(tmp_path, inductive=True, n_partitions=3)
    graph_partition(a, fg=fg, device=CPU)
    sub = induced_subgraph(fg, fg.train_mask)
    ehi = in_edge_bound(sub.in_degrees(), 3)
    total = 0
    for r in range(3):
        g, _, _ = load_partition(_store_args(tmp_path, inductive=True, n_partitions=3, graph_name=a.graph_name), r)
        assert g.num_edges() <= ehi
        total += g.num_edges()
    assert total == sub.n_edges


_SHAPES = ["tiny", "small", "synthetic-10k", "yelp"]


@pytest.fixture(scope="module")
def graphs():
    from bns_gcn_b200.data import make_graph
    return {s: make_graph(s, seed=0, device=CPU) for s in _SHAPES}


@pytest.mark.parametrize("P", [2, 4, 8])
@pytest.mark.parametrize("method", ["metis", "random"])
@pytest.mark.parametrize("shape", _SHAPES)
def test_edge_balanced_parts_are_within_both_bounds(graphs, shape, method, P):
    from bns_gcn_b200.data import assign_parts, partition_quality
    fg = graphs[shape]
    part = assign_parts(fg, P, method, 0, "vol", CPU, balance="edges")
    _assert_within(fg, part, P)
    assert torch.equal(part, assign_parts(fg, P, method, 0, "vol", CPU, balance="edges"))
    q = partition_quality(fg, part, P)
    assert q["max_in_edges"] <= _bounds(fg, P)[2] and q["min_in_edges"] > 0
    if shape != "yelp":      # the nodes default is the call without the keyword (the yelp nodes runs cost minutes)
        assert torch.equal(assign_parts(fg, P, method, 0, "vol", CPU, balance="nodes"),
                           assign_parts(fg, P, method, 0, "vol", CPU))


def test_partition_quality_counts_in_edges_by_destination_owner():
    from bns_gcn_b200.data import make_graph, partition_quality
    fg = make_graph("tiny", seed=3, device=CPU)
    part = torch.randint(0, 5, (fg.n_nodes,), generator=torch.Generator().manual_seed(1))
    q = partition_quality(fg, part, 5)
    per = torch.bincount(part[fg.dst()], minlength=5)
    assert (q["min_in_edges"], q["max_in_edges"]) == (int(per.min()), int(per.max()))
    assert int(per.sum()) == fg.n_edges


def _hub_graph():
    """A hub that receives three edges from every other node (in-degree 3/5 of the edges, above E / P for P >= 2), on
    a one-way ring, one loop per node."""
    n = 400
    i = torch.arange(n)
    src = torch.cat([i[1:], i[1:], i[1:], i, i])
    dst = torch.cat([torch.zeros(3 * (n - 1), dtype=torch.int64), (i + 1) % n, i])
    return R.graph_from_edges(n, src, dst)


@pytest.mark.parametrize("P", [2, 3, 4])
@pytest.mark.parametrize("method", ["metis", "random"])
def test_a_hub_above_e_over_p_fits_through_the_slack(method, P):
    from bns_gcn_b200.data import assign_parts
    fg = _hub_graph()
    deg = fg.in_degrees()
    assert int(deg.max()) > fg.n_edges / P
    part = assign_parts(fg, P, method, 0, "vol", CPU, balance="edges")
    _assert_within(fg, part, P)


def test_unknown_balance_is_refused():
    from bns_gcn_b200.data import assign_parts, make_graph
    with pytest.raises(ValueError, match="--partition-balance must be one of nodes, edges"):
        assign_parts(make_graph("tiny", seed=0, device=CPU), 2, "random", 0, balance="train")


def test_shed_raises_naming_the_bound_and_part():
    from bns_gcn_b200.data.partition import shed_in_edges
    deg = torch.tensor([50, 1, 1, 1])
    with pytest.raises(RuntimeError, match=r"part 0 owns 51 in-edges, above the in-edge bound 40"):
        shed_in_edges(torch.tensor([0, 0, 1, 1]), deg, 2, 40, "metis")


# ---- the multilevel partitioner's host stages ------------------------------------------------------------------------

def _coarse_graph(n, m, seed):
    """A weighted coarse-looking graph: node weights 1..6, in-edge weights with a heavy tail, symmetric edges."""
    rng = np.random.default_rng(seed)
    a, b = rng.integers(0, n, m), rng.integers(0, n, m)
    keep = a != b
    a, b = np.concatenate([a[keep], b[keep]]), np.concatenate([b[keep], a[keep]])
    key = np.unique(a * n + b)
    a, b = key // n, key % n
    indptr = np.zeros(n + 1, dtype=np.int64)
    indptr[1:] = np.cumsum(np.bincount(a, minlength=n))
    w = rng.integers(1, 5, a.shape[0]).astype(np.int64)
    nw = rng.integers(1, 7, n).astype(np.int64)
    ew = (nw * rng.pareto(1.5, n) * 10).astype(np.int64) + nw
    return indptr, b.astype(np.int64), w, nw, ew


def _coarse_bounds(nw, ew, P):
    total, etotal = int(nw.sum()), int(ew.sum())
    return max(int(0.97 * total / P), 1), int(1.03 * total / P) + 1, int(1.03 * etotal / P) + int(ew.max())


@pytest.mark.parametrize("n,m,P", [(300, 1500, 2), (300, 1500, 4), (600, 4000, 8)])
def test_initial_partition_respects_both_bounds(n, m, P):
    from bns_gcn_b200.data.multilevel import initial_partition
    indptr, idx, w, nw, ew = _coarse_graph(n, m, seed=n + P)
    lo, hi, ehi = _coarse_bounds(nw, ew, P)
    a = initial_partition(indptr, idx, w, nw, P, lo, hi, 1, 8, ew, ehi)
    assert np.array_equal(a, initial_partition(indptr, idx, w, nw, P, lo, hi, 1, 8, ew, ehi))
    sizes = np.bincount(a, weights=nw, minlength=P)
    esizes = np.bincount(a, weights=ew, minlength=P)
    assert (sizes > 0).all() and sizes.max() <= hi + nw.max() and sizes.min() >= lo - nw.max(), sizes
    assert esizes.max() <= ehi, (esizes, ehi)
    # the nodes call is the call without the in-edge weights
    assert np.array_equal(initial_partition(indptr, idx, w, nw, P, lo, hi, 1, 8),
                          initial_partition(indptr, idx, w, nw, P, lo, hi, seed=1))


@pytest.mark.parametrize("P", [2, 5, 8])
def test_block_partition_respects_both_bounds(P):
    from bns_gcn_b200.data.multilevel import block_partition
    indptr, idx, w, nw, ew = _coarse_graph(500, 3000, seed=P)
    lo, hi, ehi = _coarse_bounds(nw, ew, P)
    a = block_partition(indptr, idx, nw, P, ew, lo, hi, ehi)
    assert np.array_equal(a, block_partition(indptr, idx, nw, P, ew, lo, hi, ehi))
    sizes = np.bincount(a, weights=nw, minlength=P)
    esizes = np.bincount(a, weights=ew, minlength=P)
    assert sizes.min() >= lo and sizes.max() <= hi, (sizes, lo, hi)
    assert esizes.max() <= ehi, (esizes, ehi)


def test_cut_blocks_finds_the_only_cut_and_reports_none():
    from bns_gcn_b200.data.multilevel import cut_blocks
    nw = np.ones(8, dtype=np.int64)
    ew = np.array([9, 1, 1, 1, 1, 1, 1, 9])
    # two blocks of 3..5 nodes and at most 12 in-edges: only 4 + 4 keeps both within 12
    assert cut_blocks(nw, ew, 2, 3, 5, 12).tolist() == [0, 0, 0, 0, 1, 1, 1, 1]
    # at most 11 in-edges: 4 + 4 holds 12 each; no cut works
    assert cut_blocks(nw, ew, 2, 3, 5, 11) is None
    # heavy front: only 3 + 5 keeps the first block within 12
    ew = np.array([9, 1, 2, 5, 1, 1, 1, 1])
    assert cut_blocks(nw, ew, 2, 3, 5, 12).tolist() == [0, 0, 0, 1, 1, 1, 1, 1]


def _admit_edges_host(nodes, to, gain, wt, frm, sizes, hi, lo, ewt, esizes, ehi, need_out=None, need_eout=None):
    """multilevel.admit with in-edge weights, move by move (R.admit's rules plus the in-edge running sum per target,
    and per source: kept while its node or its in-edge excess is not yet gone)."""
    L = [dict(v=int(nodes[i]), t=int(to[i]), g=int(gain[i]), w=int(wt[i]), f=int(frm[i]), e=int(ewt[i]))
         for i in range(len(nodes))]
    kept, run, erun = [], {}, {}
    for x in sorted(L, key=lambda x: (x["t"], -x["g"], x["v"])):
        run[x["t"]] = run.get(x["t"], 0) + x["w"]
        erun[x["t"]] = erun.get(x["t"], 0) + x["e"]
        if int(sizes[x["t"]]) + run[x["t"]] <= hi and int(esizes[x["t"]]) + erun[x["t"]] <= ehi:
            kept.append(x)
    L, kept, run, erun = kept, [], {}, {}
    for x in sorted(L, key=lambda x: (x["f"], -x["g"], x["v"])):
        before, ebefore = run.get(x["f"], 0), erun.get(x["f"], 0)
        run[x["f"]], erun[x["f"]] = before + x["w"], ebefore + x["e"]
        ok = lo is None or int(sizes[x["f"]]) - run[x["f"]] >= lo
        if need_eout is not None:
            ok = ok and (ebefore < int(need_eout[x["f"]]) or before < int(need_out[x["f"]]))
        if ok:
            kept.append(x)
    return sorted((x["v"], x["t"]) for x in kept)


@pytest.mark.parametrize("mode", ["caps", "excess"])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_admit_with_in_edge_weights_matches_move_by_move(seed, mode):
    from bns_gcn_b200.data.multilevel import admit
    g = torch.Generator().manual_seed(seed)
    n, P = 400, 6
    nodes = torch.randperm(1600, generator=g)[:n]
    frm = torch.randint(0, P, (n,), generator=g)
    to = (frm + torch.randint(1, P, (n,), generator=g)) % P
    gain = torch.randint(-2, 3, (n,), generator=g)
    wt = torch.randint(1, 5, (n,), generator=g)
    ewt = torch.randint(1, 60, (n,), generator=g)
    sizes = torch.randint(90, 131, (P,), generator=g)
    esizes = torch.randint(1500, 2600, (P,), generator=g)
    kw = dict(hi=125, lo=95, ewt=ewt, esizes=esizes, ehi=2500)
    if mode == "excess":
        kw.update(need_out=(sizes - 110).clamp(min=0), need_eout=(esizes - 2200).clamp(min=0))
    mv, tt = admit(nodes, to, gain, wt, frm, sizes, **kw)
    got = sorted(zip(mv.tolist(), tt.tolist()))
    assert got == _admit_edges_host(nodes, to, gain, wt, frm, sizes, kw["hi"], kw["lo"], ewt, esizes, kw["ehi"],
                                    kw.get("need_out"), kw.get("need_eout"))
    # whatever subset is applied, no target passes either cap
    part_sizes, part_e = sizes.clone(), esizes.clone()
    for v, t in got:
        i = int((nodes == v).nonzero()[0])
        part_sizes[t] += wt[i]
        part_e[t] += ewt[i]
    assert bool((part_e <= torch.maximum(esizes, torch.tensor(2500))).all())
