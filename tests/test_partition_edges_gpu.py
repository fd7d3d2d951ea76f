"""The multilevel partitioner's kernels (csrc/partition.cuh) at the edges of what they accept, each against its plain
host restatement (tests/partition_reference.py), element for element: 33 to 64 parts (the upper half of every warp's
part table, occupancy bits 32-63, ``allowed`` masks with bit 63), rows of 19 k entries, the sort width of
``bns_part_edges`` at 2^k +- 1 output rows, int64 sums past 2^32, weighted coarse levels, the Reddit shape, and the
level loop's admission / rebalancing / refinement claims at 64 parts."""
import ctypes

import numpy as np
import pytest
import torch

from tests import partition_reference as R

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
HIGH_P = [31, 32, 33, 63, 64]
ALL64 = (1 << 64) - 1
_CACHE = {}


def _same(dev_csr, host_csr):
    for a, b in zip(dev_csr, host_csr):
        assert torch.equal(a.cpu().long(), b.long())


def _occ_bits(occ, P):
    """int64 occupancy words -> bool [n, P]."""
    return ((occ.cpu()[:, None] >> torch.arange(P)) & 1).bool()


# ---- a graph with rows of every stride class -------------------------------------------------------------------------

ROW_LENGTHS = [0, 1, 31, 32, 33, 64, 65, 4100, 19_500]
N_ROWS_GRAPH = 24_576


def _rows_graph(P):
    """CSR (indptr int64, idx int32 on the device) and a part (int32, every part populated): node i < 9 has a row of
    ROW_LENGTHS[i] distinct random columns, node 9 a row of 19,500 entries all in part P - 1 and node 10 one of 19,500
    all in part 0 (repeated columns), the rest 0 to 8 random entries."""
    if ("rows", P) not in _CACHE:
        n = N_ROWS_GRAPH
        g = torch.Generator().manual_seed(1000 + P)
        part = torch.randint(0, P, (n,), generator=g)
        part[:P] = torch.arange(P)
        top, bottom = torch.nonzero(part == P - 1)[:, 0], torch.nonzero(part == 0)[:, 0]
        rows = [torch.randperm(n, generator=g)[:k] for k in ROW_LENGTHS]
        rows.append(top[torch.randint(0, top.numel(), (19_500,), generator=g)])
        rows.append(bottom[torch.randint(0, bottom.numel(), (19_500,), generator=g)])
        lens = torch.randint(0, 9, (n - len(rows),), generator=g)
        rows += list(torch.split(torch.randint(0, n, (int(lens.sum()),), generator=g), lens.tolist()))
        indptr = torch.zeros(n + 1, dtype=torch.int64)
        indptr[1:] = torch.cumsum(torch.tensor([r.numel() for r in rows]), 0)
        idx = torch.cat(rows)
        _CACHE[("rows", P)] = (indptr.to(DEV), idx.to(DEV, torch.int32), part.to(DEV, torch.int32))
    return _CACHE[("rows", P)]


def _special_rows():
    return list(range(len(ROW_LENGTHS) + 2))


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("P", HIGH_P)
def test_conn_on_long_rows_is_exact(built, P, weighted):
    """conn, both occupancy words and (cut, vol) against the host scatter-add, on rows of 0 .. 19,500 entries, two of
    them with every entry in one part (one shared counter under contention)."""
    from bns_gcn_b200 import ops
    ip, ix, part = _rows_graph(P)
    lens = (ip[1:] - ip[:-1]).cpu()
    assert lens[:len(ROW_LENGTHS)].tolist() == ROW_LENGTHS and int(lens[9]) == int(lens[10]) == 19_500
    w = None
    if weighted:
        w = torch.randint(1, 8, (ix.numel(),), generator=torch.Generator().manual_seed(P)).to(DEV, torch.int32)
    conn, occ, q = ops.part_conn(ip, ix, w, part, P, occ=True, quality=True)
    ch, oh, qh = R.conn(ip, ix, w, part, P)
    assert torch.equal(conn.cpu(), ch) and torch.equal(occ.cpu(), oh) and tuple(q.cpu().tolist()) == qh
    # the two one-part rows: one column each, and one occupancy bit
    assert torch.nonzero(ch[9]).flatten().tolist() == [P - 1] and torch.nonzero(ch[10]).flatten().tolist() == [0]
    assert int(oh[9]) == (1 << (P - 1)) - (1 << 64 if P == 64 else 0) and int(oh[10]) == 1
    if w is None:
        assert int(ch[9, P - 1]) == int(ch[10, 0]) == 19_500
    # every variant of the kernel (with and without the table, occ, quality) writes the same
    for table, o, qq in ((False, True, False), (False, False, True), (True, False, False)):
        c2, o2, q2 = ops.part_conn(ip, ix, w, part, P, table=table, occ=o, quality=qq)
        if table:
            assert torch.equal(c2.cpu(), ch)
        if o:
            assert torch.equal(o2.cpu(), oh)
        if qq:
            assert tuple(q2.cpu().tolist()) == qh


@pytest.mark.parametrize("P", [33, 64])
def test_conn_sums_past_2_to_the_32(built, P):
    """Weighted rows with per-(node, part) sums near 2^30 (and one single entry of 2^31 - 1): the int32 table holds
    them, and the int64 cut sums past 2^32."""
    from bns_gcn_b200 import ops
    n = 512
    g = torch.Generator().manual_seed(77 + P)
    part = torch.randint(0, P, (n,), generator=g)
    part[:P] = torch.arange(P)
    members = [torch.nonzero(part == p)[:, 0] for p in range(P)]
    rows, ws = [], []
    for v in range(n):
        cols = torch.cat([m[torch.randint(0, m.numel(), (2,), generator=g)] for m in members])
        rows.append(cols)
        ws.append(torch.randint((1 << 29) - (1 << 20), (1 << 29) + 1, (cols.numel(),), generator=g))
    rows[0], ws[0] = members[P - 1][:1], torch.tensor([(1 << 31) - 1])
    indptr = torch.zeros(n + 1, dtype=torch.int64)
    indptr[1:] = torch.cumsum(torch.tensor([r.numel() for r in rows]), 0)
    ip, ix = indptr.to(DEV), torch.cat(rows).to(DEV, torch.int32)
    w, pd = torch.cat(ws).to(DEV, torch.int32), part.to(DEV, torch.int32)
    conn, occ, q = ops.part_conn(ip, ix, w, pd, P, occ=True, quality=True)
    ch, oh, qh = R.conn(ip, ix, w, pd, P)
    assert int(ch.max()) == (1 << 31) - 1 and int(ch[1:].min()) >= (1 << 30) - (1 << 21)
    assert qh[0] > 1 << 40
    assert torch.equal(conn.cpu(), ch) and torch.equal(occ.cpu(), oh) and tuple(q.cpu().tolist()) == qh


def _one_bit_table(ops, objective, part, conn, P, in_g, occ):
    """The full gain table [n, P] from P calls with one allowed part each (0 on a node's own part)."""
    n = part.numel()
    table = torch.zeros(n, P, dtype=torch.int64)
    own_all = part.cpu()
    for b in range(P):
        t, g = ops.part_gains(objective, part, conn, P, 1 << b, in_graph=in_g, occ=occ)
        t, g = t.cpu(), g.cpu()
        own = own_all == b
        assert torch.all(t[own] == -1) and torch.all(g[own] == 0) and torch.all(t[~own] == b)
        table[:, b] = g
    return table


def _tables(ops, ip, ix, part, P, objective):
    """(conn, occ, in_g, cut graph) of the objective on the by-destination CSR (ip, ix)."""
    n = part.numel()
    if objective == "cut":
        g2 = ops.part_edges(ip, ix, None, n, 2, True)
        conn, _, _ = ops.part_conn(*g2, part, P)
        return conn, None, None, g2
    out_g = ops.part_edges(ip, ix, None, n, 1, True)
    conn, occ, _ = ops.part_conn(*out_g, part, P, occ=True)
    return conn, occ, ops.part_edges(ip, ix, None, n, 0, True), out_g


def _host_gains(objective, graph, in_g, part, P, nodes):
    if objective == "cut":
        return R.cut_gains(*graph, part, P, nodes)
    return R.vol_gains(graph, in_g, part, P, nodes)


_MASKS = {
    "high-half": lambda P: ((1 << P) - 1) & ~((1 << 32) - 1),
    "low-half": lambda P: (1 << 32) - 1,
    "top-part": lambda P: 1 << (P - 1),
    "bit-63": lambda P: 1 << 63,
    "alternating-odd": lambda P: 0xAAAAAAAAAAAAAAAA,
    "alternating-even": lambda P: 0x5555555555555555,
    "every-bit": lambda P: ALL64,
    "none": lambda P: 0,
}


@pytest.mark.parametrize("objective", ["cut", "vol"])
@pytest.mark.parametrize("P", [32, 33, 64])
def test_gains_on_long_rows_and_masked_targets(built, P, objective):
    """On the long-row graph: the one-bit gain tables of the special rows and 100 random nodes against the objective's
    definition, then the best target under masks with only high bits, only bit P - 1, only bit 63, alternating bits,
    every bit and none against the choice from the table (largest gain, lowest part; -1 and 0 without a part)."""
    from bns_gcn_b200 import ops
    ip, ix, part = _rows_graph(P)
    conn, occ, in_g, graph = _tables(ops, ip, ix, part, P, objective)
    table = _one_bit_table(ops, objective, part, conn, P, in_g, occ)
    nodes = _special_rows() + torch.randperm(N_ROWS_GRAPH, generator=torch.Generator().manual_seed(5))[:100].tolist()
    host = _host_gains(objective, graph, in_g, part, P, nodes)
    assert torch.equal(table[nodes], host)
    rows = graph if objective == "cut" else in_g
    assert int((rows[0][9] - rows[0][8]).item()) >= 19_000        # node 8's row is still 19 k long after merging
    hp = part.cpu()
    for name, mask in _MASKS.items():
        allowed = mask(P)
        t, g = ops.part_gains(objective, part, conn, P, allowed, in_graph=in_g, occ=occ)
        th, gh = R.best_target(table, hp, allowed)
        assert torch.equal(t.cpu(), th) and torch.equal(g.cpu(), gh), name
        if name == "top-part":                      # no allowed part but its own: -1 and 0
            own = hp == P - 1
            assert own.any() and torch.all(t.cpu()[own] == -1) and torch.all(g.cpu()[own] == 0)
        if allowed & ((1 << P) - 1) == 0:
            assert torch.all(t.cpu() == -1) and torch.all(g.cpu() == 0)


@pytest.mark.parametrize("P", [33, 64])
def test_relabelling_permutes_every_output(built, P):
    """Independent of the host restatement: relabel the parts by p -> (p + P // 2) mod P (the halves swap at P = 64, a
    rotation at P = 33).  conn columns and occupancy bits permute exactly, cut and vol do not change, and the one-bit
    gain tables (cut and vol) agree entry for entry under the permutation."""
    from bns_gcn_b200 import ops
    ip, ix, part = _rows_graph(P)
    pi = (torch.arange(P) + P // 2) % P
    part2 = pi.to(DEV, torch.int32)[part.long()]
    for mode in (1, 2):
        g = ops.part_edges(ip, ix, None, N_ROWS_GRAPH, mode, True)
        c1, o1, q1 = ops.part_conn(*g, part, P, occ=True, quality=True)
        c2, o2, q2 = ops.part_conn(*g, part2, P, occ=True, quality=True)
        assert torch.equal(c2.cpu()[:, pi], c1.cpu())
        assert torch.equal(_occ_bits(o2, P)[:, pi], _occ_bits(o1, P))
        assert torch.equal(q1.cpu(), q2.cpu())
    for objective in ("cut", "vol"):
        conn1, occ1, in_g, _ = _tables(ops, ip, ix, part, P, objective)
        conn2, occ2, _, _ = _tables(ops, ip, ix, part2, P, objective)
        t1 = _one_bit_table(ops, objective, part, conn1, P, in_g, occ1)
        t2 = _one_bit_table(ops, objective, part2, conn2, P, in_g, occ2)
        assert torch.equal(t2[:, pi], t1), objective


# ---- bns_part_edges ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n_out", [2 ** 16 - 1, 2 ** 16, 2 ** 16 + 1, 2 ** 20 - 1, 2 ** 20, 2 ** 20 + 1])
def test_edges_at_the_sort_width_boundaries(built, n_out):
    """n_out_rows at 2^k - 1, 2^k, 2^k + 1 (the sort's end bit steps there), 2 M entries, node maps that send a tenth of
    the nodes to the top row and a twentieth to the one below it, loops present and dropped: all three modes."""
    from bns_gcn_b200 import ops
    g = torch.Generator().manual_seed(n_out)
    n_in, nnz = 200_000, 2_000_000
    rows = torch.sort(torch.randint(0, n_in, (nnz,), generator=g)).values
    idx = torch.randint(0, n_in, (nnz,), generator=g)
    loops = torch.rand(nnz, generator=g) < 0.05
    idx[loops] = rows[loops]
    indptr = torch.zeros(n_in + 1, dtype=torch.int64)
    indptr[1:] = torch.cumsum(torch.bincount(rows, minlength=n_in), 0)
    cmap = torch.randint(0, n_out, (n_in,), generator=g)
    sel = torch.randperm(n_in, generator=g)
    cmap[sel[:n_in // 10]] = n_out - 1
    cmap[sel[n_in // 10:n_in // 10 + n_in // 20]] = n_out - 2
    w = torch.randint(1, 100, (nnz,), generator=g)
    ip, ix, wd, cm = indptr.to(DEV), idx.to(DEV, torch.int32), w.to(DEV, torch.int32), cmap.to(DEV, torch.int32)
    for mode in (0, 1, 2):
        for drop in ((False, True) if mode == 2 else (True,)):
            dev = ops.part_edges(ip, ix, wd, n_out, mode, drop, row_map=cm, col_map=cm)
            host = R.edges(ip, ix, wd, n_out, mode, drop, cm, cm)
            _same(dev, host)
            top = host[0]
            assert int(top[n_out] - top[n_out - 1]) > 0 and int(top[n_out - 1] - top[n_out - 2]) > 0
    # the maps make loops (the drop key exists), and dropping them removes something
    assert int((cmap[rows] == cmap[idx]).sum()) > nnz // 50


def test_edges_every_entry_a_loop(built):
    """Every mapped entry a loop, loops dropped: no entries, an all-zero indptr of n_out_rows + 1, in every mode."""
    from bns_gcn_b200 import ops
    g = torch.Generator().manual_seed(3)
    n_in, nnz = 5_000, 300_000
    rows = torch.sort(torch.randint(0, n_in, (nnz,), generator=g)).values
    indptr = torch.zeros(n_in + 1, dtype=torch.int64)
    indptr[1:] = torch.cumsum(torch.bincount(rows, minlength=n_in), 0)
    ip, ix = indptr.to(DEV), torch.randint(0, n_in, (nnz,), generator=g).to(DEV, torch.int32)
    w = torch.randint(1, 1000, (nnz,), generator=g).to(DEV, torch.int32)
    for n_out, target in ((1, 0), (2 ** 16, 2 ** 16 - 1), (2 ** 20 + 1, 2 ** 20)):
        cmap = torch.full((n_in,), target, dtype=torch.int32, device=DEV)
        for mode in (0, 1, 2):
            indp, idx, ww = ops.part_edges(ip, ix, w, n_out, mode, True, row_map=cmap, col_map=cmap)
            assert idx.numel() == 0 and ww.numel() == 0
            assert indp.numel() == n_out + 1 and int(indp.abs().sum()) == 0


@pytest.mark.parametrize("n_out", [3, 2 ** 16 + 1])
def test_edges_long_runs_sum_exactly(built, n_out):
    """Maps that collapse 1 M entries into a handful of keys (reduce-by-key runs of ~100 k entries): the weight sums
    are exact, with and without the loops."""
    from bns_gcn_b200 import ops
    g = torch.Generator().manual_seed(n_out)
    n_in, nnz = 20_000, 1_000_000
    rows = torch.sort(torch.randint(0, n_in, (nnz,), generator=g)).values
    indptr = torch.zeros(n_in + 1, dtype=torch.int64)
    indptr[1:] = torch.cumsum(torch.bincount(rows, minlength=n_in), 0)
    ip, ix = indptr.to(DEV), torch.randint(0, n_in, (nnz,), generator=g).to(DEV, torch.int32)
    w = torch.randint(1, 1000, (nnz,), generator=g).to(DEV, torch.int32)
    cmap = torch.tensor([0, n_out - 1, n_out // 2])[torch.randint(0, 3, (n_in,), generator=g)].to(DEV, torch.int32)
    for mode in (0, 1, 2):
        for drop in (False, True):
            dev = ops.part_edges(ip, ix, w, n_out, mode, drop, row_map=cmap, col_map=cmap)
            host = R.edges(ip, ix, w, n_out, mode, drop, cmap, cmap)
            _same(dev, host)
            assert host[1].numel() == (6 if drop else 9) and int(host[2].max()) > 50_000_000


def test_edges_size_refusal(built):
    """2^30 entries in mode 2 (2^31 sort entries) and 2^31 - 1 in mode 0 are refused by the argument check, before
    anything is read or launched; the workspace query answers 0 for them."""
    from bns_gcn_b200 import _lib
    L = _lib.lib
    d = torch.zeros(64, dtype=torch.int64, device=DEV)
    for mode, nnz in ((2, 1 << 30), (0, (1 << 31) - 1), (1, 1 << 31)):
        out = ctypes.c_int64(-7)
        rc = L.bns_part_edges(4, nnz, d.data_ptr(), d.data_ptr(), None, None, None, mode, 1, 4, d.data_ptr(),
                              d.data_ptr(), d.data_ptr(), ctypes.byref(out), d.data_ptr(), 1 << 40, None)
        assert rc == -1 and out.value == -7, (mode, nnz, rc)
        assert b"2^31-1" in L.bns_last_error()
    assert L.bns_part_edges_workspace_bytes(1 << 31) == 0
    assert L.bns_part_edges_workspace_bytes((1 << 31) - 1) == 0
    assert L.bns_part_edges_workspace_bytes((1 << 31) - 2) > 0
    torch.cuda.synchronize()
    assert int(d.abs().sum()) == 0


# ---- the Reddit shape ------------------------------------------------------------------------------------------------

def _reddit():
    if "reddit" not in _CACHE:
        from bns_gcn_b200.data import make_graph
        _CACHE["reddit"] = make_graph("reddit", seed=0, with_feat=False)
    return _CACHE["reddit"]


def _reddit_csrs():
    """The CSRs ``_multilevel`` builds on the Reddit shape: {2: undirected, 1: out, 0: in}, loops dropped."""
    if "reddit-csrs" not in _CACHE:
        from bns_gcn_b200 import ops
        fg = _reddit()
        ip, ix = fg.indptr.to(DEV, torch.int64), fg.src.to(DEV, torch.int32)
        _CACHE["reddit-csrs"] = {m: ops.part_edges(ip, ix, None, fg.n_nodes, m, True) for m in (2, 1, 0)}
    return _CACHE["reddit-csrs"]


def test_reddit_edges_match_the_host(built):
    """The three CSRs of the Reddit shape (114.6 M edges, 229 M undirected entries, 18 row bits: sort end bit 50)
    against scipy's duplicate-summing COO -> CSR conversion."""
    import scipy.sparse as sp
    fg = _reddit()
    N = fg.n_nodes
    indptr = fg.indptr.cpu().numpy()
    src = fg.src.cpu().numpy().astype(np.int32)
    dst = np.repeat(np.arange(N, dtype=np.int32), np.diff(indptr))
    keep = src != dst
    A = sp.coo_matrix((np.ones(int(keep.sum()), dtype=np.int32), (dst[keep], src[keep])), shape=(N, N)).tocsr()
    del src, dst, keep
    A.sum_duplicates()
    csrs = _reddit_csrs()

    def same(dev, host):
        host.sum_duplicates()
        host.sort_indices()
        ip, ix, w = dev
        assert np.array_equal(ip.cpu().numpy(), host.indptr.astype(np.int64))
        assert np.array_equal(ix.cpu().numpy(), host.indices.astype(np.int32))
        assert np.array_equal(w.cpu().numpy(), host.data.astype(np.int32))

    same(csrs[0], A)
    At = A.T.tocsr()
    same(csrs[1], At)
    same(csrs[2], (A + At).tocsr())
    assert int(np.diff(A.indptr).max()) >= 19_000


@pytest.mark.parametrize("P", [8, 64])
def test_reddit_conn_is_exact(built, P):
    """conn, occ and (cut, vol) of a seeded random part on the Reddit shape's out- and undirected CSRs against the host
    scatter-add."""
    from bns_gcn_b200 import ops
    csrs = _reddit_csrs()
    N = _reddit().n_nodes
    part = torch.randint(0, P, (N,), generator=torch.Generator().manual_seed(P)).to(DEV, torch.int32)
    for mode in (1, 2):
        conn, occ, q = ops.part_conn(*csrs[mode], part, P, occ=True, quality=True)
        ch, oh, qh = R.conn(*csrs[mode], part, P)
        assert torch.equal(conn.cpu(), ch) and torch.equal(occ.cpu(), oh) and tuple(q.cpu().tolist()) == qh


@pytest.mark.parametrize("objective", ["cut", "vol"])
@pytest.mark.parametrize("P", [8, 64])
def test_reddit_gains_from_the_definitions(built, P, objective):
    """Every target's gain for the 5 longest rows (about 19 k entries) and 200 seeded random nodes of the Reddit shape,
    against the objective recomputed from its definition."""
    from bns_gcn_b200 import ops
    csrs = _reddit_csrs()
    N = _reddit().n_nodes
    part = torch.randint(0, P, (N,), generator=torch.Generator().manual_seed(100 + P)).to(DEV, torch.int32)
    if objective == "cut":
        graph, in_g, occ = csrs[2], None, None
        conn, _, _ = ops.part_conn(*graph, part, P)
        rows = graph
    else:
        graph, in_g = csrs[1], csrs[0]
        conn, occ, _ = ops.part_conn(*graph, part, P, occ=True)
        rows = in_g
    deg = (rows[0][1:] - rows[0][:-1]).cpu()
    longest = torch.topk(deg, 5).indices
    assert int(deg[longest].min()) >= 18_000
    nodes = longest.tolist() + torch.randperm(N, generator=torch.Generator().manual_seed(P))[:200].tolist()
    table = torch.zeros(len(nodes), P, dtype=torch.int64)
    hp = part.cpu()[nodes]
    for b in range(P):
        t, g = ops.part_gains(objective, part, conn, P, 1 << b, in_graph=in_g, occ=occ)
        t, g = t.cpu()[nodes], g.cpu()[nodes]
        assert torch.all(t[hp == b] == -1) and torch.all(t[hp != b] == b)
        table[:, b] = g
    assert torch.equal(table, _host_gains(objective, graph, in_g, part, P, nodes))


# ---- bns_part_cluster / bns_part_weights -------------------------------------------------------------------------------

SEEDS = [1, (5 * 1000003 + 11 * 7919 + 1), ((2 ** 61 + 17) * 1000003 + 3 * 7919 + 1) & ALL64, ALL64,
         0xC0FFEE1234567890]


@pytest.mark.parametrize("name", ["directed-dense", "directed-multi", "star-components", "symmetric"])
def test_weighted_cluster_step_is_exact(built, name):
    """One clustering step with node weights against its host restatement, under several label layouts (pairs, blocks,
    singletons, random labels), caps and 64-bit seeds."""
    from bns_gcn_b200 import ops
    from tests.test_partition_multilevel_gpu import _graphs
    fg = _graphs()[name]
    n = fg.n_nodes
    ip, ix = fg.indptr.to(DEV), fg.src.to(DEV, torch.int32)
    g0 = ops.part_edges(ip, ix, None, n, 2, True)
    gen = torch.Generator().manual_seed(n)
    nw = torch.randint(1, 7, (n,), generator=gen).to(DEV, torch.int32)
    layouts = {"pairs": torch.arange(n) // 2, "blocks": torch.arange(n) // 8, "singletons": torch.arange(n),
               "random": torch.randint(0, max(n // 4, 1), (n,), generator=gen)}
    moved = 0
    for lname, lab in layouts.items():
        label = lab.to(DEV, torch.int32)
        rating = ops.part_edges(*g0, n, 0, False, col_map=label)
        cw = ops.part_weights(label, nw, n)
        assert torch.equal(cw.cpu(), torch.zeros(n, dtype=torch.int64).index_add_(0, lab, nw.cpu().long()))
        for cap in (6, 15, 40):
            for seed in SEEDS:
                t, g = ops.part_cluster(rating, label, nw, cw, cap, seed)
                th, gh = R.cluster_step(rating, label, nw, cw, cap, seed)
                assert torch.equal(t.cpu(), th) and torch.equal(g.cpu(), gh), (lname, cap, seed)
                moved += int((th >= 0).sum())
    assert moved > 0


def _hash_np(x):
    x = x.astype(np.uint64)
    x ^= x >> np.uint64(33)
    x *= np.uint64(0xFF51AFD7ED558CCD)
    x ^= x >> np.uint64(33)
    x *= np.uint64(0xC4CEB9FE1A85EC53)
    x ^= x >> np.uint64(33)
    return x & np.uint64(0xFFFFFFFF)


def test_cluster_crafted_rows(built):
    """Hand-built rating rows: the cap boundary (cw + nw == cap admitted, cap + 1 refused), equal weights broken by
    part_hash(seed + c) and then by id (a real 32-bit hash collision, in one lane and across lanes), a row without the
    node's own cluster, an empty row, a tie with the own cluster (no move), an inactive node, and a rating row of
    19,500 entries; all against the host restatement as well."""
    from bns_gcn_b200 import ops
    seed, cap = 0xC0FFEE1234567890, 100
    n_pool = 1 << 18
    h = _hash_np((np.uint64(seed) + np.arange(n_pool, dtype=np.uint64)))
    vals, first, counts = np.unique(h, return_index=True, return_counts=True)
    dup = int(vals[np.nonzero(counts > 1)[0][0]])
    ca, cb = sorted(int(c) for c in np.nonzero(h == dup)[0][:2])
    assert R.part_hash(seed + ca) == R.part_hash(seed + cb) and ca < cb
    g = torch.Generator().manual_seed(11)
    pool = [int(c) for c in torch.randperm(n_pool, generator=g).tolist() if c not in (ca, cb)]
    take = iter(pool)
    K = 0x9E3779B97F4A7C15
    active = [v for v in range(4096) if R.part_hash(seed ^ ((v * K) & R.M64)) & 1]
    inactive = [v for v in range(4096) if not R.part_hash(seed ^ ((v * K) & R.M64)) & 1]
    n = 4096
    n_labels = n_pool + n
    label = torch.arange(n) + n_pool                          # every node in its own cluster, above the pool
    nw = torch.tensor([1 + (v % 5) for v in range(n)])
    cw = torch.zeros(n_labels, dtype=torch.int64)
    cw[label] = nw
    rows = {}
    expect = {}
    vs = iter(active)
    # cap boundary
    v = next(vs); c1 = next(take); cw[c1] = cap - nw[v]
    rows[v], expect[v] = [(int(label[v]), 7), (c1, 9)], (c1, 2)
    v = next(vs); c2 = next(take); cw[c2] = cap - nw[v] + 1
    rows[v], expect[v] = [(c2, 9)], (-1, 0)
    v = next(vs); c2b, c3 = next(take), next(take); cw[c2b] = cap - nw[v] + 1; cw[c3] = cap - nw[v]
    rows[v], expect[v] = [(c2b, 9), (c3, 4)], (c3, 4)
    # equal weights: the lowest hash wins
    v = next(vs); cs = [next(take) for _ in range(3)]
    win = min(cs, key=lambda c: R.part_hash(seed + c))
    rows[v], expect[v] = [(c, 5) for c in cs] + [(next(take), 1) for _ in range(40)], (win, 5)
    # equal weights and equal hashes: the lower id wins, the higher one listed first, same lane / another lane
    for pos_b, pos_a in ((4, 36), (4, 5)):
        v = next(vs)
        row = [(next(take), 1) for _ in range(40)]
        row[pos_b], row[pos_a] = (cb, 6), (ca, 6)
        rows[v], expect[v] = row, (ca, 6)
    # own cluster absent, empty row, a tie with the own cluster
    v = next(vs); c6 = next(take)
    rows[v], expect[v] = [(c6, 1)], (c6, 1)
    v = next(vs)
    rows[v], expect[v] = [], (-1, 0)
    v = next(vs); c7 = next(take)
    rows[v], expect[v] = [(int(label[v]), 5), (c7, 5)], (-1, 0)
    # an inactive node with a row it would move on
    v = inactive[0]; c8 = next(take)
    rows[v], expect[v] = [(c8, 50)], (-1, 0)
    # a rating row of 19,500 entries, the own cluster inside, some clusters full
    v = next(vs)
    cs = [next(take) for _ in range(19_499)]
    wts = torch.randint(1, 60, (19_499,), generator=g).tolist()
    for c in cs[::3]:
        cw[c] = int(torch.randint(cap - 8, cap + 1, (1,), generator=g))
    row = list(zip(cs, wts))
    row.insert(7_777, (int(label[v]), 20))
    rows[v] = row
    long_v = v
    indptr = torch.zeros(n + 1, dtype=torch.int64)
    indptr[1:] = torch.cumsum(torch.tensor([len(rows.get(u, [])) for u in range(n)]), 0)
    cid = torch.tensor([c for u in range(n) for c, _ in rows.get(u, [])], dtype=torch.int64)
    cwe = torch.tensor([w for u in range(n) for _, w in rows.get(u, [])], dtype=torch.int64)
    rating = (indptr.to(DEV), cid.to(DEV, torch.int32), cwe.to(DEV, torch.int32))
    args = (label.to(DEV, torch.int32), nw.to(DEV, torch.int32), cw.to(DEV))
    t, gn = ops.part_cluster(rating, *args, cap, seed)
    th, gh = R.cluster_step(rating, *args, cap, seed)
    assert torch.equal(t.cpu(), th) and torch.equal(gn.cpu(), gh)
    t, gn = t.cpu(), gn.cpu()
    for u, (tgt, gain) in expect.items():
        assert (int(t[u]), int(gn[u])) == (tgt, gain), (u, rows[u][:3])
    assert int(t[long_v]) >= 0 and int(gn[long_v]) > 0
    others = torch.ones(n, dtype=torch.bool)
    others[list(rows)] = False
    assert torch.all(t[others] == -1) and torch.all(gn[others] == 0)


def test_part_weights_past_2_to_the_32(built):
    """Weighted label sums past 2^32 (up to 2^51), one label holding every node, n_labels = 1, and unit weights."""
    from bns_gcn_b200 import ops
    g = torch.Generator().manual_seed(2)
    n = 1 << 20
    nw = torch.randint(1 << 30, (1 << 31) - 1, (n,), generator=g, dtype=torch.int64)
    nwd = nw.to(DEV, torch.int32)
    lab = torch.randint(0, 1000, (n,), generator=g)
    got = ops.part_weights(lab.to(DEV, torch.int32), nwd, 1000).cpu()
    want = torch.zeros(1000, dtype=torch.int64).index_add_(0, lab, nw)
    assert torch.equal(got, want) and int(want.min()) > 1 << 32
    one = torch.zeros(n, dtype=torch.int32, device=DEV)
    assert ops.part_weights(one, nwd, 1).cpu().tolist() == [int(nw.sum())] and int(nw.sum()) > 1 << 50
    assert ops.part_weights(one + 4, nwd, 5).cpu().tolist() == [0, 0, 0, 0, int(nw.sum())]
    assert ops.part_weights(one, None, 1).cpu().tolist() == [n]


# ---- the level loop at 64 parts --------------------------------------------------------------------------------------

@pytest.mark.parametrize("objective", ["cut", "vol"])
@pytest.mark.parametrize("shape", ["tiny", "small"])
def test_rebalance_from_every_node_in_part_0(built, shape, objective):
    """The worst start (every node in part 0, P = 64, unit weights): rebalance must reach the size bounds within its
    own pass limit (4 P + 8)."""
    from bns_gcn_b200 import ops
    from bns_gcn_b200.data import make_graph
    from bns_gcn_b200.data import multilevel as ml
    fg = make_graph(shape, seed=0, with_feat=False)
    N, P = fg.n_nodes, 64
    ip, ix = fg.indptr.to(DEV, torch.int64), fg.src.to(DEV, torch.int32)
    g0 = ml.Csr(*ops.part_edges(ip, ix, None, N, 2, True))
    if objective == "cut":
        lv = ml._Level(g0, None, P, "cut")
    else:
        lv = ml._Level(g0, None, P, "vol", ml.Csr(*ops.part_edges(ip, ix, None, N, 1, True)),
                       ml.Csr(*ops.part_edges(ip, ix, None, N, 0, True)))
    lo, hi = ml.size_bounds(N, P)
    part = ml.rebalance(lv, torch.zeros(N, dtype=torch.int32, device=DEV), lo, hi)
    sizes = torch.bincount(part.cpu().long(), minlength=P)
    assert sizes.numel() == P and int(sizes.min()) >= lo and int(sizes.max()) <= hi, (sizes.tolist(), lo, hi)


def test_refine_on_a_weighted_coarse_level(built):
    """refine at P = 64 on a clustered, contracted level (node weights 1 .. 4) from a balanced but unrefined start: the
    exact weighted cut never rises from one call to the next and the weighted sizes stay inside [lo, hi]."""
    from bns_gcn_b200 import ops
    from bns_gcn_b200.data import make_graph
    from bns_gcn_b200.data import multilevel as ml
    fg = make_graph("small", seed=1, with_feat=False)
    N, P = fg.n_nodes, 64
    ip, ix = fg.indptr.to(DEV, torch.int64), fg.src.to(DEV, torch.int32)
    g0 = ml.Csr(*ops.part_edges(ip, ix, None, N, 2, True))
    cmap, nc = ml.compact(ml.cluster(g0, None, 4, seed=3))
    cg, cnw = ml.contract(g0, None, cmap, nc)
    assert nc < N and int(cnw.max()) > 1 and int(cnw.sum()) == N
    w = cnw.cpu().long()
    lo, hi = ml.size_bounds(N, P)
    # longest-processing-time start: heaviest node first, into the lightest part
    start = torch.empty(nc, dtype=torch.int64)
    load = [0] * P
    for v in torch.argsort(w, descending=True, stable=True).tolist():
        p = min(range(P), key=lambda q: (load[q], q))
        start[v] = p
        load[p] += int(w[v])
    assert lo <= min(load) and max(load) <= hi
    lv = ml._Level(cg, cnw, P, "cut")
    part = start.to(DEV, torch.int32)
    cut = R.conn(*cg, part, P)[2][0]
    first = cut
    for k in range(4):
        part = ml.refine(lv, part, lo, hi, seed=k, rounds=16)
        c = R.conn(*cg, part, P)[2][0]
        sizes = torch.zeros(P, dtype=torch.int64).index_add_(0, part.cpu().long(), w)
        assert c <= cut and int(sizes.min()) >= lo and int(sizes.max()) <= hi, (k, c, cut, sizes.tolist())
        cut = c
    assert cut < first


# ---- end to end above 32 parts ---------------------------------------------------------------------------------------

def _planted(P, equal):
    if ("planted", P, equal) not in _CACHE:
        from tests.test_host_cpu import _planted_partition_graph
        make = R.equal_planted_blocks if equal else _planted_partition_graph
        _CACHE[("planted", P, equal)] = make(65536, P, 16, 2)
    return _CACHE[("planted", P, equal)]


@pytest.mark.parametrize("objective", ["cut", "vol"])
@pytest.mark.parametrize("P", [33, 48])
def test_finds_equal_planted_blocks_above_32_parts(built, P, objective):
    """65,536 nodes in P equal planted blocks (inside the size bounds), at P = 33 and 48: the bounds hold, the reported
    cut / vol is partition_quality's, and the result is no worse than the stand-in and within 1.05x of the planted
    blocks, as required at P <= 8.  Both runs go through the upper half of every part table."""
    from bns_gcn_b200.data import partition_quality
    from tests.test_partition_multilevel_gpu import _compare
    fg, blk = _planted(P, True)
    _compare(fg, partition_quality(fg, blk, P), P, objective, 1.05)


# Measured ratio to the planted blocks of _planted_partition_graph(65536, P, 16, 2) (the result is a pure function of
# graph, P, objective and seed, so these are exact).  Its blocks are drawn at random, and at P = 33 and 64 the largest
# and smallest lie outside the size bounds, so no admissible partition reaches the planted value.  The shortfall is not
# confined to P > 32: on equal blocks the partitioner finds the planted partition exactly at P = 31, 33 and 48, but not
# at P = 32 (cut 1.775x, lower half only) or 64 (1.394x), so it is the level loop's search, not the upper half of the
# kernels.  These bars keep it from getting worse.
_PLANTED_RATIO = {(33, "cut"): 1.601, (33, "vol"): 1.161, (64, "cut"): 1.369, (64, "vol"): 1.131}


@pytest.mark.parametrize("objective", ["cut", "vol"])
@pytest.mark.parametrize("P", [33, 64])
def test_finds_the_planted_blocks_above_32_parts(built, P, objective):
    """_planted_partition_graph(65536, P, 16, 2) at P = 33 and 64: the bounds hold, the reported cut / vol is
    partition_quality's, the result is no worse than the stand-in, and no worse than its measured ratio to the planted
    blocks (_PLANTED_RATIO)."""
    from bns_gcn_b200.data import partition_quality
    from tests.test_partition_multilevel_gpu import _compare
    fg, blk = _planted(P, False)
    planted = partition_quality(fg, blk, P)
    q = _compare(fg, planted, P, objective, _PLANTED_RATIO[(P, objective)] + 0.0005)
    print(f"planted P={P} {objective}: {q[objective]} / {planted[objective]} = {q[objective] / planted[objective]:.3f}")


def test_deterministic_at_64_parts(built):
    from bns_gcn_b200.data.multilevel import multilevel_partition
    fg, _ = _planted(64, False)
    for objective in ("cut", "vol"):
        a, ia = multilevel_partition(fg, 64, objective, seed=0)
        b, ib = multilevel_partition(fg, 64, objective, seed=0)
        ia.pop("seconds"), ib.pop("seconds")
        assert torch.equal(a, b) and ia == ib
