"""The sampled boundary exchange of BNS-GCN, element by element: the boundary sampler, the id exchange, the per-epoch
slot and inverse maps, the compaction of the halo matrix to the sampled columns, the feature rows sent to the peers
and the gradient rows sent back, over both transports (peer-mapped ``p2p`` and ``nccl``), and the C ABI under them.

The exchange moves data exactly: it copies rows, divides them by the sampling ratio and adds them in a fixed order.
So every comparison here is bit for bit against the host restatements of ``tests/exchange_reference.py`` (and the
Philox replay of ``oracle/philox.py``), except the compacted SpMM, which is checked against float64 per element.

Every flag wait is enqueued after the put that satisfies it (on the same stream, or after ``Buffer``'s event hand-over
between in-process ranks), so no wait here ever spins."""
import ctypes
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from tests import exchange_reference as X
from tests.layer_reference import TOL, assert_close

pytestmark = pytest.mark.gpu

# Reddit split into 8 random partitions at sampling rate 0.1 (bench.py --gpus 8), derived once on the CPU with
#     fg = data.make_graph("reddit"); parts = data.partition_graph(fg, 8, "random")
# N_IN[r] = parts[r].graph.n_in.  Every node of a partition is a halo node of every other partition:
# bincount(parts[r].node_dict["part_id"][n_in:]) is N_IN[j] for every j != r.  So rank r's boundary toward each peer
# is all its N_IN[r] inner nodes (B = 7 N_IN[r] ~ 204 K), it sends int(0.1 N_IN[r]) = 2,912 rows to each peer, and
# its halo has sum(N_IN) - N_IN[r] ~ 204 K nodes.  HALO_NNZ[r] = entries of parts[r].graph.indices that are >= n_in
# (the halo matrix A_out); the longest row of a partition has 18,164 .. MAX_DEG entries.
N_IN = [29121, 29121, 29120, 29121, 29121, 29120, 29121, 29120]
HALO_NNZ = [12495463, 12862107, 12535860, 12451271, 12533658, 12508907, 12397190, 12288058]
MAX_DEG = 19073
RATE = 0.1
PATTERN = 0x7FA5A5A5          # a NaN: slab words the exchange must not touch keep it


@pytest.fixture(scope="module")
def lib(built):
    from bns_gcn_b200._lib import lib as l
    return l


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


def _check(rc, lib, what):
    assert rc == 0, f"{what}: {lib.bns_last_error().decode()}"


# ---- layouts ------------------------------------------------------------------------------------------------------
class Layout:
    """``P`` ranks, rank ``r`` with ``n_in[r]`` inner nodes; ``halo[r][j]`` of rank r's halo nodes are owned by j.
    Rank r's boundary toward j, ``bnd[r][j]``, is ``halo[j][r]`` sorted inner ids of r.  Sizes and ratios follow
    ``train.get_send_size`` / ``get_recv_size``; rank r's halo is ordered by owner, then by the owner's id, as
    ``data.extract_partition`` orders it, and ``pos[r][j]`` is ``train.get_pos``."""

    def __init__(self, n_in, halo, rate, seed):
        P = len(n_in)
        g = np.random.default_rng(seed)
        self.P, self.n_in, self.halo = P, list(n_in), halo
        self.bnd = [[None if j == r else
                     (np.arange(n_in[r]) if halo[j][r] == n_in[r] else np.sort(g.choice(n_in[r], halo[j][r], replace=False)))
                     for j in range(P)] for r in range(P)]
        self.send = [[0 if j == r else int(rate * halo[j][r]) for j in range(P)] for r in range(P)]
        self.recv = [[0 if j == r else int(rate * halo[r][j]) for j in range(P)] for r in range(P)]
        self.ratio = [[0 if j == r else (self.send[r][j] / halo[j][r] if halo[j][r] else 1.0) for j in range(P)]
                      for r in range(P)]
        self.n_halo = [sum(halo[r][j] for j in range(P) if j != r) for r in range(P)]
        self.pos, self.pl = [], []
        for r in range(P):
            pos, pl, hb, at = [], [], n_in[r], n_in[r]
            for j in range(P):
                if j == r:
                    pos.append(None)
                    pl.append(None)
                    continue
                p = np.full(n_in[j], -1, dtype=np.int64)
                p[self.bnd[j][r]] = hb + np.arange(halo[r][j])
                hb += halo[r][j]
                pos.append(p)
                pl.append(at)
                at += self.recv[r][j]
            self.pos.append(pos)
            self.pl.append(pl)
        self.n_u = [self.n_in[r] + sum(self.recv[r]) for r in range(P)]

    def sample(self, seed):
        """One epoch's selections: ``sel[r][j]`` = ``send[r][j]`` distinct ids of ``bnd[r][j]``, in random order."""
        g = np.random.default_rng(seed)
        return [[None if j == r else g.permutation(self.bnd[r][j])[:self.send[r][j]] for j in range(self.P)]
                for r in range(self.P)]


def headline_layout():
    return Layout(N_IN, [[0 if j == r else N_IN[j] for j in range(8)] for r in range(8)], RATE, 0)


def edge_layout():
    """8 small ranks with empty samples at the first, a middle and the last peer position: rank 0 sends nothing to
    peer 1 (5 boundary nodes at rate 0.1), to peer 4 (an empty boundary) and to peer 7; rank 7 to peer 0; rank 3 to 5."""
    n_in = [300, 257, 400, 123, 350, 64, 290, 311]
    g = np.random.default_rng(5)
    halo = [[0 if j == r else int(g.integers(n_in[j] // 3, n_in[j] + 1)) for j in range(8)] for r in range(8)]
    halo[1][0], halo[4][0], halo[7][0], halo[0][7], halo[5][3] = 5, 0, 9, 0, 3
    return Layout(n_in, halo, RATE, 1)


# ---- 1. sampler ---------------------------------------------------------------------------------------------------
def _check_sampler(dev, boundary, sizes, seed, offset, offset_dev=None, replay_offset=None):
    from bns_gcn_b200 import ops
    from oracle import philox
    s = ops.BoundarySampler([torch.from_numpy(b) for b in boundary], sizes, dev)
    od = None if offset_dev is None else torch.tensor([offset_dev], dtype=torch.int64, device=dev)
    _, views = s.sample(seed, offset, od)
    ref = philox.sample_boundary(boundary, sizes, seed, offset if replay_offset is None else replay_offset)
    for i, b in enumerate(boundary):
        v = views[i].cpu().numpy()
        assert np.array_equal(v, ref[i]), (i, seed, offset)                          # exact, in order
        assert v.size == sizes[i] and np.unique(v).size == v.size, i                 # no duplicates
        assert np.isin(v, b).all(), i                                                # a subset of its segment


def test_sampler_headline(built, dev):
    """Rank 0 of the headline layout: 7 segments of 29,120 .. 29,121 ids (B = 203,847), 2,912 taken from each."""
    boundary = [np.arange(N_IN[0]) for _ in range(7)]
    sizes = [int(RATE * N_IN[0])] * 7
    for seed, off in [(0, 0), (1, 1), (0x5EED, 17)]:
        _check_sampler(dev, boundary, sizes, seed, off)


@pytest.mark.parametrize("case", ["empty-boundary", "k0", "k-eq-b", "16-segments", "255-segments"])
def test_sampler_edges(built, dev, case):
    g = np.random.default_rng(11)
    if case == "empty-boundary":
        boundary = [np.sort(g.choice(900, 300, replace=False)), np.empty(0, np.int64), np.sort(g.choice(500, 77, replace=False))]
        sizes = [30, 0, 7]
    elif case == "k0":
        boundary = [np.sort(g.choice(900, 300, replace=False)) for _ in range(5)]
        sizes = [0, 30, 0, 0, 299]
    elif case == "k-eq-b":                                          # rate 1: every boundary node, in a random order
        boundary = [np.sort(g.choice(2000, n, replace=False)) for n in (1, 513, 1024)]
        sizes = [b.size for b in boundary]
    else:
        n = 16 if case == "16-segments" else 255
        lens = g.integers(0, 400, n)
        lens[::7] = 0
        boundary = [np.sort(g.choice(5000, int(m), replace=False)) for m in lens]
        sizes = [int(g.integers(0, m + 1)) for m in lens]
    for seed, off in [(3, 0), (2 ** 32 + 5, 9), (2 ** 63 + 2 ** 40 + 1, 2 ** 32 - 1), (77, 2 ** 32), (77, 2 ** 33 + 3)]:
        _check_sampler(dev, boundary, sizes, seed, off)


def test_sampler_graph_replay_offset(built, dev):
    """``offset = 2**64 - 1`` plus ``offset_dev = e + 1`` on the device (the CUDA-graph epoch) draws epoch e's sample."""
    boundary = [np.arange(N_IN[3]) for _ in range(7)]
    sizes = [int(RATE * N_IN[3])] * 7
    for e in (0, 1, 2, 2 ** 32 - 1, 2 ** 32):
        _check_sampler(dev, boundary, sizes, 1234, 2 ** 64 - 1, offset_dev=e + 1, replay_offset=e)


# ---- 3. epoch maps, directly ----------------------------------------------------------------------------------------
def test_epoch_maps_headline(built, lib, dev):
    """``bns_epoch_maps_update`` for rank 0 of the headline layout over four epochs with different samples; the last two
    leave the first, a middle and the last peer's segment empty.  Every entry the new epoch does not set is -1 again,
    including the ones the previous epoch set."""
    from bns_gcn_b200._lib import EpochMaps
    P, n_in = 8, N_IN[0]
    peers = list(range(1, P))
    n_pos = max(N_IN)
    pos, hb = [], n_in
    for j in peers:                                  # every node of every peer is one of rank 0's halo nodes
        p = np.full(n_pos, -1, dtype=np.int64)
        p[:N_IN[j]] = hb + np.arange(N_IN[j])
        hb += N_IN[j]
        pos.append(p)
    n_halo = hb - n_in
    pos_d = [torch.from_numpy(p).to(dev) for p in pos]
    maps = torch.full((n_halo + (P - 1) * n_in,), -1, dtype=torch.int32, device=dev)
    g = np.random.default_rng(9)
    k = int(RATE * n_in)
    for epoch in range(4):
        empty = (0, 3, 6) if epoch >= 2 else ()
        sel = [np.empty(0, np.int64) if s_ in empty else g.permutation(n_in)[:k] for s_ in range(P - 1)]
        hops = [np.empty(0, np.int64) if s_ in empty else g.permutation(N_IN[j])[:int(RATE * N_IN[j])]
                for s_, j in enumerate(peers)]
        sel_cat, hops_cat = torch.from_numpy(np.concatenate(sel)).to(dev), torch.from_numpy(np.concatenate(hops)).to(dev)
        m = EpochMaps()
        m.n_seg = P - 1
        a = b = 0
        for s_ in range(P - 1):
            m.sel_begin[s_], m.hop_begin[s_] = a, b
            a += sel[s_].size
            b += hops[s_].size
            m.pos[s_] = pos_d[s_].data_ptr()
            m.inv[s_] = maps[n_halo + s_ * n_in:].data_ptr()
        m.sel_begin[P - 1], m.hop_begin[P - 1] = a, b
        m.selected_cat, m.one_hops_cat, m.slot, m.n_in = sel_cat.data_ptr(), hops_cat.data_ptr(), maps.data_ptr(), n_in
        _check(lib.bns_epoch_maps_update(ctypes.byref(m), maps.data_ptr(), maps.numel() * 4,
                                         torch.cuda.current_stream().cuda_stream), lib, "bns_epoch_maps_update")
        slot_ref, inv_ref = X.epoch_maps(n_in, n_halo, pos, hops, sel)
        got = maps.cpu().numpy()
        assert np.array_equal(got[:n_halo], slot_ref), epoch
        for s_ in range(P - 1):
            assert np.array_equal(got[n_halo + s_ * n_in:n_halo + (s_ + 1) * n_in], inv_ref[s_]), (epoch, s_)


# ---- 2, 3, 5, 6. Buffer: ids, maps, rows forward, gradient rows back ---------------------------------------------------
def _dev_view(ptr, n, typestr, dev):
    from bns_gcn_b200.helper.feature_buffer import _DevArray
    return torch.as_tensor(_DevArray(ptr, (n,), typestr), device=dev)


def _exchange_rank(comm, rank, lay, cfg, shared):
    from bns_gcn_b200._lib import lib
    from bns_gcn_b200.helper.feature_buffer import Buffer
    dev = torch.device("cuda:0")
    P, n_in, F, L = lay.P, lay.n_in[rank], cfg.F, cfg.n_comm
    p2p = cfg.backend == "p2p"
    buf = Buffer()
    buf.init_buffer(n_in, lay.ratio[rank], lay.send[rank], lay.recv[rank], [cfg.width] * (L + 1), use_pp=True,
                    backend=cfg.backend, device=dev)
    assert buf._n_u == lay.n_u[rank] and buf._pl == lay.pl[rank]
    peers = [j for j in range(P) if j != rank]
    main = torch.cuda.current_stream()
    if p2p:
        n_slot = max(lay.n_halo[rank], 1)
        maps = torch.full((n_slot + (P - 1) * n_in,), -1, dtype=torch.int32, device=dev)
        buf.set_maps(maps, n_slot, [None if j == rank else torch.from_numpy(lay.pos[rank][j]).to(dev) for j in range(P)])
        slab_ptr, slab_bytes = ctypes.c_void_p(), ctypes.c_size_t()
        flags_ptr = ctypes.c_void_p()
        lib.bns_p2p_local(buf._p2p, ctypes.byref(slab_ptr), ctypes.byref(flags_ptr), ctypes.byref(slab_bytes))
        slab_words = _dev_view(slab_ptr.value, slab_bytes.value // 4, "<i4", dev)
        flags = _dev_view(flags_ptr.value, (2 * L + 1) * P, "<i8", dev)
    n_epochs = len(cfg.samples)
    for e in range(n_epochs):
        sel = cfg.samples[e]
        buf._timer.clear()                   # the comm timer's intervals are per epoch (train.py clears it too)
        graph = e >= n_epochs - cfg.graph_epochs
        if graph:
            if not buf.graph_mode:
                buf.graph_mode = True
                buf.seq_dev = torch.zeros(1, dtype=torch.int64, device=dev)
                buf.seq_base = max(buf._seq.values())
            buf.seq_dev.add_(1)
        mine = [None if j == rank else torch.from_numpy(sel[rank][j]).to(dev) for j in range(P)]
        sel_cat = torch.cat([mine[j] for j in peers])
        buf.set_selected(mine, sel_cat)
        if p2p:
            # 2. the id lists: what each peer selected for this rank, in order, as a private copy of the slab region
            cat, views = buf.exchange_ids(sel_cat)
            main.synchronize()
            want = [sel[j][rank] for j in peers]
            for j, w in zip(peers, want):
                assert np.array_equal(views[j].cpu().numpy(), w), (rank, e, j)
            _dev_view(slab_ptr.value + buf._ids_off, max(buf._recv_total, 1), "<i8", dev).fill_(-7)
            main.synchronize()
            assert np.array_equal(cat.cpu().numpy(), np.concatenate(want)), (rank, e)
            # 3. slot map + inverse maps, rebuilt over last epoch's
            buf.update_maps(sel_cat, cat, maps[:n_slot])
            slot_ref, inv_ref = X.epoch_maps(n_in, lay.n_halo[rank], [lay.pos[rank][j] for j in peers], want,
                                             [sel[rank][j] for j in peers])
            m = maps.cpu().numpy()
            assert np.array_equal(m[:lay.n_halo[rank]], slot_ref), (rank, e)
            for s_, j in enumerate(peers):
                assert np.array_equal(m[n_slot + s_ * n_in:n_slot + (s_ + 1) * n_in], inv_ref[s_]), (rank, e, j)
            if cfg.pattern:          # nobody writes into this slab between the two barriers
                comm.barrier()
                slab_words.fill_(PATTERN)
                main.synchronize()
            comm.barrier()
        # 5. forward
        feats, hs = [], []
        for l in range(1, L + 1):
            gen = torch.Generator(device=dev).manual_seed(1000 * e + 10 * l + rank)
            x = torch.randn(n_in, F, generator=gen, device=dev)
            if cfg.inplace and p2p:
                feat = buf.input_slot(l, n_in, F)
                assert feat is not None
                feat.copy_(x)
                feat.requires_grad_(True)
            else:
                feat = x.clone().requires_grad_(True)
            feats.append(feat)
            hs.append(buf.update(l, feat))
        main.synchronize()
        if p2p and cfg.pattern:
            for l in range(L):           # the forward wrote neither the gradient regions nor the id region
                b0 = buf._bwd_off[l] // 4
                bwd = slab_words[b0:b0 + max(buf._send_total, 1) * cfg.width]
                assert bool((bwd == PATTERN).all()), (rank, e, l)
            i0 = buf._ids_off // 4
            assert bool((slab_words[i0:i0 + 2 * max(buf._recv_total, 1)] == PATTERN).all()), (rank, e)
        h_cpu = [h.detach().cpu().numpy() for h in hs]
        x_cpu = [f.detach().cpu().numpy() for f in feats]
        grads = [torch.randn(lay.n_u[rank], F, generator=torch.Generator(device=dev).manual_seed(7919 * e + 31 * l + rank),
                             device=dev) for l in range(L)]
        g_cpu = [g.cpu().numpy() for g in grads]
        shared[(e, rank)] = (x_cpu, g_cpu)
        # 6. backward: the halo rows of the gradient go back to their owners and are added at the sampled rows
        torch.autograd.backward(hs, grads)
        main.synchronize()
        d_cpu = [f.grad.cpu().numpy() for f in feats]
        comm.barrier()
        for l in range(L):
            want_h = np.empty((lay.n_u[rank], F), dtype=np.float32)
            want_h[:n_in] = x_cpu[l]
            recv = [None] * P
            for j in peers:
                a, b = lay.pl[rank][j], lay.pl[rank][j] + lay.recv[rank][j]
                want_h[a:b] = X.send_rows(shared[(e, j)][0][l], sel[j][rank], lay.ratio[j][rank])
                aj = lay.pl[j][rank]
                recv[j] = shared[(e, j)][1][l][aj:aj + lay.send[rank][j]]
            assert np.array_equal(h_cpu[l].view(np.int32), want_h.view(np.int32)), (cfg.backend, rank, e, l + 1)
            want_d = X.scatter_ring(g_cpu[l][:n_in], rank, P, sel[rank], recv, lay.ratio[rank])
            assert np.array_equal(d_cpu[l].view(np.int32), want_d.view(np.int32)), (cfg.backend, rank, e, l + 1)
        if p2p:                      # every flag of this epoch carries this epoch's value, read from the device in graph mode
            value = (buf.seq_base + int(buf.seq_dev.item())) if graph else e + 1
            fl = flags.cpu().numpy()
            for j in peers:
                for l in range(L):
                    assert fl[(2 * l) * P + j] == value and fl[(2 * l + 1) * P + j] == value, (rank, e, j, l + 1)
                assert fl[2 * L * P + j] == value, (rank, e, j)
        comm.barrier()
        if rank == 0:
            for r in range(P):
                shared.pop((e - 1, r), None)
    comm.barrier()
    return True


def _run_exchange(lay, backend, F, width=None, epochs=2, graph_epochs=0, inplace=False, pattern=False, n_comm=2):
    from bns_gcn_b200.helper.comm import run_threads
    cfg = SimpleNamespace(backend=backend, F=F, width=width or F, n_comm=n_comm, inplace=inplace, pattern=pattern,
                          graph_epochs=graph_epochs,
                          samples=[lay.sample(100 + e) for e in range(epochs + graph_epochs)])
    assert all(run_threads(lay.P, _exchange_rank, lay, cfg, {}, device="cuda:0"))


@pytest.mark.parametrize("backend", ["p2p", "nccl"])
def test_exchange_headline(built, backend):
    """Reddit / 8 partitions at F = 256: ids, maps over two epochs with different samples, rows forward, gradient rows
    back -- both transports against the same host restatement, so bit-identical to each other."""
    _run_exchange(headline_layout(), backend, 256, pattern=backend == "p2p")


@pytest.mark.parametrize("backend,F,width", [("p2p", 256, 256), ("p2p", 44, 44), ("p2p", 41, 41),
                                             ("nccl", 256, 256), ("nccl", 44, 256), ("nccl", 41, 64)])
def test_exchange_edge_layout(built, backend, F, width):
    """Empty samples at the first, a middle and the last peer position; F = 41 takes the scalar paths of the put and of
    the gradient scatter."""
    _run_exchange(edge_layout(), backend, F, width, epochs=3, pattern=backend == "p2p")


def test_exchange_input_written_in_place(built):
    """``feat`` written straight into rows [0, n_in) of the concat buffer (``Buffer.input_slot``): no copy, same bits."""
    _run_exchange(edge_layout(), "p2p", 256, inplace=True)


@pytest.mark.parametrize("lay", ["headline", "edge"])
def test_exchange_graph_mode(built, lay):
    """``graph_mode``: flag values ``seq_base + *seq_dev`` read on the device, three epochs after two eager ones."""
    _run_exchange(headline_layout() if lay == "headline" else edge_layout(), "p2p", 256 if lay == "headline" else 44,
                  epochs=2, graph_epochs=3, n_comm=1 if lay == "headline" else 2)


def test_exchange_deep_model_over_p2p(built):
    """A model of 11 layers (10 that exchange) over p2p: every layer's put has a completion ticket of its own.  The
    ticket block used to hold world + 16 entries, which refused the 9th exchanging layer in the middle of the first
    epoch."""
    lay = Layout([200, 173], [[0, 150], [120, 0]], 0.3, 2)
    _run_exchange(lay, "p2p", 64, epochs=2, n_comm=10)


# ---- 4. halo compaction ------------------------------------------------------------------------------------------------
def _random_csr(n_rows, n_cols, nnz, g, max_deg):
    """Exactly ``nnz`` entries: one row of ``max_deg``, ~5 % empty rows, the rest spread at random."""
    p = g.random(n_rows)
    p[g.random(n_rows) < 0.05] = 0
    p[n_rows // 2] = 0
    deg = g.multinomial(nnz - max_deg, p / p.sum())
    deg[n_rows // 2] = max_deg
    indptr = np.concatenate([[0], np.cumsum(deg)]).astype(np.int64)
    return indptr, g.integers(0, n_cols, int(indptr[-1])).astype(np.int32)


def _edge_csr(g, n_cols, dead, live):
    """Rows around every chunk size (0, 1, 63 .. 2000 entries), rows with no live entry, and rows whose chunks (of 256
    and of 512) hold live entries only past entry 128."""
    rows = []
    for n in [0, 1, 5, 63, 64, 65, 127, 128, 129, 255, 256, 257, 300, 511, 512, 513, 1000, 2000, 0, 0]:
        rows.append(g.integers(0, n_cols, n))
    rows.append(g.choice(dead, 700))                       # no live entry at all
    rows.append(g.choice(dead, 40))
    for chunk in (256, 512):
        k = np.arange(3 * chunk + 77)
        rows.append(np.where(k % chunk < 130, g.choice(dead, k.size), g.choice(live, k.size)))
    for _ in range(200):
        rows.append(g.integers(0, n_cols, int(g.integers(0, 90))))
    indptr = np.concatenate([[0], np.cumsum([r.size for r in rows])]).astype(np.int64)
    return indptr, np.concatenate(rows).astype(np.int32)


def _slot_map(n_cols, n_slab, g, keep_dead=(), keep_live=()):
    slot = np.full(n_cols, -1, dtype=np.int32)
    cand = np.setdiff1d(np.arange(n_cols), np.concatenate([np.asarray(keep_dead, np.int64), np.asarray(keep_live, np.int64)]))
    cols = np.concatenate([np.asarray(keep_live, np.int64), g.choice(cand, n_slab - len(keep_live), replace=False)])
    slot[cols] = g.permutation(n_slab).astype(np.int32)
    return slot


def _check_compaction(dev, c, indptr, indices, chunk_nnz, slot, scale):
    cnt, dest, cidx, cw, cpos = X.compact_cols(indptr, indices, chunk_nnz, slot, scale)
    assert c.g.n_chunks == cnt.size
    assert np.array_equal(c.chunk_cnt.cpu().numpy()[:cnt.size], cnt)
    d = torch.from_numpy(dest).to(dev)
    assert np.array_equal(c.cidx[d].cpu().numpy(), cidx)
    assert np.array_equal(c.cpos[d].cpu().numpy(), cpos)
    if scale is not None:
        assert np.array_equal(c.cw[d].cpu().numpy().view(np.int32), cw.view(np.int32))


@pytest.mark.parametrize("weights", [False, True], ids=["sage", "gcn"])
def test_compaction_headline(built, dev, weights):
    """Rank 0's halo matrix at the headline size: 29,121 rows, ~204 K columns, 12.5 M entries, one row of 19,073, at
    the library's default chunk of 256 (two passes of 128 per chunk), ~2 K sampled columns from each of 7 peers."""
    from bns_gcn_b200 import ops
    g = np.random.default_rng(21)
    n_rows, n_cols = N_IN[0], sum(N_IN) - N_IN[0]
    indptr, indices = _random_csr(n_rows, n_cols, HALO_NNZ[0], g, MAX_DEG)
    assert indices.size == HALO_NNZ[0]
    G = ops.DeviceGraph.from_csr(torch.from_numpy(indptr).to(dev), torch.from_numpy(indices).to(dev), n_cols)
    scale = (g.random(n_cols) + 0.5).astype(np.float32) if weights else None
    c = ops.CompactedCols(G, with_weights=weights, with_positions=True)
    for epoch in range(2):
        slot = _slot_map(n_cols, 7 * int(RATE * N_IN[1]), g)
        c.refresh(torch.from_numpy(slot).to(dev), 0, None if scale is None else torch.from_numpy(scale).to(dev))
        _check_compaction(dev, c, indptr, indices, 256, slot, scale)


@pytest.mark.parametrize("chunk_nnz", [64, 256, 512])
def test_compaction_edges_and_compact_spmm(built, dev, chunk_nnz):
    """Compaction of rows longer than a chunk, empty rows, rows with no live entry, and chunks whose live entries all sit
    past entry 128, over two epochs that reuse the buffers; then the compacted SpMM at F = 256 and 44, with row scale,
    GCN's column scale and accumulation, against float64 per element."""
    from bns_gcn_b200 import ops
    g = np.random.default_rng(chunk_nnz)
    n_cols, n_slab = 3000, 700
    dead, live = np.arange(0, 200), np.arange(200, 260)
    indptr, indices = _edge_csr(g, n_cols, dead, live)
    n_rows = indptr.size - 1
    G = ops.DeviceGraph.from_csr(torch.from_numpy(indptr).to(dev), torch.from_numpy(indices).to(dev), n_cols, chunk_nnz)
    scale = (g.random(n_cols) + 0.5).astype(np.float32)
    rs = (g.random(n_rows) + 0.5).astype(np.float32)
    rows = np.repeat(np.arange(n_rows), np.diff(indptr))
    worst = 0.0
    for weights in (False, True):
        c = ops.CompactedCols(G, with_weights=weights, with_positions=True)
        for epoch in range(2):
            slot = _slot_map(n_cols, n_slab, g, dead, live)
            sc = scale if weights else None
            c.refresh(torch.from_numpy(slot).to(dev), 0, None if sc is None else torch.from_numpy(sc).to(dev))
            _check_compaction(dev, c, indptr, indices, chunk_nnz, slot, sc)
            for F in (256, 44):
                x = g.standard_normal((n_slab, F)).astype(np.float32)
                y0 = g.standard_normal((n_rows, F)).astype(np.float32)
                out = torch.from_numpy(y0).to(dev)
                ops.spmm_compact(c, torch.from_numpy(x).to(dev), out, row_scale=torch.from_numpy(rs).to(dev), accumulate=True)
                m = slot[indices] >= 0
                w = torch.from_numpy(scale[indices[m]] if weights else np.ones(int(m.sum()), np.float32)).double()
                v, u = torch.from_numpy(rows[m]), torch.from_numpy(slot[indices[m]].astype(np.int64))
                xd = torch.from_numpy(x).double()
                agg = torch.zeros(n_rows, F, dtype=torch.float64).index_add_(0, v, xd[u] * w.unsqueeze(1))
                mag = torch.zeros(n_rows, F, dtype=torch.float64).index_add_(0, v, xd[u].abs() * w.unsqueeze(1))
                r = torch.from_numpy(rs).double().unsqueeze(1)
                want = torch.from_numpy(y0).double() + r * agg
                bound = torch.from_numpy(y0).double().abs() + r * mag
                worst = max(worst, assert_close(f"compact spmm chunk {chunk_nnz} F {F} gcn {weights}", out.cpu(), want,
                                                bound))
    print(f"[ratio] compact spmm chunk {chunk_nnz}: worst {worst:.3g} x TOL ({TOL:g})")


# ---- 7, 8. the C ABI directly: two and more bns_p2p_t on one GPU ----------------------------------------------------
class _P2P:
    def __init__(self, lib, rank, world, slab_bytes, n_flags, dev):
        self.lib, self.rank, self.n_flags = lib, rank, n_flags
        h = ctypes.c_void_p()
        _check(lib.bns_p2p_create(ctypes.byref(h), rank, world, slab_bytes, n_flags), lib, "bns_p2p_create")
        self.h = h
        slab, flags, nb = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_size_t()
        _check(lib.bns_p2p_local(h, ctypes.byref(slab), ctypes.byref(flags), ctypes.byref(nb)), lib, "bns_p2p_local")
        self.slab, self.flags_ptr, self.nbytes = slab.value, flags.value, nb.value
        self.words = _dev_view(self.slab, self.nbytes // 4, "<i4", dev)
        self.flags = _dev_view(self.flags_ptr, n_flags, "<i8", dev)

    def connect(self, other):
        _check(self.lib.bns_p2p_set_peer(self.h, other.rank, other.slab, other.flags_ptr, other.nbytes), self.lib,
               "bns_p2p_set_peer")

    def close(self):
        self.lib.bns_p2p_destroy(self.h)


@pytest.fixture
def fabric(lib, dev):
    """Rank 0 connected to ranks 1 and 2 of a world of 4 (rank 3 exists but is not connected)."""
    ps = [_P2P(lib, r, 4, 1 << 21, 40 if r == 0 else 8, dev) for r in range(4)]
    ps[0].connect(ps[1])
    ps[0].connect(ps[2])
    torch.cuda.synchronize()
    yield ps
    torch.cuda.synchronize()
    for p in ps:
        p.close()


def _put_all(lib, p, segs, ld_remote, H, ldh, F, idx, flag, ticket, value, value_dev=None):
    from bns_gcn_b200._lib import PutAll
    s = PutAll()
    s.n_seg = len(segs)
    at = 0
    for i, (peer, k, off, src) in enumerate(segs):
        s.row_begin[i] = at
        at += k
        s.peer[i], s.remote_off[i], s.src_begin[i], s.div[i] = peer, off, src, [3.0, 0.7, 1.5, 0.1, 2.5, 9.0][i % 6]
    s.row_begin[len(segs)] = at
    rc = lib.bns_p2p_put_all_f32(p.h, ctypes.byref(s), ld_remote, H, ldh, F, idx, flag, ticket, value, value_dev,
                                 torch.cuda.current_stream().cuda_stream)
    return rc, s


@pytest.mark.parametrize("F,ld_remote,h_shift,with_idx,off_shift", [
    (41, 41, 0, True, 0), (41, 45, 0, False, 0), (44, 48, 0, True, 0), (44, 48, 1, True, 0), (44, 44, 0, False, 4),
    (256, 260, 0, False, 0), (256, 256, 1, True, 0), (256, 256, 0, True, 0)])
def test_put_all_rows_and_untouched_words(lib, dev, fabric, F, ld_remote, h_shift, with_idx, off_shift):
    """``bns_p2p_put_all_f32`` from rank 0 into ranks 1 and 2: zero-row segments between non-empty ones, two segments
    into the same peer, an ``idx`` list or ``src_begin``, a source one float off 16-byte alignment, ``ld_remote > F``,
    destinations 4 bytes off 16-byte alignment (the scalar path).  Every written row is exact; every other word of the
    receiving slabs -- the rows past a segment, the columns past F -- keeps its sentinel."""
    p0, p1, p2 = fabric[0], fabric[1], fabric[2]
    g = np.random.default_rng(F + ld_remote + h_shift)
    n_src = 300
    Hbuf = torch.from_numpy(g.standard_normal(n_src * (F + 3) + 8).astype(np.float32)).to(dev)
    ldh = F + 3 if h_shift else F
    H = Hbuf[h_shift:h_shift + n_src * ldh].view(n_src, ldh)
    row = ld_remote * 4
    segs = [(1, 5, 16 * 5 + off_shift, 10), (2, 0, 0, 0), (1, 7, 16 * 5 + off_shift + 9 * row, 50), (2, 0, 64, 0),
            (2, 9, 16 + off_shift, 100), (1, 0, 0, 0), (2, 3, 16 + off_shift + 20 * row, 200)]
    total = sum(k for _, k, _, _ in segs)
    idx_np = g.permutation(n_src)[:total].astype(np.int64)
    idx = torch.from_numpy(idx_np).to(dev) if with_idx else None
    for p in (p1, p2):
        p.words.fill_(PATTERN)
        p.flags.zero_()
    for rep in range(2):             # the same flag value twice: the ticket is re-armed by the first launch
        if rep:
            p1.flags.zero_()
            p2.flags.zero_()
        rc, s = _put_all(lib, p0, segs, ld_remote, H.data_ptr(), ldh, F, None if idx is None else idx.data_ptr(), 3, 4 + 20,
                         11, None)
        _check(rc, lib, "bns_p2p_put_all_f32")
        torch.cuda.synchronize()
        want = {1: np.full(p1.nbytes // 4, PATTERN, np.int32), 2: np.full(p2.nbytes // 4, PATTERN, np.int32)}
        Hn, at = H.cpu().numpy(), 0
        for i, (peer, k, off, src) in enumerate(segs):
            rows = idx_np[at:at + k] if with_idx else src + np.arange(k)
            vals = Hn[rows, :F] / np.float32(s.div[i])
            for t in range(k):
                w0 = off // 4 + t * ld_remote
                want[peer][w0:w0 + F] = vals[t].view(np.int32)
            at += k
        for peer, p in ((1, p1), (2, p2)):
            got = p.words.cpu().numpy()
            bad = np.nonzero(got != want[peer])[0]
            assert bad.size == 0, (peer, rep, bad[:8])
            assert p.flags.cpu().numpy()[3] == 11


def test_flag_value_from_device_and_shared_tickets(lib, dev, fabric):
    """The published value is ``flag_value + *flag_value_dev``; a put of rows and a put of ids that share one ticket,
    with different grid sizes, each re-arm it and each publish."""
    p0, p1, p2 = fabric[0], fabric[1], fabric[2]
    IDS_OFF = 3 << 19                                      # past the 4,000 rows of 64 floats
    H = torch.randn(5000, 64, device=dev)
    vdev = torch.tensor([6], dtype=torch.int64, device=dev)
    ids = torch.arange(3000, dtype=torch.int64, device=dev) * 3
    for rep in range(3):
        for p in (p1, p2):
            p.flags.zero_()
        _check(_put_all(lib, p0, [(1, 4000, 0, 0), (2, 0, 0, 0)], 64, H.data_ptr(), 64, 64, None, 2, 7, 5,
                        vdev.data_ptr())[0], lib, "bns_p2p_put_all_f32")
        torch.cuda.synchronize()
        assert p1.flags.cpu()[2].item() == 11 and p2.flags.cpu()[2].item() == 11, rep
        begin = (ctypes.c_int64 * 3)(0, 1000, 3000)
        peers = (ctypes.c_int32 * 2)(1, 2)
        roff = (ctypes.c_uint64 * 2)(IDS_OFF, IDS_OFF)
        _check(lib.bns_p2p_put_ids_i64(p0.h, 2, begin, peers, roff, ids.data_ptr(), 5, 7, 9 + rep, None,
                                       torch.cuda.current_stream().cuda_stream), lib, "bns_p2p_put_ids_i64")
        torch.cuda.synchronize()
        assert p1.flags.cpu()[5].item() == 9 + rep and p2.flags.cpu()[5].item() == 9 + rep, rep
        got1 = _dev_view(p1.slab + IDS_OFF, 1000, "<i8", dev).cpu()
        got2 = _dev_view(p2.slab + IDS_OFF, 2000, "<i8", dev).cpu()
        assert torch.equal(got1, ids[:1000].cpu()) and torch.equal(got2, ids[1000:].cpu())
        want = (H[:4000].cpu().numpy() / np.float32(3.0)).view(np.int32)
        assert np.array_equal(p1.words[:4000 * 64].cpu().numpy().reshape(4000, 64), want)


@pytest.mark.parametrize("F,shift,n_seg", [(41, 0, 5), (44, 1, 5), (44, 0, 5), (256, 0, 5), (256, 1, 5), (8, 0, 7)],
                         ids=["41-0", "44-1", "44-0", "256-0", "256-1", "8-0-7seg"])
def test_scatter_rows_all(lib, dev, F, shift, n_seg):
    """``bns_scatter_rows_all_f32``: G[r] += recv_s[inv_s[r]] / div_s for the segments in table order, with F = 41, a
    receive buffer one float off alignment (both scalar) and the aligned 16-byte path, the latter also at F = 8 with 7
    segments, where only 2 lanes of a warp hold columns but every lane takes part in the segment shuffles."""
    g = np.random.default_rng(F + shift)
    n_rows = 3000
    ld = F + 4
    G0 = g.standard_normal((n_rows, F)).astype(np.float32)
    inv, recv, keep = [], [], []
    for s in range(n_seg):
        k = [700, 0, 1500, 1, 2999, 40, 3000][s]
        sel = g.permutation(n_rows)[:k]
        m = np.full(n_rows, -1, np.int32)
        m[sel] = np.arange(k, dtype=np.int32)
        r = g.standard_normal((max(k, 1), ld)).astype(np.float32)
        inv.append(m)
        recv.append(r)
        buf = torch.zeros(max(k, 1) * ld + 4, device=dev)
        buf[shift:shift + r.size] = torch.from_numpy(r.reshape(-1)).to(dev)
        keep.append((torch.from_numpy(m).to(dev), buf))
    div = [0.3, 1.0, 0.26, 7.0, 0.1, 3.0, 0.7][:n_seg]
    want = G0.copy()
    for s in range(n_seg):
        rows = np.nonzero(inv[s] >= 0)[0]
        want[rows] = want[rows] + recv[s][inv[s][rows], :F] / np.float32(div[s])
    G = torch.from_numpy(G0).to(dev)
    ip = (ctypes.c_void_p * n_seg)(*[m.data_ptr() for m, _ in keep])
    rp = (ctypes.c_void_p * n_seg)(*[b.data_ptr() + 4 * shift for _, b in keep])
    dv = (ctypes.c_float * n_seg)(*div)
    _check(lib.bns_scatter_rows_all_f32(G.data_ptr(), F, n_rows, F, n_seg, ip, rp, ld, dv,
                                        torch.cuda.current_stream().cuda_stream), lib, "bns_scatter_rows_all_f32")
    assert np.array_equal(G.cpu().numpy().view(np.int32), want.view(np.int32))


def test_refusals(lib, dev, fabric):
    """Every malformed call returns an error before it launches anything."""
    p0, p1 = fabric[0], fabric[1]
    H = torch.randn(64, 64, device=dev)
    n_tickets = 4 + max(p0.n_flags, 16)

    def refused(segs, flag=1, ticket=4, n_seg=None, ld=64):
        before = lib.bns_launch_count()
        from bns_gcn_b200._lib import PutAll
        if n_seg is None:
            rc = _put_all(lib, p0, segs, ld, H.data_ptr(), 64, 64, None, flag, ticket, 1)[0]
        else:
            s = PutAll()
            s.n_seg = n_seg
            rc = lib.bns_p2p_put_all_f32(p0.h, ctypes.byref(s), ld, H.data_ptr(), 64, 64, None, flag, ticket, 1, None,
                                         torch.cuda.current_stream().cuda_stream)
        return rc != 0 and lib.bns_launch_count() == before

    assert refused([(1, 8, p1.nbytes - 16 * 64, 0)])                     # remote range past the peer's slab
    assert refused([(1, 1, p1.nbytes - 240, 0)])
    assert refused([(1, 2, 2, 0)])                                        # misaligned remote_off
    assert refused([(2, 2, 6, 0)])
    assert refused([(0, 2, 0, 0)])                                        # peer == rank
    assert refused([(3, 2, 0, 0)])                                        # a peer that is not connected
    assert refused([(1, 2, 0, 0), (5, 2, 0, 0)])                          # ... or not in the world
    from bns_gcn_b200._lib import PutAll
    s = PutAll()
    s.n_seg, s.row_begin[1], s.peer[0], s.div[0] = 1, 3, 1, 0.0           # div == 0 with rows to send
    before = lib.bns_launch_count()
    assert lib.bns_p2p_put_all_f32(p0.h, ctypes.byref(s), 64, H.data_ptr(), 64, 64, None, 1, 4, 1, None, None) != 0
    assert lib.bns_launch_count() == before
    assert refused(None, n_seg=17)                                        # n_seg > BNS_MAX_PEERS
    assert refused([(1, 2, 0, 0)], flag=p0.n_flags) and refused([(1, 2, 0, 0)], flag=-1)
    assert refused([(1, 2, 0, 0)], ticket=n_tickets) and refused([(1, 2, 0, 0)], ticket=-1)
    # the ids put: the same ticket and flag bounds
    begin, peers, roff = (ctypes.c_int64 * 2)(0, 0), (ctypes.c_int32 * 1)(1), (ctypes.c_uint64 * 1)(0)
    for flag, ticket in ((p0.n_flags, 4), (0, n_tickets), (0, -1)):
        before = lib.bns_launch_count()
        assert lib.bns_p2p_put_ids_i64(p0.h, 1, begin, peers, roff, None, flag, ticket, 1, None, None) != 0
        assert lib.bns_launch_count() == before
    # with 40 flags, the last ticket is 4 + 40 - 1 (past the old limit of world + 16): accepted and published
    p1.flags.zero_()
    _check(_put_all(lib, p0, [(1, 2, 0, 0)], 64, H.data_ptr(), 64, 64, None, 1, n_tickets - 1, 13)[0], lib,
           "bns_p2p_put_all_f32")
    torch.cuda.synchronize()
    assert p1.flags.cpu()[1].item() == 13
