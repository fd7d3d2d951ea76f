"""``--comm-dtype bf16``: the boundary exchange with a bf16 wire side, on in-process ranks on one GPU.

Kernels: every new entry point bit for bit against torch -- the put against the f32 put's rows rounded by
``.to(torch.bfloat16)`` on the same device, the scatter-adds against their f32 siblings run on widened copies of the same
bf16 rows -- with NaN, +-Inf, subnormals and round-to-even ties, zero-row segments, 1 / 2 / 7 peers, F = 8 / 64 / 256
with rows wider than F; malformed arguments return BNS_E_INVALID before anything launches.

Exchange: ``Buffer`` over both transports against the host restatements of ``tests/exchange_reference.py``: the received
halo rows are the bf16 rounding of the reference rows, and the owners' gradients the reference scatter of the rounded
returned rows, bit for bit.

Layers: ``SageConvFn`` / ``GcnConvFn``, wide and narrow, fed the inner rows and a bf16 halo table, against the float64
restatement of ``tests/layer_reference.py`` on the widened rows: output, inner and halo gradients, parameter gradients.

Training step: with ``--agg-dtype bf16`` the wide layers' forward is bit-identical between ``--comm-dtype f32`` and
``bf16``; at one partition the flag changes nothing; the benchmark's model trains on the Reddit shape with 4 ranks."""
import ctypes
import functools
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from tests import exchange_reference as X
from tests.test_boundary_exchange_gpu import PATTERN, Layout, _P2P, _dev_view, edge_layout, headline_layout
from tests.test_spmm_bf16_gpu import _specials

pytestmark = pytest.mark.gpu

E_INVALID = -1


@pytest.fixture(scope="module")
def lib(built):
    from bns_gcn_b200._lib import lib as l
    return l


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


def _check(rc, lib, what):
    assert rc == 0, f"{what}: {lib.bns_last_error().decode()}"


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _f32_rows(n, ld, seed, dev):
    """f32 rows of random bit patterns (every exponent), the special values, and ties: column 0 holds values whose low 16
    bits are 0x8000 (halfway between two bf16), even and odd."""
    gen = torch.Generator().manual_seed(seed)
    bits = torch.randint(-2 ** 31, 2 ** 31, (n, ld), generator=gen, dtype=torch.int64).to(torch.int32)
    x = bits.view(torch.float32)
    sp = _specials()
    k = min(sp.numel(), x.numel() // 3)
    x.view(-1)[:k * 3:3] = sp[:k]
    ties = torch.randint(-2 ** 31, 2 ** 31, (n,), generator=gen, dtype=torch.int64).to(torch.int32) & ~0xffff | 0x8000
    x[:, 0] = ties.view(torch.float32)
    return x.to(dev)


def _bf16_rows(n, ld, seed, dev):
    """bf16 rows of random bit patterns (NaN, +-Inf, subnormals and zeros included)."""
    gen = torch.Generator().manual_seed(seed)
    bits = torch.randint(-2 ** 15, 2 ** 15, (n, ld), generator=gen, dtype=torch.int32).to(torch.int16)
    sp = torch.tensor([0x7FC0, 0x7F81, 0xFFC1 - 65536, 0x7F80, 0xFF80 - 65536, 0x0001, 0x8001 - 65536, 0x007F, 0, -32768],
                      dtype=torch.int16)
    k = min(sp.numel(), (bits.numel() + 4) // 5)
    bits.view(-1)[:k * 5:5] = sp[:k]
    return bits.view(torch.bfloat16).to(dev)


# ---- kernels -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("with_idx", [True, False], ids=["idx", "src-begin"])
@pytest.mark.parametrize("F", [8, 64, 256])
@pytest.mark.parametrize("n_peers", [1, 2, 7])
def test_put_all_bf16_is_the_rounded_f32_put(lib, dev, n_peers, F, with_idx):
    """Rank 0 puts into ``n_peers`` peers, each with a zero-row segment beside its rows (two segments per peer), rows
    ``ld = F + 8`` wide; the divisors include 1 (ties reach the rounding unchanged).  The bf16 rows equal the f32 put's
    rows rounded on the device, and every other half-word of the receiving slabs keeps its sentinel."""
    from bns_gcn_b200._lib import PutAll
    world, ld = n_peers + 1, F + 8
    ps = [_P2P(lib, r, world, 1 << 21, 8, dev) for r in range(world)]
    try:
        for p in ps[1:]:
            ps[0].connect(p)
        g = np.random.default_rng(100 * n_peers + F)
        counts = [(int(g.integers(1, 40)), 0) for _ in range(n_peers)]
        counts[0] = (0, int(g.integers(1, 40)))                 # a zero-row segment first
        total = sum(a + b for a, b in counts)
        n_src = 3 * total + 200                                 # src_begin of a segment is 3 * (its first row) + 1
        H = torch.empty(n_src, F + 8, device=dev)[:, :F].copy_(_f32_rows(n_src, F, F + int(with_idx), dev))
        idx = torch.from_numpy(g.permutation(n_src)[:total].astype(np.int64)).to(dev)
        divs = [1.0, 0.3, 7.0, 0.1, 2.5, 1.0, 0.7]
        F32_OFF, BF_OFF = 0, 1 << 20

        def segs(bf16):
            s, at, i = PutAll(), 0, 0
            for j in range(n_peers):
                for h, k in enumerate(counts[j]):
                    s.row_begin[i] = at
                    s.peer[i] = j + 1
                    s.src_begin[i] = 3 * at + 1
                    s.div[i] = divs[(j + h) % len(divs)]
                    row0 = sum(counts[j][:h])
                    s.remote_off[i] = (BF_OFF + row0 * ld * 2) if bf16 else (F32_OFF + row0 * ld * 4)
                    at += k
                    i += 1
            s.n_seg, s.row_begin[i] = i, at
            return s
        for p in ps[1:]:
            p.words.fill_(PATTERN)
            p.flags.zero_()
        ip = idx.data_ptr() if with_idx else None
        _check(lib.bns_p2p_put_all_f32(ps[0].h, ctypes.byref(segs(False)), ld, H.data_ptr(), H.stride(0), F, ip, 1,
                                       world, 5, None, _stream()), lib, "bns_p2p_put_all_f32")
        _check(lib.bns_p2p_put_all_bf16(ps[0].h, ctypes.byref(segs(True)), ld, H.data_ptr(), H.stride(0), F, ip, 2,
                                        world + 1, 6, None, _stream()), lib, "bns_p2p_put_all_bf16")
        torch.cuda.synchronize()
        for j in range(n_peers):
            p, n = ps[j + 1], sum(counts[j])
            f32 = p.words[:n * ld].view(torch.float32).view(max(n, 1), ld)[:n] if n else None
            half = p.words.view(torch.int16)
            want = torch.full((half.numel(),), 0, dtype=torch.int16, device=dev)
            want.view(torch.int32).fill_(PATTERN)
            if n:
                want[(BF_OFF // 2):(BF_OFF // 2) + n * ld].view(n, ld)[:, :F] = f32[:, :F].to(torch.bfloat16).view(torch.int16)
                want[:n * ld * 2] = half[:n * ld * 2]                                         # the f32 region
            assert torch.equal(half, want), (j, n)
            fl = p.flags.cpu()
            assert fl[1].item() == 5 and fl[2].item() == 6, j
    finally:
        torch.cuda.synchronize()
        for p in ps:
            p.close()


@pytest.mark.parametrize("F", [8, 64, 256])
@pytest.mark.parametrize("n_seg", [1, 2, 7])
def test_scatter_rows_all_bf16_is_the_f32_scatter_of_widened_rows(lib, dev, n_seg, F):
    """Segments with 0 / 1 / many / all rows selected, ``ld_recv = F + 8``: the bf16 scatter equals the segments added
    in order with one f32 division and one f32 add per element, and (F = 256) ``bns_scatter_rows_all_f32`` over
    ``recv.float()``, bit for bit."""
    g = np.random.default_rng(n_seg * 1000 + F)
    n_rows, ld = 2000, F + 8
    G0 = _f32_rows(n_rows, F, F, dev).clone()
    G0[G0.isnan() | G0.isinf()] = 1.5                        # keep the destination finite; the rows carry the specials
    invs, rb, rf = [], [], []
    for s in range(n_seg):
        k = [700, 0, 1, n_rows, 33, 1500, 2][s]
        m = np.full(n_rows, -1, np.int32)
        m[g.permutation(n_rows)[:k]] = np.arange(k, dtype=np.int32)
        invs.append(torch.from_numpy(m).to(dev))
        r = _bf16_rows(max(k, 1), ld, 10 * s + F, dev)
        rb.append(r)
        rf.append(r.float())
    divs = [0.3, 1.0, 7.0, 0.26, 1.0, 3.0, 0.1][:n_seg]
    div = (ctypes.c_float * n_seg)(*divs)
    inv = (ctypes.c_void_p * n_seg)(*[m.data_ptr() for m in invs])
    G2 = G0.clone()
    _check(lib.bns_scatter_rows_all_bf16(G2.data_ptr(), F, n_rows, F, n_seg, inv,
                                         (ctypes.c_void_p * n_seg)(*[r.data_ptr() for r in rb]), ld, div, _stream()),
           lib, "bns_scatter_rows_all_bf16")
    want = G0.clone()                       # the segments in order, one f32 division and one f32 add per element
    for s in range(n_seg):
        rows = (invs[s] >= 0).nonzero().squeeze(1)
        r = rf[s][invs[s][rows].long(), :F]
        want[rows] = want[rows] + r / torch.full_like(r, divs[s])        # a true division (a scalar one multiplies)
    assert torch.equal(G2.view(torch.int32), want.view(torch.int32))
    if F >= 128:
        # the f32 sibling on the widened rows; it is only run where every lane of its warp takes part in its shuffles
        G1 = G0.clone()
        _check(lib.bns_scatter_rows_all_f32(G1.data_ptr(), F, n_rows, F, n_seg, inv,
                                            (ctypes.c_void_p * n_seg)(*[r.data_ptr() for r in rf]), ld, div, _stream()),
               lib, "bns_scatter_rows_all_f32")
        assert torch.equal(G1.view(torch.int32), G2.view(torch.int32))


@pytest.mark.parametrize("F", [8, 64, 256])
def test_staged_pack_and_scatter_bf16(lib, dev, F):
    """The staged transport: ``bns_gather_div_bf16`` is ``bns_gather_div_f32`` rounded on the device, and
    ``bns_scatter_add_div_bf16`` is ``bns_scatter_add_div_f32`` over the widened rows; rows ``F + 8`` wide."""
    from bns_gcn_b200 import ops
    g = np.random.default_rng(F)
    ld = F + 8
    H = torch.empty(500, ld, device=dev)[:, :F].copy_(_f32_rows(500, F, F, dev))
    idx = torch.from_numpy(g.permutation(500)[:300].astype(np.int64)).to(dev)
    for div in (1.0, 0.37, 3.0):
        out32 = torch.empty(300, ld, device=dev)[:, :F]
        out16 = torch.full((300, ld), -7.0, dtype=torch.bfloat16, device=dev)
        ops.gather_div(H, idx, div, out=out32)
        ops.gather_div(H, idx, div, out=out16[:, :F])
        assert torch.equal(out16[:, :F].view(torch.int16), out32.to(torch.bfloat16).view(torch.int16)), div
        assert torch.all(out16[:, F:] == -7.0)
        src = _bf16_rows(300, ld, F + int(10 * div), dev)[:, :F]
        G0 = torch.empty(500, ld, device=dev)[:, :F].copy_(torch.randn(500, F, device=dev))
        G1, G2 = G0.clone(), G0.clone()
        ops.scatter_add_div(G1, idx, src.float(), div)
        ops.scatter_add_div(G2, idx, src, div)
        assert torch.equal(G1.view(torch.int32), G2.view(torch.int32)), div


@pytest.mark.parametrize("F,lds,ldd", [(256, 256, 256), (256, 264, 260), (64, 72, 64), (8, 8, 8), (41, 43, 45)])
def test_cvt_rows_bf16_f32_is_exact(built, dev, F, lds, ldd):
    from bns_gcn_b200 import ops
    src = _bf16_rows(3000, lds, F, dev)
    dst = torch.full((3000, ldd), -7.0, device=dev)
    ops.cvt_rows_f32(src[:, :F], out=dst[:, :F])
    assert torch.equal(dst[:, :F].view(torch.int32), src[:, :F].float().view(torch.int32))
    assert torch.all(dst[:, F:] == -7.0)


def test_refusals(lib, dev):
    """Non-multiple-of-8 widths and strides, a misaligned source, destination offset or receive row: BNS_E_INVALID,
    nothing launched."""
    from bns_gcn_b200._lib import PutAll
    ps = [_P2P(lib, r, 2, 1 << 20, 8, dev) for r in range(2)]
    try:
        ps[0].connect(ps[1])
        H = torch.randn(64, 72, device=dev)

        def put(F=64, ldh=72, ld=64, off=0, h=H.data_ptr()):
            s = PutAll()
            s.n_seg, s.row_begin[1], s.peer[0], s.div[0], s.remote_off[0] = 1, 4, 1, 1.0, off
            before = lib.bns_launch_count()
            rc = lib.bns_p2p_put_all_bf16(ps[0].h, ctypes.byref(s), ld, h, ldh, F, None, 1, 2, 1, None, _stream())
            return rc == E_INVALID and lib.bns_launch_count() == before
        assert put(F=60) and put(F=12, ld=16) and put(ldh=68) and put(ld=68) and put(off=8) and put(off=4)
        assert put(h=H.data_ptr() + 4)
        assert put(off=(1 << 20) - 64 * 2 * 3)                       # past the peer's slab
        assert not put() and torch.cuda.synchronize() is None       # the well-formed call goes through
        G = torch.zeros(100, 72, device=dev)
        inv = torch.full((100,), -1, dtype=torch.int32, device=dev)
        rb = torch.zeros(8, 72, dtype=torch.bfloat16, device=dev)
        one_f = (ctypes.c_float * 1)(1.0)

        def scat(F=64, ldg=72, ld=72, g=G.data_ptr(), r=rb.data_ptr()):
            before = lib.bns_launch_count()
            rc = lib.bns_scatter_rows_all_bf16(g, ldg, 100, F, 1, (ctypes.c_void_p * 1)(inv.data_ptr()),
                                               (ctypes.c_void_p * 1)(r), ld, one_f, _stream())
            return rc == E_INVALID and lib.bns_launch_count() == before
        assert scat(F=60) and scat(ldg=70) and scat(ld=68) and scat(g=G.data_ptr() + 8) and scat(r=rb.data_ptr() + 2)
        idx = torch.arange(8, dtype=torch.int64, device=dev)
        out = torch.zeros(8, 72, dtype=torch.bfloat16, device=dev)
        before = lib.bns_launch_count()
        for h, ldh, F, o, ldo in ((H.data_ptr(), 72, 60, out.data_ptr(), 72), (H.data_ptr(), 68, 64, out.data_ptr(), 72),
                                  (H.data_ptr(), 72, 64, out.data_ptr(), 68), (H.data_ptr() + 4, 72, 64, out.data_ptr(), 72),
                                  (H.data_ptr(), 72, 64, out.data_ptr() + 2, 72)):
            assert lib.bns_gather_div_bf16(h, ldh, F, idx.data_ptr(), 8, 1.0, o, ldo, _stream()) == E_INVALID
        for g_, ldg, F, src, lds in ((G.data_ptr(), 72, 60, out.data_ptr(), 72), (G.data_ptr(), 68, 64, out.data_ptr(), 72),
                                     (G.data_ptr(), 72, 64, out.data_ptr(), 68), (G.data_ptr() + 4, 72, 64, out.data_ptr(), 72),
                                     (G.data_ptr(), 72, 64, out.data_ptr() + 2, 72)):
            assert lib.bns_scatter_add_div_bf16(g_, ldg, F, idx.data_ptr(), 8, 1.0, src, lds, _stream()) == E_INVALID
        assert lib.bns_launch_count() == before
    finally:
        torch.cuda.synchronize()
        for p in ps:
            p.close()


# ---- exchange --------------------------------------------------------------------------------------------------------
def _exchange_rank(comm, rank, lay, cfg, shared):
    from bns_gcn_b200.helper.feature_buffer import Buffer
    dev = torch.device("cuda:0")
    P, n_in, F, L = lay.P, lay.n_in[rank], cfg.F, cfg.n_comm
    p2p = cfg.backend == "p2p"
    buf = Buffer()
    buf.init_buffer(n_in, lay.ratio[rank], lay.send[rank], lay.recv[rank], [F] * (L + 1), use_pp=True,
                    backend=cfg.backend, device=dev, comm_dtype="bf16")
    peers = [j for j in range(P) if j != rank]
    n_halo = lay.n_u[rank] - n_in
    if p2p:
        n_slot = max(lay.n_halo[rank], 1)
        maps = torch.full((n_slot + (P - 1) * n_in,), -1, dtype=torch.int32, device=dev)
        buf.set_maps(maps, n_slot, [None if j == rank else torch.from_numpy(lay.pos[rank][j]).to(dev) for j in range(P)])
    for e in range(cfg.epochs):
        sel = cfg.samples[e]
        buf._timer.clear()
        mine = [None if j == rank else torch.from_numpy(sel[rank][j]).to(dev) for j in range(P)]
        sel_cat = torch.cat([mine[j] for j in peers])
        buf.set_selected(mine, sel_cat)
        if p2p:
            cat, _ = buf.exchange_ids(sel_cat)
            buf.update_maps(sel_cat, cat, maps[:n_slot])
            comm.barrier()
        feats, outs, halos, grads = [], [], [], []
        for l in range(1, L + 1):
            x = torch.randn(n_in, F, generator=torch.Generator(device=dev).manual_seed(1000 * e + 10 * l + rank),
                            device=dev)
            if cfg.inplace and p2p:
                feat = buf.input_slot(l, n_in, F)
                feat.copy_(x)
                feat.requires_grad_(True)
            else:
                feat = x.clone().requires_grad_(True)
            h = buf.update(l, feat)
            assert h.shape == (n_in, F) and h._bns_halo.dtype == torch.bfloat16 and h._bns_halo.shape == (n_halo, F)
            feats.append(feat)
            outs.append(h)
        torch.cuda.current_stream().synchronize()
        halos = [h._bns_halo.float().cpu() for h in outs]        # the slab region is rewritten next epoch
        x_cpu = [f.detach().cpu().numpy() for f in feats]
        for l in range(L):
            gg = torch.randn(lay.n_u[rank], F, generator=torch.Generator(device=dev).manual_seed(7919 * e + 31 * l + rank),
                             device=dev)
            grads.append(gg.cpu().numpy())
            shared[(e, rank, l)] = (x_cpu[l], grads[l])
        # backward, last layer first (as the model's): the halo rows leave through begin_backward
        d_cpu = [None] * L
        for l in reversed(range(L)):
            gg = torch.from_numpy(grads[l]).to(dev)
            buf.begin_backward(l + 1, gg)
            torch.autograd.backward(outs[l], gg[:n_in])
            d_cpu[l] = feats[l].grad.cpu().numpy()
        torch.cuda.current_stream().synchronize()
        comm.barrier()
        for l in range(L):
            want_h = np.zeros((n_halo, F), dtype=np.float32)
            recv = [None] * P
            for j in peers:
                a = lay.pl[rank][j] - n_in
                rows = X.send_rows(shared[(e, j, l)][0], sel[j][rank], lay.ratio[j][rank])
                want_h[a:a + lay.recv[rank][j]] = torch.from_numpy(rows).to(dev).to(torch.bfloat16).float().cpu().numpy()
                aj = lay.pl[j][rank]
                back = shared[(e, j, l)][1][aj:aj + lay.send[rank][j]]
                recv[j] = torch.from_numpy(np.ascontiguousarray(back)).to(dev).to(torch.bfloat16).float().cpu().numpy()
            assert np.array_equal(halos[l].numpy().view(np.int32), want_h.view(np.int32)), (cfg.backend, rank, e, l + 1)
            want_d = X.scatter_ring(grads[l][:n_in], rank, P, sel[rank], recv, lay.ratio[rank])
            assert np.array_equal(d_cpu[l].view(np.int32), want_d.view(np.int32)), (cfg.backend, rank, e, l + 1)
        comm.barrier()
        if rank == 0:
            for r in range(P):
                for l in range(L):
                    shared.pop((e - 1, r, l), None)
    comm.barrier()
    return True


def _run_exchange(lay, backend, F, epochs=2, inplace=False, n_comm=2):
    from bns_gcn_b200.helper.comm import run_threads
    cfg = SimpleNamespace(backend=backend, F=F, n_comm=n_comm, inplace=inplace, epochs=epochs,
                          samples=[lay.sample(100 + e) for e in range(epochs)])
    assert all(run_threads(lay.P, _exchange_rank, lay, cfg, {}, device="cuda:0"))


@pytest.mark.parametrize("backend", ["p2p", "nccl"])
def test_exchange_headline_bf16(built, backend):
    """Reddit / 8 partitions at F = 256, two epochs with different samples."""
    _run_exchange(headline_layout(), backend, 256)


@pytest.mark.parametrize("backend,F", [("p2p", 64), ("nccl", 64), ("nccl", 8)])
def test_exchange_edge_layout_bf16(built, backend, F):
    """Empty samples at the first, a middle and the last peer position, three epochs."""
    _run_exchange(edge_layout(), backend, F, epochs=3)


@pytest.mark.parametrize("P", [2, 4])
def test_exchange_input_written_in_place_bf16(built, P):
    """``feat`` written into the slab's inner rows by its producer (``Buffer.input_slot``), 1 and 3 peers."""
    g = np.random.default_rng(P)
    n_in = [int(x) for x in g.integers(150, 400, P)]
    halo = [[0 if j == r else int(g.integers(n_in[j] // 3, n_in[j] + 1)) for j in range(P)] for r in range(P)]
    _run_exchange(Layout(n_in, halo, 0.3, P), "p2p", 256, inplace=True)


# ---- layers -----------------------------------------------------------------------------------------------------------
class _Exchange:
    """Stands in for ``feature_buffer.Buffer``: keeps a copy of the halo gradient rows it is handed."""

    def __init__(self, n_in):
        self.n_in, self.calls = n_in, []

    def begin_backward(self, layer, grad):
        self.calls.append((layer, grad[self.n_in:].clone()))


LAYER_CASES = ([(kind, 256, fout, variant) for kind in ("sage", "gcn") for fout in (256, 41)
                for variant in ("sampled10", "sampled50", "colmap", "nothing-received", "no-halo-matrix")]
               + [("gcn", 256, fout, "colmap-unweighted") for fout in (256, 41)])


@pytest.mark.parametrize("kind,fin,fout,variant", LAYER_CASES)
def test_layer_with_bf16_halo_matches_float64(built, monkeypatch, kind, fin, fout, variant):
    """``SageConvFn`` / ``GcnConvFn`` fed the way ``Buffer.update`` feeds them under ``--comm-dtype bf16`` (inner rows as
    the input, the halo rows as a bf16 table beside it, the exchange stand-in taking the halo gradient), wide (256 -> 256)
    and narrow (256 -> 41, transform first), ``--agg-dtype f32``: output, inner-row gradient, the halo gradient handed to
    the exchange and every parameter gradient agree with the float64 restatement of the layer on ``[h_in ; widened
    halo]`` -- the operands the mode rounds, rounded, nothing else -- within the f32 layers' bar, on the partitions of
    tests/test_fused_layers_gpu.py (10 % / 50 % samples, the slot-map fallback, GCN's unweighted compaction, nothing
    received, no halo matrix)."""
    from tests import layer_reference as R
    from tests.test_fused_layers_gpu import _case, _inputs, _layer, _reference, _setup
    from bns_gcn_b200 import fused
    case = _case(kind, _setup(monkeypatch, variant, True))
    layer, arena = _layer(kind, fin, fout)
    h_u, dout = _inputs(case, fin, fout, seed=23)
    n_in = case.n_in
    halo = h_u[n_in:].to(torch.bfloat16)
    h_ref = torch.cat([h_u[:n_in], halo.float()])
    ex = _Exchange(n_in)
    feat = h_u[:n_in].clone().requires_grad_(True)
    feat._bns_halo, feat._bns_exchange = halo, (ex, 2)
    holder = fused.Transient()
    arena.flat_g.fill_(float("nan"))
    norms = (case.in_norm,) if kind == "sage" else (case.in_norm, case.out_norm)
    layer(case.g, feat, *norms, fused=(arena, 0.0, 0, holder))
    holder.value.backward(dout)
    torch.cuda.synchronize()
    want, bound = _reference(case, layer, arena, h_ref, dout)
    label = f"{kind} {fin}->{fout} {variant} bf16-halo"
    R.assert_close(f"{label} out", holder.value, want[0], bound[0])
    assert feat.grad.shape == (n_in, fin)
    R.assert_close(f"{label} d h_in", feat.grad, want[1][:n_in], bound[1][:n_in])
    assert len(ex.calls) == 1 and ex.calls[0][0] == 2
    assert ex.calls[0][1].shape == (case.n_u - n_in, fin)
    if case.n_u > n_in:                                     # (nothing received: an empty halo gradient)
        R.assert_close(f"{label} d halo", ex.calls[0][1], want[1][n_in:], bound[1][n_in:])
    for (name, p), w, b in zip(layer.named_parameters(), want[2:], bound[2:]):
        g = arena.grad_padded(p)
        R.assert_close(f"{label} d {name}", g, w, b)
        assert torch.all(g[p.shape[0]:] == 0), f"{label}: pad of the gradient of {name} is not 0"


# ---- training step -----------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _parts(shape, P):
    from bns_gcn_b200.data import make_graph, partition_graph
    dev = torch.device("cuda:0")
    return partition_graph(make_graph(shape, seed=0, device=dev), P, "random", seed=0, device=dev)


@pytest.mark.parametrize("backend", ["p2p", "nccl"])
@pytest.mark.parametrize("model", ["graphsage", "gcn"])
def test_wide_layers_bit_identical_with_agg_bf16(built, model, backend):
    """4 partitions of the ``small`` shape, 4 layers at hidden 256 (two wide exchanging layers, then the narrow class
    layer), ``--agg-dtype bf16``: the first epoch's outputs of both wide layers are bit-identical between
    ``--comm-dtype f32`` and ``bf16``; the loss stays close."""
    from tests.harness import make_args, run_product
    parts = _parts("small", 4)
    if model == "gcn" and parts[0].meta["n_feat"] % 4:
        pytest.skip("the fused GCN step needs a feature width that is a multiple of 4")
    res = {}
    for cd in ("f32", "bf16"):
        a = make_args(dataset="small", model=model, n_layers=4, n_hidden=256, sampling_rate=0.3, dropout=0.5,
                      backend=backend, agg_dtype="bf16", comm_dtype=cd, n_partitions=4)
        res[cd] = run_product(parts, a, "cuda:0", 1)
    for r in range(4):
        for name in ("layer1", "layer2"):
            x, y = res["f32"][r]["layers"][name], res["bf16"][r]["layers"][name]
            assert torch.equal(x.view(torch.int32), y.view(torch.int32)), (r, name)
        lf, lb = res["f32"][r]["loss"][0], res["bf16"][r]["loss"][0]
        assert abs(lf - lb) <= 1e-2 * abs(lf), (r, lf, lb)


@pytest.mark.parametrize("model", ["graphsage", "gcn"])
def test_one_partition_is_f32(built, model):
    """At one partition nothing is exchanged: ``--comm-dtype bf16`` gives the f32 run's losses and weights, bit for bit."""
    from tests.harness import make_args, run_product
    parts = _parts("small", 1)
    if model == "gcn" and parts[0].meta["n_feat"] % 4:
        pytest.skip("the fused GCN step needs a feature width that is a multiple of 4")
    res = {}
    for cd in ("f32", "bf16"):
        a = make_args(dataset="small", model=model, n_hidden=256, dropout=0.5, comm_dtype=cd)
        res[cd] = run_product(parts, a, "cuda:0", 3, capture=False)
    assert res["f32"][0]["loss"] == res["bf16"][0]["loss"]
    for x, y in zip(res["f32"][0]["params"], res["bf16"][0]["params"]):
        assert torch.equal(x, y)


@pytest.mark.parametrize("backend", ["p2p", "nccl"])
def test_training_converges_like_f32(built, backend):
    """The ``small`` shape at 4 partitions, 3-layer GraphSAGE at hidden 256, 12 epochs: with bf16 boundary rows the
    summed loss stays within 2 % of the f32 run's at every epoch."""
    from tests.harness import make_args, run_product
    parts = _parts("small", 4)
    res = {}
    for cd in ("f32", "bf16"):
        a = make_args(dataset="small", n_hidden=256, sampling_rate=0.3, dropout=0.5, backend=backend, comm_dtype=cd,
                      n_partitions=4)
        res[cd] = run_product(parts, a, "cuda:0", 12, capture=False)
    lf = [sum(res["f32"][r]["loss"][e] for r in range(4)) for e in range(12)]
    lb = [sum(res["bf16"][r]["loss"][e] for r in range(4)) for e in range(12)]
    for x, y in zip(lf, lb):
        assert abs(x - y) <= 2e-2 * abs(x), (lf, lb)


@pytest.mark.parametrize("model", ["graphsage", "gcn"])
def test_reddit_shape_epoch(built, model):
    """The benchmark's model (3 layers, hidden 256, --use-pp, LayerNorm, dropout 0.5) on the Reddit shape with 4
    in-process ranks over p2p, ``--comm-dtype bf16``: two epochs run and give finite losses."""
    from tests.harness import make_args, run_product
    parts = _parts("reddit", 4)
    if model == "gcn" and parts[0].meta["n_feat"] % 4:
        pytest.skip("the fused GCN step needs a feature width that is a multiple of 4")
    a = make_args(dataset="reddit", model=model, n_hidden=256, sampling_rate=0.1, dropout=0.5, backend="p2p",
                  comm_dtype="bf16", n_partitions=4)
    res = run_product(parts, a, "cuda:0", 2, capture=False)
    for r in range(4):
        assert all(np.isfinite(x) for x in res[r]["loss"]), res[r]["loss"]
