"""``--comm-dtype fp8``: the boundary exchange with an fp8 wire side, on in-process ranks on one GPU.

Kernels: every new entry point bit for bit -- the put's codes and scales against ``tests/fp8_reference.py`` applied to
the f32 put's rows, the scatters against their f32 siblings run on the dequantized rows -- with NaN, +-Inf, zero rows,
subnormal quotients, e4m3 ties and row maxima of exactly 448 * 2^k, zero-row segments, 1 / 2 / 7 peers and
F = 16 / 64 / 256 / 1024 with rows wider than F; malformed arguments return BNS_E_INVALID before anything launches.

Exchange: ``Buffer`` over both transports against the host restatements of ``tests/exchange_reference.py``: the received
halo codes and scales are the fp8 rows of the reference rows, and the owners' gradients the reference scatter of the
dequantized returned rows, bit for bit.

Layers: ``SageConvFn`` / ``GcnConvFn``, wide and narrow, fed the inner rows and an ``Fp8Rows`` halo table, against the
float64 restatement of ``tests/layer_reference.py`` on the dequantized rows.

Training step: with ``--agg-dtype fp8`` the wide layers' forward is bit-identical between ``--comm-dtype f32`` and
``fp8``; the loss follows f32's; a resume is bit-exact; the benchmark's model trains on the Reddit shape with 4 ranks."""
import ctypes
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from tests import exchange_reference as X
from tests import fp8_reference as Q
from tests.test_boundary_exchange_gpu import PATTERN, Layout, _P2P, edge_layout, headline_layout
from tests.test_comm_bf16_gpu import _Exchange, _parts, LAYER_CASES

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


def _rows(n, F, seed, dev):
    """f32 rows of eight kinds (row r is kind r % 8): random values over a wide range of exponents; one NaN; one +Inf or
    -Inf; zeros (with -0.0); subnormal values; e4m3 ties (400, 432, 3 * 2^-10 beside a max of 448) times 2^k; a max of
    exactly 448 * 2^k; random bit patterns (every exponent, the specials included)."""
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(n, F, generator=gen) * torch.exp2(torch.randint(-40, 40, (n, 1), generator=gen).float())
    k = torch.exp2(torch.randint(-20, 20, (n,), generator=gen).float())
    col = torch.randint(0, F, (n,), generator=gen)
    for r in range(n):
        kind = r % 8
        if kind == 1:
            x[r, col[r]] = float("nan")
        elif kind == 2:
            x[r, col[r]] = float("inf") if r % 16 < 8 else -float("inf")
        elif kind == 3:
            x[r] = 0.0
            x[r, col[r]] = -0.0
        elif kind == 4:
            x[r] = torch.randn(F, generator=gen) * 1e-41
        elif kind == 5:
            x[r, :4] = torch.tensor([448.0, 400.0, 432.0, 3 * 2.0 ** -10])
            x[r, 4:] = x[r, 4:].clamp(-300, 300)
            x[r] *= k[r]
        elif kind == 6:
            x[r] = x[r].clamp(-440, 440)
            x[r, col[r]] = -448.0 if r % 16 < 8 else 448.0
            x[r] *= k[r]
        elif kind == 7:
            x[r] = torch.randint(-2 ** 31, 2 ** 31, (F,), generator=gen, dtype=torch.int64).to(torch.int32).view(torch.float32)
    return x.to(dev)


def _same_f32(a, b):
    """Bitwise equal, except that NaN may have any payload on both sides."""
    na, nb = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb) and torch.equal(a.masked_fill(na, 0).view(torch.int32), b.masked_fill(nb, 0).view(torch.int32))


def _u8(codes):
    return codes.view(torch.uint8)


# ---- kernels -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("with_idx", [True, False], ids=["idx", "src-begin"])
@pytest.mark.parametrize("F", [16, 64, 256, 1024])
@pytest.mark.parametrize("n_peers", [1, 2, 7])
def test_put_all_fp8_is_the_quantized_f32_put(lib, dev, n_peers, F, with_idx):
    """Rank 0 puts into ``n_peers`` peers, each with a zero-row segment beside its rows, ``ldh = F + 16`` and
    ``ld_remote = F + 16``; the divisors include 1 (crafted rows reach the rule unchanged) and 0.1.  The codes and scales
    equal ``quantize_rows`` of the f32 put's rows, and every other byte of the receiving slabs keeps its sentinel."""
    from bns_gcn_b200._lib import PutAll
    world, ld = n_peers + 1, F + 16
    ps = [_P2P(lib, r, world, 1 << 22, 8, dev) for r in range(world)]
    try:
        for p in ps[1:]:
            ps[0].connect(p)
        g = np.random.default_rng(100 * n_peers + F)
        counts = [(int(g.integers(1, 40)), 0) for _ in range(n_peers)]
        counts[0] = (0, int(g.integers(1, 40)))                 # a zero-row segment first
        total = sum(a + b for a, b in counts)
        n_src = 3 * total + 200                                 # src_begin of a segment is 3 * (its first row) + 1
        H = torch.empty(n_src, ld, device=dev)[:, :F].copy_(_rows(n_src, F, F + int(with_idx), dev))
        idx = torch.from_numpy(g.permutation(n_src)[:total].astype(np.int64)).to(dev)
        divs = [1.0, 0.1, 7.0, 1.0, 2.5, 0.1, 0.7]
        F32_OFF, CODE_OFF, SCALE_OFF = 0, 1 << 21, (1 << 21) + (1 << 20)

        def segs(fp8):
            s, at, i = PutAll(), 0, 0
            so = (ctypes.c_uint64 * (2 * n_peers))()
            for j in range(n_peers):
                for h, k in enumerate(counts[j]):
                    s.row_begin[i] = at
                    s.peer[i] = j + 1
                    s.src_begin[i] = 3 * at + 1
                    s.div[i] = divs[(j + h) % len(divs)]
                    row0 = sum(counts[j][:h])
                    s.remote_off[i] = (CODE_OFF + row0 * ld) if fp8 else (F32_OFF + row0 * ld * 4)
                    so[i] = SCALE_OFF + row0 * 4
                    at += k
                    i += 1
            s.n_seg, s.row_begin[i] = i, at
            return s, so
        for p in ps[1:]:
            p.words.fill_(PATTERN)
            p.flags.zero_()
        ip = idx.data_ptr() if with_idx else None
        s32, _ = segs(False)
        s8, so = segs(True)
        _check(lib.bns_p2p_put_all_f32(ps[0].h, ctypes.byref(s32), ld, H.data_ptr(), H.stride(0), F, ip, 1,
                                       world, 5, None, _stream()), lib, "bns_p2p_put_all_f32")
        _check(lib.bns_p2p_put_all_fp8(ps[0].h, ctypes.byref(s8), so, ld, H.data_ptr(), H.stride(0), F, ip, 2,
                                       world + 1, 6, None, _stream()), lib, "bns_p2p_put_all_fp8")
        torch.cuda.synchronize()
        for j in range(n_peers):
            p, n = ps[j + 1], sum(counts[j])
            raw = _u8(p.words)
            want = torch.empty_like(p.words).fill_(PATTERN).view(torch.uint8)
            f32 = p.words[:n * ld].view(n, ld)[:, :F].view(torch.float32) if n else None
            if n:
                codes, scale = Q.quantize_rows(f32)
                want[:n * ld * 4] = raw[:n * ld * 4]                                           # the f32 region
                want[CODE_OFF:CODE_OFF + n * ld].view(n, ld)[:, :F] = _u8(codes)
                want[SCALE_OFF:SCALE_OFF + n * 4] = scale.view(torch.uint8)
            assert torch.equal(raw, want), (j, n)
            fl = p.flags.cpu()
            assert fl[1].item() == 5 and fl[2].item() == 6, j
    finally:
        torch.cuda.synchronize()
        for p in ps:
            p.close()


def _fp8_table(n, ld, F, seed, dev):
    """An fp8 table of ``n`` rows (the fp8 rows of ``_rows``, NaN-scale rows included), code rows ``ld`` bytes apart."""
    from bns_gcn_b200 import ops
    t = ops.Fp8Rows(torch.zeros(n, ld, dtype=torch.float8_e4m3fn, device=dev)[:, :F],
                    torch.empty(n, dtype=torch.float32, device=dev))
    return ops.cvt_rows_fp8(_rows(n, F, seed, dev), out=t)


@pytest.mark.parametrize("F", [16, 64, 256, 1024])
@pytest.mark.parametrize("n_seg", [1, 2, 7])
def test_scatter_rows_all_fp8_is_the_f32_scatter_of_dequantized_rows(lib, dev, n_seg, F):
    """Segments with 0 / 1 / many / all rows selected, ``ld_recv = F + 16``, NaN-scale rows among the received ones:
    the fp8 scatter equals ``bns_scatter_rows_all_f32`` over the dequantized rows, bit for bit."""
    g = np.random.default_rng(n_seg * 1000 + F)
    n_rows, ld = 2000, F + 16
    G0 = torch.randn(n_rows, F, device=dev) * 3
    invs, tabs, deq = [], [], []
    for s in range(n_seg):
        k = [700, 0, 1, n_rows, 33, 1500, 2][s]
        m = np.full(n_rows, -1, np.int32)
        m[g.permutation(n_rows)[:k]] = np.arange(k, dtype=np.int32)
        invs.append(torch.from_numpy(m).to(dev))
        t = _fp8_table(max(k, 1), ld, F, 10 * s + F, dev)
        tabs.append(t)
        d = torch.zeros(max(k, 1), ld, device=dev)
        d[:, :F] = t.codes.float() * t.scale.unsqueeze(1)          # exact: a power-of-two scale
        deq.append(d)
    divs = [0.3, 1.0, 7.0, 0.26, 1.0, 3.0, 0.1][:n_seg]
    div = (ctypes.c_float * n_seg)(*divs)
    inv = (ctypes.c_void_p * n_seg)(*[m.data_ptr() for m in invs])
    G8 = G0.clone()
    _check(lib.bns_scatter_rows_all_fp8(G8.data_ptr(), F, n_rows, F, n_seg, inv,
                                        (ctypes.c_void_p * n_seg)(*[t.codes.data_ptr() for t in tabs]),
                                        (ctypes.c_void_p * n_seg)(*[t.scale.data_ptr() for t in tabs]), ld, div,
                                        _stream()), lib, "bns_scatter_rows_all_fp8")
    G1 = G0.clone()
    _check(lib.bns_scatter_rows_all_f32(G1.data_ptr(), F, n_rows, F, n_seg, inv,
                                        (ctypes.c_void_p * n_seg)(*[d.data_ptr() for d in deq]), ld, div, _stream()),
           lib, "bns_scatter_rows_all_f32")
    torch.cuda.synchronize()
    assert _same_f32(G8, G1)


@pytest.mark.parametrize("F", [16, 64, 256, 1024])
def test_staged_pack_and_scatter_fp8(lib, dev, F):
    """The staged transport: ``bns_gather_div_fp8`` is the fp8 rows of ``bns_gather_div_f32``'s rows, and
    ``bns_scatter_add_div_fp8`` is ``bns_scatter_add_div_f32`` over the dequantized rows; rows ``F + 16`` wide."""
    from bns_gcn_b200 import ops
    g = np.random.default_rng(F)
    ld = F + 16
    H = torch.empty(500, ld, device=dev)[:, :F].copy_(_rows(500, F, F, dev))
    idx = torch.from_numpy(g.permutation(500)[:300].astype(np.int64)).to(dev)
    for div in (1.0, 0.1, 3.0):
        out32 = torch.empty(300, ld, device=dev)[:, :F]
        ops.gather_div(H, idx, div, out=out32)
        codes = torch.full((300, ld), 0x5A, dtype=torch.uint8, device=dev)
        out8 = ops.Fp8Rows(codes.view(torch.float8_e4m3fn)[:, :F], torch.empty(300, device=dev))
        ops.gather_div(H, idx, div, out=out8)
        qc, qs = Q.quantize_rows(out32)
        assert torch.equal(_u8(out8.codes), _u8(qc)), div
        assert torch.equal(out8.scale.view(torch.int32), qs.view(torch.int32)), div
        assert torch.all(codes[:, F:] == 0x5A)
        src = _fp8_table(300, ld, F, F + int(10 * div), dev)
        G0 = torch.empty(500, ld, device=dev)[:, :F].copy_(torch.randn(500, F, device=dev))
        G1, G2 = G0.clone(), G0.clone()
        ops.scatter_add_div(G1, idx, src.dequantize(), div)
        ops.scatter_add_div(G2, idx, src, div)
        assert _same_f32(G1, G2), div


@pytest.mark.parametrize("F,ldc,ldd", [(256, 256, 256), (256, 272, 260), (64, 80, 64), (16, 16, 16), (1024, 1024, 1028)])
def test_cvt_rows_fp8_f32_is_exact(built, dev, F, ldc, ldd):
    from bns_gcn_b200 import ops
    src = _fp8_table(3000, ldc, F, F, dev)
    dst = torch.full((3000, ldd), -7.0, device=dev)
    ops.cvt_rows_f32(src, out=dst[:, :F])
    assert _same_f32(dst[:, :F], src.codes.float() * src.scale.unsqueeze(1))
    # exact wherever the value is an f32; a code rounded up past the top of the f32 range (a row whose max lies within
    # one e4m3 step of 2^128) is +-Inf, as every f32 sum over the table makes it
    d64 = Q.dequantize(src.codes, src.scale)
    fits = d64.abs() <= torch.finfo(torch.float32).max
    assert torch.equal(dst[:, :F].double()[fits], d64[fits])
    assert torch.isinf(dst[:, :F][~fits & ~torch.isnan(d64)]).all() and torch.isnan(dst[:, :F][torch.isnan(d64)]).all()
    assert torch.all(dst[:, F:] == -7.0)


def test_refusals(lib, dev):
    """Widths, strides and offsets off the 16-byte grid, F past 1024, misaligned scales, a code or scale range past the
    peer's slab, NULL scale tables: BNS_E_INVALID, nothing launched."""
    from bns_gcn_b200._lib import PutAll
    ps = [_P2P(lib, r, 2, 1 << 20, 8, dev) for r in range(2)]
    try:
        ps[0].connect(ps[1])
        H = torch.randn(64, 1056, device=dev)

        def put(F=64, ldh=80, ld=64, off=0, soff=4096, h=H.data_ptr(), null_scales=False):
            s = PutAll()
            s.n_seg, s.row_begin[1], s.peer[0], s.div[0], s.remote_off[0] = 1, 4, 1, 1.0, off
            so = (ctypes.c_uint64 * 1)(soff)
            before = lib.bns_launch_count()
            rc = lib.bns_p2p_put_all_fp8(ps[0].h, ctypes.byref(s), None if null_scales else so, ld, h, ldh, F, None, 1,
                                         2, 1, None, _stream())
            return rc == E_INVALID and lib.bns_launch_count() == before
        assert put(F=56) and put(F=8, ld=16) and put(ldh=72) and put(ld=72) and put(off=8) and put(soff=2)
        assert put(F=1040, ldh=1056, ld=1040)
        assert put(h=H.data_ptr() + 4) and put(null_scales=True)
        assert put(off=(1 << 20) - 64 * 3)                          # codes past the peer's slab
        assert put(soff=(1 << 20) - 4 * 3)                          # scales past the peer's slab
        assert not put() and torch.cuda.synchronize() is None       # the well-formed call goes through
        assert not put(F=1024, ldh=1056, ld=1024) and torch.cuda.synchronize() is None
        G = torch.zeros(100, 80, device=dev)
        inv = torch.full((100,), -1, dtype=torch.int32, device=dev)
        rb = torch.zeros(8, 80, dtype=torch.uint8, device=dev)
        sc = torch.ones(8, device=dev)
        one_f = (ctypes.c_float * 1)(1.0)

        def scat(F=64, ldg=80, ld=80, g=G.data_ptr(), r=rb.data_ptr(), s=sc.data_ptr()):
            before = lib.bns_launch_count()
            rc = lib.bns_scatter_rows_all_fp8(g, ldg, 100, F, 1, (ctypes.c_void_p * 1)(inv.data_ptr()),
                                              (ctypes.c_void_p * 1)(r), (ctypes.c_void_p * 1)(s), ld, one_f, _stream())
            return rc == E_INVALID and lib.bns_launch_count() == before
        assert scat(F=56) and scat(ldg=78) and scat(ld=72) and scat(g=G.data_ptr() + 8) and scat(r=rb.data_ptr() + 8)
        assert scat(s=sc.data_ptr() + 2) and scat(s=None)
        assert not scat() and torch.cuda.synchronize() is None
        idx = torch.arange(8, dtype=torch.int64, device=dev)
        out = torch.zeros(8, 80, dtype=torch.uint8, device=dev)
        before = lib.bns_launch_count()
        for h, ldh, F, o, ldo, s in ((H.data_ptr(), 80, 56, out.data_ptr(), 80, sc.data_ptr()),
                                     (H.data_ptr(), 72, 64, out.data_ptr(), 80, sc.data_ptr()),
                                     (H.data_ptr(), 80, 64, out.data_ptr(), 72, sc.data_ptr()),
                                     (H.data_ptr() + 4, 80, 64, out.data_ptr(), 80, sc.data_ptr()),
                                     (H.data_ptr(), 80, 64, out.data_ptr() + 8, 80, sc.data_ptr()),
                                     (H.data_ptr(), 80, 64, out.data_ptr(), 80, sc.data_ptr() + 2),
                                     (H.data_ptr(), 1056, 1040, out.data_ptr(), 1040, sc.data_ptr())):
            assert lib.bns_gather_div_fp8(h, ldh, F, idx.data_ptr(), 8, 1.0, o, ldo, s, _stream()) == E_INVALID
        for g_, ldg, F, src, lds, s in ((G.data_ptr(), 80, 56, out.data_ptr(), 80, sc.data_ptr()),
                                        (G.data_ptr(), 78, 64, out.data_ptr(), 80, sc.data_ptr()),
                                        (G.data_ptr(), 80, 64, out.data_ptr(), 72, sc.data_ptr()),
                                        (G.data_ptr() + 4, 80, 64, out.data_ptr(), 80, sc.data_ptr()),
                                        (G.data_ptr(), 80, 64, out.data_ptr() + 8, 80, sc.data_ptr()),
                                        (G.data_ptr(), 80, 64, out.data_ptr(), 80, sc.data_ptr() + 2)):
            assert lib.bns_scatter_add_div_fp8(g_, ldg, F, idx.data_ptr(), 8, 1.0, src, lds, s, _stream()) == E_INVALID
        for c, ldc, F, d, ldd in ((out.data_ptr(), 80, 56, G.data_ptr(), 80), (out.data_ptr(), 72, 64, G.data_ptr(), 80),
                                  (out.data_ptr() + 8, 80, 64, G.data_ptr(), 80),
                                  (out.data_ptr(), 80, 64, G.data_ptr() + 4, 80)):
            assert lib.bns_cvt_rows_fp8_f32(c, ldc, sc.data_ptr(), d, ldd, 8, F, _stream()) == E_INVALID
        assert lib.bns_launch_count() == before
    finally:
        torch.cuda.synchronize()
        for p in ps:
            p.close()


# ---- exchange --------------------------------------------------------------------------------------------------------
def _exchange_rank(comm, rank, lay, cfg, shared):
    from bns_gcn_b200 import ops
    from bns_gcn_b200.helper.feature_buffer import Buffer
    dev = torch.device("cuda:0")
    P, n_in, F, L = lay.P, lay.n_in[rank], cfg.F, cfg.n_comm
    p2p = cfg.backend == "p2p"
    buf = Buffer()
    buf.init_buffer(n_in, lay.ratio[rank], lay.send[rank], lay.recv[rank], [F] * (L + 1), use_pp=True,
                    backend=cfg.backend, device=dev, comm_dtype="fp8")
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
        feats, outs, grads = [], [], []
        for l in range(1, L + 1):
            x = torch.randn(n_in, F, generator=torch.Generator(device=dev).manual_seed(1000 * e + 10 * l + rank),
                            device=dev)
            x *= torch.exp2(torch.randint(-8, 8, (n_in, 1), device=dev,
                                          generator=torch.Generator(device=dev).manual_seed(e + l + rank)).float())
            feat = x.clone().requires_grad_(True)
            h = buf.update(l, feat)
            assert isinstance(h._bns_halo, ops.Fp8Rows) and h.shape == (n_in, F) and h._bns_halo.shape == (n_halo, F)
            feats.append(feat)
            outs.append(h)
        torch.cuda.current_stream().synchronize()
        halos = [(h._bns_halo.codes.view(torch.uint8).cpu(), h._bns_halo.scale.cpu()) for h in outs]
        x_cpu = [f.detach().cpu().numpy() for f in feats]
        for l in range(L):
            gg = torch.randn(lay.n_u[rank], F, generator=torch.Generator(device=dev).manual_seed(7919 * e + 31 * l + rank),
                             device=dev)
            grads.append(gg.cpu().numpy())
            shared[(e, rank, l)] = (x_cpu[l], grads[l])
        d_cpu = [None] * L
        for l in reversed(range(L)):
            gg = torch.from_numpy(grads[l]).to(dev)
            buf.begin_backward(l + 1, gg)
            torch.autograd.backward(outs[l], gg[:n_in])
            d_cpu[l] = feats[l].grad.cpu().numpy()
        torch.cuda.current_stream().synchronize()
        comm.barrier()
        for l in range(L):
            want_c = torch.zeros(n_halo, F, dtype=torch.uint8)
            want_s = torch.zeros(n_halo)
            recv = [None] * P
            for j in peers:
                a = lay.pl[rank][j] - n_in
                rows = torch.from_numpy(X.send_rows(shared[(e, j, l)][0], sel[j][rank], lay.ratio[j][rank]))
                c, s = Q.quantize_rows(rows.to(dev))
                want_c[a:a + lay.recv[rank][j]] = _u8(c).cpu()
                want_s[a:a + lay.recv[rank][j]] = s.cpu()
                aj = lay.pl[j][rank]
                back = torch.from_numpy(np.ascontiguousarray(shared[(e, j, l)][1][aj:aj + lay.send[rank][j]])).to(dev)
                bc, bs = Q.quantize_rows(back)
                recv[j] = (bc.float() * bs.unsqueeze(1)).cpu().numpy()
            assert torch.equal(halos[l][0], want_c), (cfg.backend, rank, e, l + 1)
            assert torch.equal(halos[l][1].view(torch.int32), want_s.view(torch.int32)), (cfg.backend, rank, e, l + 1)
            want_d = X.scatter_ring(grads[l][:n_in], rank, P, sel[rank], recv, lay.ratio[rank])
            assert np.array_equal(d_cpu[l].view(np.int32), want_d.view(np.int32)), (cfg.backend, rank, e, l + 1)
        comm.barrier()
        if rank == 0:
            for r in range(P):
                for l in range(L):
                    shared.pop((e - 1, r, l), None)
    comm.barrier()
    return True


def _run_exchange(lay, backend, F, epochs=2, n_comm=2):
    from bns_gcn_b200.helper.comm import run_threads
    cfg = SimpleNamespace(backend=backend, F=F, n_comm=n_comm, epochs=epochs,
                          samples=[lay.sample(100 + e) for e in range(epochs)])
    assert all(run_threads(lay.P, _exchange_rank, lay, cfg, {}, device="cuda:0"))


@pytest.mark.parametrize("backend", ["p2p", "nccl"])
def test_exchange_headline_fp8(built, backend):
    """Reddit / 8 partitions at F = 256, two epochs with different samples."""
    _run_exchange(headline_layout(), backend, 256)


@pytest.mark.parametrize("backend,F", [("p2p", 64), ("nccl", 64), ("nccl", 16)])
def test_exchange_edge_layout_fp8(built, backend, F):
    """Empty samples at the first, a middle and the last peer position, three epochs."""
    _run_exchange(edge_layout(), backend, F, epochs=3)


@pytest.mark.parametrize("P", [2, 4])
def test_exchange_small_worlds_fp8(built, P):
    """1 and 3 peers over p2p at F = 256."""
    g = np.random.default_rng(P)
    n_in = [int(x) for x in g.integers(150, 400, P)]
    halo = [[0 if j == r else int(g.integers(n_in[j] // 3, n_in[j] + 1)) for j in range(P)] for r in range(P)]
    _run_exchange(Layout(n_in, halo, 0.3, P), "p2p", 256)


# ---- layers -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,fin,fout,variant", LAYER_CASES)
def test_layer_with_fp8_halo_matches_float64(built, monkeypatch, kind, fin, fout, variant):
    """``SageConvFn`` / ``GcnConvFn`` fed the way ``Buffer.update`` feeds them under ``--comm-dtype fp8`` (inner rows as
    the input, the halo rows as an ``Fp8Rows`` table beside it, the exchange stand-in taking the halo gradient), wide
    (256 -> 256) and narrow (256 -> 41): output, inner-row gradient, the halo gradient handed to the exchange and every
    parameter gradient agree with the float64 restatement of the layer on ``[h_in ; dequantized halo]`` within the f32
    layers' bar."""
    from tests import layer_reference as R
    from tests.test_fused_layers_gpu import _case, _inputs, _layer, _reference, _setup
    from bns_gcn_b200 import fused, ops
    case = _case(kind, _setup(monkeypatch, variant, True))
    layer, arena = _layer(kind, fin, fout)
    h_u, dout = _inputs(case, fin, fout, seed=29)
    n_in = case.n_in
    halo = ops.cvt_rows_fp8(h_u[n_in:].contiguous())
    h_ref = torch.cat([h_u[:n_in], halo.dequantize()])
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
    label = f"{kind} {fin}->{fout} {variant} fp8-halo"
    R.assert_close(f"{label} out", holder.value, want[0], bound[0])
    assert feat.grad.shape == (n_in, fin)
    R.assert_close(f"{label} d h_in", feat.grad, want[1][:n_in], bound[1][:n_in])
    assert len(ex.calls) == 1 and ex.calls[0][0] == 2
    assert ex.calls[0][1].shape == (case.n_u - n_in, fin)
    if case.n_u > n_in:
        R.assert_close(f"{label} d halo", ex.calls[0][1], want[1][n_in:], bound[1][n_in:])
    for (name, p), w, b in zip(layer.named_parameters(), want[2:], bound[2:]):
        g = arena.grad_padded(p)
        R.assert_close(f"{label} d {name}", g, w, b)
        assert torch.all(g[p.shape[0]:] == 0), f"{label}: pad of the gradient of {name} is not 0"


# ---- training step -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("backend", ["p2p", "nccl"])
@pytest.mark.parametrize("model", ["graphsage", "gcn"])
def test_wide_layers_bit_identical_with_agg_fp8(built, model, backend):
    """4 partitions of the ``small`` shape, 4 layers at hidden 256 (two wide exchanging layers, then the narrow class
    layer), ``--agg-dtype fp8``: the first epoch's outputs of both wide layers are bit-identical between
    ``--comm-dtype f32`` and ``fp8``; the loss stays close."""
    from tests.harness import make_args, run_product
    parts = _parts("small", 4)
    if model == "gcn" and parts[0].meta["n_feat"] % 4:
        pytest.skip("the fused GCN step needs a feature width that is a multiple of 4")
    res = {}
    for cd in ("f32", "fp8"):
        a = make_args(dataset="small", model=model, n_layers=4, n_hidden=256, sampling_rate=0.3, dropout=0.5,
                      backend=backend, agg_dtype="fp8", comm_dtype=cd, n_partitions=4)
        res[cd] = run_product(parts, a, "cuda:0", 1)
    for r in range(4):
        for name in ("layer1", "layer2"):
            x, y = res["f32"][r]["layers"][name], res["fp8"][r]["layers"][name]
            assert torch.equal(x.view(torch.int32), y.view(torch.int32)), (r, name)
        lf, lb = res["f32"][r]["loss"][0], res["fp8"][r]["loss"][0]
        assert abs(lf - lb) <= 2e-2 * abs(lf), (r, lf, lb)


@pytest.mark.parametrize("backend,extra", [("p2p", {}), ("nccl", {}),
                                           ("p2p", {"agg_dtype": "fp8", "dense_dtype": "bf16"})],
                         ids=["p2p", "nccl", "p2p-agg-fp8-dense-bf16"])
def test_training_converges_like_f32(built, backend, extra):
    """The ``small`` shape at 4 partitions, 3-layer GraphSAGE at hidden 256, 12 epochs: with fp8 boundary rows (and, in
    the last case, fp8 gather tables and bf16 GEMMs) the summed loss stays within 2 % of the f32 run's at every epoch."""
    from tests.harness import make_args, run_product
    parts = _parts("small", 4)
    res = {}
    for cd in ("f32", "fp8"):
        a = make_args(dataset="small", n_hidden=256, sampling_rate=0.3, dropout=0.5, backend=backend, n_partitions=4,
                      **({"comm_dtype": "f32"} if cd == "f32" else {"comm_dtype": "fp8", **extra}))
        res[cd] = run_product(parts, a, "cuda:0", 12, capture=False)
    lf = [sum(res["f32"][r]["loss"][e] for r in range(4)) for e in range(12)]
    l8 = [sum(res["fp8"][r]["loss"][e] for r in range(4)) for e in range(12)]
    for x, y in zip(lf, l8):
        assert abs(x - y) <= 2e-2 * abs(x), (lf, l8)


@pytest.mark.parametrize("backend", ["p2p", "nccl"])
def test_resume_is_bit_exact(built, tmp_path, monkeypatch, backend):
    """4 in-process ranks: 6 epochs against 3, a save, a teardown, a resume and 3 more, with ``--comm-dtype fp8``."""
    from tests.test_resume_gpu import _args, _check_resume
    _check_resume(_args(4, backend=backend, comm_dtype="fp8"), tmp_path, monkeypatch, fused=True)


@pytest.mark.parametrize("model", ["graphsage", "gcn"])
def test_reddit_shape_epoch(built, model):
    """The benchmark's model (3 layers, hidden 256, --use-pp, LayerNorm, dropout 0.5) on the Reddit shape with 4
    in-process ranks over p2p, ``--comm-dtype fp8``: one epoch runs and gives finite losses."""
    from tests.harness import make_args, run_product
    parts = _parts("reddit", 4)
    if model == "gcn" and parts[0].meta["n_feat"] % 4:
        pytest.skip("the fused GCN step needs a feature width that is a multiple of 4")
    a = make_args(dataset="reddit", model=model, n_hidden=256, sampling_rate=0.1, dropout=0.5, backend="p2p",
                  comm_dtype="fp8", n_partitions=4)
    res = run_product(parts, a, "cuda:0", 1, capture=False)
    for r in range(4):
        assert all(np.isfinite(x) for x in res[r]["loss"]), res[r]["loss"]
