"""GAT's training attention (``graph.GatAttention``) against a float64 restatement, on one crafted partition graph.

The staged kernels (``bns_gat_scores_f32`` -> weighted SpMM per head; SDDMM -> ``bns_gat_softmax_bwd_f32`` ->
``bns_gat_colsum_f32`` -> transposed SpMM) run every case, with 1 to 8 heads and up to 1024 columns.  The graph has rows
of degree 0, 1, 31, 32, 33 and 4100 (the long one ordered so that its running maximum grows at every block of 32), halo-only rows,
rows whose halo entries are all unsampled, and a halo row whose chunks hold 0, 1, 31, 32 and 33 sampled entries.  The
scores reach 120, where exp overflows float32 without the max subtraction, and some are exactly 0.  Also: dropout
against a replay of its Philox mask, degenerate partitions, determinism, argument rejection, and ``GATConv``'s training call (padded per-head widths
included) against float64."""
import types

import numpy as np
import pytest
import torch

from tests.gat_reference import gat_attention_reference

pytestmark = pytest.mark.gpu

SLOPE = 0.2
N_IN, N_HALO, N_SLAB = 700, 900, 400
# chunk_nnz of the halo matrix: small, so that halo rows span many chunks, and above 32, so that one chunk can hold
# 33 sampled entries (chunk sizes are rounded up to multiples of 32)
HALO_CHUNK = 64
CHUNK_COUNTS = (0, 1, 31, 32, 33)
# special rows: no entry; inner degree 1, 31, 32, 33; halo only (100 sampled entries over two chunks); halo only and
# all unsampled; 7 inner entries and 50 unsampled halo ones; the chunk row; the long sorted row; scores of exactly 0
R_EMPTY, R_D1, R_D31, R_D32, R_D33, R_HALO, R_UNSAMPLED, R_INNER_UNSAMPLED, R_CHUNKS, R_LONG, R_ZERO = range(11)
LIVE_SPECIAL = (R_D1, R_D31, R_D32, R_D33, R_HALO, R_INNER_UNSAMPLED, R_CHUNKS, R_LONG, R_ZERO)


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / b.norm().clamp(min=1e-30)).item()


def _grid(n, H, gen, lim=60):
    """Multiples of 1/64 in [-lim, lim]: el + er is exact in float32, so only the kernels' own rounding counts."""
    return torch.round((torch.rand(n, H, generator=gen) * 2 * lim - lim) * 64) / 64


def _csr(rows):
    indptr = torch.zeros(len(rows) + 1, dtype=torch.int64)
    indptr[1:] = torch.cumsum(torch.tensor([len(r) for r in rows], dtype=torch.int64), 0)
    return indptr, torch.cat([torch.as_tensor(r, dtype=torch.int64) for r in rows])


def _crafted_host(H, seed):
    """The crafted partition (CSR of the inner and the halo matrix, slot map, el, er) and the reference's entry lists:
    the inner entries, then the sampled halo entries, with their positions in the two CSRs."""
    gen = torch.Generator().manual_seed(seed)
    slot = torch.full((N_HALO,), -1, dtype=torch.int32)
    perm = torch.randperm(N_HALO, generator=gen)
    live, dead = perm[:N_SLAB], perm[N_SLAB:]
    slot[live] = torch.randperm(N_SLAB, generator=gen).int()
    n_u = N_IN + N_SLAB
    el, er = _grid(n_u, H, gen), _grid(N_IN, H, gen)

    def pick(pool, k):
        return pool[torch.randint(0, len(pool), (k,), generator=gen)]

    def inner_cols(k):
        return torch.randint(0, N_IN, (k,), generator=gen)

    empty = torch.empty(0, dtype=torch.int64)
    inner, halo = [empty] * N_IN, [empty] * N_IN
    inner[R_D1], inner[R_D31], inner[R_D32], inner[R_D33] = (inner_cols(k) for k in (1, 31, 32, 33))
    halo[R_HALO] = pick(live, 100)
    halo[R_UNSAMPLED] = pick(dead, 40)
    inner[R_INNER_UNSAMPLED], halo[R_INNER_UNSAMPLED] = inner_cols(7), pick(dead, 50)
    chunks = []
    for cnt in CHUNK_COUNTS:
        c = torch.cat([pick(live, cnt), pick(dead, HALO_CHUNK - cnt)])
        chunks.append(c[torch.randperm(HALO_CHUNK, generator=gen)])
    inner[R_CHUNKS], halo[R_CHUNKS] = inner_cols(3), torch.cat(chunks)
    # raw scores of exactly 0 (inner and halo entries) next to scores 1/64 .. 3/64 either side of it, so that the
    # entries at 0 carry a large share of the row's attention
    er[R_ZERO] = _grid(1, H, gen, lim=30)[0]
    z = torch.randperm(N_IN, generator=gen)[:8]
    el[z] = -er[R_ZERO] + torch.tensor([0., 0., 0., 0., 1., 3., -1., -2.]).unsqueeze(1) / 64
    el[N_IN + slot[live[:2]].long()] = -er[R_ZERO]
    inner[R_ZERO], halo[R_ZERO] = z, live[:2]
    s = inner_cols(4100)                    # (after el is final) in increasing order of el[:, 0]
    inner[R_LONG] = s[torch.argsort(el[s, 0], stable=True)]
    for r in range(R_ZERO + 1, N_IN):
        if torch.rand(1, generator=gen).item() < 0.05:
            continue
        inner[r] = inner_cols(int(torch.poisson(torch.tensor(6.0), generator=gen)))
        halo[r] = torch.randint(0, N_HALO, (int(torch.poisson(torch.tensor(8.0), generator=gen)),), generator=gen)
    ip_in, ix_in = _csr(inner)
    ip_out, ix_out = _csr(halo)
    rows_in = torch.repeat_interleave(torch.arange(N_IN), ip_in[1:] - ip_in[:-1])
    rows_out = torch.repeat_interleave(torch.arange(N_IN), ip_out[1:] - ip_out[:-1])
    x = slot[ix_out].long()
    sampled = x >= 0
    u = torch.cat([ix_in, N_IN + x[sampled]])
    v = torch.cat([rows_in, rows_out[sampled]])
    live_deg = torch.bincount(v, minlength=N_IN)
    assert [int(live_deg[r]) for r in (R_EMPTY, R_UNSAMPLED)] == [0, 0]
    return types.SimpleNamespace(H=H, n_u=n_u, slot=slot, el=el, er=er, ip_in=ip_in, ix_in=ix_in, ip_out=ip_out,
                                 ix_out=ix_out, u=u, v=v, pos_in=torch.arange(ix_in.numel()),
                                 pos_out=torch.nonzero(sampled).squeeze(1), gen=gen)


def _crafted(H, seed):
    """``_crafted_host`` plus its ``PartitionGraph`` on the device, compacted to this sample with positions."""
    from bns_gcn_b200 import ops
    from bns_gcn_b200.graph import PartitionGraph
    dev = torch.device("cuda:0")
    case = _crafted_host(H, seed)
    a_in = ops.DeviceGraph.from_csr(case.ip_in.to(dev), case.ix_in.int().to(dev), N_IN)
    a_out = ops.DeviceGraph.from_csr(case.ip_out.to(dev), case.ix_out.int().to(dev), N_HALO, HALO_CHUNK)
    g = PartitionGraph(N_IN, N_HALO, a_in, a_out, dev)
    g.want_positions = True
    g.slot.copy_(case.slot.to(dev))
    g.refresh_compaction()
    # the chunk row really has chunks with 0, 1, 31, 32 and 33 sampled entries
    n_chunks = torch.clamp((case.ip_out[1:] - case.ip_out[:-1] + HALO_CHUNK - 1) // HALO_CHUNK, min=1)
    c0 = int(n_chunks[:R_CHUNKS].sum())
    assert g.compact.chunk_cnt[c0:c0 + len(CHUNK_COUNTS)].tolist() == list(CHUNK_COUNTS)
    case.g = g
    return case


def _run(g, ft, el, er, d, H, Fo, p, seed):
    """GatAttention forward and backward on the device: (rst, d ft, d el, d er) on the CPU."""
    from bns_gcn_b200.graph import GatAttention
    dev = torch.device("cuda:0")
    ftg, elg, erg = (t.to(dev).requires_grad_(True) for t in (ft, el, er))
    out = GatAttention.apply(ftg, elg, erg, g, H, Fo, SLOPE, p, seed)
    out.backward(d.to(dev))
    torch.cuda.synchronize()
    return out.detach().cpu(), ftg.grad.cpu(), elg.grad.cpu(), erg.grad.cpu()


def _check(got, want, v, special=LIVE_SPECIAL):
    """Whole tensors, then each special row on its own; a row without live entries gives exactly 0 and d er = 0.
    ``v``: the row of each of the reference's entries."""
    out, d_ft, d_el, d_er = got
    r_out, r_ft, r_el, r_er, _, a_da = want
    assert _rel(out, r_out) < 2e-5
    assert _rel(d_ft, r_ft) < 2e-5
    assert _rel(d_el, r_el) < 5e-5
    assert _rel(d_er, r_er) < 5e-5
    # d er_v sums a[k] * (d a[k] - sum over the row of a * d a) over row v, which is 0 when the row's entries share one
    # LeakyReLU branch: one row's d er is measured against the size of the products that cancel in it, the sum over
    # the row of |a * d a|, where that is larger than d er itself
    scale = torch.zeros(out.shape[0], a_da.shape[1], dtype=torch.float64).index_add(0, v, a_da.abs())
    for r in special:
        assert _rel(out[r], r_out[r]) < 2e-5, r
        err = (d_er[r].double() - r_er[r]).norm().item()
        assert err <= 5e-5 * max(r_er[r].norm().item(), scale[r].norm().item()), r
    dead = torch.bincount(v, minlength=out.shape[0]) == 0
    assert torch.all(out[dead] == 0) and torch.all(d_er[dead] == 0)


CASES = [(1, 64), (3, 68), (5, 80), (8, 128), (1, 512), (5, 16), (3, 300)]
assert {1, 3, 5, 8} <= {H for H, _ in CASES}


@pytest.mark.parametrize("H,Fo", CASES)
def test_attention_matches_float64_on_crafted_rows(built, H, Fo):
    """Forward, d ft, d el and d er against the float64 restatement, on the whole graph and
    on each special row; scores beyond exp's float32 range, of exactly 0, and on both sides of 0."""
    case = _crafted(H, 10 * H + Fo)
    ft = torch.randn(case.n_u, H * Fo, generator=case.gen)
    d = torch.randn(N_IN, H * Fo, generator=case.gen)
    want = gat_attention_reference(ft, case.el, case.er, case.u, case.v, N_IN, H, Fo, d, SLOPE)
    e = want[4]
    assert e.max().item() > 89.0 and (e == 0).any() and (e < 0).any() and (e > 0).any()
    got = _run(case.g, ft, case.el, case.er, d, H, Fo, 0.0, 1)
    _check(got, want, case.v)


def _philox_keep(gid, H, seed, offset, p):
    """Replay of gat_keep (csrc/gat.cuh): one Philox4x32-10 call per (entry, group of 4 heads); word h % 4 of the call
    keyed by h // 4 decides head h."""
    from oracle.philox import philox4x32_10
    gid = gid.numpy().astype(np.uint64)
    lo, hi = (gid & np.uint64(0xFFFFFFFF)).astype(np.uint32), (gid >> np.uint64(32)).astype(np.uint32)
    keep = np.empty((gid.size, H), dtype=bool)
    for g4 in range((H + 3) // 4):
        r = philox4x32_10(lo, hi ^ np.uint32(0x47415400) ^ np.uint32(g4), np.full_like(lo, offset & 0xFFFFFFFF),
                          np.full_like(lo, offset >> 32), seed & 0xFFFFFFFF, seed >> 32)
        for h in range(4 * g4, min(H, 4 * g4 + 4)):
            keep[:, h] = r[h & 3].astype(np.float32) * np.float32(2.3283064365386963e-10) >= np.float32(p)
    return torch.from_numpy(keep)


@pytest.mark.parametrize("H", [5, 8])
@pytest.mark.parametrize("p", [0.1, 0.5])
def test_attention_dropout_mask_and_gradients(built, H, p):
    """bns_gat_scores_f32, called as GatAttention.forward calls it, gives P and W = P * mask / (1 - p); the mask is the
    Philox replay, keeps 1 - p of every head, and heads h and h + 4 draw independent masks.  GatAttention under that
    mask equals the float64 restatement, forward and backward."""
    from bns_gcn_b200 import ops
    from bns_gcn_b200._lib import check, lib
    dev = torch.device("cuda:0")
    Fo, seed, offset = 16, (3 << 40) + 77, (1 << 33) + 5
    case = _crafted(H, 1000 + H)
    g, c = case.g, case.g.compact
    nnz_in, nnz_out = case.ix_in.numel(), case.ix_out.numel()
    el, er = case.el.to(dev), case.er.to(dev)
    p_in, w_in = torch.zeros(nnz_in, H, device=dev), torch.zeros(nnz_in, H, device=dev)
    p_out, w_out, wc = (torch.zeros(nnz_out, H, device=dev) for _ in range(3))
    ops.RNG.update(offset=offset, offset_dev=None)
    try:
        check(lib.bns_gat_scores_f32(g.a_in._h, g.a_out._h, c.cidx.data_ptr(), c.chunk_cnt.data_ptr(), c.cpos.data_ptr(),
                                     N_IN, H, el.data_ptr(), er.data_ptr(), SLOPE, p, seed, ops.RNG["offset"], None,
                                     p_in.data_ptr(), p_out.data_ptr(), w_in.data_ptr(), w_out.data_ptr(), wc.data_ptr(),
                                     torch.cuda.current_stream().cuda_stream), "bns_gat_scores_f32")
        P = torch.cat([p_in.cpu(), p_out.cpu()[case.pos_out]])          # the reference's entries: inner, sampled halo
        W = torch.cat([w_in.cpu(), w_out.cpu()[case.pos_out]])
        mask = W != 0
        ks = torch.tensor(1.0) / (torch.tensor(1.0) - torch.tensor(p, dtype=torch.float32))
        assert torch.allclose(W, torch.where(mask, P * ks, torch.zeros(())), rtol=1e-6, atol=0)
        live = P != 0                                 # (a probability that underflowed to 0 hides its mask bit)
        assert live.float().mean().item() > 0.5
        gid = torch.cat([case.pos_in, nnz_in + case.pos_out])
        assert torch.equal(mask, _philox_keep(gid, H, seed, offset, p) & live)
        n = live.sum(0)
        for h in range(H):
            rate = mask[:, h][live[:, h]].float().mean().item()
            assert abs(rate - (1 - p)) < 5 * (p * (1 - p) / n[h].item()) ** 0.5, (h, rate)
        q = (1 - p) ** 2
        for h in range(H - 4):
            both = live[:, h] & live[:, h + 4]
            frac = (mask[:, h] & mask[:, h + 4])[both].float().mean().item()
            assert abs(frac - q) < 5 * (q * (1 - q) / both.sum().item()) ** 0.5, (h, frac)
        ft = torch.randn(case.n_u, H * Fo, generator=case.gen)
        d = torch.randn(N_IN, H * Fo, generator=case.gen)
        want = gat_attention_reference(ft, case.el, case.er, case.u, case.v, N_IN, H, Fo, d, SLOPE, keep=mask, p=p)
        _check(_run(g, ft, case.el, case.er, d, H, Fo, p, seed), want, case.v)
    finally:
        ops.RNG.update(seed=0, offset=0, offset_dev=None)


def _plain_partition(n_in, n_halo, n_slab, inner_deg, halo_deg, seed):
    """A random partition: inner degree ~ Poisson(inner_deg) (0: no inner entry at all), halo degree ~ Poisson(halo_deg),
    n_slab of the n_halo halo nodes sampled."""
    from bns_gcn_b200 import ops
    from bns_gcn_b200.graph import PartitionGraph
    dev = torch.device("cuda:0")
    gen = torch.Generator().manual_seed(seed)
    inner = [torch.randint(0, n_in, (int(torch.poisson(torch.tensor(float(inner_deg)), generator=gen)),), generator=gen)
             for _ in range(n_in)]
    halo = [torch.randint(0, n_halo, (int(torch.poisson(torch.tensor(float(halo_deg)), generator=gen)),), generator=gen)
            for _ in range(n_in)]
    ip_in, ix_in = _csr(inner)
    ip_out, ix_out = _csr(halo)
    slot = torch.full((n_halo,), -1, dtype=torch.int32)
    slot[torch.randperm(n_halo, generator=gen)[:n_slab]] = torch.randperm(n_slab, generator=gen).int()
    a_in = ops.DeviceGraph.from_csr(ip_in.to(dev), ix_in.int().to(dev), n_in)
    a_out = ops.DeviceGraph.from_csr(ip_out.to(dev), ix_out.int().to(dev), n_halo, HALO_CHUNK)
    g = PartitionGraph(n_in, n_halo, a_in, a_out, dev)
    g.want_positions = True
    g.slot.copy_(slot.to(dev))
    g.refresh_compaction()
    rows_in = torch.repeat_interleave(torch.arange(n_in), ip_in[1:] - ip_in[:-1])
    rows_out = torch.repeat_interleave(torch.arange(n_in), ip_out[1:] - ip_out[:-1])
    x = slot[ix_out].long()
    return g, (ix_in, rows_in), (n_in + x[x >= 0], rows_out[x >= 0]), gen


def test_attention_on_degenerate_partitions(built):
    """A partition without inner entries (every row fed by the halo alone), and a halo matrix while no halo node is
    received (ft has only the n_in inner rows, so the halo entries are left out), against the float64 restatement."""
    H, Fo, n_in, n_slab = 3, 24, 300, 150
    g, _, (u, v), gen = _plain_partition(n_in, 400, n_slab, 0, 9, seed=5)
    assert g.a_in.nnz == 0
    el, er = _grid(n_in + n_slab, H, gen), _grid(n_in, H, gen)
    ft, d = torch.randn(n_in + n_slab, H * Fo, generator=gen), torch.randn(n_in, H * Fo, generator=gen)
    want = gat_attention_reference(ft, el, er, u, v, n_in, H, Fo, d, SLOPE)
    _check(_run(g, ft, el, er, d, H, Fo, 0.0, 1), want, v, ())
    g, (u, v), _, gen = _plain_partition(n_in, 400, n_slab, 7, 9, seed=6)
    el, er = _grid(n_in, H, gen), _grid(n_in, H, gen)
    ft, d = torch.randn(n_in, H * Fo, generator=gen), torch.randn(n_in, H * Fo, generator=gen)
    want = gat_attention_reference(ft, el, er, u, v, n_in, H, Fo, d, SLOPE)
    _check(_run(g, ft, el, er, d, H, Fo, 0.0, 1), want, v, ())


def test_attention_repeats_bit_identically(built):
    """Forward and backward launched twice on the same inputs (dropout on, 8 heads) give bit-identical results."""
    from bns_gcn_b200 import ops
    H, Fo = 8, 32
    case = _crafted(H, 4321)
    ft = torch.randn(case.n_u, H * Fo, generator=case.gen)
    d = torch.randn(N_IN, H * Fo, generator=case.gen)
    ops.RNG.update(offset=9, offset_dev=None)
    try:
        first = _run(case.g, ft, case.el, case.er, d, H, Fo, 0.3, 99)
        second = _run(case.g, ft, case.el, case.er, d, H, Fo, 0.3, 99)
    finally:
        ops.RNG.update(seed=0, offset=0, offset_dev=None)
    for a, b in zip(first, second):
        assert torch.equal(a, b)


def test_attention_kernels_and_gatconv_reject_bad_arguments(built):
    """Heads outside 1..8, a width that is not a multiple of 4, more than 1024 columns and p = 1 are answered with
    BNS_E_INVALID and a message naming the function.  GATConv builds exactly when graph.gat_unsupported accepts its
    heads and width, and that is exactly when bns_gat_scores_f32 takes the heads and bns_gat_proj_f32 the padded width."""
    from bns_gcn_b200 import ops
    from bns_gcn_b200._lib import lib
    from bns_gcn_b200.graph import gat_padded_width, gat_unsupported
    from bns_gcn_b200.module.gat import GATConv
    dev = torch.device("cuda:0")
    a = ops.DeviceGraph.from_csr(torch.tensor([0, 1, 2], dtype=torch.int64, device=dev),
                                 torch.tensor([1, 0], dtype=torch.int32, device=dev), 2)
    aT = a.transpose()
    LD = 1040                                                   # wide enough that only the width limit rejects 1028
    ft, attn = torch.zeros(2, LD, device=dev), torch.zeros(LD, device=dev)
    el, er, P, dE, d_er = (torch.zeros(2, 8, device=dev) for _ in range(5))
    proj_out = torch.zeros(2, 16, device=dev)
    st = torch.cuda.current_stream().cuda_stream

    def scores(H=2, p=0.0):
        return lib.bns_gat_scores_f32(a._h, None, None, None, None, 2, H, el.data_ptr(), er.data_ptr(), SLOPE, p, 1, 0,
                                      None, P.data_ptr(), None, dE.data_ptr(), None, None, st)

    def softmax_bwd(H=2, p=0.0):
        return lib.bns_gat_softmax_bwd_f32(a._h, None, None, None, None, 2, H, el.data_ptr(), er.data_ptr(), SLOPE, p, 1,
                                           0, None, P.data_ptr(), None, dE.data_ptr(), None, d_er.data_ptr(), st)

    def colsum(H=2):
        return lib.bns_gat_colsum_f32(aT._h, dE.data_ptr(), H, None, 0, d_er.data_ptr(), st)

    def proj(H=2, Fo=8):
        return lib.bns_gat_proj_f32(ft.data_ptr(), LD, 2, H, Fo, attn.data_ptr(), proj_out.data_ptr(), st)

    bad = {scores: [dict(H=0), dict(H=9), dict(p=1.0)],
           softmax_bwd: [dict(H=0), dict(H=9), dict(p=1.0)],
           colsum: [dict(H=0), dict(H=9)],
           proj: [dict(H=0), dict(Fo=6), dict(H=1, Fo=1028), dict(H=2, Fo=516), dict(H=8, Fo=132)]}
    for fn, cases in bad.items():
        assert fn() == 0, fn.__name__                             # the same call with good arguments runs
        name = {scores: b"bns_gat_scores_f32", softmax_bwd: b"bns_gat_softmax_bwd_f32", colsum: b"bns_gat_colsum_f32",
                proj: b"bns_gat_proj_f32"}[fn]
        for kw in cases:
            assert fn(**kw) == -1 and name in lib.bns_last_error(), (fn.__name__, kw)
    for H in range(0, 10):
        for Fo in (-4, 0, 1, 2, 4, 5, 6, 8, 12, 41, 100, 126, 127, 128, 129, 256, 340, 341, 512, 1021, 1024, 1028):
            ok = gat_unsupported(H, Fo) is None
            assert ok == (scores(H) == 0 and proj(H, gat_padded_width(Fo)) == 0), (H, Fo)
            try:
                GATConv(4, Fo, H)
                built_layer = True
            except NotImplementedError as e:
                built_layer = False
                assert gat_unsupported(H, Fo) in str(e), (H, Fo)
            assert built_layer == ok, (H, Fo)
    torch.cuda.synchronize()


def test_gatconv_training_matches_float64(built):
    """GATConv's training call layer(g, (h_src, h_dst)) on a partition graph -- fc, el / er, the attention and the bias,
    with a per-head width padded to a multiple of 4 where it is not one -- against a float64 restatement: the output
    and the gradients of both inputs, fc.weight, attn_l, attn_r and bias.  Heads x width: a width that is a multiple
    of 4, and two padded layouts (one head of 41 like Reddit's classes, two heads of 5)."""
    for H, Fo in ((3, 40), (1, 41), (2, 5)):
        _check_gatconv_training(H, Fo)


def _check_gatconv_training(H, Fo):
    from bns_gcn_b200.module import gat
    dev = torch.device("cuda:0")
    F_in = 24
    case = _crafted(H, 77 + Fo)
    torch.manual_seed(Fo)
    layer = gat.GATConv(F_in, Fo, H, 0.0, 0.0).to(dev).train()
    gen = torch.Generator().manual_seed(78)
    with torch.no_grad():
        layer.bias.copy_(torch.randn(H * Fo, generator=gen))          # (initialised to 0)
    h_src = torch.randn(case.n_u, F_in, generator=gen)
    h_dst = torch.randn(N_IN, F_in, generator=gen)
    d = torch.randn(N_IN, H, Fo, generator=gen)
    hs, hd = h_src.to(dev).requires_grad_(True), h_dst.to(dev).requires_grad_(True)
    out = layer(case.g, (hs, hd))
    out.backward(d.to(dev))
    got = [out, hs.grad, hd.grad, layer.fc.weight.grad, layer.attn_l.grad, layer.attn_r.grad, layer.bias.grad]
    # float64: fc and el / er under autograd; the attention's own gradients (d ft, d el, d er) from the restatement,
    # carried back through fc and the projections as the gradient of <ft, d ft> + <el, d el> + <er, d er>
    w, al, ar, b = (t.detach().double().cpu().requires_grad_(True)
                    for t in (layer.fc.weight, layer.attn_l, layer.attn_r, layer.bias))
    xs, xd = h_src.double().requires_grad_(True), h_dst.double().requires_grad_(True)
    ft_src, ft_dst = xs @ w.t(), xd @ w.t()
    el = (ft_src.view(-1, H, Fo) * al).sum(-1)
    er = (ft_dst.view(-1, H, Fo) * ar).sum(-1)
    rst, d_ft, d_el, d_er = gat_attention_reference(ft_src.detach(), el.detach(), er.detach(), case.u, case.v, N_IN, H,
                                                    Fo, d.reshape(N_IN, H * Fo), SLOPE)[:4]
    want_out = rst.view(-1, H, Fo) + b.detach().view(H, Fo)
    ((ft_src * d_ft).sum() + (el * d_el).sum() + (er * d_er).sum()).backward()
    want = [want_out, xs.grad, xd.grad, w.grad, al.grad, ar.grad, d.double().sum(0).reshape(-1)]
    names = ["out", "d h_src", "d h_dst", "d fc.weight", "d attn_l", "d attn_r", "d bias"]
    for name, g_, w_ in zip(names, got, want):
        assert g_ is not None and g_.shape == w_.shape, (H, Fo, name)
        assert _rel(g_, w_) < (2e-5 if name == "out" else 5e-5), (H, Fo, name, _rel(g_, w_))
