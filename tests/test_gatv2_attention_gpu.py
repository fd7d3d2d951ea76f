"""GATv2's attention kernels against the float64 restatement in ``tests/gatv2_reference.py``.

Training (``graph.Gatv2Attention``: ``bns_gatv2_scores_f32`` -> weighted SpMM per head; SDDMM ->
``bns_gatv2_softmax_bwd_f32`` -> transposed SpMM + ``bns_gatv2_colsum_f32``) runs on GAT's crafted partition graph
(``test_gat_train_attention_gpu._crafted``): rows of degree 0, 1, 31, 32, 33 and 4100, halo-only rows, rows whose halo
entries are all unsampled, and a halo row whose chunks hold 0, 1, 31, 32 and 33 sampled entries.  1 to 8 heads, padded
widths up to 1024, scores up to 120 in magnitude, exact zeros and both LeakyReLU branches.  Also: the dropout mask
against a Philox replay, two runs bit-identical, malformed arguments refused, and the inference kernel and its block
variant."""
import pytest
import torch

from tests.gatv2_reference import gatv2_attention_reference, gatv2_infer_reference
from tests.test_gat_train_attention_gpu import N_IN, R_LONG, R_ZERO, SLOPE, _crafted, _philox_keep

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / b.norm().clamp(min=1e-30)).item()


def _inputs(case, H, Fp, gen, s_max=120.0):
    """z_src, z_dst, attn and d rst.  attn is scaled so that the largest |score| of the case is ``s_max``; the first two
    inner entries of row R_ZERO get z_src[u] = -z_dst[v], a score of exactly 0."""
    zs = torch.randn(case.n_u, H * Fp, generator=gen)
    zd = torch.randn(N_IN, H * Fp, generator=gen)
    zero_u = case.u[case.v == R_ZERO][:2]
    zs[zero_u] = -zd[R_ZERO]
    attn = torch.randn(H * Fp, generator=gen)
    from tests.gatv2_reference import gatv2_scores_reference
    s = gatv2_scores_reference(zs, zd, attn, case.u, case.v, H, Fp, SLOPE)
    attn = (attn.double() * (s_max / s.abs().max())).float()
    d = torch.randn(N_IN, H * Fp, generator=gen)
    return zs, zd, attn, d


def _run(g, zs, zd, attn, d, H, Fp, p, seed):
    from bns_gcn_b200.graph import Gatv2Attention
    zsg, zdg, ag = (t.to(DEV).requires_grad_(True) for t in (zs, zd, attn.view(1, H, Fp)))
    out = Gatv2Attention.apply(zsg, zdg, ag, g, H, Fp, SLOPE, p, seed)
    out.backward(d.to(DEV))
    torch.cuda.synchronize()
    return out.detach().cpu(), zsg.grad.cpu(), zdg.grad.cpu(), ag.grad.cpu().reshape(-1)


def _check(got, want, v):
    out, d_zs, d_zd, d_at = got
    r_out, r_zs, r_zd, r_at, _ = want
    assert _rel(out, r_out) < 2e-5
    assert _rel(d_zs, r_zs) < 5e-5
    assert _rel(d_zd, r_zd) < 5e-5
    assert _rel(d_at, r_at) < 5e-5
    for r in (R_LONG, R_ZERO):
        assert _rel(out[r], r_out[r]) < 2e-5, r
    dead = torch.bincount(v, minlength=out.shape[0]) == 0
    assert dead.any() and torch.all(out[dead] == 0) and torch.all(d_zd[dead] == 0)


CASES = [(1, 64), (2, 4), (3, 68), (5, 80), (8, 128), (1, 512), (4, 256), (5, 16), (3, 300)]


@pytest.mark.parametrize("H,Fp", CASES)
def test_gatv2_attention_matches_float64_on_crafted_rows(built, H, Fp):
    case = _crafted(H, 7 * H + Fp)
    zs, zd, attn, d = _inputs(case, H, Fp, case.gen)
    want = gatv2_attention_reference(zs, zd, attn, case.u, case.v, N_IN, H, Fp, d, SLOPE)
    s = want[4]
    assert s.abs().max().item() > 119.0 and (s == 0).any() and (s < 0).any() and (s > 0).any()
    z = zs[case.u].view(-1, H, Fp) + zd[case.v].view(-1, H, Fp)
    assert (z > 0).any() and (z < 0).any()                         # both LeakyReLU branches
    _check(_run(case.g, zs, zd, attn, d, H, Fp, 0.0, 1), want, case.v)


@pytest.mark.parametrize("H,p", [(5, 0.1), (8, 0.5)])
def test_gatv2_dropout_mask_is_the_philox_replay(built, H, p):
    """P and W = P * mask / (1 - p) from bns_gatv2_scores_f32; the mask is GAT's Philox stream (gat_keep), replayed
    on the host; Gatv2Attention under that mask equals the float64 restatement, forward and backward."""
    from bns_gcn_b200 import ops
    from bns_gcn_b200._lib import check, lib
    Fp, seed, offset = 16, (5 << 40) + 3, (1 << 33) + 7
    case = _crafted(H, 2000 + H)
    g, c = case.g, case.g.compact
    zs, zd, attn, d = _inputs(case, H, Fp, case.gen, s_max=8.0)
    nnz_in, nnz_out = case.ix_in.numel(), case.ix_out.numel()
    zsd, zdd, ad = zs.to(DEV), zd.to(DEV), attn.to(DEV)
    p_in, w_in = torch.zeros(nnz_in, H, device=DEV), torch.zeros(nnz_in, H, device=DEV)
    p_out, w_out, wc = (torch.zeros(nnz_out, H, device=DEV) for _ in range(3))
    ops.RNG.update(offset=offset, offset_dev=None)
    try:
        check(lib.bns_gatv2_scores_f32(g.a_in._h, g.a_out._h, c.cidx.data_ptr(), c.chunk_cnt.data_ptr(),
                                       c.cpos.data_ptr(), N_IN, H, Fp, zsd.data_ptr(), zsd.stride(0), zdd.data_ptr(),
                                       zdd.stride(0), ad.data_ptr(), SLOPE, p, seed, offset, None, p_in.data_ptr(),
                                       p_out.data_ptr(), w_in.data_ptr(), w_out.data_ptr(), wc.data_ptr(),
                                       torch.cuda.current_stream().cuda_stream), "bns_gatv2_scores_f32")
        P = torch.cat([p_in.cpu(), p_out.cpu()[case.pos_out]])
        W = torch.cat([w_in.cpu(), w_out.cpu()[case.pos_out]])
        mask = W != 0
        ks = torch.tensor(1.0) / (torch.tensor(1.0) - torch.tensor(p, dtype=torch.float32))
        assert torch.allclose(W, torch.where(mask, P * ks, torch.zeros(())), rtol=1e-6, atol=0)
        live = P != 0
        assert live.float().mean().item() > 0.5
        gid = torch.cat([case.pos_in, nnz_in + case.pos_out])
        assert torch.equal(mask, _philox_keep(gid, H, seed, offset, p) & live)
        want = gatv2_attention_reference(zs, zd, attn, case.u, case.v, N_IN, H, Fp, d, SLOPE, keep=mask, p=p)
        _check(_run(g, zs, zd, attn, d, H, Fp, p, seed), want, case.v)
    finally:
        ops.RNG.update(seed=0, offset=0, offset_dev=None)


def test_gatv2_attention_repeats_bit_identically(built):
    from bns_gcn_b200 import ops
    H, Fp = 8, 32
    case = _crafted(H, 777)
    zs, zd, attn, d = _inputs(case, H, Fp, case.gen)
    ops.RNG.update(offset=9, offset_dev=None)
    try:
        first = _run(case.g, zs, zd, attn, d, H, Fp, 0.3, 99)
        second = _run(case.g, zs, zd, attn, d, H, Fp, 0.3, 99)
    finally:
        ops.RNG.update(seed=0, offset=0, offset_dev=None)
    for a, b in zip(first, second):
        assert torch.equal(a, b)


def _infer_graph(n_rows, n_src, degrees, gen):
    ip = torch.zeros(n_rows + 1, dtype=torch.int64)
    ip[1:] = torch.cumsum(torch.as_tensor(degrees, dtype=torch.int64), 0)
    ix = torch.randint(0, n_src, (int(ip[-1]),), generator=gen, dtype=torch.int64).int()
    return ip, ix


@pytest.mark.parametrize("H,Fp", [(1, 4), (1, 64), (3, 68), (8, 128), (2, 512), (4, 256)])
def test_gatv2_infer_and_block_match_float64(built, H, Fp):
    """One pass (bns_gatv2_infer_f32) and the inner block plus 3 peer blocks (bns_gatv2_infer_block_f32) against the
    float64 forward; rows of degree 0, 1, 31, 32, 33 and 4100; scores up to 120."""
    from bns_gcn_b200 import ops
    from bns_gcn_b200.graph import gatv2_infer, gatv2_infer_block
    gen = torch.Generator().manual_seed(31 * H + Fp)
    n_rows, n_src = 600, 900
    deg = torch.poisson(torch.full((n_rows,), 7.0), generator=gen).long()
    deg[:6] = torch.tensor([0, 1, 31, 32, 33, 4100])
    ip, ix = _infer_graph(n_rows, n_src, deg, gen)
    zs, zd = torch.randn(n_src, H * Fp, generator=gen), torch.randn(n_rows, H * Fp, generator=gen)
    attn = torch.randn(H * Fp, generator=gen)
    from tests.gatv2_reference import gatv2_scores_reference
    v = torch.repeat_interleave(torch.arange(n_rows), ip[1:] - ip[:-1])
    s = gatv2_scores_reference(zs, zd, attn, ix.long(), v, H, Fp, SLOPE)
    attn = (attn.double() * (120.0 / s.abs().max())).float()
    want = gatv2_infer_reference(ip, ix, zs, zd, attn, H, Fp, SLOPE)
    a = ops.DeviceGraph.from_csr(ip.to(DEV), ix.to(DEV), n_src)
    one = gatv2_infer(a, zs.to(DEV), zd.to(DEV), attn.to(DEV), H, Fp, SLOPE).cpu()
    assert _rel(one, want) < 2e-5
    assert torch.all(one[0] == 0)
    # split the columns into 4 blocks: the same rows, disjoint source ranges
    bounds = [0, 200, 500, 501, n_src]
    m = torch.empty(n_rows, H, device=DEV)
    l, acc = torch.empty_like(m), torch.empty(n_rows, H * Fp, device=DEV)
    rows = torch.repeat_interleave(torch.arange(n_rows), ip[1:] - ip[:-1])
    for k in range(4):
        b0, b1 = bounds[k], bounds[k + 1]
        sel = (ix >= b0) & (ix < b1)
        ipb = torch.zeros(n_rows + 1, dtype=torch.int64)
        ipb[1:] = torch.cumsum(torch.bincount(rows[sel], minlength=n_rows), 0)
        blk = ops.DeviceGraph.from_csr(ipb.to(DEV), (ix[sel] - b0).int().to(DEV), b1 - b0)
        gatv2_infer_block(blk, zs[b0:b1].to(DEV), zd.to(DEV), attn.to(DEV), H, Fp, SLOPE, m, l, acc, k == 0, k == 3,
                          acc)
    got = acc.cpu()
    assert _rel(got, want) < 2e-5
    for r in range(1, 6):
        assert _rel(got[r], want[r]) < 2e-5, r
    two = gatv2_infer(a, zs.to(DEV), zd.to(DEV), attn.to(DEV), H, Fp, SLOPE).cpu()
    assert torch.equal(one, two)


def test_gatv2_kernels_reject_bad_arguments(built):
    """Every malformed argument is refused with BNS_E_INVALID naming the entry point, before any launch."""
    from bns_gcn_b200 import ops
    from bns_gcn_b200._lib import BnsError, lib
    from bns_gcn_b200.graph import gatv2_infer, gatv2_infer_block
    st = torch.cuda.current_stream().cuda_stream
    ip = torch.tensor([0, 2, 3], dtype=torch.int64, device=DEV)
    ix = torch.tensor([0, 1, 1], dtype=torch.int32, device=DEV)
    a = ops.DeviceGraph.from_csr(ip, ix, 2)
    z = torch.zeros(2, 64, device=DEV)
    at = torch.zeros(64, device=DEV)
    P = torch.zeros(3, 8, device=DEV)

    def scores(H=2, Fp=8, zs=z, ldzs=64, attn=at, p=0.0, P_in=P, W_in=None):
        return lib.bns_gatv2_scores_f32(a._h, None, None, None, None, 2, H, Fp, ops._ptr(zs), ldzs, z.data_ptr(), 64,
                                        ops._ptr(attn), SLOPE, p, 0, 0, None, ops._ptr(P_in), None, ops._ptr(W_in),
                                        None, None, st)
    assert scores() == 0
    torch.cuda.synchronize()
    for kw in (dict(H=0), dict(H=9), dict(Fp=6), dict(H=8, Fp=132), dict(zs=None), dict(attn=None), dict(P_in=None),
               dict(ldzs=6), dict(ldzs=8, H=4), dict(p=1.0), dict(p=0.5),
               dict(zs=z[:, 1:])):
        assert scores(**kw) == -1, kw
        assert b"bns_gatv2_scores_f32" in lib.bns_last_error(), kw
    ws = torch.zeros(1 << 20, dtype=torch.uint8, device=DEV)
    dz = torch.zeros(2, 64, device=DEV)
    da = torch.zeros(64, device=DEV)

    def bwd(Fp=8, d_zd=dz, d_attn=da, ws_bytes=None, ldd=64):
        return lib.bns_gatv2_softmax_bwd_f32(a._h, None, None, None, None, 2, 2, Fp, z.data_ptr(), 64, z.data_ptr(), 64,
                                             at.data_ptr(), SLOPE, 0.0, 0, 0, None, P.data_ptr(), None, P.data_ptr(),
                                             None, ops._ptr(d_zd), ldd, ops._ptr(d_attn), ws.data_ptr(),
                                             ws.numel() if ws_bytes is None else ws_bytes, st)
    assert bwd() == 0
    torch.cuda.synchronize()
    for kw in (dict(Fp=5), dict(d_zd=None), dict(d_attn=None), dict(ldd=6), dict(d_attn=da[1:])):
        assert bwd(**kw) == -1, kw
        assert b"bns_gatv2_softmax_bwd_f32" in lib.bns_last_error(), kw
    assert bwd(ws_bytes=0) != 0
    aT = a.transpose()
    assert lib.bns_gatv2_colsum_f32(a._h, P.data_ptr(), 2, 8, z.data_ptr(), 64, z.data_ptr(), 64, at.data_ptr(), SLOPE,
                                    None, 0, dz.data_ptr(), 64, st) == -1                  # not a transpose
    assert b"bns_gatv2_colsum_f32" in lib.bns_last_error()
    assert lib.bns_gatv2_colsum_f32(aT._h, P.data_ptr(), 2, 8, z.data_ptr(), 64, z.data_ptr(), 64, at.data_ptr(), SLOPE,
                                    None, 0, None, 64, st) == -1
    assert lib.bns_gatv2_infer_f32(a._h, z.data_ptr(), 64, z.data_ptr(), 64, at.data_ptr(), 9, 8, SLOPE, dz.data_ptr(),
                                   64, st) == -1
    assert b"bns_gatv2_infer_f32" in lib.bns_last_error()
    m = torch.zeros(2, 2, device=DEV)
    assert lib.bns_gatv2_infer_block_f32(a._h, z.data_ptr(), 64, z.data_ptr(), 64, at.data_ptr(), 2, 8, SLOPE, None,
                                         m.data_ptr(), dz.data_ptr(), 64, 1, 1, dz.data_ptr(), 64, st) == -1
    assert b"bns_gatv2_infer_block_f32" in lib.bns_last_error()
    with pytest.raises(BnsError, match="gatv2_infer"):
        gatv2_infer(a, z[:, :12], z[:, :12], at[:12], 2, 6, SLOPE)
    with pytest.raises(BnsError, match="zs must be"):
        gatv2_infer(a, z[:1, :16], z[:, :16], at[:16], 2, 8, SLOPE)
    with pytest.raises(BnsError, match="needs zs"):
        gatv2_infer_block(a, None, z[:, :16], at[:16], 2, 8, SLOPE, m, m.clone(), dz[:, :16], True, True, dz[:, :16])
    with pytest.raises(BnsError, match="needs rst"):
        gatv2_infer_block(a, z[:, :16], z[:, :16], at[:16], 2, 8, SLOPE, m, m.clone(), dz[:, :16], True, True)
    torch.cuda.synchronize()
