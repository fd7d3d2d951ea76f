"""The graph transformer layer's attention kernels against the float64 restatement in ``tests/transformer_reference.py``.

Training (``graph.TconvAttention``: ``bns_tconv_scores_f32`` -> weighted SpMM per head on the value columns; SDDMM ->
``bns_tconv_softmax_bwd_f32`` -> transposed SpMMs for d v and d k) runs on GAT's crafted partition graph
(``test_gat_train_attention_gpu._crafted``): rows of degree 0, 1, 31, 32, 33 and 4100, halo-only rows, rows whose halo
entries are all unsampled, and a halo row whose chunks hold 0, 1, 31, 32 and 33 sampled entries.  1 to 8 heads, padded
widths 4 to 1024, head widths C that are not a multiple of 4 (zero pad columns, scale 1/sqrt(C)), scores up to 120 in
magnitude and exact zeros (q_v orthogonal to k_u).  Also: the dropout mask against a Philox replay, two runs
bit-identical, malformed arguments refused, and the inference kernel and its block variant under several splits."""
import math

import pytest
import torch

from tests.test_gat_train_attention_gpu import N_IN, R_LONG, R_ZERO, _crafted, _philox_keep
from tests.transformer_reference import tconv_attention_reference, tconv_infer_reference, tconv_scores_reference

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / b.norm().clamp(min=1e-30)).item()


def _pad(t, H, C, Fp):
    """``[n, H * C]`` -> ``[n, H * Fp]`` with zero pad columns."""
    return torch.nn.functional.pad(t.view(-1, H, C), (0, Fp - C)).reshape(-1, H * Fp)


def _inputs(case, H, C, Fp, gen, s_max=120.0):
    """q, k, v and d rst, head widths C padded to Fp with zeros.  q is scaled so that the largest |score| of the case
    is ``s_max``; the first two inner entries of row R_ZERO get k[u] orthogonal to q[R_ZERO] (disjoint supports), a
    score of exactly 0."""
    q = torch.randn(N_IN, H * C, generator=gen)
    k = torch.randn(case.n_u, H * C, generator=gen)
    val = torch.randn(case.n_u, H * C, generator=gen)
    zero_u = case.u[case.v == R_ZERO][:2]
    even = torch.arange(H * C) % 2 == 0
    q[R_ZERO, ~even] = 0
    k[zero_u.unsqueeze(1), even.nonzero().squeeze(1)] = 0
    q, k, val = (_pad(t, H, C, Fp) for t in (q, k, val))
    s = tconv_scores_reference(q, k, case.u, case.v, H, Fp, 1.0 / math.sqrt(C))
    q = (q.double() * (s_max / s.abs().max())).float()
    d = _pad(torch.randn(N_IN, H * C, generator=gen), H, C, Fp)
    return q, k, val, d


def _run(g, q, k, val, d, H, Fp, scale, p, seed):
    from bns_gcn_b200.graph import TconvAttention
    qg = q.to(DEV).requires_grad_(True)
    kvg = torch.cat([k, val], 1).to(DEV).requires_grad_(True)
    out = TconvAttention.apply(qg, kvg, g, H, Fp, scale, p, seed)
    out.backward(d.to(DEV))
    torch.cuda.synchronize()
    HF = H * Fp
    return out.detach().cpu(), qg.grad.cpu(), kvg.grad[:, :HF].cpu(), kvg.grad[:, HF:].cpu()


def _check(got, want, v):
    out, d_q, d_k, d_v = got
    r_out, r_q, r_k, r_v, _ = want
    assert _rel(out, r_out) < 2e-5
    assert _rel(d_q, r_q) < 5e-5
    assert _rel(d_k, r_k) < 5e-5
    assert _rel(d_v, r_v) < 5e-5
    for r in (R_LONG, R_ZERO):            # (d q of one row can be all cancellation: a saturated softmax)
        assert _rel(out[r], r_out[r]) < 2e-5, r
    dead = torch.bincount(v, minlength=out.shape[0]) == 0
    assert dead.any() and torch.all(out[dead] == 0) and torch.all(d_q[dead] == 0)


# (H, C, Fp): padded widths 4 to 1024, and C = 5, 41, 126 padded to 8, 44, 128
CASES = [(1, 4, 4), (1, 64, 64), (2, 4, 4), (3, 68, 68), (5, 80, 80), (8, 128, 128), (1, 1024, 1024), (4, 256, 256),
         (2, 512, 512), (3, 300, 300), (3, 5, 8), (1, 41, 44), (8, 126, 128)]


@pytest.mark.parametrize("H,C,Fp", CASES)
def test_tconv_attention_matches_float64_on_crafted_rows(built, H, C, Fp):
    case = _crafted(H, 7 * H + Fp)
    q, k, val, d = _inputs(case, H, C, Fp, case.gen)
    scale = 1.0 / math.sqrt(C)
    want = tconv_attention_reference(q, k, val, case.u, case.v, N_IN, H, Fp, d, scale)
    s = want[4]
    assert s.abs().max().item() > 119.0 and (s < 0).any() and (s > 0).any()
    assert (s[(case.v == R_ZERO).nonzero().squeeze(1)[:2]] == 0).all()
    got = _run(case.g, q, k, val, d, H, Fp, scale, 0.0, 1)
    _check(got, want, case.v)
    if Fp != C:                                             # pad columns of d q and d k stay 0
        pad = torch.arange(H * Fp) % Fp >= C
        assert torch.all(got[1][:, pad] == 0) and torch.all(got[2][:, pad] == 0)


@pytest.mark.parametrize("H,p", [(5, 0.1), (8, 0.5)])
def test_tconv_dropout_mask_is_the_philox_replay(built, H, p):
    """P and W = P * mask / (1 - p) from bns_tconv_scores_f32; the mask is GAT's Philox stream (gat_keep), replayed on
    the host; TconvAttention under that mask equals the float64 restatement, forward and backward."""
    from bns_gcn_b200 import ops
    from bns_gcn_b200._lib import check, lib
    C = Fp = 16
    seed, offset = (5 << 40) + 3, (1 << 33) + 7
    scale = 1.0 / math.sqrt(C)
    case = _crafted(H, 2000 + H)
    g, c = case.g, case.g.compact
    q, k, val, d = _inputs(case, H, C, Fp, case.gen, s_max=8.0)
    nnz_in, nnz_out = case.ix_in.numel(), case.ix_out.numel()
    qd, kd = q.to(DEV), k.to(DEV)
    p_in, w_in = torch.zeros(nnz_in, H, device=DEV), torch.zeros(nnz_in, H, device=DEV)
    p_out, w_out, wc = (torch.zeros(nnz_out, H, device=DEV) for _ in range(3))
    ops.RNG.update(offset=offset, offset_dev=None)
    try:
        check(lib.bns_tconv_scores_f32(g.a_in._h, g.a_out._h, c.cidx.data_ptr(), c.chunk_cnt.data_ptr(),
                                       c.cpos.data_ptr(), N_IN, H, Fp, qd.data_ptr(), qd.stride(0), kd.data_ptr(),
                                       kd.stride(0), scale, p, seed, offset, None, p_in.data_ptr(), p_out.data_ptr(),
                                       w_in.data_ptr(), w_out.data_ptr(), wc.data_ptr(),
                                       torch.cuda.current_stream().cuda_stream), "bns_tconv_scores_f32")
        P = torch.cat([p_in.cpu(), p_out.cpu()[case.pos_out]])
        W = torch.cat([w_in.cpu(), w_out.cpu()[case.pos_out]])
        mask = W != 0
        ks = torch.tensor(1.0) / (torch.tensor(1.0) - torch.tensor(p, dtype=torch.float32))
        assert torch.allclose(W, torch.where(mask, P * ks, torch.zeros(())), rtol=1e-6, atol=0)
        live = P != 0
        assert live.float().mean().item() > 0.5
        gid = torch.cat([case.pos_in, nnz_in + case.pos_out])
        assert torch.equal(mask, _philox_keep(gid, H, seed, offset, p) & live)
        want = tconv_attention_reference(q, k, val, case.u, case.v, N_IN, H, Fp, d, scale, keep=mask, p=p)
        _check(_run(g, q, k, val, d, H, Fp, scale, p, seed), want, case.v)
    finally:
        ops.RNG.update(seed=0, offset=0, offset_dev=None)


def test_tconv_attention_repeats_bit_identically(built):
    from bns_gcn_b200 import ops
    H, C = 8, 32
    case = _crafted(H, 777)
    q, k, val, d = _inputs(case, H, C, C, case.gen)
    ops.RNG.update(offset=9, offset_dev=None)
    try:
        first = _run(case.g, q, k, val, d, H, C, 1.0 / math.sqrt(C), 0.3, 99)
        second = _run(case.g, q, k, val, d, H, C, 1.0 / math.sqrt(C), 0.3, 99)
    finally:
        ops.RNG.update(seed=0, offset=0, offset_dev=None)
    for a, b in zip(first, second):
        assert torch.equal(a, b)


def _infer_graph(n_rows, n_src, degrees, gen):
    ip = torch.zeros(n_rows + 1, dtype=torch.int64)
    ip[1:] = torch.cumsum(torch.as_tensor(degrees, dtype=torch.int64), 0)
    ix = torch.randint(0, n_src, (int(ip[-1]),), generator=gen, dtype=torch.int64).int()
    return ip, ix


SPLITS = {"one": [0, 900], "four": [0, 200, 500, 501, 900], "empty-middle": [0, 450, 450, 900],
          "seven": [0, 1, 2, 3, 100, 101, 899, 900]}


@pytest.mark.parametrize("H,C,Fp", [(1, 4, 4), (1, 64, 64), (3, 68, 68), (8, 128, 128), (2, 512, 512),
                                    (4, 256, 256), (1, 1024, 1024), (3, 5, 8)])
def test_tconv_infer_and_every_block_split_match_float64(built, H, C, Fp):
    """One pass (bns_tconv_infer_f32) and the inner block plus peer blocks (bns_tconv_infer_block_f32) under several
    splits of the source columns, one of them with an empty block, against the float64 forward; rows of degree 0, 1,
    31, 32, 33 and 4100; scores up to 120."""
    from bns_gcn_b200 import ops
    from bns_gcn_b200.graph import tconv_infer, tconv_infer_block
    gen = torch.Generator().manual_seed(31 * H + Fp)
    n_rows, n_src = 600, 900
    scale = 1.0 / math.sqrt(C)
    deg = torch.poisson(torch.full((n_rows,), 7.0), generator=gen).long()
    deg[:6] = torch.tensor([0, 1, 31, 32, 33, 4100])
    ip, ix = _infer_graph(n_rows, n_src, deg, gen)
    q = _pad(torch.randn(n_rows, H * C, generator=gen), H, C, Fp)
    k, val = (_pad(torch.randn(n_src, H * C, generator=gen), H, C, Fp) for _ in range(2))
    v = torch.repeat_interleave(torch.arange(n_rows), ip[1:] - ip[:-1])
    s = tconv_scores_reference(q, k, ix.long(), v, H, Fp, scale)
    q = (q.double() * (120.0 / s.abs().max())).float()
    want = tconv_infer_reference(ip, ix, q, k, val, H, Fp, scale)
    kv = torch.cat([k, val], 1).to(DEV)
    a = ops.DeviceGraph.from_csr(ip.to(DEV), ix.to(DEV), n_src)
    one = tconv_infer(a, q.to(DEV), kv, H, Fp, scale).cpu()
    assert _rel(one, want) < 2e-5
    assert torch.all(one[0] == 0)
    for r in range(1, 6):
        assert _rel(one[r], want[r]) < 2e-5, r
    for name, bounds in SPLITS.items():
        m = torch.empty(n_rows, H, device=DEV)
        l, acc = torch.empty_like(m), torch.empty(n_rows, H * Fp, device=DEV)
        nb = len(bounds) - 1
        for j in range(nb):
            b0, b1 = bounds[j], bounds[j + 1]
            sel = (ix >= b0) & (ix < b1)
            ipb = torch.zeros(n_rows + 1, dtype=torch.int64)
            ipb[1:] = torch.cumsum(torch.bincount(v[sel], minlength=n_rows), 0)
            blk = ops.DeviceGraph.from_csr(ipb.to(DEV), (ix[sel] - b0).int().to(DEV), b1 - b0)
            tconv_infer_block(blk, q.to(DEV), kv[b0:b1] if b1 > b0 else None, H, Fp, scale, m, l, acc, j == 0,
                              j == nb - 1, acc)
        got = acc.cpu()
        assert _rel(got, want) < 2e-5, name
        assert torch.all(got[0] == 0), name
        for r in range(1, 6):
            assert _rel(got[r], want[r]) < 2e-5, (name, r)
    two = tconv_infer(a, q.to(DEV), kv, H, Fp, scale).cpu()
    assert torch.equal(one, two)


def test_tconv_kernels_reject_bad_arguments(built):
    """Every malformed argument is refused with BNS_E_INVALID naming the entry point, before any launch."""
    from bns_gcn_b200 import ops
    from bns_gcn_b200._lib import BnsError, lib
    from bns_gcn_b200.graph import tconv_infer, tconv_infer_block
    st = torch.cuda.current_stream().cuda_stream
    ip = torch.tensor([0, 2, 3], dtype=torch.int64, device=DEV)
    ix = torch.tensor([0, 1, 1], dtype=torch.int32, device=DEV)
    a = ops.DeviceGraph.from_csr(ip, ix, 2)
    z = torch.zeros(2, 64, device=DEV)
    P = torch.zeros(3, 8, device=DEV)

    def scores(H=2, Fp=8, k=z, ldk=64, q=z, scale=0.5, p=0.0, P_in=P, W_in=None):
        return lib.bns_tconv_scores_f32(a._h, None, None, None, None, 2, H, Fp, ops._ptr(q), 64, ops._ptr(k), ldk,
                                        scale, p, 0, 0, None, ops._ptr(P_in), None, ops._ptr(W_in), None, None, st)
    assert scores() == 0
    torch.cuda.synchronize()
    for kw in (dict(H=0), dict(H=9), dict(Fp=6), dict(H=8, Fp=132), dict(k=None), dict(q=None), dict(P_in=None),
               dict(ldk=6), dict(ldk=8, H=4), dict(p=1.0), dict(p=0.5), dict(k=z[:, 1:]), dict(scale=0.0),
               dict(scale=float("inf"))):
        assert scores(**kw) == -1, kw
        assert b"bns_tconv_scores_f32" in lib.bns_last_error(), kw
    dq = torch.zeros(2, 64, device=DEV)

    def bwd(Fp=8, d_q=dq, ldd=64, dE=P):
        return lib.bns_tconv_softmax_bwd_f32(a._h, None, None, None, None, 2, 2, Fp, z.data_ptr(), 64, z.data_ptr(), 64,
                                             0.5, 0.0, 0, 0, None, P.data_ptr(), None, ops._ptr(dE), None,
                                             ops._ptr(d_q), ldd, st)
    assert bwd() == 0
    torch.cuda.synchronize()
    for kw in (dict(Fp=5), dict(d_q=None), dict(ldd=6), dict(d_q=dq[:, 1:]), dict(dE=None)):
        assert bwd(**kw) == -1, kw
        assert b"bns_tconv_softmax_bwd_f32" in lib.bns_last_error(), kw
    kv = torch.zeros(2, 128, device=DEV)
    assert lib.bns_tconv_infer_f32(a._h, z.data_ptr(), 64, kv.data_ptr(), 128, kv.data_ptr() + 256, 128, 9, 8, 0.5,
                                   dq.data_ptr(), 64, st) == -1
    assert b"bns_tconv_infer_f32" in lib.bns_last_error()
    assert lib.bns_tconv_infer_f32(a._h, z.data_ptr(), 64, kv.data_ptr(), 128, None, 128, 2, 8, 0.5, dq.data_ptr(), 64,
                                   st) == -1
    m = torch.zeros(2, 2, device=DEV)
    assert lib.bns_tconv_infer_block_f32(a._h, z.data_ptr(), 64, kv.data_ptr(), 128, kv.data_ptr() + 64, 128, 2, 8,
                                         0.5, None, m.data_ptr(), dq.data_ptr(), 64, 1, 1, dq.data_ptr(), 64,
                                         st) == -1
    assert b"bns_tconv_infer_block_f32" in lib.bns_last_error()
    with pytest.raises(BnsError, match="tconv_infer"):
        tconv_infer(a, z[:, :12], kv[:, :24], 2, 6, 0.5)
    with pytest.raises(BnsError, match="kv must be"):
        tconv_infer(a, z[:, :16], kv[:, :16], 2, 8, 0.5)
    with pytest.raises(BnsError, match="needs kv"):
        tconv_infer_block(a, z[:, :16], None, 2, 8, 0.5, m, m.clone(), dq[:, :16], True, True, dq[:, :16])
    with pytest.raises(BnsError, match="needs rst"):
        tconv_infer_block(a, z[:, :16], kv[:, :32], 2, 8, 0.5, m, m.clone(), dq[:, :16], True, True)
    torch.cuda.synchronize()
