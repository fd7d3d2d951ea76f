"""The bf16 dense GEMMs of ``csrc/dense_tc.cuh`` (``bns_dense_tn_bf16``, ``bns_dense_nt_bf16``, ``--dense-dtype bf16``)
against float64, element by element, and their rounding bit for bit against torch's.

Reference and bound: the float64 product of the operands rounded by torch (``.to(torch.bfloat16)``, nearest even), plus
the f32 epilogue terms, within ``layer_reference.TOL`` of ``|A_bf| |B_bf|^T + |bias| + |addend|`` (times
``|row_scale|``).  What is left after the rounding is the kernel's f32 accumulation, so the bar is the 3xTF32 kernels'.
Operands are NaN-fenced views and outputs sentinel-filled views (``tests/test_dense_gemm_gpu.py``), so a read or a
store outside a view is seen."""
import pytest
import torch

from tests.test_dense_gemm_gpu import (BENCH_ROWS, EPILOGUES, _ceil4, _check_tn, _close, _dev, _gen, _lib,
                                       _nt_data, _operand, _output, _report, _spread, _splits, _stream, _untouched,
                                       _vector, CHUNK)

pytestmark = pytest.mark.gpu

TWO_LEVEL_ROWS = 13_900_000      # papers100M's per-rank node count: the two-level split-K reduce


@pytest.fixture(scope="module")
def dense(built):
    from bns_gcn_b200.module import dense as d
    return d


def _bf(t):
    """``t`` rounded to bf16 (nearest even) by torch, widened back to f32."""
    return t.to(torch.bfloat16).float()


# ---- TN -----------------------------------------------------------------------------------------------------------
def _tn_case(dense, worst, key, M, N, K, lda, ldc, seed, bias=False, addend=False, row_scale=False, in_place=False):
    g = _gen(seed)
    ad, bd = _spread(M, K, g), _spread(N, K, g)
    a, b = _operand(ad, lda), _operand(bd, _ceil4(K) + 4)
    bi = _vector(_spread(1, N, g, row_scale=False)[0]) if bias else None
    rs = None
    if row_scale:
        rv = torch.randn(M, generator=g, device=_dev())
        rv[::7] = 0.0
        rs = _vector(rv)
    label = f"TN bf16 (M, N, K, lda, ldc) = ({M}, {N}, {K}, {lda}, {ldc}) bias={bias} addend={addend} row_scale={row_scale}"
    buf, out = _output(M, N, ldc)
    add = add0 = None
    if addend:
        add0 = _spread(M, N, g)
        if in_place:
            out.copy_(add0)
            add = out
            label += " in place"
        else:
            add = _operand(add0, _ceil4(N) + 12)
    got = dense.tc_mm_tn(a, b, bias=bi, addend=add, row_scale=rs, out=out, bf16=True)
    _check_tn(worst, key, label, got, _bf(a), _bf(b), bi, add0, rs)
    _untouched(buf, M, N, label)
    if not in_place:                  # two runs, the same bits
        buf2, out2 = _output(M, N, ldc)
        dense.tc_mm_tn(a, b, bias=bi, addend=add, row_scale=rs, out=out2, bf16=True)
        assert torch.equal(out.view(torch.int32), out2.view(torch.int32)), f"{label}: not bit-reproducible"
    return got


def test_tn_edge_shapes(dense):
    """M / N / K that are not multiples of the 128 x 128 x 32 tile, K = 4 and 44 among them, wider ``lda``; the epilogue
    cycles through its 8 combinations."""
    worst = {}
    i = 0
    for M in (1, 127, 129, 4099):
        for N in (1, 3, 44, 129, 256):
            for K in (1, 4, 31, 33, 44, 1204):
                for lda in (_ceil4(K), _ceil4(K) + 8):
                    bias, add, rs = EPILOGUES[i % 8]
                    _tn_case(dense, worst, "TN bf16 edges", M, N, K, lda, _ceil4(N) + 4, seed=i, bias=bias, addend=add,
                             row_scale=rs)
                    i += 1
    _report(worst)


def test_tn_epilogue_combinations(dense):
    """bias / addend / row_scale in all 8 combinations, the addend at its own leading dimension and aliasing the output."""
    worst = {}
    i = 7000
    for N in (3, 44, 256):
        for bias, add, rs in EPILOGUES:
            _tn_case(dense, worst, "TN bf16 epilogue", 4099, N, 602, 604, _ceil4(N) + 4, seed=i, bias=bias, addend=add,
                     row_scale=rs)
            i += 1
            if add:
                _tn_case(dense, worst, "TN bf16 epilogue", 4099, N, 602, 604, _ceil4(N) + 4, seed=i, bias=bias,
                         addend=True, row_scale=rs, in_place=True)
                i += 1
    _report(worst)


@pytest.mark.parametrize("K,N", [(1204, 256), (256, 256), (256, 44), (44, 256)])
def test_tn_bench_shapes(dense, K, N):
    """The benchmark's dense products at its one-partition row count (Reddit shape, 232,965 rows)."""
    worst = {}
    _tn_case(dense, worst, f"TN bf16 bench {K}->{N}", BENCH_ROWS, N, K, _ceil4(K), _ceil4(N), seed=K + N, bias=N == 256)
    _report(worst)


# ---- NT -----------------------------------------------------------------------------------------------------------
def _nt_call(a, b, out, ws_fill):
    from bns_gcn_b200._lib import check
    R_, N1 = a.shape
    N2 = b.shape[1]
    need = _lib().bns_dense_nt_workspace_bytes(R_, N1, N2)
    ws = torch.full((need // 4 + 128 * N2 + 64,), ws_fill, device=_dev())
    check(_lib().bns_dense_nt_bf16(a.data_ptr(), a.stride(0), b.data_ptr(), b.stride(0), out.data_ptr(), out.stride(0),
                                   R_, N1, N2, ws.data_ptr() if need else None, need, _stream()), "bns_dense_nt_bf16")


def _nt_case(worst, key, R_, N1, N2, seed, repeat=True, data=None):
    ad, bd = _nt_data(R_, N1, N2, seed) if data is None else data
    a, b = _operand(ad, _ceil4(N1) + 4), _operand(bd, N2 + 8)
    del ad, bd
    buf, out = _output(N1, N2, N2 + 4)
    s = _splits(R_, N1, N2)
    label = f"NT bf16 (R, N1, N2) = ({R_}, {N1}, {N2}) splits={s}"
    _nt_call(a, b, out, float("nan"))
    ref = torch.zeros(N1, N2, dtype=torch.float64, device=_dev())
    bnd = torch.zeros_like(ref)
    for r0 in range(0, R_, CHUNK):
        ac, bc = _bf(a[r0:r0 + CHUNK]).double(), _bf(b[r0:r0 + CHUNK]).double()
        ref += ac.t() @ bc
        bnd += ac.abs().t() @ bc.abs()
    _close(worst, key, label, out, ref, bnd)
    _untouched(buf, N1, N2, label)
    if repeat:
        first = out.clone()
        for fill in (0.0, float("nan")):
            _nt_call(a, b, out, fill)
            assert torch.equal(out.view(torch.int32), first.view(torch.int32)), f"{label}: not bit-reproducible"
        _untouched(buf, N1, N2, label)
    return s


def test_nt_sweep(dense):
    worst = {}
    i = 0
    for N1 in (1, 44, 129, 256):
        for N2 in (4, 44, 132, 1204):
            for R_ in (1, 37, 3000):
                _nt_case(worst, "NT bf16 sweep", R_, N1, N2, seed=100 + i, repeat=False)
                i += 1
    _report(worst)


def test_nt_split_regimes(dense):
    """One slice straight into C, a slice per k-block, slices of unequal length, and the benchmark's weight gradients
    (more than 100 slices) -- the plan and workspace of the 3xTF32 kernel; each run again must give the same bits."""
    worst = {}
    nkb = lambda r: (r + 31) // 32                                  # noqa: E731
    assert _splits(32, 128, 128) == 1
    _nt_case(worst, "NT bf16 one slice", 32, 128, 128, seed=1)
    assert _splits(64, 128, 128) == nkb(64) == 2
    _nt_case(worst, "NT bf16 slice per k-block", 64, 128, 128, seed=2)
    uneven = [c for c in ((5000, 256, 1204), (3001, 128, 128), (10000, 44, 256), (7777, 256, 256))
              if _splits(*c) > 1 and nkb(c[0]) % _splits(*c) != 0]
    assert uneven
    _nt_case(worst, "NT bf16 unequal slices", *uneven[0], seed=3)
    for j, (N1, N2) in enumerate(((256, 1204), (256, 256), (44, 256))):
        assert _splits(BENCH_ROWS, N1, N2) > 100
        _nt_case(worst, f"NT bf16 bench {N1}x{N2}", BENCH_ROWS, N1, N2, seed=10 + j)
    _report(worst)


def test_nt_two_level_reduce(dense):
    """R = 13.9 M rows (papers100M's per-rank nodes): more than 1,024 slices, summed in groups of 64 first."""
    free, _ = torch.cuda.mem_get_info(0)
    if free < (40 << 30):
        pytest.skip("needs ~40 GB of free device memory")
    R_, N1, N2 = TWO_LEVEL_ROWS, 44, 256
    assert _splits(R_, N1, N2) > 1024
    g = _gen(41)
    worst = {}
    _nt_case(worst, "NT bf16 two-level", R_, N1, N2, seed=0, repeat=False,
             data=(_spread(R_, N1, g, row_scale=False, col_scale=True), _spread(R_, N2, g, row_scale=False, col_scale=True)))
    _report(worst)


# ---- rounding, bit for bit ------------------------------------------------------------------------------------------
def _rounding_values(n, g):
    """f32 values whose low 16 bits are an exact tie (0x8000), just below / above one, 0, all ones or random, under odd
    and even kept halves; one in ten has a kept mantissa of all ones, so rounding up carries into the exponent.  The
    first four: 0x477FFFFF (carries to 65536), 0xC77F8000 (a tie on an odd half: carries to -65536), 0x3F7FFFFF
    (carries to 1.0) and 0x3F808000 (a tie on an even half: stays 1.0039).  No value rounds to Inf: Inf * 0 would turn
    the row's other outputs into NaN (``test_special_values`` covers Inf)."""
    dev = _dev()
    sign = torch.randint(0, 2, (n,), generator=g, device=dev)
    expo = torch.randint(0x60, 0xA0, (n,), generator=g, device=dev)
    mant = torch.randint(0, 0x80, (n,), generator=g, device=dev)
    mant = torch.where(torch.rand(n, generator=g, device=dev) < 0.1, torch.full_like(mant, 0x7F), mant)
    lo = torch.tensor([0x8000, 0x7FFF, 0x8001, 0x0000, 0xFFFF], device=dev)[torch.randint(0, 5, (n,), generator=g,
                                                                                            device=dev)]
    lo = torch.where(torch.rand(n, generator=g, device=dev) < 0.2,
                     torch.randint(0, 1 << 16, (n,), generator=g, device=dev), lo)
    bits = (((sign << 15) | (expo << 7) | mant) << 16) | lo
    bits[:4] = torch.tensor([0x477FFFFF, 0xC77F8000, 0x3F7FFFFF, 0x3F808000], device=dev)
    return torch.where(bits >= 1 << 31, bits - (1 << 32), bits).to(torch.int32).view(torch.float32)


def test_rounding_bit_exact(dense):
    """B of one-hot rows: C = bf16(A) exactly (the products are x * 1 and x * 0, the sums add zeros), compared bit for
    bit with torch's rounding of A, ties to even and exponent carries included; the same through NT with a one-hot
    A."""
    M, K, N = 1000, 256, 256
    g = _gen(55)
    ad = _rounding_values(M * K, g).view(M, K)
    perm = torch.randperm(K, generator=g, device=_dev())
    onehot = torch.zeros(N, K, device=_dev())
    onehot[torch.arange(N, device=_dev()), perm] = 1.0
    a, b = _operand(ad, K), _operand(onehot, K)
    buf, out = _output(M, N, N)
    dense.tc_mm_tn(a, b, out=out, bf16=True)
    want = _bf(ad)[:, perm]
    assert (ad.view(torch.int32) & 0xFFFF == 0x8000).any() and want[0, perm.argsort()[1]] == -65536.0
    assert torch.equal(out.view(torch.int32), want.view(torch.int32)), "TN: rounding differs from torch's"
    _untouched(buf, M, N, "TN rounding")
    # NT: C[n1, :] = bf16(B[perm[n1], :])
    R_, N1, N2 = K, 128, 1000
    bd = _rounding_values(R_ * N2, g).view(R_, N2)
    oh = torch.zeros(R_, N1, device=_dev())
    oh[perm[:N1], torch.arange(N1, device=_dev())] = 1.0
    a2, b2 = _operand(oh, N1), _operand(bd, N2)
    buf2, out2 = _output(N1, N2, N2)
    _nt_call(a2, b2, out2, float("nan"))
    assert torch.equal(out2.view(torch.int32), _bf(bd)[perm[:N1]].view(torch.int32)), "NT: rounding differs"
    _untouched(buf2, N1, N2, "NT rounding")


def test_special_values(dense):
    """NaN stays NaN and +-Inf stays +-Inf through the rounding: each special value of A meets exactly one 1 of the
    one-hot B (its other products are Inf * 0 = NaN, so only that output column is checked)."""
    M, K = 64, 64
    a = torch.randn(M, K, device=_dev())
    specials = [float("nan"), float("inf"), float("-inf")]
    cols = torch.arange(M, device=_dev()) % K
    for i in range(M):
        a[i, cols[i]] = specials[i % 3]
    b = torch.eye(K, device=_dev())
    out = dense.tc_mm_tn(a, b, bf16=True)
    got = out[torch.arange(M, device=_dev()), cols]
    assert torch.isnan(got[0::3]).all()
    assert (got[1::3] == float("inf")).all() and (got[2::3] == float("-inf")).all()


# ---- argument checks ----------------------------------------------------------------------------------------------
def test_rejections_match_3xtf32(dense):
    """Every argument the 3xTF32 entry points refuse, the bf16 ones refuse with the same code, before any launch."""
    lib = _lib()
    st = _stream()
    m = torch.zeros(64, 64, device=_dev())
    c = torch.zeros(64, 64, device=_dev())
    p = m.data_ptr()
    ws = torch.zeros(1 << 20, device=_dev())

    def tn(fn, A=p, lda=64, B=p, ldb=64, bias=None, add=None, ldadd=0, C=c.data_ptr(), ldc=64, M=8, N=8, K=8):
        return fn(A, lda, B, ldb, bias, add, ldadd, None, C, ldc, M, N, K, st)

    assert tn(lib.bns_dense_tn_bf16) == 0
    torch.cuda.synchronize()
    n0 = lib.bns_launch_count()
    for what, kw in [("misaligned A", dict(A=p + 4)), ("misaligned B", dict(B=p + 8)), ("misaligned C", dict(C=p + 4)),
                     ("misaligned bias", dict(bias=p + 4)), ("misaligned addend", dict(add=p + 4, ldadd=64)),
                     ("lda % 4", dict(lda=10)), ("ldb % 4", dict(ldb=10)), ("ldc % 4", dict(ldc=10)),
                     ("ldadd % 4", dict(add=p, ldadd=10)), ("lda < K", dict(K=12, lda=8)),
                     ("ldb < K", dict(K=12, lda=12, ldb=8)), ("ldc < N", dict(N=12, ldc=8)),
                     ("ldadd < N", dict(add=p, ldadd=4)), ("M = 0", dict(M=0)), ("N = 0", dict(N=0)),
                     ("K = 0", dict(K=0)), ("NULL A", dict(A=None))]:
        rc = tn(lib.bns_dense_tn_bf16, **kw)
        assert rc == -1 and b"bns_dense_tn_bf16" in lib.bns_last_error(), f"TN {what}: {rc}"
        assert rc == tn(lib.bns_dense_tn_3xtf32, **kw), f"TN {what}"
    need = lib.bns_dense_nt_workspace_bytes(4096, 128, 128)
    assert need > 0

    def nt(fn, A=p, lda=64, B=p, ldb=64, C=p, ldc=64, R_=8, N1=8, N2=8, w=ws.data_ptr(), wb=ws.numel() * 4):
        return fn(A, lda, B, ldb, C, ldc, R_, N1, N2, w, wb, st)

    big = dict(R_=4096, N1=128, N2=128, lda=128, ldb=128, ldc=128)
    for what, kw, code in [("misaligned A", dict(A=p + 4), -1), ("misaligned B", dict(B=p + 4), -1),
                           ("misaligned C", dict(C=p + 4), -1), ("lda % 4", dict(lda=10), -1),
                           ("ldb % 4", dict(ldb=10), -1), ("ldc % 4", dict(ldc=10), -1),
                           ("lda < N1", dict(N1=12, lda=8), -1), ("ldb < N2", dict(N2=12, ldb=8), -1),
                           ("ldc < N2", dict(N2=12, ldb=12, ldc=8), -1), ("N2 % 4", dict(N2=6), -1),
                           ("R = 0", dict(R_=0), -1), ("N1 = 0", dict(N1=0), -1), ("N2 = 0", dict(N2=0), -1),
                           ("workspace too small", dict(big, wb=need - 4), -3),
                           ("workspace NULL", dict(big, w=None), -3),
                           ("workspace misaligned", dict(big, w=ws.data_ptr() + 4), -3)]:
        rc = nt(lib.bns_dense_nt_bf16, **kw)
        assert rc == code and b"bns_dense_nt_bf16" in lib.bns_last_error(), f"NT {what}: {rc}"
        assert rc == nt(lib.bns_dense_nt_3xtf32, **kw), f"NT {what}"
    assert lib.bns_launch_count() == n0, "a rejected call launched a kernel"
    torch.cuda.synchronize()
