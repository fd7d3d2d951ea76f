"""The dense 3xTF32 GEMMs of ``csrc/dense_tc.cuh`` (``bns_dense_tn_3xtf32``, ``bns_dense_nt_3xtf32`` with its split-K
reduce) and the bias-gradient column sum ``bns_colsum_f32`` against float64, element by element.

Reference and bound (``layer_reference.assert_close``, ``|got - ref| <= TOL * bound``):
  TN  ref = (A B^T + bias + addend) * row_scale,  bound = (|A| |B|^T + |bias| + |addend|) * |row_scale|
  NT  ref = A^T B,                                bound = |A|^T |B|
  colsum  ref = sum_r x[r, :],                     bound = sum_r |x[r, :]|
The bound is what f32 rounding (and the 3xTF32 split, ~2^-20 per product) is relative to, element by element, so a
small output row or column is held to its own scale: the operands' rows and columns are scaled by powers of two from
2^-20 to 2^20, so a misplaced tile, row or column exceeds its element's bound even when it is tiny next to max|C|.
Some outputs cancel exactly (paired operand rows of opposite sign), and one case has all operands positive, where the
bound equals |C| and the printed ratio is the kernel's real error over TOL.

Every operand is a view into a larger NaN-filled buffer (columns between the row and the leading dimension, rows
after the view, the pads of bias / addend / row_scale), so a read outside the view turns its output NaN.  Every output
is a view into a buffer filled with a NaN bit pattern that must be unchanged outside the view afterwards, so a store
outside it is seen.  Each split-K regime of NT is asserted from ``bns_dense_nt_workspace_bytes`` on the running GPU."""
import contextlib
import io

import pytest
import torch

from tests import layer_reference as R

pytestmark = pytest.mark.gpu

BENCH_ROWS = 232_965            # inner nodes of the benchmark's single partition (Reddit shape, README configs[1])
PART8_ROWS = 29_121             # the same graph cut into 8 partitions
SENTINEL = 0x7FA5A5A5           # a NaN payload no kernel computes: the output buffers' out-of-view contents
EXP = 20                        # operand rows / columns are scaled by 2^e, e in [-EXP, EXP]
CHUNK = 1 << 15                 # rows per float64 reference chunk at the large shapes


@pytest.fixture(scope="module")
def dense(built):
    from bns_gcn_b200.module import dense as d
    return d


def _lib():
    from bns_gcn_b200._lib import lib
    return lib


def _dev():
    return torch.device("cuda:0")


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _ceil4(n):
    return (n + 3) // 4 * 4


# ---- operands and outputs -----------------------------------------------------------------------------------------
def _gen(seed):
    return torch.Generator(device=_dev()).manual_seed(seed)


def _pow2(n, g):
    """``n`` powers of two with exponents uniform in ``[-EXP, EXP]``."""
    return torch.exp2(torch.randint(-EXP, EXP + 1, (n,), generator=g, device=_dev()).float())


def _spread(rows, cols, g, row_scale=True, col_scale=False, positive=False):
    """``[rows, cols]`` of magnitude ~1 (uniform in (0, 1] when ``positive``), rows and / or columns scaled by
    ``2^e``."""
    if positive:
        x = 1.0 - torch.rand(rows, cols, generator=g, device=_dev())
    else:
        x = torch.randn(rows, cols, generator=g, device=_dev())
    if row_scale:
        x *= _pow2(rows, g)[:, None]
    if col_scale:
        x *= _pow2(cols, g)[None, :]
    return x


def _operand(data, ld, extra_rows=3):
    """``data`` copied into the ``[rows, cols]`` corner of a NaN-filled ``[rows + extra_rows, ld]`` buffer."""
    rows, cols = data.shape
    buf = torch.full((rows + extra_rows, ld), float("nan"), device=_dev())
    v = buf[:rows, :cols]
    v.copy_(data)
    return v


def _vector(data, pad=8):
    buf = torch.full((data.numel() + pad,), float("nan"), device=_dev())
    buf[:data.numel()] = data
    return buf[:data.numel()]


def _output(rows, cols, ld, extra_rows=3):
    """``(buffer, view)``: a ``[rows, cols]`` view of a ``[rows + extra_rows, ld]`` buffer holding ``SENTINEL``."""
    buf = torch.full((rows + extra_rows, ld), SENTINEL, dtype=torch.int32, device=_dev()).view(torch.float32)
    return buf, buf[:rows, :cols]


def _untouched(buf, rows, cols, label):
    """The buffer outside its ``[rows, cols]`` view still holds ``SENTINEL``."""
    bits = buf.view(torch.int32)
    outside = torch.ones(bits.shape, dtype=torch.bool, device=bits.device)
    outside[:rows, :cols] = False
    bad = outside & (bits != SENTINEL)
    n = int(bad.sum())
    assert n == 0, f"{label}: {n} stores outside the output view, first at {torch.nonzero(bad)[:4].tolist()}"


def _close(worst, key, label, got, want, bound):
    with contextlib.redirect_stdout(io.StringIO()):
        r = R.assert_close(label, got, want, bound)
    worst[key] = max(worst.get(key, 0.0), r)


def _report(worst):
    for k, v in worst.items():
        print(f"[ratio] {k}: {v:.3g}")


# ---- TN -----------------------------------------------------------------------------------------------------------
def _check_tn(worst, key, label, got, a, b, bias=None, addend=None, row_scale=None):
    """``got`` against the float64 reference, ``CHUNK`` rows at a time; ``addend``: its values before the call."""
    bd = b.double()
    bda = bd.abs()
    for r0 in range(0, a.shape[0], CHUNK):
        r1 = min(r0 + CHUNK, a.shape[0])
        ad = a[r0:r1].double()
        ref, bnd = ad @ bd.t(), ad.abs() @ bda.t()
        if bias is not None:
            ref += bias.double()
            bnd += bias.double().abs()
        if addend is not None:
            ref += addend[r0:r1].double()
            bnd += addend[r0:r1].double().abs()
        if row_scale is not None:
            rs = row_scale[r0:r1].double()[:, None]
            ref *= rs
            bnd *= rs.abs()
        _close(worst, key, f"{label} rows {r0}:{r1}", got[r0:r1], ref, bnd)


def _tn_case(dense, worst, key, M, N, K, lda, ldc, seed, bias=False, addend=False, row_scale=False, ldadd=None,
             in_place=False, positive=False, cancel=True):
    """One TN product through ``tc_mm_tn`` on NaN-padded operand views and a sentinel-filled output view."""
    g = _gen(seed)
    ad = _spread(M, K, g, positive=positive, row_scale=not positive)
    bd = _spread(N, K, g, positive=positive, row_scale=not positive)
    if cancel and K >= 2 and M >= 4:
        # the first quarter of A's rows: second half of the contraction = -(first half), and B repeats its first half
        # in the second, so those output rows are exactly 0 while their bound is not
        h = K // 2
        ad[:M // 4, h:2 * h] = -ad[:M // 4, :h]
        bd[:, h:2 * h] = bd[:, :h]
    a, b = _operand(ad, lda), _operand(bd, _ceil4(K) + 4)
    bi = _vector(_spread(1, N, g, row_scale=False, positive=positive)[0]) if bias else None
    rs = None
    if row_scale:
        rv = torch.randn(M, generator=g, device=_dev())
        rv[::7] = 0.0
        rs = _vector(rv)
    label = f"TN (M, N, K, lda, ldc) = ({M}, {N}, {K}, {lda}, {ldc}) bias={bias} addend={addend} row_scale={row_scale}"
    buf, out = _output(M, N, ldc)
    add = add0 = None
    if addend:
        av = _spread(M, N, g, row_scale=True, positive=positive)
        if in_place:
            out.copy_(av)
            add = out
            label += " in place"
        else:
            add = _operand(av, ldadd if ldadd is not None else ldc + 4)
            label += f" ldadd={add.stride(0)}"
        add0 = av
    got = dense.tc_mm_tn(a, b, bias=bi, addend=add, row_scale=rs, out=out)
    assert got.data_ptr() == out.data_ptr()
    _check_tn(worst, key, label, got, a, b, bi, add0, rs)
    _untouched(buf, M, N, label)
    return got


TN_M = (1, 64, 127, 128, 129, 4099)
TN_N = (1, 2, 3, 4, 5, 44, 127, 128, 129, 256)
TN_K = (1, 4, 8, 31, 32, 33, 44, 602, 1204)
EPILOGUES = [(bias, add, rs) for bias in (False, True) for add in (False, True) for rs in (False, True)]


def test_tn_edge_sweep(dense):
    """Every (M, N, K) of the edge lists, with ``lda = ceil4(K)`` and a wider ``lda``, ``ldc > N`` (odd N reaches the
    scalar tail of the epilogue); the epilogue combination cycles through all 8 across the sweep."""
    worst = {}
    i = 0
    for M in TN_M:
        for N in TN_N:
            for K in TN_K:
                for lda in (_ceil4(K), _ceil4(K) + 8):
                    bias, add, rs = EPILOGUES[i % 8]
                    _tn_case(dense, worst, "TN edges", M, N, K, lda, _ceil4(N) + 4, seed=i, bias=bias, addend=add,
                             row_scale=rs)
                    i += 1
    _report(worst)


def test_tn_epilogue_combinations(dense):
    """bias / addend / row_scale in all 8 combinations at N = 3, 44, 256: ``C = (A B^T + bias + addend) * row_scale``
    in that order, with row_scale holding 0 and negative values, the addend at its own leading dimension and aliasing
    the output in place (the input-gradient accumulation of ``fused.py``)."""
    worst = {}
    i = 1000
    for N in (3, 44, 256):
        for bias, add, rs in EPILOGUES:
            for M, K in ((129, 44), (4099, 602)):
                _tn_case(dense, worst, "TN epilogue", M, N, K, _ceil4(K), _ceil4(N) + 4, seed=i, bias=bias,
                         addend=add, row_scale=rs, ldadd=_ceil4(N) + 12)
                i += 1
                if add:
                    _tn_case(dense, worst, "TN epilogue", M, N, K, _ceil4(K), _ceil4(N) + 4, seed=i, bias=bias,
                             addend=True, row_scale=rs, in_place=True)
                    i += 1
    _report(worst)


@pytest.mark.parametrize("M", [BENCH_ROWS, PART8_ROWS])
def test_tn_bench_shapes(dense, M):
    """The benchmark's dense products (3-layer GraphSAGE, hidden 256, 602 features, 41 classes padded to 44): the three
    forward products, the second with the bias sum and the fused addend, and the input gradient with row_scale =
    1 / deg, plus its in-place accumulation.  Far more output tiles than SMs: persistent CTAs walk many items."""
    assert (M + 127) // 128 * 2 > _sms()
    worst = {}
    cases = [dict(N=256, K=1204, bias=True), dict(N=256, K=256, bias=True, addend=True), dict(N=44, K=256),
             dict(N=256, K=44, row_scale=True), dict(N=256, K=44, addend=True, in_place=True)]
    for j, c in enumerate(cases):
        N, K = c.pop("N"), c.pop("K")
        if c.get("row_scale"):
            g = _gen(77)
            deg = torch.randint(1, 500, (M,), generator=g, device=_dev()).float()
            _tn_deg(dense, worst, M, N, K, 1.0 / deg, seed=j)
        else:
            _tn_case(dense, worst, "TN bench shapes", M, N, K, _ceil4(K), _ceil4(N), seed=5000 + j, **c)
    _report(worst)


def _tn_deg(dense, worst, M, N, K, rs_values, seed):
    """dY [M, K] x (W^T) [N, K]^T * (1 / deg): GCN's pre-scaled input gradient."""
    g = _gen(seed)
    a, b = _operand(_spread(M, K, g), _ceil4(K)), _operand(_spread(N, K, g), _ceil4(K))
    rs = _vector(rs_values)
    buf, out = _output(M, N, _ceil4(N))
    label = f"TN (M, N, K, lda, ldc) = ({M}, {N}, {K}, {a.stride(0)}, {out.stride(0)}) row_scale = 1/deg"
    got = dense.tc_mm_tn(a, b, row_scale=rs, out=out)
    _check_tn(worst, "TN bench shapes", label, got, a, b, row_scale=rs)
    _untouched(buf, M, N, label)
    return got


# ---- NT -----------------------------------------------------------------------------------------------------------
def _splits(R_, N1, N2):
    """The slice count the library picks on this GPU: the workspace holds one ``[N1, N2]`` partial per slice."""
    return max(1, _lib().bns_dense_nt_workspace_bytes(R_, N1, N2) // (4 * N1 * N2))


def _nt_call(a, b, out, ws_fill):
    """``bns_dense_nt_3xtf32`` with a fresh workspace (filled with ``ws_fill``) sized one tile row beyond the
    requirement, so a store past a slice stays inside the allocation."""
    from bns_gcn_b200._lib import check
    R_, N1 = a.shape
    N2 = b.shape[1]
    need = _lib().bns_dense_nt_workspace_bytes(R_, N1, N2)
    ws = torch.full((need // 4 + 128 * N2 + 64,), ws_fill, device=_dev())
    check(_lib().bns_dense_nt_3xtf32(a.data_ptr(), a.stride(0), b.data_ptr(), b.stride(0), out.data_ptr(), out.stride(0),
                                     R_, N1, N2, ws.data_ptr() if need else None, need, _stream()), "bns_dense_nt_3xtf32")


def _nt_data(R_, N1, N2, seed, positive=False):
    """A [R, N1], B [R, N2] with the columns (the output's rows / columns) scaled by powers of two, and the first
    quarter of the contraction rows cancelled exactly by the second quarter."""
    g = _gen(seed)
    ad = _spread(R_, N1, g, row_scale=False, col_scale=not positive, positive=positive)
    bd = _spread(R_, N2, g, row_scale=False, col_scale=not positive, positive=positive)
    q = R_ // 4
    if q and not positive:
        ad[q:2 * q] = -ad[:q]
        bd[q:2 * q] = bd[:q]
    return ad, bd


def _nt_case(worst, key, R_, N1, N2, seed, positive=False, repeat=False):
    ad, bd = _nt_data(R_, N1, N2, seed, positive)
    a, b = _operand(ad, _ceil4(N1) + 4), _operand(bd, N2 + 8)
    buf, out = _output(N1, N2, N2 + 4)
    s = _splits(R_, N1, N2)
    label = f"NT (R, N1, N2) = ({R_}, {N1}, {N2}) splits={s}"
    _nt_call(a, b, out, float("nan"))
    ref = torch.zeros(N1, N2, dtype=torch.float64, device=_dev())
    bnd = torch.zeros_like(ref)
    for r0 in range(0, R_, CHUNK):
        ac, bc = a[r0:r0 + CHUNK].double(), b[r0:r0 + CHUNK].double()
        ref += ac.t() @ bc
        bnd += ac.abs().t() @ bc.abs()
    _close(worst, key, label, out, ref, bnd)
    _untouched(buf, N1, N2, label)
    if repeat:
        first = out.clone()
        for fill in (0.0, float("nan")):           # another workspace, other contents: the same bits
            _nt_call(a, b, out, fill)
            assert torch.equal(out.view(torch.int32), first.view(torch.int32)), f"{label}: not bit-reproducible"
        _untouched(buf, N1, N2, label)
    return s


def test_nt_sweep(dense):
    worst = {}
    seen = set()
    i = 0
    for N1 in (1, 41, 44, 129, 256):
        for N2 in (4, 44, 128, 132, 1204):
            for R_ in (1, 37, 3000):
                seen.add(_nt_case(worst, "NT sweep", R_, N1, N2, seed=i))
                i += 1
    print(f"[splits] NT sweep: {sorted(seen)}")
    _report(worst)


def test_nt_split_regimes(dense):
    """Each split-K regime, asserted on this GPU: one slice written straight to the strided C; as many slices as
    k-blocks; slices of unequal length; more than 100 slices at the benchmark's two weight gradients.  Every case is
    run again with other workspaces and must give the same bits."""
    worst = {}
    nkb = lambda r: (r + 31) // 32                                  # noqa: E731  (k-blocks of 32 contraction rows)
    assert _splits(32, 128, 128) == 1
    _nt_case(worst, "NT one slice", 32, 128, 128, seed=1, repeat=True)
    assert _splits(64, 128, 128) == nkb(64) == 2
    _nt_case(worst, "NT slice per k-block", 64, 128, 128, seed=2, repeat=True)
    uneven = [c for c in ((5000, 256, 1204), (3001, 128, 128), (10000, 44, 256), (7777, 256, 256), (150000, 256, 256))
              if _splits(*c) > 1 and nkb(c[0]) % _splits(*c) != 0]
    assert uneven, "no candidate shape has slices of unequal length on this GPU"
    for j, c in enumerate(uneven[:2]):
        s = _nt_case(worst, "NT unequal slices", *c, seed=3 + j, repeat=True)
        print(f"[splits] NT unequal slices (R, N1, N2) = {c}: {s} slices over {nkb(c[0])} k-blocks")
    for j, (N1, N2) in enumerate(((256, 1204), (44, 256))):
        s = _splits(BENCH_ROWS, N1, N2)
        assert s > 100, (N1, N2, s)
        _nt_case(worst, "NT bench shapes", BENCH_ROWS, N1, N2, seed=10 + j, repeat=True)
        print(f"[splits] NT bench (R, N1, N2) = ({BENCH_ROWS}, {N1}, {N2}): {s} slices over {nkb(BENCH_ROWS)} k-blocks, "
              f"{nkb(BENCH_ROWS) % s} of them one k-block longer")
        _nt_case(worst, "NT bench shapes", PART8_ROWS, N1, N2, seed=20 + j)
    _report(worst)


def test_no_cancellation_error(dense):
    """All operands positive: the bound is |C| itself and the ratio is the kernel's real relative error over TOL (the
    3xTF32 split and the tensor cores' accumulation chains, no cancellation to hide or to amplify it).  Measured on an
    H100 80GB HBM3: 0.74 (TN, K = 1204) and 0.82 (NT, R = 232,965), a relative error of 1.5e-5 and 1.6e-5.  That is
    far above the split's ~2^-20 per product and leaves little room under TOL, though it is 6x below the 1e-4
    parity bar of the layer outputs."""
    worst = {}
    _tn_case(dense, worst, "no cancellation TN", BENCH_ROWS, 256, 1204, 1204, 256, seed=31, positive=True, cancel=False)
    _nt_case(worst, "no cancellation NT", BENCH_ROWS, 256, 1204, seed=32, positive=True)
    _report(worst)


# ---- colsum -------------------------------------------------------------------------------------------------------
def test_colsum(dense):
    """``bns_colsum_f32`` on strided NaN-padded inputs, both outputs written, bound sum |x|."""
    from bns_gcn_b200._lib import check
    lib = _lib()
    worst = {}
    for cols in (4, 44, 256, 1024):
        for rows in (1, 31, BENCH_ROWS):
            g = _gen(rows + cols)
            x = _operand(_spread(rows, cols, g, row_scale=True, col_scale=True), cols + 8)
            bufs = [_output(1, cols, cols + 4) for _ in range(2)]
            need = lib.bns_colsum_workspace_bytes(cols)
            ws = torch.full((need // 4 + 64,), float("nan"), device=_dev())
            check(lib.bns_colsum_f32(x.data_ptr(), x.stride(0), rows, cols, bufs[0][1].data_ptr(), bufs[1][1].data_ptr(),
                                     ws.data_ptr(), need, _stream()), "bns_colsum_f32")
            xd = x.double()
            label = f"colsum (rows, cols, ld) = ({rows}, {cols}, {x.stride(0)})"
            for k, (buf, out) in enumerate(bufs):
                _close(worst, "colsum", f"{label} out{k + 1}", out[0], xd.sum(0), xd.abs().sum(0))
                _untouched(buf, 1, cols, label)
            assert torch.equal(bufs[0][1], bufs[1][1])
    _report(worst)


# ---- argument checks ----------------------------------------------------------------------------------------------
def _rejected(what, rc):
    lib = _lib()
    assert rc != 0, f"{what}: accepted"
    assert lib.bns_last_error(), what


def test_rejections(dense):
    """Every argument check of the three entry points refuses on the host, before any launch."""
    lib = _lib()
    st = _stream()
    m = torch.zeros(64, 64, device=_dev())
    c = torch.zeros(64, 64, device=_dev())
    p = m.data_ptr()
    ws = torch.zeros(1 << 20, device=_dev())

    def tn(A=p, lda=64, B=p, ldb=64, bias=None, add=None, ldadd=0, C=c.data_ptr(), ldc=64, M=8, N=8, K=8):
        return lib.bns_dense_tn_3xtf32(A, lda, B, ldb, bias, add, ldadd, None, C, ldc, M, N, K, st)

    assert tn() == 0                          # the baseline call is valid (and launches once)
    n0 = lib.bns_launch_count()
    for what, kw in [("TN misaligned A", dict(A=p + 4)), ("TN misaligned B", dict(B=p + 8)),
                     ("TN misaligned C", dict(C=p + 4)), ("TN misaligned bias", dict(bias=p + 4)),
                     ("TN misaligned addend", dict(add=p + 4, ldadd=64)), ("TN lda % 4", dict(lda=10)),
                     ("TN ldb % 4", dict(ldb=10)), ("TN ldc % 4", dict(ldc=10)), ("TN ldadd % 4", dict(add=p, ldadd=10)),
                     ("TN lda < K", dict(K=12, lda=8)), ("TN ldb < K", dict(K=12, lda=12, ldb=8)),
                     ("TN ldc < N", dict(N=12, ldc=8)), ("TN ldadd < N", dict(add=p, ldadd=4)),
                     ("TN M = 0", dict(M=0)), ("TN N = 0", dict(N=0)), ("TN K = 0", dict(K=0)),
                     ("TN NULL A", dict(A=None))]:
        _rejected(what, tn(**kw))

    need = lib.bns_dense_nt_workspace_bytes(4096, 128, 128)
    assert need > 0

    def nt(A=p, lda=64, B=p, ldb=64, C=p, ldc=64, R_=8, N1=8, N2=8, w=ws.data_ptr(), wb=ws.numel() * 4):
        return lib.bns_dense_nt_3xtf32(A, lda, B, ldb, C, ldc, R_, N1, N2, w, wb, st)

    for what, kw in [("NT misaligned A", dict(A=p + 4)), ("NT misaligned B", dict(B=p + 4)),
                     ("NT misaligned C", dict(C=p + 4)), ("NT lda % 4", dict(lda=10)), ("NT ldb % 4", dict(ldb=10)),
                     ("NT ldc % 4", dict(ldc=10)), ("NT lda < N1", dict(N1=12, lda=8)),
                     ("NT ldb < N2", dict(N2=12, ldb=8)), ("NT ldc < N2", dict(N2=12, ldb=12, ldc=8)),
                     ("NT N2 % 4", dict(N2=6)), ("NT R = 0", dict(R_=0)), ("NT N1 = 0", dict(N1=0)),
                     ("NT N2 = 0", dict(N2=0)),
                     ("NT workspace too small", dict(R_=4096, N1=128, N2=128, lda=128, ldb=128, ldc=128, wb=need - 4)),
                     ("NT workspace NULL", dict(R_=4096, N1=128, N2=128, lda=128, ldb=128, ldc=128, w=None)),
                     ("NT workspace misaligned", dict(R_=4096, N1=128, N2=128, lda=128, ldb=128, ldc=128,
                                                      w=ws.data_ptr() + 4))]:
        _rejected(what, nt(**kw))

    cneed = lib.bns_colsum_workspace_bytes(64)

    def cs(X=p, ld=64, rows=8, cols=64, out=p, out2=None, w=ws.data_ptr(), wb=cneed):
        return lib.bns_colsum_f32(X, ld, rows, cols, out, out2, w, wb, st)

    for what, kw in [("colsum misaligned X", dict(X=p + 4)), ("colsum misaligned out", dict(out=p + 4)),
                     ("colsum misaligned out2", dict(out2=p + 4)), ("colsum ld % 4", dict(ld=66)),
                     ("colsum ld < cols", dict(ld=60)), ("colsum cols % 4", dict(cols=62)),
                     ("colsum cols > 1024", dict(cols=1028, ld=1028)), ("colsum rows = 0", dict(rows=0)),
                     ("colsum cols = 0", dict(cols=0)), ("colsum workspace too small", dict(wb=cneed - 16)),
                     ("colsum workspace misaligned", dict(w=ws.data_ptr() + 4)), ("colsum NULL X", dict(X=None))]:
        _rejected(what, cs(**kw))
    assert lib.bns_launch_count() == n0, "a rejected call launched a kernel"
    torch.cuda.synchronize()
