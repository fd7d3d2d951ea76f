"""The fp8 kernels of ``--dense-dtype fp8``: ``bns_cvt_rows_f32_fp8_any`` and ``bns_dropout_fp8`` bit for bit against
the host rule (``tests/fp8_reference.py``) and ``bns_dropout_f32``; ``bns_dense_tn_fp8`` against the float64 product of
its codes and scales (``tests/dense_fp8_reference.py``) within 1e-3 of the magnitude sum of its terms; the derived fp8
weights of ``ParamArena`` bit for bit against the host rule after every optimizer step and after a reload.

Operands are code views of larger buffers whose pad bytes (between K and the row stride) and extra rows hold random
garbage, so a read outside a view shows as a wrong result; outputs are sentinel-filled views
(``tests/test_dense_gemm_gpu.py``), so a store outside one is seen."""
import contextlib
import io

import pytest
import torch

from tests import dense_fp8_reference as D
from tests import fp8_reference as Q
from tests import layer_reference as R
from tests.test_dense_gemm_gpu import (BENCH_ROWS, CHUNK, EPILOGUES, _dev, _gen, _lib, _output, _report, _spread,
                                       _stream, _untouched, _vector)

pytestmark = pytest.mark.gpu

# Hopper's e4m3 wgmma sums its products with fewer mantissa bits than f32: on an H100 the worst error measured here was
# 3.3e-4 of the magnitude sum at K = 44 (one 128-code block) and 5.8e-4 at K = 8192, so the bar is 1e-3, not the 1e-5
# that f32 sums of the same products would meet.
TOL = 1e-3


def _close(worst, key, label, got, want, bound, tol):
    with contextlib.redirect_stdout(io.StringIO()):
        r = R.assert_close(label, got, want, bound, tol=tol)
    worst[key] = max(worst.get(key, 0.0), r)


@pytest.fixture(scope="module")
def mods(built):
    from bns_gcn_b200 import fused, ops
    from bns_gcn_b200.module import dense
    return ops, dense, fused


def _same_rows(got, codes, scale, label):
    """``got`` (``ops.Fp8Rows``) holds exactly ``codes`` / ``scale`` (codes as bytes, scales as bits)."""
    assert torch.equal(got.codes.view(torch.uint8), codes.view(torch.uint8)), f"{label}: codes differ"
    assert torch.equal(got.scale.view(torch.int32), scale.view(torch.int32)), f"{label}: scales differ"


def _special_rows(F, g):
    """Rows of magnitude ~1 scaled by 2^e, then crafted rows: NaN, +Inf, -Inf, zero, subnormal-only, tiny (codes that
    are e4m3 subnormals), exact ties between two e4m3 values, and maxima of exactly 448 * 2^k."""
    x = _spread(64, F, g)
    x[0, F // 2] = float("nan")
    x[1, 0] = float("inf")
    x[2, F - 1] = float("-inf")
    x[3] = 0.0
    x[4] = torch.randn(F, generator=g, device=_dev()) * 1e-39           # f32 subnormals
    x[5] = torch.randn(F, generator=g, device=_dev()) * 2.0 ** -130
    x[6, :] = 1.0 + 2.0 ** -4                                            # halfway between two e4m3 values: ties
    x[6, ::2] = 1.0 + 3 * 2.0 ** -4
    x[6, 0] = 448.0
    for i, k in enumerate((-10, 0, 3, 20)):
        x[7 + i, 0] = -448.0 * 2.0 ** k
    return x


@pytest.mark.parametrize("F", [4, 44, 1024, 1204])
def test_quantizer_any_width_bit_exact(mods, F):
    ops, _, _ = mods
    x = _special_rows(F, _gen(F))
    buf = torch.full((x.shape[0] + 2, F + 12), float("nan"), device=_dev())
    src = buf[:x.shape[0], :F]
    src.copy_(x)
    got = ops.cvt_rows_fp8_any(src)
    codes, scale = Q.quantize_rows(x)
    _same_rows(got, codes, scale, f"F={F}")
    assert torch.isnan(got.scale[:3]).all() and not torch.isnan(got.scale[3:]).any()
    if F % 16 == 0:                                      # the same rows as the F % 16 quantizer
        _same_rows(got, *(lambda t: (t.codes, t.scale))(ops.cvt_rows_fp8(src)), f"F={F} vs cvt_rows_fp8")


@pytest.mark.parametrize("p", [0.0, 0.5])
def test_dropout_fp8_bit_exact(mods, p):
    """Both outputs: the f32 rows bit for bit against ``bns_dropout_f32`` (same seed, same epoch offset), their fp8 rows
    against the host rule applied to those rows."""
    ops, _, fused = mods
    n, F = 5000, 1204
    x = _spread(n, F, _gen(7))
    x[3, 5] = float("inf")
    ops.RNG.update(seed=11, offset=3)
    want = fused.dropout(x, p, 99)
    y, q = fused.dropout_fp8(x, p, 99)
    assert torch.equal(y.view(torch.int32), want.view(torch.int32))
    codes, scale = Q.quantize_rows(want)
    _same_rows(q, codes, scale, f"dropout p={p}")


# ---- the GEMM ---------------------------------------------------------------------------------------------------------
def _fp8_operand(ops, data, pad=16, extra_rows=3, seed=0):
    """``data``'s fp8 rows in a buffer whose row stride exceeds the row by ``pad`` bytes (rounded up to 16), the pad
    bytes and ``extra_rows`` more rows random garbage; scales in a NaN-fenced vector."""
    rows, K = data.shape
    ld = (K + pad + 15) // 16 * 16
    codes, scale = Q.quantize_rows(data)
    g = torch.Generator(device=_dev()).manual_seed(seed)
    buf = torch.randint(0, 256, (rows + extra_rows, ld), dtype=torch.uint8, generator=g, device=_dev())
    buf[:rows, :K] = codes.view(torch.uint8)
    return ops.Fp8Rows(buf[:rows, :K].view(torch.float8_e4m3fn), _vector(scale)), codes, scale


def _tn_case(mods, worst, key, M, N, K, seed, bias=False, addend=False, row_scale=False, in_place=False, positive=False,
             ldc=None):
    ops, dense, _ = mods
    g = _gen(seed)
    a, qa, sa = _fp8_operand(ops, _spread(M, K, g, positive=positive, row_scale=not positive), seed=seed)
    b, qb, sb = _fp8_operand(ops, _spread(N, K, g, positive=positive, row_scale=not positive), pad=48, seed=seed + 1)
    bi = _vector(_spread(1, N, g, row_scale=False)[0]) if bias else None
    rs = None
    if row_scale:
        rv = torch.randn(M, generator=g, device=_dev())
        rv[::7] = 0.0
        rs = _vector(rv)
    ldc = ldc or (N + 3) // 4 * 4 + 4
    label = f"TN fp8 (M, N, K) = ({M}, {N}, {K}) bias={bias} addend={addend} row_scale={row_scale}"
    buf, out = _output(M, N, ldc)
    add = add0 = None
    if addend:
        add0 = _spread(M, N, g)
        if in_place:
            out.copy_(add0)
            add = out
            label += " in place"
        else:
            abuf = torch.full((M + 2, (N + 3) // 4 * 4 + 12), float("nan"), device=_dev())
            add = abuf[:M, :N]
            add.copy_(add0)
    got = dense.tc_mm_tn_fp8(a, b, bias=bi, addend=add, row_scale=rs, out=out)
    for r0 in range(0, M, CHUNK):
        r1 = min(r0 + CHUNK, M)
        ref, bnd = D.tn(qa[r0:r1], sa[r0:r1], qb, sb, bi, None if add0 is None else add0[r0:r1],
                        None if rs is None else rs[r0:r1])
        _close(worst, key, f"{label} rows {r0}:{r1}", got[r0:r1], ref, bnd, TOL)
    _untouched(buf, M, N, label)
    if not in_place:
        buf2, out2 = _output(M, N, ldc)
        dense.tc_mm_tn_fp8(a, b, bias=bi, addend=add, row_scale=rs, out=out2)
        assert torch.equal(out.view(torch.int32), out2.view(torch.int32)), f"{label}: not bit-reproducible"
    return got


def test_tn_edge_shapes(mods):
    """M, N, K off the 128 x 128 x 128 tile, K in {1, 16, 44, 1204}; the epilogue cycles through its 8 combinations."""
    worst = {}
    i = 0
    for M in (1, 127, 129, 4099):
        for N in (1, 3, 44, 129, 256):
            for K in (1, 16, 44, 1204):
                bias, add, rs = EPILOGUES[i % 8]
                _tn_case(mods, worst, "TN fp8 edges", M, N, K, seed=i, bias=bias, addend=add, row_scale=rs)
                i += 1
    _report(worst)


def test_tn_epilogue_combinations(mods):
    """bias / addend / row_scale in all 8 combinations, the addend at its own leading dimension and aliasing C."""
    worst = {}
    i = 7000
    for N in (3, 44, 256):
        for bias, add, rs in EPILOGUES:
            _tn_case(mods, worst, "TN fp8 epilogue", 4099, N, 602, seed=i, bias=bias, addend=add, row_scale=rs)
            i += 1
            if add:
                _tn_case(mods, worst, "TN fp8 epilogue", 4099, N, 602, seed=i, bias=bias, addend=True, row_scale=rs,
                         in_place=True)
                i += 1
    _report(worst)


@pytest.mark.parametrize("K,N", [(1204, 256), (256, 256), (256, 44), (44, 256)])
def test_tn_bench_shapes(mods, K, N):
    """The benchmark's forward and input-gradient products at its one-partition row count."""
    worst = {}
    _tn_case(mods, worst, f"TN fp8 bench {K}->{N}", BENCH_ROWS, N, K, seed=K + N, bias=N == 256)
    _report(worst)


PAPERS_ROWS = 13_900_000         # papers100M's per-rank node count


def test_tn_papers100m_rows(mods):
    """M = 13.9 M rows (papers100M's per-rank nodes), K = N = 256, bias and an addend aliasing C: the A rows (a 14 GB f32
    matrix, quantized by ``cvt_rows_fp8_any`` in one call, bit-exact against the host rule at both ends) and C lie past
    2^31 bytes, so a 32-bit row offset anywhere in the quantizer, the tensor map, the scale index or the epilogue
    shows.  Checked in row chunks against ``dense_fp8_reference.tn``."""
    ops, dense, _ = mods
    free, _ = torch.cuda.mem_get_info(0)
    if free < (40 << 30):
        pytest.skip("needs ~40 GB of free device memory")
    M, K, N, step = PAPERS_ROWS, 256, 256, 1 << 20
    addend = lambda i: _spread(min(step, M - i), N, _gen(1000 + i // step))   # noqa: E731
    a32 = torch.empty(M, K, device=_dev())
    for i in range(0, M, step):
        a32[i:i + step] = _spread(min(step, M - i), K, _gen(7 + i // step))
    a = ops.cvt_rows_fp8_any(a32)
    for rows in (slice(0, 4096), slice(M - 4096, M)):
        _same_rows(a[rows], *Q.quantize_rows(a32[rows]), f"13.9M rows {rows}")
    del a32
    torch.cuda.empty_cache()
    g = _gen(5)
    b = ops.cvt_rows_fp8_any(_spread(N, K, g))
    bias = _vector(_spread(1, N, g, row_scale=False)[0])
    out = torch.empty(M, N, device=_dev())
    for i in range(0, M, step):
        out[i:i + step] = addend(i)                        # regenerated below for the reference
    dense.tc_mm_tn_fp8(a, b, bias=bias, addend=out, out=out)
    worst, big = {}, 1 << 18
    for r0 in range(0, M, big):
        r1 = min(r0 + big, M)
        i = r0 // step * step                              # big divides step: one addend chunk holds [r0, r1)
        add = addend(i)[r0 - i:r1 - i]
        ref, bnd = D.tn(a.codes[r0:r1], a.scale[r0:r1], b.codes, b.scale, bias, add)
        _close(worst, "TN fp8 13.9M", f"TN fp8 13.9M rows {r0}:{r1}", out[r0:r1], ref, bnd, TOL)
    _report(worst)


def test_tn_long_k_promotes_to_f32(mods):
    """K = 8192 with all operands positive, where the bound equals |C| and every rounding error adds up: the kernel
    promotes each 128-code block's sums to f32 (a chain of 64 blocks summed on the tensor cores keeps fewer bits)."""
    worst = {}
    _tn_case(mods, worst, "TN fp8 long K", 512, 256, 8192, seed=77, positive=True)
    _report(worst)


def test_special_scales_poison_only_their_row_and_column(mods):
    ops, dense, _ = mods
    g = _gen(9)
    a, b = _spread(300, 200, g), _spread(140, 200, g)
    a[5, 7], b[130, 0] = float("nan"), float("-inf")
    out = dense.tc_mm_tn_fp8(ops.cvt_rows_fp8_any(a), ops.cvt_rows_fp8_any(b))
    nan = torch.isnan(out)
    assert nan[5].all() and nan[:, 130].all()
    assert int(nan.sum()) == 140 + 300 - 1


def test_rejections(mods):
    """Every malformed argument is refused with the bf16 entry points' code (-1) before anything launches."""
    lib = _lib()
    st = _stream()
    codes = torch.zeros(64, 64, dtype=torch.uint8, device=_dev())
    sc = torch.ones(64, device=_dev())
    c = torch.zeros(64, 64, device=_dev())
    p, s = codes.data_ptr(), sc.data_ptr()

    def tn(A=p, lda=64, sa=s, B=p, ldb=64, sb=s, bias=None, add=None, ldadd=0, C=c.data_ptr(), ldc=64, M=8, N=8, K=8):
        return lib.bns_dense_tn_fp8(A, lda, sa, B, ldb, sb, bias, add, ldadd, None, C, ldc, M, N, K, st)

    assert tn() == 0
    torch.cuda.synchronize()
    n0 = lib.bns_launch_count()
    for what, kw in [("misaligned A", dict(A=p + 8)), ("misaligned B", dict(B=p + 4)), ("misaligned C", dict(C=p + 4)),
                     ("misaligned a_scale", dict(sa=s + 2)), ("misaligned b_scale", dict(sb=s + 1)),
                     ("misaligned bias", dict(bias=s + 4)), ("misaligned addend", dict(add=c.data_ptr() + 4, ldadd=64)),
                     ("lda % 16", dict(lda=24)), ("ldb % 16", dict(ldb=40)), ("ldc % 4", dict(ldc=10)),
                     ("ldadd % 4", dict(add=c.data_ptr(), ldadd=10)), ("lda < K", dict(K=20, lda=16)),
                     ("ldb < K", dict(K=20, lda=32, ldb=16)), ("ldc < N", dict(N=12, ldc=8)),
                     ("ldadd < N", dict(add=c.data_ptr(), ldadd=4)), ("M = 0", dict(M=0)), ("N = 0", dict(N=0)),
                     ("K = 0", dict(K=0)), ("NULL A", dict(A=None)), ("NULL a_scale", dict(sa=None)),
                     ("NULL b_scale", dict(sb=None))]:
        rc = tn(**kw)
        assert rc == -1 and b"bns_dense_tn_fp8" in lib.bns_last_error(), f"{what}: {rc}"
    f = torch.zeros(8, 8, device=_dev())
    for fn, args in (("bns_cvt_rows_f32_fp8_any", (f.data_ptr(), 8, p, 64, s, 8, 6, st)),       # F % 4
                     ("bns_cvt_rows_f32_fp8_any", (f.data_ptr(), 8, p, 24, s, 8, 8, st)),      # ldc % 16
                     ("bns_dropout_fp8", (f.data_ptr(), 8, 8, 8, 0.5, 1, 0, None, f.data_ptr(), 8, p, 8, s, st)),
                     ("bns_dropout_fp8", (f.data_ptr(), 8, 8, 8, 1.0, 1, 0, None, f.data_ptr(), 8, p, 64, s, st))):
        assert getattr(lib, fn)(*args) == -1, fn
    assert lib.bns_launch_count() == n0, "a rejected call launched a kernel"


# ---- derived fp8 weights ------------------------------------------------------------------------------------------------
def test_derived_weights_follow_every_step_and_a_reload(mods):
    """``fp8_rows(W)`` / ``fp8_rows(W, transposed=True)`` equal the host rule applied to ``padded(W)`` /
    ``transposed(W)`` after creation, after each Adam step and after the weights are reloaded; pad rows have zero
    codes."""
    _, _, fused = mods
    torch.manual_seed(0)
    model = torch.nn.Sequential(torch.nn.Linear(1204, 256), torch.nn.Linear(256, 41)).to(_dev())
    arena = fused.ParamArena(model)
    opt = fused.FusedAdam(arena, lr=1e-2)
    ws = [model[0].weight, model[1].weight]
    views = [(w, t, arena.fp8_rows(w, t)) for w in ws for t in (False, True)]

    def check(label):
        torch.cuda.synchronize()
        for w, t, q in views:
            src = arena.transposed(w) if t else arena.padded(w)
            _same_rows(q, *Q.quantize_rows(src), f"{label} {tuple(w.shape)} transposed={t}")
        q = arena.fp8_rows(model[1].weight)
        assert q.shape == (44, 256) and (q.codes[41:].view(torch.uint8) == 0).all()

    check("created")
    for step in range(3):
        for p in arena.params:                           # the pads' gradients stay zero, as every backward leaves them
            arena.unpadded(arena.flat_g, p).copy_(torch.randn(p.shape, device=_dev()))
        opt.step()
        check(f"step {step}")
    sd = {k: v.clone() * 0.5 for k, v in model.state_dict().items()}
    model.load_state_dict(sd)
    arena.refresh(advance=None)
    check("reload")
