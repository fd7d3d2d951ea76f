"""The fp8 gather tables of ``--agg-dtype fp8``: ``bns_cvt_rows_f32_fp8``, ``bns_spmm_sum_fp8`` and
``bns_spmm_compact_fp8``, element by element.

The conversion is bit-exact (codes and scales) against the host restatement of tests/fp8_reference.py, at strided rows,
with ties, subnormal codes, the 448 edge, zero rows, rows below 2^-126 and rows holding NaN or +-Inf.  Every SpMM result
is compared with a float64 sum of the DEQUANTIZED table (codes times row scale, exact), within 1e-5 of the sum of the
magnitudes of its terms: every column slab (256, 128, 64, 32 and automatic), row and column maps, row / column scales
and per-entry weights, accumulation, rows of degree 0, 1, 256, 257 and >= 4096 (split over several chunks), source-row
blocks and the compacted halo pass.  Two runs are bit-identical.  One case gathers from a table past 2^31 bytes at the
papers100M per-rank shape (13.9 M rows of 256 codes)."""
import pytest
import torch

from tests import fp8_reference as Q
from tests import layer_reference as R
from tests.test_spmm_bf16_gpu import _csr, _degrees, _graph, _reference

pytestmark = pytest.mark.gpu

TOL = 1e-5


def _dev():
    return torch.device("cuda:0")


def _table(n, F, seed, pad=16, spread=True):
    """An fp8 table of ``n`` random rows ``[n, F]`` (row stride padded by ``pad`` codes), and its f64 values.  ``spread``:
    row magnitudes over many binades, so that the row scales differ."""
    from bns_gcn_b200 import ops
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(n, F, generator=gen)
    if spread:
        x = x * torch.exp2(torch.randint(-20, 12, (n, 1), generator=gen).float())
    x = x.to(_dev())
    out = ops.Fp8Rows(torch.empty(n, F + pad, dtype=torch.float8_e4m3fn, device=_dev())[:, :F],
                      torch.empty(n, dtype=torch.float32, device=_dev()))
    t = ops.cvt_rows_fp8(x, out)
    return t, Q.dequantize(t.codes, t.scale)


def _crafted_rows(F):
    """Rows that exercise the scale rule and the rounding: ties, subnormal codes, the 448 edge, zeros, tiny maxima,
    non-finite values."""
    rows = []
    r = torch.zeros(F)
    r[0], r[1], r[2], r[3] = 448.0, -448.0, 400.0, 17.0                          # 400: a tie between 384 and 416
    rows.append(r)
    r = torch.zeros(F)
    r[0], r[1], r[2], r[3] = 449.0, 1.0, 2.0 ** -9, 3 * 2.0 ** -11              # max just above 448 -> e = 1
    rows.append(r)
    r = torch.linspace(-1, 1, F) * 2.0 ** -9                                    # subnormal codes after scaling
    r[0] = 1.0
    rows.append(r)
    rows.append(torch.zeros(F))                                                  # zeros: scale 1
    rows.append(-torch.zeros(F))                                                 # -0: codes 0x80
    r = torch.zeros(F)
    r[5], r[6] = 1e-39, -3e-42                                                  # max below 2^-126: e clamps to -126
    rows.append(r)
    r = torch.randn(F)
    r[7] = float("nan")
    rows.append(r)
    r = torch.randn(F)
    r[F - 1] = float("inf")
    rows.append(r)
    r = torch.randn(F)
    r[3] = -float("inf")
    rows.append(r)
    r = torch.full((F,), 3.0e38)                                                 # near the f32 maximum: e = 120
    r[1] = 1.0
    rows.append(r)
    # halfway cases between adjacent codes at several binades, both signs
    m = torch.tensor([1.0625, 1.1875, 1.3125, 1.4375]).repeat(F // 4) * torch.exp2(torch.arange(F) % 9 - 4.0)
    m[0] = 256.0
    rows.append(m * torch.where(torch.arange(F) % 2 == 0, 1.0, -1.0))
    return torch.stack(rows)


@pytest.mark.parametrize("F,lds,ldc", [(256, 256, 256), (256, 300, 272), (48, 52, 64), (16, 16, 16), (272, 276, 288)])
def test_cvt_rows_fp8_bit_exact(built, F, lds, ldc):
    from bns_gcn_b200 import ops
    dev = _dev()
    gen = torch.Generator().manual_seed(F + lds)
    n = 3000
    x = torch.randn(n, lds, generator=gen) * torch.exp2(torch.randint(-140, 120, (n, 1), generator=gen).float())
    c = _crafted_rows(lds)
    x[:c.shape[0]] = c
    src = x.to(dev)
    codes = torch.full((n, ldc), 0x5a, dtype=torch.uint8, device=dev)
    scale = torch.full((n + 1,), -7.0, device=dev)
    t = ops.cvt_rows_fp8(src[:, :F], ops.Fp8Rows(codes.view(torch.float8_e4m3fn)[:, :F], scale[:n]))
    want_c, want_s = Q.quantize_rows(x[:, :F])
    assert torch.equal(t.codes.view(torch.uint8).cpu(), want_c.view(torch.uint8))
    assert torch.equal(t.scale.cpu().view(torch.int32), want_s.view(torch.int32))     # NaN bits included
    assert torch.all(codes[:, F:] == 0x5a) and float(scale[n]) == -7.0                # nothing past the view
    auto = ops.cvt_rows_fp8(src[:, :F])
    assert auto.codes.stride(0) % 16 == 0 and auto.codes.data_ptr() % 16 == 0
    assert torch.equal(auto.codes.view(torch.uint8).cpu(), want_c.view(torch.uint8))


def test_cvt_rows_fp8_rules(built):
    """The crafted rows' scales and codes, stated directly."""
    from bns_gcn_b200 import ops
    F = 16
    x = _crafted_rows(F)
    t = ops.cvt_rows_fp8(x.to(_dev()))
    s = t.scale.cpu()
    c = t.codes.view(torch.uint8).cpu()
    assert s[0] == 1.0 and c[0, 0] == 0x7e and c[0, 1] == 0xfe and c[0, 2] == 0x7c     # 400 ties to 384 (even)
    assert s[1] == 2.0
    assert s[2] == 2.0 ** -8                                                           # max 1 -> 256 <= 448 < 512
    assert s[3] == 1.0 and torch.all(c[3] == 0)
    assert torch.all(c[4] == 0x80)
    assert s[5] == 2.0 ** -126
    assert torch.isnan(s[6:9]).all() and torch.all(c[6:9] == 0)
    assert s[9] == 2.0 ** 120


def test_cvt_rows_fp8_refusals(built):
    from bns_gcn_b200 import _lib, ops
    dev = _dev()
    x = torch.zeros(10, 64, device=dev)
    with pytest.raises(_lib.BnsError, match="F % 16 == 0"):
        ops.cvt_rows_fp8(x[:, :24])
    bad = ops.Fp8Rows(torch.empty(10, 72, dtype=torch.float8_e4m3fn, device=dev)[:, :32],
                      torch.empty(10, device=dev))
    with pytest.raises(_lib.BnsError, match="ldc % 16 == 0"):
        ops.cvt_rows_fp8(x[:, :32], bad)
    with pytest.raises(_lib.BnsError, match="16-byte aligned"):
        ops.cvt_rows_fp8(x[:, 1:33])
    assert _lib.lib.bns_cvt_rows_f32_fp8(x.data_ptr(), 64, None, 64, None, 10, 64, None) == -1      # BNS_E_INVALID


@pytest.mark.parametrize("F", [256, 128, 48])
@pytest.mark.parametrize("slab", [0, 256, 128, 64, 32])
def test_spmm_fp8_slabs(built, F, slab):
    from bns_gcn_b200 import ops
    n_cols = 3000
    ip, ix = _csr(_degrees(1200, 1), n_cols, 2)
    g = _graph(ip, ix, n_cols)
    assert g.n_split_rows >= 3
    t, xd = _table(n_cols, F, 3)
    rs = (torch.rand(ip.numel() - 1, generator=torch.Generator().manual_seed(4)) + 0.5).to(_dev())
    y = ops.spmm(g, t, row_scale=rs, slab=slab)
    want, bound = _reference(xd, ip, ix, g.n_rows, rs=rs)
    R.assert_close(f"fp8 F={F} slab={slab}", y, want, bound, tol=TOL)
    assert torch.all(y[torch.tensor([0, 8], device=_dev())] == 0)           # degree-0 rows
    assert torch.equal(y, ops.spmm(g, t, row_scale=rs, slab=slab))         # repeatable, bit for bit


@pytest.mark.parametrize("slab", [256, 128, 64, 32])
@pytest.mark.parametrize("variant", ["row_map", "col_map", "col_map+col_scale", "col_scale", "edge_weight", "accumulate"])
def test_spmm_fp8_maps_scales_accumulate(built, variant, slab):
    from bns_gcn_b200 import ops
    dev = _dev()
    F, n_rows, n_direct, n_cols = 256, 900, 1000, 3000
    ip, ix = _csr(_degrees(n_rows, 5), n_cols, 6)
    g = _graph(ip, ix, n_cols)
    gen = torch.Generator().manual_seed(7)
    kw, ref_kw = {}, {}
    n_out, x_rows = n_rows, n_cols
    if variant == "row_map":
        perm = torch.randperm(n_rows, generator=gen)
        rm = torch.where(torch.rand(n_rows, generator=gen) < 0.2, -1, perm).int().to(dev)
        kw.update(row_map=rm, out=torch.zeros(n_out, F, device=dev))
        ref_kw.update(row_map=rm)
    if variant.startswith("col_map"):
        n_halo = n_cols - n_direct
        n_sampled = n_halo // 3
        cm = torch.full((n_halo,), -1, dtype=torch.int32)
        cm[torch.randperm(n_halo, generator=gen)[:n_sampled]] = n_direct + torch.randperm(n_sampled, generator=gen).int()
        cm = cm.to(dev)
        x_rows = n_direct + n_sampled
        kw.update(col_map=cm, n_direct=n_direct)
        ref_kw.update(col_map=cm, n_direct=n_direct)
    if variant.endswith("col_scale"):
        cs = (torch.rand(n_cols, generator=gen) + 0.25).to(dev)
        kw.update(col_scale=cs)
        ref_kw.update(cs=cs)
    if variant == "edge_weight":
        ew = torch.rand(ix.numel(), generator=gen).to(dev)
        kw.update(edge_weight=ew)
        ref_kw.update(ew=ew)
    t, xd = _table(x_rows, F, 8)
    rs = (torch.rand(n_rows, generator=gen) + 0.5).to(dev)
    if variant == "accumulate":
        y0 = torch.randn(n_rows, F, generator=gen).to(dev)
        y = y0.clone()
        ops.spmm(g, t, y, row_scale=rs, accumulate=True, slab=slab)
        ref_kw.update(y0=y0)
    else:
        y = ops.spmm(g, t, row_scale=rs, slab=slab, **kw)
    want, bound = _reference(xd, ip, ix, n_out, rs=rs, **ref_kw)
    if variant == "row_map":
        skipped = torch.ones(n_out, dtype=torch.bool, device=dev)
        skipped[kw["row_map"][kw["row_map"] >= 0].long()] = False
        assert torch.all(y[skipped] == 0)
    R.assert_close(f"fp8 {variant} slab={slab}", y, want, bound, tol=TOL)


def test_spmm_fp8_split_rows(built):
    """Rows of degree 0 / 1 / 256 / 257 / 4100 with the default 256-entry chunks: the long ones go through the f32
    partial sums and the fix-up pass."""
    from bns_gcn_b200 import ops
    n_cols = 5000
    degrees = [0, 1, 256, 257, 4100, 0, 1, 256, 257, 4100, 3]
    ip, ix = _csr(degrees, n_cols, 21)
    g = _graph(ip, ix, n_cols)
    assert g.n_split_rows >= 4
    t, xd = _table(n_cols, 256, 22)
    y = ops.spmm(g, t)
    want, bound = _reference(xd, ip, ix, g.n_rows)
    R.assert_close("fp8 split rows", y, want, bound, tol=TOL)
    assert torch.all(y[0] == 0) and torch.all(y[5] == 0)


def test_spmm_fp8_nonfinite_row_poisons_its_sums(built):
    from bns_gcn_b200 import ops
    dev = _dev()
    x = torch.randn(40, 32)
    x[3, 5] = float("inf")
    t = ops.cvt_rows_fp8(x.to(dev))
    ip = torch.tensor([0, 2, 4, 5], dtype=torch.int64)
    ix = torch.tensor([0, 3, 1, 2, 3])
    y = ops.spmm(_graph(ip, ix, 40), t)
    assert torch.isnan(y[0]).all() and torch.isfinite(y[1]).all() and torch.isnan(y[2]).all()


@pytest.mark.parametrize("n_blocks", [2, 3, 4])
def test_spmm_fp8_source_row_blocks(built, monkeypatch, n_blocks):
    """``ops.spmm_auto`` cuts the fp8 table (codes and scales) into ``n_blocks`` source-row blocks."""
    from bns_gcn_b200 import ops
    monkeypatch.setenv("BNS_SPMM_COLBLOCKS", str(n_blocks))
    n_cols = 4000
    ip, ix = _csr(_degrees(1500, 9), n_cols, 10)
    g = _graph(ip, ix, n_cols)
    t, xd = _table(n_cols, 256, 11, pad=0)
    rs = (torch.rand(g.n_rows, generator=torch.Generator().manual_seed(12)) + 0.5).to(_dev())
    y = ops.spmm_auto(g, t, row_scale=rs)
    assert len(g._col_blocks) == n_blocks
    want, bound = _reference(xd, ip, ix, g.n_rows, rs=rs)
    R.assert_close(f"fp8 {n_blocks} blocks", y, want, bound, tol=TOL)


def test_plan_col_blocks_fp8(built):
    """An fp8 table is a quarter of the f32 one: a quarter of the source-row blocks for the same graph."""
    from bns_gcn_b200 import ops

    class G:
        n_rows, nnz = 1000, 1000 * 100
    G.n_cols = 4 * ops.BLOCK_TABLE_BYTES // 512          # 4 blocks of 128 f32 columns
    assert ops.plan_col_blocks(G, 256) == 4
    assert ops.plan_col_blocks(G, 256, 1) == 1


@pytest.mark.parametrize("weighted", [False, True], ids=["unweighted", "cw"])
def test_spmm_compact_fp8_chunk_counts(built, weighted):
    """The compacted halo pass over chunks holding 0 / 1 / 31 / 32 / 33 sampled entries, and the column-mapped pass on
    the same table, against the f64 sum; the compacted pass twice, bit for bit.  The row scale follows the row of X each
    entry gathers."""
    from bns_gcn_b200 import ops
    dev = _dev()
    F, chunk, n_rows = 256, 64, 250
    counts = [0, 1, 31, 32, 33]
    degrees = [chunk] * n_rows
    degrees[7], degrees[100] = 300, 5 * chunk
    ip = torch.cat([torch.zeros(1, dtype=torch.int64), torch.tensor(degrees).cumsum(0)])
    n_cols = int(ip[-1])
    ix = torch.arange(n_cols)
    gen = torch.Generator().manual_seed(13)
    sampled = torch.zeros(n_cols, dtype=torch.bool)
    for r in range(n_rows):
        k = counts[r % len(counts)] if degrees[r] == chunk else int(degrees[r] * 0.4)
        sampled[int(ip[r]) + torch.randperm(degrees[r], generator=gen)[:k]] = True
    n_s = int(sampled.sum())
    col_map = torch.full((n_cols,), -1, dtype=torch.int32)
    col_map[sampled] = torch.randperm(n_s, generator=gen).int()
    col_map = col_map.to(dev)
    g = _graph(ip, ix, n_cols, chunk)
    cs = (torch.rand(n_cols, generator=gen) + 0.25).to(dev) if weighted else None
    c = ops.CompactedCols(g, with_weights=weighted)
    c.refresh(col_map, 0, cs)
    t, xd = _table(n_s, F, 14)
    rs = (torch.rand(n_rows, generator=gen) + 0.5).to(dev)
    y0 = torch.randn(n_rows, F, generator=gen).to(dev)
    y = y0.clone()
    ops.spmm_compact(c, t, y, row_scale=rs, accumulate=True)
    y_map = y0.clone()
    ops.spmm(g, t, y_map, row_scale=rs, col_scale=cs, col_map=col_map, n_direct=0, accumulate=True)
    want, bound = _reference(xd, ip, ix, n_rows, rs=rs, cs=cs, col_map=col_map, n_direct=0, y0=y0)
    R.assert_close(f"fp8 compact {'cw' if weighted else 'plain'}", y, want, bound, tol=TOL)
    # the column-mapped pass meets the same bar; with two 16-lane row groups per warp at the 256-column slab it need not
    # add the entries in the same order as the compacted pass
    R.assert_close(f"fp8 col_map {'cw' if weighted else 'plain'}", y_map, want, bound, tol=TOL)
    y2 = y0.clone()
    ops.spmm_compact(c, t, y2, row_scale=rs, accumulate=True)
    assert torch.equal(y, y2)


def test_spmm_fp8_refuses_misaligned_tables(built):
    from bns_gcn_b200 import _lib, ops
    dev = _dev()
    n_cols = 100
    ip, ix = _csr([3] * 50, n_cols, 15)
    g = _graph(ip, ix, n_cols)
    codes = torch.zeros(n_cols, 72, dtype=torch.float8_e4m3fn, device=dev)
    sc = torch.ones(n_cols, device=dev)
    with pytest.raises(_lib.BnsError, match="F % 16 == 0"):
        ops.spmm(g, ops.Fp8Rows(codes[:, :24], sc))
    with pytest.raises(_lib.BnsError, match="ldx % 16 == 0"):
        ops.spmm(g, ops.Fp8Rows(codes[:, :32], sc))
    with pytest.raises(_lib.BnsError, match="16-byte aligned"):
        ops.spmm(g, ops.Fp8Rows(torch.zeros(n_cols, 64, dtype=torch.float8_e4m3fn, device=dev)[:, 8:40], sc))
    with pytest.raises(_lib.BnsError, match="one contiguous scale per row"):
        ops.spmm(g, ops.Fp8Rows(torch.zeros(n_cols, 64, dtype=torch.float8_e4m3fn, device=dev), sc[:10]))


def test_spmm_fp8_large_table(built):
    """13.9 M rows of 256 codes (3.6 GB: byte offsets past 2^31), the gathered rows spread over the whole table and
    concentrated at its end; a sample of the conversion checked against the host rule at rows past 2^31 bytes."""
    from bns_gcn_b200 import ops
    dev = _dev()
    n_x, F = 13_900_000, 256
    free, _ = torch.cuda.mem_get_info()
    if free < 24 << 30:
        pytest.skip(f"needs 24 GiB of free device memory, {free >> 30} GiB free")
    codes = torch.empty(n_x, F, dtype=torch.float8_e4m3fn, device=dev)
    scale = torch.empty(n_x, dtype=torch.float32, device=dev)
    gen = torch.Generator(device=dev).manual_seed(31)
    step = 1_000_000
    for r0 in range(0, n_x, step):
        r1 = min(n_x, r0 + step)
        x = torch.randn(r1 - r0, F, device=dev, generator=gen)
        x *= torch.exp2(torch.randint(-10, 10, (r1 - r0, 1), device=dev, generator=gen).float())
        ops.cvt_rows_fp8(x, ops.Fp8Rows(codes[r0:r1], scale[r0:r1]))
        if r1 == n_x:                                    # the last rows: past 2^31 bytes of codes
            wc, ws = Q.quantize_rows(x[-2000:].cpu())
            assert torch.equal(codes[n_x - 2000:].view(torch.uint8).cpu(), wc.view(torch.uint8))
            assert torch.equal(scale[n_x - 2000:].cpu(), ws)
        del x
    n_rows = 3000
    g0 = torch.Generator().manual_seed(32)
    ip = torch.cat([torch.zeros(1, dtype=torch.int64), torch.randint(0, 40, (n_rows,), generator=g0).cumsum(0)])
    nnz = int(ip[-1])
    ix = torch.where(torch.rand(nnz, generator=g0) < 0.5, torch.randint(0, n_x, (nnz,), generator=g0),
                     torch.randint(n_x - 100_000, n_x, (nnz,), generator=g0))
    assert int(ix.max()) * F >= 2 ** 31
    g = _graph(ip, ix, n_x)
    t = ops.Fp8Rows(codes, scale)
    y = ops.spmm(g, t)
    used = torch.unique(ix)
    rows_d = Q.dequantize(codes[used.to(dev)], scale[used.to(dev)])
    remap = torch.full((n_x,), -1, dtype=torch.int64)
    remap[used] = torch.arange(used.numel())
    want, bound = _reference(rows_d, ip, remap[ix], g.n_rows)                # only the gathered rows, widened
    R.assert_close("fp8 large table", y, want, bound, tol=TOL)
