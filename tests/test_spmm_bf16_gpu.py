"""The bf16 gather tables of ``--agg-dtype bf16``: ``bns_spmm_sum_bf16``, ``bns_spmm_compact_bf16`` and
``bns_cvt_rows_f32_bf16``, element by element.

Every SpMM result is compared with a float64 sum of the bf16-ROUNDED inputs (torch's ``.to(torch.bfloat16)``, round to
nearest even), within 1e-5 of the sum of the magnitudes of its terms (tests/layer_reference.py): every column slab
(automatic, 256, 128, 64) at F = 256 and 128, row and column maps, row / column scales and per-entry weights,
accumulation, rows of degree 0, 1, 255, 256, 257 and >= 4096 (rows longer than a chunk go through the partial sums and the
fix-up pass), 2 to 4 source-row blocks, and the compacted halo pass with chunks holding 0 / 1 / 31 / 32 / 33 sampled
entries, with and without per-entry weights.  The conversion is bit-exact against torch's on the same device, ±0,
subnormals, ±inf, NaN and halfway cases included."""
import pytest
import torch

from tests import layer_reference as R

pytestmark = pytest.mark.gpu

TOL = 1e-5
DEGREES = [0, 1, 255, 256, 257, 4096, 5000, 3, 0, 17]


def _dev():
    return torch.device("cuda:0")


def _csr(degrees, n_cols, seed):
    gen = torch.Generator().manual_seed(seed)
    deg = torch.tensor(degrees, dtype=torch.int64)
    ip = torch.cat([torch.zeros(1, dtype=torch.int64), deg.cumsum(0)])
    ix = torch.randint(0, n_cols, (int(ip[-1]),), generator=gen)
    return ip, ix


def _degrees(n_rows, seed):
    """``DEGREES`` first, then random degrees (mostly short rows, some longer than a 256-entry chunk)."""
    gen = torch.Generator().manual_seed(seed)
    rest = torch.poisson(torch.full((n_rows - len(DEGREES),), 20.0), generator=gen).long()
    rest[torch.rand(rest.shape[0], generator=gen) < 0.02] = 600
    return DEGREES + rest.tolist()


def _graph(ip, ix, n_cols, chunk=0):
    from bns_gcn_b200 import ops
    dev = _dev()
    return ops.DeviceGraph.from_csr(ip.to(dev), ix.int().to(dev), n_cols, chunk)


def _reference(xb, ip, ix, n_out, *, rs=None, cs=None, ew=None, row_map=None, col_map=None, n_direct=None, y0=None):
    """``(value, bound)`` in float64 of ``bns_spmm_sum_*`` on the bf16 table ``xb``."""
    dev = _dev()
    x = xb.double()
    n_rows = ip.numel() - 1
    rows = torch.repeat_interleave(torch.arange(n_rows), ip[1:] - ip[:-1]).to(dev)
    cols = ix.to(dev)
    w = torch.ones(cols.numel(), dtype=torch.float64, device=dev)
    if cs is not None:
        w = w * cs.double()[cols]
    if ew is not None:
        w = w * ew.double()
    xr = cols
    if col_map is not None:
        mapped = col_map.long()[(cols - n_direct).clamp(min=0)]
        xr = torch.where(cols < n_direct, cols, mapped)
    live = xr >= 0
    F = x.shape[1]
    val = torch.zeros(n_rows, F, dtype=torch.float64, device=dev)
    bnd = torch.zeros_like(val)
    if bool(live.any()):
        term = x[xr[live]] * w[live].unsqueeze(1)
        val.index_add_(0, rows[live], term)
        bnd.index_add_(0, rows[live], term.abs())
    if rs is not None:
        val, bnd = val * rs.double().unsqueeze(1), bnd * rs.double().abs().unsqueeze(1)
    orow = torch.arange(n_rows, device=dev) if row_map is None else row_map.long()
    keep = orow >= 0
    out_v = torch.zeros(n_out, F, dtype=torch.float64, device=dev) if y0 is None else y0.double().clone()
    out_b = torch.zeros_like(out_v) if y0 is None else y0.double().abs()
    out_v[orow[keep]] = out_v[orow[keep]] + val[keep] if y0 is not None else val[keep]
    out_b[orow[keep]] = out_b[orow[keep]] + bnd[keep] if y0 is not None else bnd[keep]
    return out_v, out_b


def _table(n, F, seed, pad=8):
    """A bf16 table ``[n, F]`` at a row stride padded by ``pad`` elements (a multiple of 8), and the f32 values it rounds."""
    from bns_gcn_b200 import ops
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(n, F + pad, generator=gen).to(_dev())[:, :F]
    return ops.cvt_rows_bf16(x), x


@pytest.mark.parametrize("F", [256, 128])
@pytest.mark.parametrize("slab", [0, 256, 128, 64])
def test_spmm_bf16_slabs(built, F, slab):
    from bns_gcn_b200 import ops
    n_cols = 3000
    ip, ix = _csr(_degrees(1200, 1), n_cols, 2)
    g = _graph(ip, ix, n_cols)
    assert g.n_split_rows >= 3
    xb, x = _table(n_cols, F, 3)
    assert torch.equal(xb, x.to(torch.bfloat16))
    rs = (torch.rand(ip.numel() - 1, generator=torch.Generator().manual_seed(4)) + 0.5).to(_dev())
    y = ops.spmm(g, xb, row_scale=rs, slab=slab)
    want, bound = _reference(xb, ip, ix, g.n_rows, rs=rs)
    R.assert_close(f"bf16 F={F} slab={slab}", y, want, bound, tol=TOL)
    assert torch.all(y[torch.tensor([0, 8], device=_dev())] == 0)           # degree-0 rows
    # the rounding happened in the table, not in the sum: the f32 table gives another result
    assert not torch.equal(y, ops.spmm(g, x.contiguous(), row_scale=rs, slab=slab))


@pytest.mark.parametrize("variant", ["row_map", "col_map", "col_map+col_scale", "edge_weight", "accumulate"])
def test_spmm_bf16_maps_scales_accumulate(built, variant):
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
        n_out = n_rows
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
    xb, _ = _table(x_rows, F, 8)
    rs = (torch.rand(n_rows, generator=gen) + 0.5).to(dev)
    if variant == "accumulate":
        y0 = torch.randn(n_rows, F, generator=gen).to(dev)
        y = y0.clone()
        ops.spmm(g, xb, y, row_scale=rs, accumulate=True)
        ref_kw.update(y0=y0)
    else:
        y = ops.spmm(g, xb, row_scale=rs, **kw)
    want, bound = _reference(xb, ip, ix, n_out, rs=rs, **ref_kw)
    if variant == "row_map":
        skipped = torch.ones(n_out, dtype=torch.bool, device=dev)
        skipped[kw["row_map"][kw["row_map"] >= 0].long()] = False
        assert torch.all(y[skipped] == 0)
    R.assert_close(f"bf16 {variant}", y, want, bound, tol=TOL)


@pytest.mark.parametrize("n_blocks", [2, 3, 4])
def test_spmm_bf16_source_row_blocks(built, monkeypatch, n_blocks):
    """``ops.spmm_auto`` cuts the bf16 table into ``n_blocks`` source-row blocks, each pass accumulating."""
    from bns_gcn_b200 import ops
    monkeypatch.setenv("BNS_SPMM_COLBLOCKS", str(n_blocks))
    n_cols = 4000
    ip, ix = _csr(_degrees(1500, 9), n_cols, 10)
    g = _graph(ip, ix, n_cols)
    xb, _ = _table(n_cols, 256, 11, pad=0)
    rs = (torch.rand(g.n_rows, generator=torch.Generator().manual_seed(12)) + 0.5).to(_dev())
    y = ops.spmm_auto(g, xb, row_scale=rs)
    assert len(g._col_blocks) == n_blocks
    want, bound = _reference(xb, ip, ix, g.n_rows, rs=rs)
    R.assert_close(f"bf16 {n_blocks} blocks", y, want, bound, tol=TOL)


def test_plan_col_blocks_sizes_from_element_size(built):
    """A bf16 table is half as large: half as many source-row blocks for the same graph."""
    from bns_gcn_b200 import ops

    class G:
        n_rows, nnz = 1000, 1000 * 100
    G.n_cols = 3 * ops.BLOCK_TABLE_BYTES // 512          # 3 blocks of 128 f32 columns
    assert ops.plan_col_blocks(G, 256) == 3 == ops.plan_col_blocks(G, 256, 4)
    assert ops.plan_col_blocks(G, 256, 2) == 2


@pytest.mark.parametrize("weighted", [False, True], ids=["unweighted", "cw"])
def test_spmm_compact_bf16_chunk_counts(built, weighted):
    """One 64-entry chunk per row whose sampled entries number 0, 1, 31, 32 or 33, plus rows split over several chunks:
    the compacted pass equals the f64 sum and the column-mapped pass on the same table, bit for bit."""
    from bns_gcn_b200 import ops
    dev = _dev()
    F, chunk, n_rows = 256, 64, 250
    counts = [0, 1, 31, 32, 33]
    degrees = [chunk] * n_rows
    degrees[7], degrees[100] = 300, 5 * chunk
    ip = torch.cat([torch.zeros(1, dtype=torch.int64), torch.tensor(degrees).cumsum(0)])
    n_cols = int(ip[-1])
    ix = torch.arange(n_cols)                                 # every entry its own column: the map decides the count
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
    per_chunk = c.chunk_cnt.cpu()
    for k in counts:
        assert int((per_chunk == k).sum()) > 0, k
    xb, _ = _table(n_s, F, 14)
    rs = (torch.rand(n_rows, generator=gen) + 0.5).to(dev)
    y0 = torch.randn(n_rows, F, generator=gen).to(dev)
    y = y0.clone()
    ops.spmm_compact(c, xb, y, row_scale=rs, accumulate=True)
    y_map = y0.clone()
    ops.spmm(g, xb, y_map, row_scale=rs, col_scale=cs, col_map=col_map, n_direct=0, accumulate=True)
    want, bound = _reference(xb, ip, ix, n_rows, rs=rs, cs=cs, col_map=col_map, n_direct=0, y0=y0)
    R.assert_close(f"bf16 compact {'cw' if weighted else 'plain'}", y, want, bound, tol=TOL)
    assert torch.equal(y, y_map)


def test_spmm_bf16_refuses_misaligned_tables(built):
    from bns_gcn_b200 import _lib, ops
    n_cols = 100
    ip, ix = _csr([3] * 50, n_cols, 15)
    g = _graph(ip, ix, n_cols)
    x = torch.zeros(n_cols, 36, dtype=torch.bfloat16, device=_dev())
    with pytest.raises(_lib.BnsError, match="F % 8 == 0"):
        ops.spmm(g, x[:, :12])                                 # F = 12
    with pytest.raises(_lib.BnsError, match="ldx % 8 == 0"):
        ops.spmm(g, x[:, 4:20])                                # 8-byte aligned start, ldx 36


def _specials():
    bits = torch.tensor([0x00000000, 0x80000000, 0x00000001, 0x80000001, 0x007fffff, 0x00400000, 0x00008000,
                         0x00018000, 0x7f800000, 0xff800000, 0x7fc00000, 0xffc00000, 0x7f800001, 0x7fbfffff,
                         0x3f808000, 0x3f818000, 0x3f808001, 0x3f807fff, 0x7f7fffff, 0xff7fffff, 0x7f7f8000,
                         0x00800000, 0x3f800000], dtype=torch.int64)
    return bits.to(torch.int32).view(torch.float32)


@pytest.mark.parametrize("F,lds,ldd", [(256, 256, 256), (256, 300, 264), (44, 48, 48), (7, 9, 8)])
def test_cvt_rows_bit_exact(built, F, lds, ldd):
    """Every f32 exponent with random mantissas, the special values, and ties (even and odd), strided in and out; the
    columns past F of the destination are not written."""
    from bns_gcn_b200 import ops
    dev = _dev()
    gen = torch.Generator().manual_seed(F)
    n = 4096
    bits = torch.randint(-2 ** 31, 2 ** 31, (n, lds), generator=gen, dtype=torch.int64).to(torch.int32)
    src = bits.view(torch.float32)
    sp = _specials()
    src.view(-1)[:sp.numel() * 7:7] = sp
    ties = torch.randint(-2 ** 31, 2 ** 31, (n,), generator=gen, dtype=torch.int64).to(torch.int32) & ~0xffff | 0x8000
    src[:, 0] = ties.view(torch.float32)
    src = src.to(dev)
    dst = torch.full((n, ldd), -7.0, dtype=torch.bfloat16, device=dev)
    ops.cvt_rows_bf16(src[:, :F], out=dst[:, :F])
    want = src[:, :F].to(torch.bfloat16)
    assert torch.equal(dst[:, :F].view(torch.int16), want.view(torch.int16))
    assert torch.all(dst[:, F:] == -7.0)
    auto = ops.cvt_rows_bf16(src[:, :F])
    assert auto.stride(0) % 8 == 0 and torch.equal(auto.view(torch.int16), want.view(torch.int16))
