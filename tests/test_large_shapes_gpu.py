"""The training step's kernels at the papers100M per-rank shape (BASELINE.json configs[4], 8 ranks): tensors past 2^31
elements and 4 GiB, and reductions over 13.9 M rows, against float64.

Per rank: 13,882,494 inner nodes (111,059,956 / 8), ~9.7 M sampled halo rows in the layer-0 gather table, ~97 M halo
nodes, ~200 M local entries, hidden width 256, 172 classes.  At that shape every ``row * ld`` of an activation passes
2^31 (row 8,259,552 at ld = 260), the gather table passes 2^32 elements, and the f32 reductions of the weight and bias
gradients and of LayerNorm's dgamma / dbeta run over 13.9 M rows.

Method, for every case:
  * outputs are checked on sampled rows: the first and last, the rows on either side of every multiple of 2^30
    elements of each operand's leading dimension (every 2^31 / 2^32 element and every 4 GiB byte boundary of f32 and
    bf16 matrices), the heavy rows, and 4,000 seeded random rows; every column of those rows.  The float64 reference is
    computed on the GPU from exactly the entries / rows that feed them.  Small outputs (dW, colsum, dgamma, dbeta, the
    loss) are checked in full against a float64 reduction over every row;
  * comparison: ``layer_reference.assert_close`` with its ``TOL`` and bound = the operation applied to |operands|; a
    failure names the global rows that are out.  The worst ratio per case is printed (pytest -s);
  * operands are views into buffers whose padding columns hold NaN (a wrapped read turns its output NaN), outputs are
    views into buffers holding the ``SENTINEL`` NaN pattern of test_dense_gemm_gpu.py past the view (pad columns and
    three extra rows), checked afterwards (a wrapped store lands where it is seen);
  * each test states its device-memory need and skips, naming it, when less is free.

What is not reached: the SpMM partial-sum workspace holds one F-wide row per chunk of a row longer than one chunk, so
it passes 2^31 elements only with ~2 G entries in split rows, which the int32 entry ids of the transpose exclude."""
import contextlib
import io

import numpy as np
import pytest
import torch

from tests import layer_reference as R

pytestmark = pytest.mark.gpu

N_IN = 111_059_956 // 8           # inner nodes of one of 8 ranks (papers100M)
N_SAMP = 9_700_000                # sampled halo rows of the layer-0 gather table (10 % of the halo)
N_HALO = 97_000_000               # halo nodes of one rank
F = 256                           # hidden width (and the layer-0 input concat(feat, mean))
LD = F + 4                        # leading dimension of every f32 operand: 4 NaN pad columns
AVG_DEG = 14                      # ~200 M local entries / 13.9 M rows
HEAVY = 100_000                   # entries of a power-law hub row: ~390 chunks of 256
N_CLASS = 172
TRAIN_FRAC = 0.011
SENTINEL = 0x7FA5A5A5             # NaN payload no kernel computes (as in test_dense_gemm_gpu.py)
N_RANDOM_ROWS = 4000
GB = 1 << 30


def _dev():
    return torch.device("cuda:0")


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _lib():
    from bns_gcn_b200._lib import lib
    return lib


def _check_rc(rc, what):
    from bns_gcn_b200._lib import check
    check(rc, what)


def _need(gb):
    """Skip, naming the need, when less than ``gb`` GB of device memory is free (after returning this process's cached
    blocks: earlier tests' tensors are gone, their memory may still be held by the allocator)."""
    import gc
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info(0)
    if free < gb * GB:
        pytest.skip(f"needs ~{gb} GB of free device memory, {free / GB:.1f} GB free")
    print(f"[memory] needs ~{gb} GB, {free / GB:.1f} GB free")


def _gen(seed):
    return torch.Generator(device=_dev()).manual_seed(seed)


# ---- buffers ----------------------------------------------------------------------------------------------------------
def _operand(rows, cols, ld, fill_fn=None, extra_rows=3):
    """``[rows, cols]`` view of a NaN-filled ``[rows + extra_rows, ld]`` buffer, the view filled by ``fill_fn(view)``."""
    buf = torch.full((rows + extra_rows, ld), float("nan"), device=_dev())
    v = buf[:rows, :cols]
    if fill_fn is not None:
        fill_fn(v)
    return v


def _output(rows, cols, ld, extra_rows=3):
    """``(buffer, view)``: a ``[rows, cols]`` view of a ``[rows + extra_rows, ld]`` buffer holding ``SENTINEL``."""
    buf = torch.full((rows + extra_rows, ld), SENTINEL, dtype=torch.int32, device=_dev()).view(torch.float32)
    return buf, buf[:rows, :cols]


def _untouched(buf, rows, cols, label):
    """Outside its ``[rows, cols]`` view the buffer still holds ``SENTINEL`` (pad columns of every row, extra rows)."""
    bits = buf.view(torch.int32)
    bad_cols = int((bits[:rows, cols:] != SENTINEL).sum()) if bits.shape[1] > cols else 0
    bad_tail = int((bits[rows:] != SENTINEL).sum())
    assert bad_cols == 0 and bad_tail == 0, \
        f"{label}: stores outside the output view: {bad_cols} in the pad columns, {bad_tail} in the rows past it"


def _fill_randn(g, scale_rows=False):
    def f(v):
        for r0 in range(0, v.shape[0], 1 << 22):
            c = v[r0:r0 + (1 << 22)]
            c.normal_(generator=g)
            if scale_rows:
                c.mul_(torch.exp2(torch.randint(-8, 9, (c.shape[0], 1), generator=g, device=_dev()).float()))
    return f


def _fill_positive(g):
    def f(v):
        for r0 in range(0, v.shape[0], 1 << 22):
            c = v[r0:r0 + (1 << 22)]
            c.uniform_(generator=g)
            c.neg_().add_(1.0)              # (0, 1]
    return f


# ---- sampled rows and the comparison ----------------------------------------------------------------------------------
def sample_rows(n, lds=(), extra=(), seed=0, k=N_RANDOM_ROWS):
    """Sorted unique int64 rows (device): first, last, both sides of every multiple of 2^30 elements for each leading
    dimension in ``lds``, ``extra``, and ``k`` seeded random rows."""
    s = {0, n - 1}
    for ld in lds:
        m = 1 << 30
        while m // ld <= n:
            r = m // ld
            s |= {r - 1, r, r + 1}
            m += 1 << 30
    s |= {int(r) for r in extra}
    s = sorted(r for r in s if 0 <= r < n)
    rnd = torch.randint(0, n, (k,), generator=torch.Generator().manual_seed(seed))
    return torch.unique(torch.cat([torch.tensor(s, dtype=torch.int64), rnd])).to(_dev())


def _close(worst, key, label, got, want, bound, rows=None):
    """``assert_close`` on sampled rows; a failure also names the GLOBAL rows (``rows[i]``) that are out."""
    try:
        with contextlib.redirect_stdout(io.StringIO()):
            r = R.assert_close(label, got, want, bound)
    except AssertionError as e:
        if rows is None:
            raise
        err = (got.double() - want).abs()
        bad = ~(err <= R.TOL * bound + 1e-30)
        local = torch.unique(torch.nonzero(bad)[:, 0])
        raise AssertionError(f"{e}\n  global rows out: {rows[local][:16].tolist()} ({local.numel()} rows)") from None
    worst[key] = max(worst.get(key, 0.0), r)
    return r


def _report(worst):
    for k, v in worst.items():
        print(f"[ratio] {k}: {v:.3g}")


def _bits_equal(label, got, want, rows=None):
    a, b = got.contiguous().view(torch.int32), want.contiguous().view(torch.int32)
    bad = a != b
    if bool(bad.any()):
        local = torch.unique(torch.nonzero(bad)[:, 0])
        where = rows[local][:16].tolist() if rows is not None else local[:16].tolist()
        raise AssertionError(f"{label}: {int(bad.sum())} elements differ, rows {where}")


# ---- sparse structure -------------------------------------------------------------------------------------------------
def make_csr(n_rows, n_cols, heavy_rows, seed, tail_cols):
    """Degrees uniform in [1, 2 AVG_DEG), the ``heavy_rows`` with ``HEAVY`` entries, columns uniform in
    ``[0, n_cols)`` and every 1009th entry one of ``tail_cols`` (the last rows of the gather table)."""
    g = _gen(seed)
    deg = torch.randint(1, 2 * AVG_DEG, (n_rows,), generator=g, device=_dev())
    deg[torch.tensor(heavy_rows, device=_dev())] = HEAVY
    indptr = torch.zeros(n_rows + 1, dtype=torch.int64, device=_dev())
    indptr[1:] = torch.cumsum(deg, 0)
    nnz = int(indptr[-1])
    idx = torch.randint(0, n_cols, (nnz,), generator=g, device=_dev(), dtype=torch.int32)
    t = torch.as_tensor(tail_cols, dtype=torch.int32, device=_dev())
    sl = idx[::1009]
    sl.copy_(t[torch.arange(sl.numel(), device=_dev()) % t.numel()])
    return indptr, idx


def entries_of(indptr, rows):
    """``(owner, pos)``: for the entries of ``rows`` (in CSR order), the index into ``rows`` and the CSR position."""
    s, e = indptr[rows], indptr[rows + 1]
    cnt = e - s
    owner = torch.repeat_interleave(torch.arange(rows.numel(), device=rows.device), cnt)
    first = torch.repeat_interleave(torch.cumsum(cnt, 0) - cnt, cnt)
    pos = torch.arange(owner.numel(), device=rows.device) - first + torch.repeat_interleave(s, cnt)
    return owner, pos


def check_structure(g, gt, indptr, idx, trows):
    """Exact integer checks of ``bns_graph_create`` / ``bns_graph_transpose``: the copied CSR, the chunk and split-row
    counts of both (a row without entries has one chunk), the transpose's row lengths = column counts, and on the
    transpose's rows ``trows``: every entry's permutation points at a source entry of that column, its id is that
    entry's row, in source order."""
    ip, ix = g.csr()
    assert torch.equal(ip, indptr) and torch.equal(ix, idx), "bns_graph_copy_csr"
    del ip, ix
    for h, ptr in ((g, indptr), (gt, None)):
        if ptr is None:
            ptr = gt.csr()[0]
            assert int(ptr[-1]) == idx.numel()
            assert torch.equal(ptr[1:] - ptr[:-1], torch.bincount(idx.long(), minlength=g.n_cols)), "transpose row lengths"
        deg = ptr[1:] - ptr[:-1]
        assert h.n_chunks == int(((deg + 255) // 256).clamp(min=1).sum()), "chunk count"
        assert h.n_split_rows == int((deg > 256).sum()), "split-row count"
    ipT, ixT = gt.csr()
    perm = gt.perm()
    owner, pos = entries_of(ipT, trows)
    src = perm[pos].long()
    assert torch.equal(idx[src].long(), trows[owner]), "transpose: perm points at an entry of another column"
    src_row = torch.searchsorted(indptr, src, right=True) - 1
    assert torch.equal(ixT[pos].long(), src_row), "transpose: row id differs from the source entry's row"
    same = owner[1:] == owner[:-1]
    assert bool((src[1:][same] > src[:-1][same]).all()), "transpose: entries of a column not in source order"


def spmm_reference(indptr, indices, rows, x, xrow=None, col_scale=None, row_scale=None, y0=None, max_entries=1 << 20):
    """float64 ``(ref, bound)`` of ``y[r] = y0[r] + row_scale[r] * sum_k col_scale[c_k] x[xrow(c_k)]`` for ``rows``
    (entries whose ``xrow`` is negative skipped); bound = the same over absolute values."""
    n = rows.numel()
    ref = torch.zeros(n, x.shape[1], dtype=torch.float64, device=x.device)
    bnd = torch.zeros_like(ref)
    deg = (indptr[rows + 1] - indptr[rows]).cpu()
    i0 = 0
    while i0 < n:
        i1, tot = i0, 0
        while i1 < n and (i1 == i0 or tot + int(deg[i1]) <= max_entries):
            tot += int(deg[i1])
            i1 += 1
        owner, pos = entries_of(indptr, rows[i0:i1])
        c = indices[pos].long()
        xr = c if xrow is None else xrow(c)
        live = xr >= 0
        owner, c, xr = owner[live], c[live], xr[live]
        v = x[xr].double()
        if col_scale is not None:
            v *= col_scale[c].double()[:, None]
        ref[i0:i1].index_add_(0, owner, v)
        bnd[i0:i1].index_add_(0, owner, v.abs())
        i0 = i1
    if row_scale is not None:
        rs = row_scale[rows].double()[:, None]
        ref *= rs
        bnd *= rs.abs()
    if y0 is not None:
        ref += y0.double()
        bnd += y0.double().abs()
    return ref, bnd


# ---- SpMM over a plain matrix, source-row blocked, the transpose ---------------------------------------------------
def test_spmm_f32_plain_blocked_and_transposed(built, monkeypatch):
    """Layer 0's aggregation over the inner + sampled-halo gather table (23.6 M rows, past 2^32 elements) into 13.9 M
    output rows (past 2^31), heavy rows of 100,000 entries (~390 chunks: partial sums + fix-up), entries at the last
    table rows; with row scale, column scale and ``accumulate``, then through two forced source-row blocks
    (``BNS_SPMM_COLBLOCKS``), then the backward's transposed pass with a row map into a 23.6 M-row output.  The
    transpose's CSR, entry permutation and chunk counts are checked exactly on sampled rows."""
    from bns_gcn_b200 import ops
    _need(58)
    C = N_IN + N_SAMP
    assert C * LD > 1 << 32 and N_IN * LD > 1 << 31
    worst = {}
    heavy = [0, (1 << 31) // LD, N_IN // 2 + 7, N_IN - 1]
    tail = list(range(C - 16, C))
    indptr, idx = make_csr(N_IN, C, heavy, seed=1, tail_cols=tail)
    nnz = idx.numel()
    assert nnz > 180_000_000, nnz
    g = ops.DeviceGraph.from_csr(indptr, idx, C)
    deg = indptr[1:] - indptr[:-1]
    assert g.n_chunks == int(((deg + 255) // 256).sum()) and g.n_split_rows == int((deg > 256).sum())
    gen = _gen(2)
    x = _operand(C, F, LD, _fill_randn(gen, scale_rows=True))
    rs = torch.rand(N_IN, generator=gen, device=_dev()) + 0.5
    cs = torch.rand(C, generator=gen, device=_dev()) + 0.5
    rows = sample_rows(N_IN, lds=(LD,), extra=heavy, seed=3)

    # (a) spmm_auto, one block: out = y0 + rs * A (cs * x)
    buf, y = _output(N_IN, F, LD)
    _fill_randn(gen)(y)
    y0 = y[rows].clone()
    assert ops.plan_col_blocks(g, F) == 1
    ops.spmm_auto(g, x, y, row_scale=rs, col_scale=cs, accumulate=True)
    ref, bnd = spmm_reference(indptr, idx, rows, x, col_scale=cs, row_scale=rs, y0=y0)
    _close(worst, "spmm f32 rs+cs+accumulate", "spmm f32 rs+cs+accumulate", y[rows], ref, bnd, rows)
    _untouched(buf, N_IN, F, "spmm f32 rs+cs+accumulate")

    # (b) forced source-row blocks, fresh output
    monkeypatch.setenv("BNS_SPMM_COLBLOCKS", "2")
    assert ops.plan_col_blocks(g, F) == 2
    buf.view(torch.int32).fill_(SENTINEL)
    ops.spmm_auto(g, x, y, row_scale=rs)
    monkeypatch.delenv("BNS_SPMM_COLBLOCKS")
    ref, bnd = spmm_reference(indptr, idx, rows, x, row_scale=rs)
    _close(worst, "spmm f32 two source-row blocks", "spmm f32 blocks", y[rows], ref, bnd, rows)
    _untouched(buf, N_IN, F, "spmm f32 blocks")
    g.__dict__.pop("_col_blocks", None)

    # (c) the transpose: exact structure on sampled rows, then dX[row_map[c]] = sum_r A[r, c] dY[r]
    gt = g.transpose()
    trows = sample_rows(C, lds=(LD,), extra=tail, seed=4)
    check_structure(g, gt, indptr, idx, trows)
    obuf = torch.as_strided(x, (C + 3, LD), (LD, 1))  # the table's memory becomes the output (view at offset 0)
    del x
    torch.cuda.empty_cache()
    obuf.view(torch.int32).fill_(SENTINEL)
    out = obuf[:C, :F]
    gen = _gen(5)
    y.normal_(generator=gen)                          # dY
    row_map = torch.randperm(C, generator=gen, device=_dev()).to(torch.int32)
    skip = torch.rand(C, generator=gen, device=_dev()) < 0.1
    skip[torch.tensor(tail, device=_dev())] = False
    row_map[skip] = -1
    ops.spmm(gt, y, out, row_map=row_map, n_out_rows=C)
    orows = row_map[trows].long()
    live = orows >= 0
    ipT, ixT = gt.csr()
    ref, bnd = spmm_reference(ipT, ixT, trows[live], y)
    _close(worst, "spmm f32 transposed, row-mapped", "spmm f32 transposed", out[orows[live]], ref, bnd, trows[live])
    skipped_out = torch.ones(C, dtype=torch.bool, device=_dev())
    skipped_out[row_map[row_map >= 0].long()] = False
    srows = torch.nonzero(skipped_out)[:, 0][:N_RANDOM_ROWS]
    assert bool((obuf[srows].view(torch.int32) == SENTINEL).all()), "transposed pass wrote rows no entry maps to"
    _untouched(obuf, C, F, "spmm f32 transposed")
    _report(worst)


# ---- the column-mapped halo form, its compaction, the bf16 table ------------------------------------------------------
def test_spmm_halo_col_map_compact_and_bf16(built):
    """A [13.9 M, 13.9 M + 97 M] with halo columns mapped through ``slot`` (built by ``halo_slot_update`` over 97 M
    halo nodes, checked exactly) into a 9.7 M-row slab after the inner rows: ``spmm`` with ``col_map`` / ``n_direct``
    and column scale, ``CompactedCols.refresh`` + ``spmm_compact`` (bit-identical to it), then the same table in bf16
    (``cvt_rows_bf16``, bit-exact against torch on the sampled rows; 23.6 M x 264 bf16 elements, past 2^32 and 8 GiB)
    through ``spmm`` and ``spmm_compact``."""
    from bns_gcn_b200 import ops
    _need(58)
    n_cols = N_IN + N_HALO
    C = N_IN + N_SAMP
    assert n_cols < 2 ** 31 - 1 and C * LD > 1 << 32
    worst = {}
    gen = _gen(11)
    # slot[h] = N_IN + k for the k-th sampled halo node (one_hops in the order a peer sent them), else -1
    one_hops = torch.randperm(N_HALO, generator=gen, device=_dev())[:N_SAMP]
    pos = torch.arange(N_HALO, device=_dev()) + N_IN          # owner-local id -> my local id (identity peer here)
    slot = torch.empty(N_HALO, dtype=torch.int32, device=_dev())
    ops.fill_i32(slot, -1)
    ops.halo_slot_update(pos, one_hops, N_IN, N_IN, slot)
    want = torch.full((N_HALO,), -1, dtype=torch.int32, device=_dev())
    want[one_hops] = (N_IN + torch.arange(N_SAMP, device=_dev())).to(torch.int32)
    assert torch.equal(slot, want), "halo_slot_update"
    del want, pos
    top = one_hops[-16:] + N_IN                                # halo columns whose rows are the last slab rows
    heavy = [0, (1 << 31) // LD, N_IN - 1]
    indptr, idx = make_csr(N_IN, n_cols, heavy, seed=12, tail_cols=top.tolist())
    g = ops.DeviceGraph.from_csr(indptr, idx, n_cols)
    x = _operand(C, F, LD, _fill_randn(gen))
    cs = torch.rand(n_cols, generator=gen, device=_dev()) + 0.5
    rs = torch.rand(N_IN, generator=gen, device=_dev()) + 0.5
    rows = sample_rows(N_IN, lds=(LD,), extra=heavy, seed=13)

    def xrow(c):
        h = (c - N_IN).clamp_(min=0)
        return torch.where(c < N_IN, c, slot[h].long())

    buf, y = _output(N_IN, F, LD)
    ops.spmm(g, x, y, row_scale=rs, col_scale=cs, col_map=slot, n_direct=N_IN)
    ref, bnd = spmm_reference(indptr, idx, rows, x, xrow=xrow, col_scale=cs, row_scale=rs)
    _close(worst, "spmm f32 col_map", "spmm f32 col_map", y[rows], ref, bnd, rows)
    _untouched(buf, N_IN, F, "spmm f32 col_map")
    y_map = y[rows].clone()

    cc = ops.CompactedCols(g, with_weights=True)
    cc.refresh(slot, n_direct=N_IN, col_scale=cs)
    buf.view(torch.int32).fill_(SENTINEL)
    ops.spmm_compact(cc, x, y, row_scale=rs)
    _bits_equal("spmm_compact f32 vs col_map", y[rows], y_map, rows)
    _close(worst, "spmm f32 compact", "spmm f32 compact", y[rows], ref, bnd, rows)
    _untouched(buf, N_IN, F, "spmm f32 compact")
    del ref, bnd, y_map

    # bf16 table: NaN (0x7FC0) in the pad columns and rows
    ldb = F + 8
    xh_buf = torch.full((C + 3, ldb), 0x7FC0, dtype=torch.int16, device=_dev()).view(torch.bfloat16)
    xh = xh_buf[:C, :F]
    ops.cvt_rows_bf16(x, xh)
    assert C * ldb > 1 << 32
    xrows = sample_rows(C, lds=(ldb, LD), extra=range(C - 16, C), seed=14)
    _bits_equal("cvt_rows_bf16", xh[xrows], x[xrows].to(torch.bfloat16), xrows)
    assert bool((xh_buf[:, F:].view(torch.int16) == 0x7FC0).all()) and bool((xh_buf[C:].view(torch.int16) == 0x7FC0).all()), \
        "cvt_rows_bf16 wrote outside its view"
    del x, buf, y
    torch.cuda.empty_cache()
    xf = xh                                                       # reference input: the bf16 values, exact in f64
    buf, y = _output(N_IN, F, LD)
    ops.spmm(g, xh, y, row_scale=rs, col_scale=cs, col_map=slot, n_direct=N_IN)
    ref, bnd = spmm_reference(indptr, idx, rows, xf, xrow=xrow, col_scale=cs, row_scale=rs)
    _close(worst, "spmm bf16 col_map", "spmm bf16 col_map", y[rows], ref, bnd, rows)
    _untouched(buf, N_IN, F, "spmm bf16 col_map")
    y_map = y[rows].clone()
    buf.view(torch.int32).fill_(SENTINEL)
    ops.spmm_compact(cc, xh, y, row_scale=rs)
    _bits_equal("spmm_compact bf16 vs col_map", y[rows], y_map, rows)
    _untouched(buf, N_IN, F, "spmm bf16 compact")
    _report(worst)


# ---- dense ------------------------------------------------------------------------------------------------------------
def _tn(a, b, out, bias=None, addend=None, row_scale=None):
    lib = _lib()
    _check_rc(lib.bns_dense_tn_3xtf32(a.data_ptr(), a.stride(0), b.data_ptr(), b.stride(0),
                                      None if bias is None else bias.data_ptr(),
                                      None if addend is None else addend.data_ptr(),
                                      0 if addend is None else addend.stride(0),
                                      None if row_scale is None else row_scale.data_ptr(), out.data_ptr(), out.stride(0),
                                      a.shape[0], b.shape[0], a.shape[1], _stream()), "bns_dense_tn_3xtf32")


def test_dense_tn_13m_rows(built):
    """``bns_dense_tn_3xtf32`` with M = 13.9 M, K = 256: N = 256 with bias, the addend aliasing the output (the
    input-gradient accumulation) and row_scale; N = 44 with bias, a separate addend and row_scale.  Output rows past
    8.26 M (2^31 / 260) must be right."""
    _need(36)
    M, K = N_IN, F
    assert M * LD > 1 << 31 and M < 2 ** 31
    worst = {}
    gen = _gen(21)
    a = _operand(M, K, LD, _fill_randn(gen, scale_rows=True))
    rows = sample_rows(M, lds=(LD,), seed=22)
    rs = torch.randn(M, generator=gen, device=_dev())
    for N in (256, 44):
        b = _operand(N, K, K + 4, _fill_randn(gen))
        bias = torch.randn(N + 4, generator=gen, device=_dev())[:N]
        ldc = N + 4
        buf, out = _output(M, N, ldc)
        if N == 256:
            _fill_randn(gen)(out)
            add0 = out[rows].clone()
            _tn(a, b, out, bias=bias, addend=out, row_scale=rs)
            label = f"TN M={M} N={N} bias + addend in place + row_scale"
        else:
            add = _operand(M, N, N + 8, _fill_randn(gen))
            add0 = add[rows].clone()
            _tn(a, b, out, bias=bias, addend=add, row_scale=rs)
            label = f"TN M={M} N={N} bias + addend + row_scale"
        ad, bd = a[rows].double(), b.double()
        ref = (ad @ bd.t() + bias.double() + add0.double()) * rs[rows].double()[:, None]
        bnd = (ad.abs() @ bd.abs().t() + bias.double().abs() + add0.double().abs()) * rs[rows].double().abs()[:, None]
        _close(worst, label, label, out[rows], ref, bnd, rows)
        _untouched(buf, M, N, label)
        del buf, out
        torch.cuda.empty_cache()
    _report(worst)


def _nt(a, b, out, ws):
    lib = _lib()
    R_, N1 = a.shape
    N2 = b.shape[1]
    need = lib.bns_dense_nt_workspace_bytes(R_, N1, N2)
    _check_rc(lib.bns_dense_nt_3xtf32(a.data_ptr(), a.stride(0), b.data_ptr(), b.stride(0), out.data_ptr(), out.stride(0),
                                      R_, N1, N2, ws.data_ptr(), need, _stream()), "bns_dense_nt_3xtf32")


def test_weight_and_bias_gradients_13m_rows(built):
    """``bns_dense_nt_3xtf32`` dW = dY^T X over R = 13.9 M rows (N1 x N2 = 256 x 256 and 256 x 44), every element of
    dW, all operands positive so that the bound is |dW| and the ratio is the kernel's real error over TOL; the slice
    count (~9,000: chains of at most 48 k-blocks, summed by ``splitk_reduce_kernel``) asserted from
    ``bns_dense_nt_workspace_bytes``.  ``bns_colsum_f32`` of the same dY over 13.9 M rows, every column."""
    lib = _lib()
    _need(36)
    R_ = N_IN
    worst = {}
    gen = _gen(31)
    a = _operand(R_, F, LD, _fill_positive(gen))
    b = _operand(R_, F, LD, _fill_positive(gen))
    nkb = (R_ + 31) // 32
    for N2 in (256, 44):
        bb = b[:, :N2]
        if N2 < F:
            b[:, N2:N2 + 4].fill_(float("nan"))           # NaN right after the narrower operand's row
        need = lib.bns_dense_nt_workspace_bytes(R_, F, N2)
        splits = need // (4 * F * N2)
        # a contraction this long is cut into chains of at most 48 k-blocks (more than kTwoLevelSlices = 1,024 slices)
        assert splits >= (nkb + 47) // 48 and splits > 1024, (splits, nkb)
        ws = torch.full((need // 4 + 128 * N2,), float("nan"), device=_dev())
        buf, out = _output(F, N2, N2 + 4)
        _nt(a, bb, out, ws)
        ref = torch.zeros(F, N2, dtype=torch.float64, device=_dev())
        for r0 in range(0, R_, 1 << 19):
            ref += a[r0:r0 + (1 << 19)].double().t() @ bb[r0:r0 + (1 << 19)].double()
        label = f"NT R={R_} N1={F} N2={N2} splits={splits} (positive: ratio = relative error / TOL)"
        # where the error comes from: the slices themselves (tensor-core chains) or their f32 sum (splitk_reduce)
        parts = ws[:need // 4].view(splits, F, N2)
        psum = torch.zeros(F, N2, dtype=torch.float64, device=_dev())
        for s0 in range(0, splits, 512):
            psum += parts[s0:s0 + 512].double().sum(0)
        print(f"[nt-error] {label}: slices {((psum - ref).abs() / ref).max().item():.3g}, "
              f"reduce {((out.double() - psum).abs() / ref).max().item():.3g} (max relative)")
        _close(worst, label, label, out, ref, ref)
        _untouched(buf, F, N2, label)
        assert bool(ws[need // 4:].isnan().all()), f"{label}: stores past the workspace's slices"
        print(f"[splits] NT (R, N1, N2) = ({R_}, {F}, {N2}): {splits} slices over {nkb} k-blocks")
        del ws, buf, out
        torch.cuda.empty_cache()
    # colsum over the same 13.9 M rows
    need = lib.bns_colsum_workspace_bytes(F)
    ws = torch.full((need // 4 + 64,), float("nan"), device=_dev())
    bufs = [_output(1, F, F + 4) for _ in range(2)]
    _check_rc(lib.bns_colsum_f32(a.data_ptr(), a.stride(0), R_, F, bufs[0][1].data_ptr(), bufs[1][1].data_ptr(),
                                 ws.data_ptr(), need, _stream()), "bns_colsum_f32")
    ref = torch.zeros(F, dtype=torch.float64, device=_dev())
    for r0 in range(0, R_, 1 << 21):
        ref += a[r0:r0 + (1 << 21)].double().sum(0)
    for k, (buf, out) in enumerate(bufs):
        label = f"colsum rows={R_} cols={F} out{k + 1} (positive: ratio = relative error / TOL)"
        _close(worst, "colsum", label, out[0], ref, ref)
        _untouched(buf, 1, F, label)
    _report(worst)


# ---- row-wise kernels -------------------------------------------------------------------------------------------------
EPS = 1e-5
P_DROP = 0.5
SEED = (1 << 40) + 12345
OFFSET = (1 << 33) + 7


def keep_mask_np(seed, offset, rows, Fw, p):
    """bool ``[len(rows), Fw]`` keep mask of ``drop_mask4`` for the given rows, from ``oracle.philox`` (numpy)."""
    from oracle.philox import philox4x32_10
    nv = (Fw + 3) // 4
    r = rows.cpu().numpy().astype(np.uint64)
    rr = np.broadcast_to(r[:, None], (r.size, nv))
    vec = np.broadcast_to(np.arange(nv, dtype=np.uint64)[None, :], (r.size, nv))
    m = np.uint64(0xFFFFFFFF)
    out = philox4x32_10((rr & m).astype(np.uint32), ((rr >> np.uint64(32)) ^ ((vec << np.uint64(8)) & m)).astype(np.uint32),
                        np.full(rr.shape, offset & 0xFFFFFFFF, dtype=np.uint32),
                        np.full(rr.shape, offset >> 32, dtype=np.uint32), seed & 0xFFFFFFFF, seed >> 32)
    u = np.stack(out, -1).astype(np.float32) * np.float32(2.0 ** -32)
    return torch.from_numpy((u >= np.float32(p)).reshape(r.size, 4 * nv)[:, :Fw].copy()).to(_dev())


def test_row_wise_kernels_13m_rows(built):
    """``bns_ln_relu_dropout_fwd_f32`` / ``bwd_f32`` at 13.9 M x 256, p = 0.5: y, dx and the mask on sampled rows (the
    mask against ``oracle.philox``, rows above 2^23 included); dgamma / dbeta in full against a float64 sum over every
    row (mask = where the forward's y is non-zero, itself checked on the sampled rows).  Then ``bns_dropout_f32`` and
    ``bns_scale_rows_f32`` at the same size."""
    lib = _lib()
    _need(50)
    n = N_IN
    assert n * LD > 1 << 31 and n > 1 << 23
    worst = {}
    gen = _gen(41)
    x = _operand(n, F, LD, _fill_randn(gen))
    x[::7].add_(3.0)
    gamma = torch.rand(F, generator=gen, device=_dev()) + 0.5
    beta = torch.randn(F, generator=gen, device=_dev()) * 0.3
    rows = sample_rows(n, lds=(LD,), extra=(1 << 23, (1 << 23) + 1, (1 << 24) - 1), seed=42)
    ks = float(np.float32(1.0) / (np.float32(1.0) - np.float32(P_DROP)))
    keep = keep_mask_np(SEED, OFFSET, rows, F, P_DROP)

    ybuf, y = _output(n, F, LD)
    mean = torch.empty(n, device=_dev())
    rstd = torch.empty(n, device=_dev())
    _check_rc(lib.bns_ln_relu_dropout_fwd_f32(x.data_ptr(), x.stride(0), n, F, gamma.data_ptr(), beta.data_ptr(), EPS,
                                              P_DROP, SEED, OFFSET, None, y.data_ptr(), y.stride(0), mean.data_ptr(),
                                              rstd.data_ptr(), _stream()), "bns_ln_relu_dropout_fwd_f32")
    _untouched(ybuf, n, F, "ln fwd")
    gd, bd = gamma.double(), beta.double()
    xd = x[rows].double()
    xc = xd - xd.mean(1, keepdim=True)
    rsd = ((xc * xc).mean(1, keepdim=True) + EPS).rsqrt()
    xh = xc * rsd
    z = xh * gd + bd
    a_ = xh.abs() + rsd * xd.abs().mean(1, keepdim=True)
    bz = gd.abs() * a_ + bd.abs()
    yk = y[rows]
    act = (yk != 0) | ((z > 0) & ~keep)
    flip = (act != (z > 0)) & keep
    assert bool((z[flip].abs() <= R.TOL * bz[flip]).all()), "ln fwd: a ReLU side differs from float64 beyond the margin"
    assert not bool(((yk != 0) & ~keep).any()), "ln fwd: an element the Philox mask drops is non-zero"
    m = (act & keep).double() * ks
    _close(worst, "ln fwd y", "ln fwd y", yk, z * m, bz * keep.double() * ks, rows)
    ynz = y != 0                                                # the forward's kept, active set (bool, 3.6 GB)
    del ybuf, y, yk
    torch.cuda.empty_cache()

    dy = _operand(n, F, LD, _fill_randn(gen))
    dxbuf, dx = _output(n, F, LD)
    dgamma = torch.full((F,), float("nan"), device=_dev())
    dbeta = torch.full((F,), float("nan"), device=_dev())
    ws = torch.empty(lib.bns_ln_bwd_workspace_bytes(F), dtype=torch.uint8, device=_dev())
    _check_rc(lib.bns_ln_relu_dropout_bwd_f32(dy.data_ptr(), dy.stride(0), x.data_ptr(), x.stride(0), n, F,
                                              gamma.data_ptr(), beta.data_ptr(), mean.data_ptr(), rstd.data_ptr(), EPS,
                                              P_DROP, SEED, OFFSET, None, dx.data_ptr(), dx.stride(0), dgamma.data_ptr(),
                                              dbeta.data_ptr(), ws.data_ptr(), ws.numel(), _stream()),
              "bns_ln_relu_dropout_bwd_f32")
    _untouched(dxbuf, n, F, "ln bwd")
    g_ = dy[rows].double() * m
    gz = g_ * gd
    agz = gz.abs()
    want = rsd * (gz - gz.mean(1, keepdim=True) - xh * (gz * xh).mean(1, keepdim=True))
    bound = rsd * (agz + agz.mean(1, keepdim=True) + xh.abs() * (agz * a_).mean(1, keepdim=True)
                   + a_ * (agz * xh.abs()).mean(1, keepdim=True))
    _close(worst, "ln bwd dx", "ln bwd dx", dx[rows], want, bound, rows)
    sums = torch.zeros(4, F, dtype=torch.float64, device=_dev())
    ch = 1 << 18
    for r0 in range(0, n, ch):
        xd = x[r0:r0 + ch].double()
        xc = xd - xd.mean(1, keepdim=True)
        rsd = ((xc * xc).mean(1, keepdim=True) + EPS).rsqrt()
        xh = xc * rsd
        a_ = xh.abs() + rsd * xd.abs().mean(1, keepdim=True)
        g_ = dy[r0:r0 + ch].double() * (ynz[r0:r0 + ch].double() * ks)
        sums += torch.stack([(g_ * xh).sum(0), (g_.abs() * a_).sum(0), g_.sum(0), g_.abs().sum(0)])
    _close(worst, "ln bwd dgamma (13.9 M rows)", "ln bwd dgamma", dgamma, sums[0], sums[1])
    _close(worst, "ln bwd dbeta (13.9 M rows)", "ln bwd dbeta", dbeta, sums[2], sums[3])
    del dy, ynz, xd, xc, g_
    torch.cuda.empty_cache()

    # layer 0's input dropout: y = x * keep * (1 / (1 - p)) exactly, one multiply
    dxbuf.view(torch.int32).fill_(SENTINEL)
    _check_rc(lib.bns_dropout_f32(x.data_ptr(), x.stride(0), n, F, P_DROP, SEED, OFFSET, None, dx.data_ptr(),
                                  dx.stride(0), _stream()), "bns_dropout_f32")
    _untouched(dxbuf, n, F, "dropout")
    xs = x[rows]
    _bits_equal("dropout", dx[rows], torch.where(keep, xs * ks, torch.zeros_like(xs)), rows)
    # y = x * row_scale + bias
    dxbuf.view(torch.int32).fill_(SENTINEL)
    rs = torch.randn(n, generator=gen, device=_dev())
    bias = torch.randn(F, generator=gen, device=_dev())
    _check_rc(lib.bns_scale_rows_f32(x.data_ptr(), x.stride(0), n, F, rs.data_ptr(), bias.data_ptr(), dx.data_ptr(),
                                     dx.stride(0), _stream()), "bns_scale_rows_f32")
    _untouched(dxbuf, n, F, "scale_rows")
    xd = xs.double()
    r_ = rs[rows].double()[:, None]
    _close(worst, "scale_rows", "scale_rows", dx[rows], xd * r_ + bias.double(), (xd * r_).abs() + bias.double().abs(),
           rows)
    _report(worst)


def test_xent_13m_rows(built):
    """``bns_xent_f32`` over 13.9 M rows, C = 172 (ld 176), a 1.1 % train mask: the loss against a float64 sum over
    every train row, d(logits) on sampled rows (train rows among them) against float64, zeros on unmasked rows and in
    the pad columns, nothing written past them."""
    lib = _lib()
    _need(24)
    n, C = N_IN, N_CLASS
    ld, cp = 176, 176                    # logits row, dlogits row: 172 classes padded to a multiple of 4
    assert n * ld > 1 << 31
    worst = {}
    gen = _gen(51)
    logits = _operand(n, C, ld, lambda v: [v[r0:r0 + (1 << 22)].normal_(generator=gen).mul_(3.0)
                                           for r0 in range(0, n, 1 << 22)])
    labels = torch.randint(0, C, (n,), generator=gen, device=_dev())
    mask = torch.rand(n, generator=gen, device=_dev()) < TRAIN_FRAC
    mask[n - 1] = True
    train = torch.nonzero(mask)[:, 0]
    n_train = train.numel()
    scale = 1.0 / n_train
    buf, dl = _output(n, cp, cp + 4)
    loss = torch.full((1,), float("nan"), device=_dev())
    ws = torch.zeros(lib.bns_xent_workspace_bytes(), dtype=torch.uint8, device=_dev())
    _check_rc(lib.bns_xent_f32(logits.data_ptr(), logits.stride(0), n, C, labels.data_ptr(), None, 0,
                               mask.view(torch.uint8).data_ptr(), scale, loss.data_ptr(), dl.data_ptr(), dl.stride(0), cp,
                               ws.data_ptr(), ws.numel(), _stream()), "bns_xent_f32")
    _untouched(buf, n, cp, "xent")
    ref = torch.zeros((), dtype=torch.float64, device=_dev())
    for i0 in range(0, n_train, 1 << 16):
        t = train[i0:i0 + (1 << 16)]
        lp = torch.log_softmax(logits[t].double(), 1)
        ref -= lp.gather(1, labels[t][:, None]).sum()
    _close(worst, "xent loss", f"xent loss over {n_train} train rows of {n}", loss[0], ref, ref.abs())
    rng = torch.Generator().manual_seed(52)
    extra = train[torch.randint(0, n_train, (N_RANDOM_ROWS,), generator=rng).to(_dev())].tolist()
    rows = sample_rows(n, lds=(ld, cp + 4), extra=extra + [int(train[-1])], seed=53)
    sm = torch.softmax(logits[rows].double(), 1)
    onehot = torch.zeros_like(sm).scatter_(1, labels[rows][:, None], 1.0)
    mk = mask[rows].double()[:, None]
    want = (sm - onehot) * scale * mk
    bound = (sm + onehot) * scale * mk
    _close(worst, "xent dlogits", "xent dlogits", dl[rows, :C], want, bound, rows)
    assert bool((dl[rows][~mask[rows]] == 0).all()), "xent: an unmasked row's gradient is not 0"
    assert bool((dl[rows, C:] == 0).all()), "xent: a pad column's gradient is not 0"
    _report(worst)


# ---- exchange ---------------------------------------------------------------------------------------------------------
def test_gather_scatter_13m_rows(built):
    """``gather_div`` / ``scatter_add_div`` with selected ids in the last rows of a 13.9 M x 256 matrix (and around the
    2^31-element rows), exact: one f32 division (and one addition) per element.  ``bns_scatter_rows_all_f32`` with
    two segments whose inverse maps cover the last rows."""
    import ctypes
    from bns_gcn_b200 import ops
    lib = _lib()
    _need(34)
    n = N_IN
    assert n * LD > 1 << 31
    gen = _gen(61)
    h = _operand(n, F, LD, _fill_randn(gen))
    base = sample_rows(n, lds=(LD,), extra=range(n - 2048, n), seed=62, k=0)
    idx = torch.unique(torch.cat([base, torch.randperm(n, generator=gen, device=_dev())[:200_000]]))
    idx = idx[torch.randperm(idx.numel(), generator=gen, device=_dev())]
    k = idx.numel()
    div = 3.0
    obuf, out = _output(k, F, LD)
    ops.gather_div(h, idx, div, out)
    _untouched(obuf, k, F, "gather_div")
    # the f32 quotient, correctly rounded (torch multiplies by the reciprocal when dividing by a scalar)
    q = lambda t, d: (t.double() / d).float()                   # noqa: E731
    _bits_equal("gather_div", out, q(h[idx], div), idx)
    h0 = h[idx].clone()
    ops.scatter_add_div(h, idx, out, div)
    _bits_equal("scatter_add_div", h[idx], h0 + q(out, div), idx)
    assert bool((torch.as_strided(h, (n + 3, LD), (LD, 1))[:, F:].isnan()).all()), "scatter_add_div wrote a pad column"
    del obuf, out, h0
    # scatter_rows_all: G[r] += recv_s[inv_s[r]] / div_s, segment 0 then 1
    G = h
    segs = []
    for s_ in range(2):
        sel = idx[s_::2]
        inv = torch.full((n,), -1, dtype=torch.int32, device=_dev())
        inv[sel] = torch.arange(sel.numel(), device=_dev(), dtype=torch.int32)
        recv = torch.randn(sel.numel(), LD, generator=gen, device=_dev())
        segs.append((sel, inv, recv, 2.0 + s_))
    probe = torch.unique(torch.cat([idx, sample_rows(n, lds=(LD,), seed=63)]))
    g0 = G[probe].clone()
    ip = (ctypes.c_void_p * 2)(*[s[1].data_ptr() for s in segs])
    rp = (ctypes.c_void_p * 2)(*[s[2].data_ptr() for s in segs])
    dv = (ctypes.c_float * 2)(*[s[3] for s in segs])
    _check_rc(lib.bns_scatter_rows_all_f32(G.data_ptr(), G.stride(0), n, F, 2, ip, rp, LD, dv, _stream()),
              "bns_scatter_rows_all_f32")
    want = g0.clone()
    for sel, inv, recv, d in segs:
        i = inv[probe].long()
        hit = i >= 0
        want[hit] = want[hit] + q(recv[i[hit], :F], d)
    _bits_equal("scatter_rows_all", G[probe], want, probe)
    gb = torch.as_strided(G, (n + 3, LD), (LD, 1))
    assert bool(gb[:, F:].isnan().all()) and bool(gb[n:].isnan().all()), "scatter_rows_all wrote outside G's view"


def _dev_view(ptr, n, typestr):
    from bns_gcn_b200.helper.feature_buffer import _DevArray
    return torch.as_tensor(_DevArray(ptr, (n,), typestr), device=_dev())


def test_p2p_put_all_past_4gib(built):
    """``bns_p2p_put_all_f32`` from rank 0 into rank 1 (two in-process ranks on one GPU) with a 4.06 GiB receive slab:
    one segment whose rows straddle the 4 GiB byte offset, one at ``remote_off`` past 4 GiB, rows gathered from the
    last rows of a 13.9 M x 256 matrix.  Every written word is exact (one f32 division); every other word of the slab
    keeps its sentinel."""
    import ctypes
    from bns_gcn_b200._lib import PutAll
    lib = _lib()
    _need(24)
    n = N_IN
    slab_bytes = (1 << 32) + (64 << 20)
    ps = []
    for rank, nb in ((0, 1 << 20), (1, slab_bytes)):
        h = ctypes.c_void_p()
        _check_rc(lib.bns_p2p_create(ctypes.byref(h), rank, 2, nb, 4), "bns_p2p_create")
        slab, flags, got = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_size_t()
        _check_rc(lib.bns_p2p_local(h, ctypes.byref(slab), ctypes.byref(flags), ctypes.byref(got)), "bns_p2p_local")
        ps.append((h, slab.value, flags.value, got.value))
    try:
        (h0, _, _, _), (h1, slab1, flags1, nb1) = ps
        assert nb1 >= slab_bytes
        _check_rc(lib.bns_p2p_set_peer(h0, 1, slab1, flags1, nb1), "bns_p2p_set_peer")
        words = _dev_view(slab1, nb1 // 4, "<i4")
        words.fill_(SENTINEL)
        fl = _dev_view(flags1, 4, "<i8")
        fl.zero_()
        gen = _gen(71)
        hm = _operand(n, F, LD, _fill_randn(gen))
        row = LD * 4
        k0, k1 = 4000, 3000
        off0 = (1 << 32) - 1000 * row                      # rows 1000.. of this segment lie past 4 GiB
        off1 = (1 << 32) + (16 << 20) + 16
        assert off1 + k1 * row <= nb1 and off0 + k0 * row > 1 << 32
        idx = torch.cat([torch.arange(n - k0, n, device=_dev()),
                         torch.randperm(n, generator=gen, device=_dev())[:k1]])
        s = PutAll()
        s.n_seg = 2
        s.row_begin[0], s.row_begin[1], s.row_begin[2] = 0, k0, k0 + k1
        for i_, (off, d) in enumerate(((off0, 3.0), (off1, 0.7))):
            s.peer[i_], s.remote_off[i_], s.src_begin[i_], s.div[i_] = 1, off, 0, d
        _check_rc(lib.bns_p2p_put_all_f32(h0, ctypes.byref(s), LD, hm.data_ptr(), hm.stride(0), F, idx.data_ptr(), 1, 2,
                                          5, None, _stream()), "bns_p2p_put_all_f32")
        torch.cuda.synchronize()
        assert int(fl[1]) == 5, "the flag was not published"
        written = torch.zeros(nb1 // 4, dtype=torch.bool, device=_dev())
        for (off, k, d, ids) in ((off0, k0, 3.0, idx[:k0]), (off1, k1, 0.7, idx[k0:])):
            w0 = off // 4
            got = words[w0:w0 + k * LD].view(k, LD)[:, :F]
            want = (hm[ids].double() / float(np.float32(d))).float()
            _bits_equal(f"p2p put_all at byte offset {off}", got.view(torch.float32), want, ids)
            written[w0:w0 + k * LD].view(k, LD)[:, :F] = True
        stray = int(((words != SENTINEL) & ~written).sum())
        assert stray == 0, f"p2p put_all: {stray} words of the slab outside the segments changed"
    finally:
        torch.cuda.synchronize()
        for h, *_ in ps:
            lib.bns_p2p_destroy(h)


def test_epoch_maps_97m_halo(built):
    """``bns_epoch_maps_update`` for one rank of 8 at the papers100M shape: 97 M halo nodes (the slot map), seven
    inverse maps of 13.9 M inner nodes, 10 % sampled each way.  The whole allocation is compared exactly with a torch
    restatement (every entry not set is -1)."""
    from bns_gcn_b200._lib import EpochMaps
    import ctypes
    lib = _lib()
    _need(8)
    n_in, P = N_IN, 8
    peer_n = N_HALO // (P - 1)
    n_halo = peer_n * (P - 1)
    gen = _gen(81)
    maps = torch.empty(n_halo + (P - 1) * n_in, dtype=torch.int32, device=_dev())
    assert maps.numel() > 1 << 27 and n_halo > 9 * 10 ** 7
    pos, sel, hops = [], [], []
    for s_ in range(P - 1):
        p = torch.full((peer_n + 16,), -1, dtype=torch.int64, device=_dev())
        p[:peer_n] = n_in + s_ * peer_n + torch.arange(peer_n, device=_dev())
        pos.append(p)
        # random distinct ids, the last four first (the last inner rows / the last halo nodes)
        for lst, n_ in ((sel, n_in), (hops, peer_n)):
            last = torch.arange(n_ - 4, n_, device=_dev())
            rest = torch.randperm(n_ - 4, generator=gen, device=_dev())[:n_ // 10 - 4]
            lst.append(torch.cat([last, rest]))
    sel_cat, hop_cat = torch.cat(sel), torch.cat(hops)
    m = EpochMaps()
    m.n_seg = P - 1
    a = b = 0
    for s_ in range(P - 1):
        m.sel_begin[s_], m.hop_begin[s_] = a, b
        a += sel[s_].numel()
        b += hops[s_].numel()
        m.pos[s_] = pos[s_].data_ptr()
        m.inv[s_] = maps[n_halo + s_ * n_in:].data_ptr()
    m.sel_begin[P - 1], m.hop_begin[P - 1] = a, b
    m.selected_cat, m.one_hops_cat, m.slot, m.n_in = sel_cat.data_ptr(), hop_cat.data_ptr(), maps.data_ptr(), n_in
    maps.fill_(12345)
    _check_rc(lib.bns_epoch_maps_update(ctypes.byref(m), maps.data_ptr(), maps.numel() * 4, _stream()),
              "bns_epoch_maps_update")
    want = torch.full_like(maps, -1)
    want[torch.cat([pos[s_][hops[s_]] for s_ in range(P - 1)]) - n_in] = torch.arange(b, device=_dev(), dtype=torch.int32)
    for s_ in range(P - 1):
        want[n_halo + s_ * n_in + sel[s_]] = torch.arange(sel[s_].numel(), device=_dev(), dtype=torch.int32)
    bad = torch.nonzero(maps != want)[:, 0]
    assert bad.numel() == 0, f"epoch maps: {bad.numel()} entries differ, first at {bad[:8].tolist()}"


def _philox_torch(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 on int64 GPU tensors of uint32 values (pinned to ``oracle.philox`` below)."""
    M = 0xFFFFFFFF

    def mulhilo(m, c):
        t1, t2 = m * (c & 0xFFFF), m * (c >> 16)
        s = t1 + ((t2 & 0xFFFF) << 16)
        return (t2 >> 16) + (s >> 32), s & M
    k0, k1 = k0 & M, k1 & M
    for _ in range(10):
        hi0, lo0 = mulhilo(0xD2511F53, c0)
        hi1, lo1 = mulhilo(0xCD9E8D57, c2)
        c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
        k0, k1 = (k0 + 0x9E3779B9) & M, (k1 + 0xBB67AE85) & M
    return c0, c1, c2, c3


def test_boundary_sampler_per_rank_size(built):
    """``BoundarySampler`` for one rank of 8 at the papers100M shape: seven boundary lists of ~11.8 M inner nodes
    (B ~ 83 M: an inner node with 14 random neighbours borders a given peer with probability ~0.85), 10 % drawn from
    each.  Every selected id is compared with the sampler's contract replayed in torch (Philox keys, stable sort per
    segment), whose Philox is pinned to ``oracle.philox`` on sampled counters."""
    from bns_gcn_b200 import ops
    from oracle.philox import philox4x32_10
    _need(12)
    P, seed, offset = 8, (1 << 35) + 99, (1 << 32) + 3
    gen = _gen(91)
    boundary = [None]
    for _ in range(P - 1):
        b = torch.nonzero(torch.rand(N_IN, generator=gen, device=_dev()) < 0.85)[:, 0]
        boundary.append(b)
    sizes = [0] + [b.numel() // 10 for b in boundary[1:]]
    sampler = ops.BoundarySampler(boundary, sizes, _dev())
    B = sampler.B
    assert B > 8 * 10 ** 7, B
    sel, _ = sampler.sample(seed, offset)
    i = torch.arange(B, dtype=torch.int64, device=_dev())
    r0, r1, _, _ = _philox_torch(i & 0xFFFFFFFF, i >> 32, torch.full_like(i, offset & 0xFFFFFFFF),
                                 torch.full_like(i, offset >> 32), seed & 0xFFFFFFFF, seed >> 32)
    probe = sample_rows(B, seed=92).cpu().numpy().astype(np.uint64)
    w = philox4x32_10((probe & np.uint64(0xFFFFFFFF)).astype(np.uint32), (probe >> np.uint64(32)).astype(np.uint32),
                      np.full(probe.size, offset & 0xFFFFFFFF, np.uint32), np.full(probe.size, offset >> 32, np.uint32),
                      seed & 0xFFFFFFFF, seed >> 32)
    pr = torch.from_numpy(probe.astype(np.int64)).to(_dev())
    assert torch.equal(r0[pr].cpu(), torch.from_numpy(w[0].astype(np.int64))) and \
        torch.equal(r1[pr].cpu(), torch.from_numpy(w[1].astype(np.int64))), "torch Philox differs from oracle.philox"
    key = (r0 << 24) | (r1 >> 8)
    del r0, r1
    segb = sampler.seg_begin
    seg = torch.searchsorted(segb, i, right=True) - 1
    key |= seg << 56
    order = torch.sort(key, stable=True)[1]
    del key, seg, i
    want = torch.cat([sampler.cat[order[int(segb[s_]):int(segb[s_]) + k]] for s_, k in enumerate(sampler.sizes)])
    bad = torch.nonzero(sel != want)[:, 0]
    assert bad.numel() == 0, f"sampler: {bad.numel()} of {sel.numel()} ids differ, first at positions {bad[:8].tolist()}"


def test_papers100m_partition_structure(built):
    """Rank 0 of 8 of ``data.make_local_partition("papers100m", 0, 8, scale=1.0)`` (the real generator's degree
    distribution: 13.9 M inner rows, 216 M entries, 67 M halo columns): ``bns_graph_create`` / ``transpose``
    checked exactly (``check_structure``) on sampled transpose rows, the last columns included."""
    from bns_gcn_b200 import ops
    from bns_gcn_b200.data.synthetic import make_local_partition
    _need(30)
    part = make_local_partition("papers100m", 0, 8, device=_dev(), scale=1.0)
    lg = part.graph
    part.node_dict.clear()
    n_cols = lg.n_in + lg.n_halo
    indptr, idx = lg.indptr, lg.indices.to(torch.int32)
    del part, lg
    torch.cuda.empty_cache()
    print(f"[shape] papers100m rank 0 of 8: {indptr.numel() - 1} inner rows, {n_cols - indptr.numel() + 1} halo "
          f"columns, {idx.numel()} entries, max degree {int((indptr[1:] - indptr[:-1]).max())}")
    assert indptr.numel() - 1 > 1.3e7 and idx.numel() > 1.9e8 and int(idx.max()) == n_cols - 1
    g = ops.DeviceGraph.from_csr(indptr, idx, n_cols)
    gt = g.transpose()
    trows = sample_rows(n_cols, extra=range(n_cols - 16, n_cols), seed=101)
    check_structure(g, gt, indptr, idx, trows)
