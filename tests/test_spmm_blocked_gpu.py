"""``ops.spmm_auto`` with its source rows cut into blocks (``plan_col_blocks`` / ``make_col_blocks``, forced through
``BNS_SPMM_COLBLOCKS``) against float64, element by element (tests/layer_reference.py), and against the unblocked pass.

On one GPU at the Reddit shape the F = 256 and F = 128 aggregations run as 2 blocks.  The graph here has heavy rows
whose entries span every block, rows whose entries all lie in the first or the last block, empty rows, and a column
range without entries, so that with 4 blocks one block is empty; a second family of graphs has fewer columns than
blocks, so that some blocks have no columns at all.  Each pass runs with a row scale, a column scale (sliced per
block), accumulation into a non-zero output, ``n_out_rows`` and a strided (``fused.gather_friendly``) source and
output, at F = 256, 128, 44 and 602; also the transposed pass of the backward, and the rebuild of the cached blocks
when the block count changes."""
import functools
import types

import pytest
import torch

from tests import layer_reference as R

pytestmark = pytest.mark.gpu

N_ROWS, N_COLS = 2500, 4000
EMPTY_COLS = (2000, 3000)                  # no entry has its column here: block 2 of 4
HEAVY = {5: 4500, 1700: 3200, N_ROWS - 1: 2600}
FIRST_BLOCK_ROWS, LAST_BLOCK_ROWS = range(100, 200), range(300, 400)


def _dev():
    return torch.device("cuda:0")


def _host_csr(n_rows, n_cols, gen, avg=20.0, heavy=None, confined=()):
    """Rows of ~``avg`` entries (5 % empty); ``heavy``: row -> entry count; ``confined``: (rows, lo, hi) whose entries
    lie in ``[lo, hi)``; no column lies in ``EMPTY_COLS``."""
    deg = torch.poisson(torch.full((n_rows,), avg), generator=gen).long()
    deg[torch.rand(n_rows, generator=gen) < 0.05] = 0
    for row, d in (heavy or {}).items():
        deg[row] = d
    lo = torch.zeros(n_rows, dtype=torch.int64)
    hi = torch.full((n_rows,), n_cols, dtype=torch.int64)
    for rows, a, b in confined:
        lo[list(rows)], hi[list(rows)] = a, b
    rows = torch.repeat_interleave(torch.arange(n_rows), deg)
    span = hi[rows] - lo[rows]
    # rows whose range covers EMPTY_COLS draw from the columns outside it (ranges that do not touch it are kept)
    gap = (lo[rows] <= EMPTY_COLS[0]) & (hi[rows] >= EMPTY_COLS[1])
    span = torch.where(gap, span - (EMPTY_COLS[1] - EMPTY_COLS[0]), span)
    col = lo[rows] + (torch.rand(rows.numel(), generator=gen, dtype=torch.float64) * span).long()
    col = torch.where(gap & (col >= EMPTY_COLS[0]), col + (EMPTY_COLS[1] - EMPTY_COLS[0]), col)
    indptr = torch.cat([torch.zeros(1, dtype=torch.int64), deg.cumsum(0)])
    return indptr, col, rows


@functools.lru_cache(maxsize=None)
def _graph(n_rows=N_ROWS, n_cols=N_COLS):
    from bns_gcn_b200 import ops
    gen = torch.Generator().manual_seed(n_rows + n_cols)
    if n_cols == N_COLS:
        ip, col, rows = _host_csr(n_rows, n_cols, gen, heavy=HEAVY,
                                  confined=((FIRST_BLOCK_ROWS, 0, 900), (LAST_BLOCK_ROWS, 3100, 3900)))
        assert not bool(((col >= EMPTY_COLS[0]) & (col < EMPTY_COLS[1])).any())
    else:
        ip, col, rows = _host_csr(n_rows, n_cols, gen, avg=6.0, heavy={0: 700})
    dev = _dev()
    g = ops.DeviceGraph.from_csr(ip.to(dev), col.int().to(dev), n_cols)
    return types.SimpleNamespace(g=g, n_rows=n_rows, n_cols=n_cols, rows=rows.to(dev), cols=col.to(dev))


def _reference(case, x, rs=None, cs=None, y0=None, transpose=False):
    """``y0 + rs * (A (cs * x))`` (``A^T`` with ``transpose``) in float64, and its bound."""
    v, u, n = (case.cols, case.rows, case.n_cols) if transpose else (case.rows, case.cols, case.n_rows)

    def run(x, rs, cs, y0):
        y = R.aggregate(x.double(), v, u, n, None if cs is None else cs.double()[u])
        if rs is not None:
            y = y * rs.double().unsqueeze(1)
        return y if y0 is None else y + y0.double()
    return run(x, rs, cs, y0), run(x.abs(), rs, cs, None if y0 is None else y0.abs())


def _forms(case, F, gen):
    """``(name, call(spmm_fn) -> result rows, reference, bound)`` for every argument form of ``spmm_auto``."""
    from bns_gcn_b200 import fused
    dev = _dev()
    x = torch.randn(case.n_cols, F, generator=gen).to(dev)
    rs = (torch.rand(case.n_rows, generator=gen) + 0.5).to(dev)
    cs = (torch.rand(case.n_cols, generator=gen) + 0.5).to(dev)
    y0 = torch.randn(case.n_rows, F, generator=gen).to(dev)
    xs = fused.gather_friendly(case.n_cols, F, dev)
    xs.copy_(x)
    ys = fused.gather_friendly(case.n_rows, F, dev)

    def accumulate(spmm):
        out = y0.clone()
        spmm(case.g, x, out, row_scale=rs, col_scale=cs, accumulate=True)
        return out

    def n_out_rows(spmm):
        out = spmm(case.g, x, col_scale=cs, n_out_rows=case.n_rows + 5)
        assert out.shape == (case.n_rows + 5, F)
        return out[:case.n_rows]

    def strided(spmm):
        ys.copy_(y0)
        spmm(case.g, xs, ys, row_scale=rs, accumulate=True)
        return ys.clone()

    return [
        ("row_scale", lambda spmm: spmm(case.g, x, row_scale=rs), *_reference(case, x, rs=rs)),
        ("col_scale", lambda spmm: spmm(case.g, x, row_scale=rs, col_scale=cs), *_reference(case, x, rs, cs)),
        ("accumulate", accumulate, *_reference(case, x, rs, cs, y0)),
        ("n_out_rows", n_out_rows, *_reference(case, x, cs=cs)),
        ("gather_friendly", strided, *_reference(case, x, rs=rs, y0=y0)),
    ]


def _unblocked(g, x, out=None, *, row_scale=None, n_out_rows=None, accumulate=False, col_scale=None):
    from bns_gcn_b200 import ops
    return ops.spmm(g, x, out, row_scale=row_scale, n_out_rows=n_out_rows, accumulate=accumulate, col_scale=col_scale)


@pytest.mark.parametrize("F", [256, 128, 44, 602])
@pytest.mark.parametrize("n_blocks", [1, 2, 3, 4])
def test_blocked_spmm_matches_float64(built, monkeypatch, n_blocks, F):
    """Every argument form against float64 and against one unblocked pass; a repeat is bit-identical."""
    from bns_gcn_b200 import ops
    monkeypatch.setenv("BNS_SPMM_COLBLOCKS", str(n_blocks))
    case = _graph()
    assert ops.plan_col_blocks(case.g, F) == n_blocks
    for name, call, want, bound in _forms(case, F, torch.Generator().manual_seed(F)):
        label = f"spmm_auto {n_blocks} blocks F={F} {name}"
        got = call(ops.spmm_auto)
        torch.cuda.synchronize()
        if n_blocks > 1:
            assert len(case.g._col_blocks) == n_blocks
        R.assert_close(label, got, want, bound)
        R.assert_close(f"{label} vs unblocked", got, call(_unblocked).double(), bound)
        assert torch.equal(got, call(ops.spmm_auto)), f"{label}: a repeat differs"


def test_blocks_are_rebuilt_when_the_count_changes(built, monkeypatch):
    """``g._col_blocks`` follows the block count: ranges that tile ``[0, n_cols)``, every entry in exactly one block
    with its column shifted into the block, and a correct result after each change."""
    from bns_gcn_b200 import ops
    case = _graph()
    g = case.g
    gen = torch.Generator().manual_seed(1)
    x = torch.randn(N_COLS, 128, generator=gen).to(_dev())
    rs = (torch.rand(N_ROWS, generator=gen) + 0.5).to(_dev())
    want, bound = _reference(case, x, rs=rs)
    for nb in (2, 3, 2, 4):
        monkeypatch.setenv("BNS_SPMM_COLBLOCKS", str(nb))
        got = ops.spmm_auto(g, x, row_scale=rs)
        blocks = g._col_blocks
        assert len(blocks) == nb
        assert [(c0, c1) for _, c0, c1 in blocks] == [(N_COLS * b // nb, N_COLS * (b + 1) // nb) for b in range(nb)]
        assert sum(gb.nnz for gb, _, _ in blocks) == g.nnz
        for gb, c0, c1 in blocks:
            assert gb.n_rows == N_ROWS and gb.n_cols == c1 - c0
            ip, ix = gb.csr()
            in_block = (case.cols >= c0) & (case.cols < c1)
            assert torch.equal(torch.diff(ip), torch.bincount(case.rows[in_block], minlength=N_ROWS))
            assert torch.equal(ix.long(), case.cols[in_block] - c0)
        if nb == 4:
            assert blocks[2][0].nnz == 0                    # the empty column range
        R.assert_close(f"rebuild {nb} blocks", got, want, bound)


@pytest.mark.parametrize("F", [256, 44])
@pytest.mark.parametrize("n_cols,n_blocks", [(3, 4), (1, 2), (2, 3)])
def test_blocks_without_columns(built, monkeypatch, n_cols, n_blocks, F):
    """More blocks than columns: the leading blocks have no columns, the first of them still zeroes the output."""
    from bns_gcn_b200 import ops
    monkeypatch.setenv("BNS_SPMM_COLBLOCKS", str(n_blocks))
    case = _graph(300, n_cols)
    gen = torch.Generator().manual_seed(n_cols)
    x = torch.randn(n_cols, F, generator=gen).to(_dev())
    rs = (torch.rand(300, generator=gen) + 0.5).to(_dev())
    cs = (torch.rand(n_cols, generator=gen) + 0.5).to(_dev())
    out = torch.full((300, F), float("nan"), device=_dev())
    ops.spmm_auto(case.g, x, out, row_scale=rs, col_scale=cs)
    assert [c1 - c0 for _, c0, c1 in case.g._col_blocks].count(0) == n_blocks - n_cols
    R.assert_close(f"{n_cols} columns in {n_blocks} blocks F={F}", out, *_reference(case, x, rs, cs))
    y0 = torch.randn(300, F, generator=gen).to(_dev())
    acc = y0.clone()
    ops.spmm_auto(case.g, x, acc, col_scale=cs, accumulate=True)
    R.assert_close(f"{n_cols} columns in {n_blocks} blocks F={F} accumulate", acc, *_reference(case, x, cs=cs, y0=y0))


@pytest.mark.parametrize("F", [256, 44])
def test_transposed_pass_at_two_blocks(built, monkeypatch, F):
    """The backward's ``spmm_auto(a_in_t, dys, du[:n_in], row_scale=cs_in)``: the transpose cut into 2 blocks of its
    source rows, writing the head rows of a larger gradient (the rows after them stay untouched)."""
    from bns_gcn_b200 import fused, ops
    monkeypatch.setenv("BNS_SPMM_COLBLOCKS", "2")
    case = _graph()
    gt = case.g.transpose()
    gen = torch.Generator().manual_seed(F + 2)
    dys = fused.gather_friendly(N_ROWS, F, _dev())
    dys.copy_(torch.randn(N_ROWS, F, generator=gen))
    cs = (torch.rand(N_COLS, generator=gen) + 0.5).to(_dev())
    du = torch.full((N_COLS + 300, F), float("nan"), device=_dev())
    ops.spmm_auto(gt, dys, du[:N_COLS], row_scale=cs)
    assert len(gt._col_blocks) == 2
    want, bound = _reference(case, dys, rs=cs, transpose=True)
    R.assert_close(f"transposed 2 blocks F={F}", du[:N_COLS], want, bound)
    assert torch.all(du[N_COLS:].isnan())
    empty = torch.zeros(N_COLS, dtype=torch.bool)
    empty[EMPTY_COLS[0]:EMPTY_COLS[1]] = True
    assert torch.all(du[:N_COLS][empty.to(_dev())] == 0)
