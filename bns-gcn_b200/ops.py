"""torch-facing wrappers over the C ABI (``include/bnsgcn.h``): device memory and streams come from
PyTorch, every kernel comes from ``libbnsgcn.so``.  Nothing here computes on the CPU.

* ``DeviceGraph``      a static CSR matrix in HBM (``bns_graph_t``) + its transpose
* ``spmm``             ``bns_spmm_sum_f32``
* ``AggregateSum``     autograd Function: the DGL ``update_all(copy_u, sum)`` of module/layer.py:35-37, 88-90
                       with the degree / norm scalings of :34, :38, :91 fused in
* ``gather_div`` / ``scatter_add_div`` / ``sample_boundary`` / ``halo_slot_update``
"""
from __future__ import annotations

import ctypes
from typing import Dict, Optional

import torch

from . import _lib
from ._lib import check, lib


# bench.py sets this to a list to collect (start_event, end_event, algorithmic_bytes, nnz, F, live_nnz) per launch
PROFILE = None


def _stream_ptr() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _req(t: torch.Tensor, dtype, name: str) -> torch.Tensor:
    if not t.is_cuda:
        raise _lib.BnsError(f"{name} must be a CUDA tensor (there is no CPU path)")
    if t.dtype != dtype:
        raise _lib.BnsError(f"{name} must be {dtype}, got {t.dtype}")
    return t


def device_info() -> dict:
    name = ctypes.create_string_buffer(256)
    sms, l2, maj, mnr = ctypes.c_int(), ctypes.c_int64(), ctypes.c_int(), ctypes.c_int()
    check(lib.bns_device_info(name, 256, ctypes.byref(sms), ctypes.byref(l2), ctypes.byref(maj), ctypes.byref(mnr)),
          "bns_device_info")
    return {"name": name.value.decode(), "sm_count": sms.value, "l2_bytes": l2.value, "cc": (maj.value, mnr.value)}


class DeviceGraph:
    """A static sparse 0/1 matrix ``[n_rows, n_cols]`` in CSR, resident on the GPU.

    Row ``r`` lists the columns whose feature rows are summed into output row ``r``.
    """

    def __init__(self, handle: int, device: torch.device):
        self._h = ctypes.c_void_p(handle)
        self.device = device
        nr, nc, nnz, nch, nsp = (ctypes.c_int64() for _ in range(5))
        check(lib.bns_graph_info(self._h, ctypes.byref(nr), ctypes.byref(nc), ctypes.byref(nnz), ctypes.byref(nch),
                                 ctypes.byref(nsp)), "bns_graph_info")
        self.n_rows, self.n_cols, self.nnz = nr.value, nc.value, nnz.value
        self.n_chunks, self.n_split_rows = nch.value, nsp.value
        self._t: Optional["DeviceGraph"] = None
        self._ws: Dict[int, torch.Tensor] = {}

    @classmethod
    def from_csr(cls, indptr: torch.Tensor, indices: torch.Tensor, n_cols: int, chunk_nnz: int = 0) -> "DeviceGraph":
        _req(indptr, torch.int64, "indptr")
        _req(indices, torch.int32, "indices")
        indptr, indices = indptr.contiguous(), indices.contiguous()
        out = ctypes.c_void_p()
        with torch.cuda.device(indptr.device):
            check(lib.bns_graph_create(ctypes.byref(out), indptr.numel() - 1, n_cols, indices.numel(),
                                       indptr.data_ptr(), indices.data_ptr() if indices.numel() else None,
                                       chunk_nnz, _stream_ptr()), "bns_graph_create")
        return cls(out.value, indptr.device)

    def transpose(self) -> "DeviceGraph":
        if self._t is None:
            out = ctypes.c_void_p()
            with torch.cuda.device(self.device):
                check(lib.bns_graph_transpose(self._h, ctypes.byref(out), _stream_ptr()), "bns_graph_transpose")
            self._t = DeviceGraph(out.value, self.device)
            self._t._t = self
        return self._t

    def csr(self):
        """Copies of the library-owned CSR (for tests)."""
        indptr = torch.empty(self.n_rows + 1, dtype=torch.int64, device=self.device)
        indices = torch.empty(self.nnz, dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            check(lib.bns_graph_copy_csr(self._h, indptr.data_ptr(), indices.data_ptr() if self.nnz else None,
                                         _stream_ptr()), "bns_graph_copy_csr")
        return indptr, indices

    def perm(self) -> torch.Tensor:
        """For a transpose: ``perm[k]`` = position in the source graph's CSR of the entry that is entry ``k`` here."""
        if getattr(self, "_perm", None) is None:
            p = torch.empty(self.nnz, dtype=torch.int32, device=self.device)
            with torch.cuda.device(self.device):
                check(lib.bns_graph_copy_perm(self._h, p.data_ptr(), _stream_ptr()), "bns_graph_copy_perm")
            self._perm = p
        return self._perm

    def workspace(self, F: int) -> Optional[torch.Tensor]:
        need = lib.bns_spmm_workspace_bytes(self._h, F)
        if need == 0:
            return None
        ws = self._ws.get(F)
        if ws is None or ws.numel() < need:
            ws = torch.empty(need, dtype=torch.uint8, device=self.device)
            self._ws[F] = ws
        return ws

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            try:
                lib.bns_graph_destroy(h)
            except Exception:   # interpreter shutdown
                pass


class Fp8Rows:
    """An fp8 gather table (``--agg-dtype fp8``, ``cvt_rows_fp8``): e4m3 ``codes`` ``[rows, F]`` (``float8_e4m3fn``, row
    stride a multiple of 16 bytes) and one power-of-two f32 ``scale`` per row; row ``r`` stands for
    ``codes[r].float() * scale[r]``.  Slicing takes rows."""

    __slots__ = ("codes", "scale")

    def __init__(self, codes: torch.Tensor, scale: torch.Tensor):
        self.codes, self.scale = codes, scale

    @property
    def shape(self):
        return self.codes.shape

    @property
    def device(self):
        return self.codes.device

    def element_size(self) -> int:
        return 1

    def __getitem__(self, rows: slice) -> "Fp8Rows":
        return Fp8Rows(self.codes[rows], self.scale[rows])

    def dequantize(self) -> torch.Tensor:
        """The f32 rows the SpMM sums (for tests and diagnostics)."""
        return self.codes.float() * self.scale.unsqueeze(1)


def _table(x, name: str = "x"):
    """``(kind, data pointer, row stride, scale pointer)`` of a gather table: f32, bf16 or ``Fp8Rows``."""
    if isinstance(x, Fp8Rows):
        c = x.codes
        _req(c, torch.float8_e4m3fn, name + ".codes")
        _req(x.scale, torch.float32, name + ".scale")
        if c.dim() != 2 or c.stride(1) != 1 or x.scale.dim() != 1 or x.scale.shape[0] != c.shape[0] or \
                x.scale.stride(0) != 1:
            raise _lib.BnsError(f"{name}: codes must be a row-major 2-D tensor with one contiguous scale per row")
        return "fp8", c.data_ptr(), c.stride(0), x.scale.data_ptr()
    if x.dtype == torch.bfloat16:
        if not x.is_cuda:
            raise _lib.BnsError(f"{name} must be a CUDA tensor (there is no CPU path)")
        kind = "bf16"
    else:
        _req(x, torch.float32, name)
        kind = "f32"
    if x.dim() != 2 or x.stride(1) != 1:
        raise _lib.BnsError(f"{name} must be a row-major 2-D tensor")
    return kind, x.data_ptr(), x.stride(0), None


def _table_bytes(x, F: int) -> int:
    return x.element_size() * F * x.shape[0] + (4 * x.shape[0] if isinstance(x, Fp8Rows) else 0)


def spmm(g: DeviceGraph, x: torch.Tensor, out: Optional[torch.Tensor] = None, *, n_out_rows: Optional[int] = None,
         row_scale: Optional[torch.Tensor] = None, col_scale: Optional[torch.Tensor] = None,
         row_map: Optional[torch.Tensor] = None, col_map: Optional[torch.Tensor] = None, n_direct: int = 0,
         accumulate: bool = False, slab: int = 0, edge_weight: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``bns_spmm_sum_f32``: ``out[orow(r)] (+)= row_scale[r] * sum_k col_scale[c_k] * x[xrow(c_k)]``.  A bf16 ``x``
    (``cvt_rows_bf16``) takes ``bns_spmm_sum_bf16``, an ``Fp8Rows`` ``x`` (``cvt_rows_fp8``) ``bns_spmm_sum_fp8``: the
    same sum, accumulated and written in f32."""
    kind, xp, ldx, xs = _table(x)
    F = x.shape[1]
    if out is None:
        if accumulate:
            raise _lib.BnsError("accumulate=True needs an output tensor")
        rows = g.n_rows if n_out_rows is None else n_out_rows
        out = torch.empty(rows, F, dtype=torch.float32, device=x.device)
    _req(out, torch.float32, "out")
    if out.dim() != 2 or out.stride(1) != 1 or out.shape[1] != F:
        raise _lib.BnsError("out must be row-major [*, F]")
    for t, n, nm in ((row_scale, torch.float32, "row_scale"), (col_scale, torch.float32, "col_scale"),
                     (row_map, torch.int32, "row_map"), (col_map, torch.int32, "col_map")):
        if t is not None:
            _req(t, n, nm)
    ws = g.workspace(F)
    prof = PROFILE
    if prof is not None:
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record(torch.cuda.current_stream(x.device))
    name = "bns_spmm_sum_" + kind
    xargs = (xp, xs, ldx) if kind == "fp8" else (xp, ldx)
    with torch.cuda.device(x.device):
        check(getattr(lib, name)(g._h, *xargs, F, out.data_ptr(), out.stride(0),
                                 _ptr(row_scale), _ptr(col_scale), _ptr(edge_weight), _ptr(row_map), _ptr(col_map),
                                 n_direct, x.shape[0], slab, 1 if accumulate else 0, _ptr(ws),
                                 0 if ws is None else ws.numel(), _stream_ptr()), name)
    if prof is not None:
        ev1.record(torch.cuda.current_stream(x.device))
        # SURVEY.md §8(d): every distinct operand byte once -- row offsets, column ids, source rows, output rows
        alg = 8 * (g.n_rows + 1) + 4 * g.nnz + _table_bytes(x, F) + 4 * F * out.shape[0]
        # entries whose source row is really gathered: all of them, or (sampled halo) the mapped fraction
        live = g.nnz
        if col_map is not None and g.n_cols > n_direct:
            live = int(g.nnz * min(1.0, max(x.shape[0] - 0, 0) / max(g.n_cols - n_direct, 1)))
        if row_map is not None:
            live = int(g.nnz * min(1.0, out.shape[0] / max(g.n_rows, 1)))
        prof.append((ev0, ev1, alg, g.nnz, F, live))
    return out


# ---- source-row blocking ------------------------------------------------------------------------------------------
# Column slabs (csrc: pick_slab) cut the gather table by columns; cutting the SOURCE ROWS into blocks as well makes
# every pass gather from a smaller table, so more of it stays in L2.  Only worth it where rows are re-read often (high
# average degree) and few blocks suffice -- each extra block costs one read-modify-write of the output.  On an H100 SXM
# (700 W) the Reddit-shape F = 256 launch takes 9.4 ms with two blocks of <= 60 MB and 15.5 ms unblocked.
BLOCK_TABLE_BYTES = 60 << 20
BLOCK_MIN_AVG_DEGREE = 64
BLOCK_MAX = 4


def plan_col_blocks(g: DeviceGraph, F: int, elem_bytes: int = 4) -> int:
    """Number of source-row blocks for width ``F`` (1 = no blocking); ``elem_bytes``: 4 for an f32 table, 2 for bf16,
    1 for fp8 (its row scales are not counted)."""
    import os
    forced = os.environ.get("BNS_SPMM_COLBLOCKS")
    if forced:
        return max(1, int(forced))
    if F < 128 or g.n_rows == 0 or g.nnz / max(g.n_rows, 1) < BLOCK_MIN_AVG_DEGREE:
        return 1
    b = -(-g.n_cols * 128 * elem_bytes // BLOCK_TABLE_BYTES)     # a 128-column slab of every source row
    return b if 1 < b <= BLOCK_MAX else 1


def make_col_blocks(g: DeviceGraph, n_blocks: int, chunk_nnz: int = 0):
    """``[(sub-graph, c0, c1)]``: block ``b`` holds the entries whose column lies in ``[c0, c1)``, columns shifted to 0."""
    ip, ix = g.csr()
    dev = g.device
    rows = torch.repeat_interleave(torch.arange(g.n_rows, device=dev), ip[1:] - ip[:-1])
    out = []
    for b in range(n_blocks):
        c0, c1 = (g.n_cols * b) // n_blocks, (g.n_cols * (b + 1)) // n_blocks
        m = (ix >= c0) & (ix < c1)
        ipb = torch.zeros(g.n_rows + 1, dtype=torch.int64, device=dev)
        ipb[1:] = torch.cumsum(torch.bincount(rows[m], minlength=g.n_rows), 0)
        out.append((DeviceGraph.from_csr(ipb, (ix[m] - c0).to(torch.int32), c1 - c0, chunk_nnz), c0, c1))
    return out


def spmm_auto(g: DeviceGraph, x: torch.Tensor, out: Optional[torch.Tensor] = None, *, row_scale=None,
              n_out_rows: Optional[int] = None, accumulate: bool = False, col_scale=None) -> torch.Tensor:
    """``spmm`` of a plain matrix (no maps, no weights), source-row blocked when ``plan_col_blocks`` says so: one pass
    per block, each accumulating into ``out``.  Counts as ONE launch in bench.py's roofline bookkeeping."""
    global PROFILE
    F = x.shape[1]
    nb = plan_col_blocks(g, F, x.element_size())
    if nb <= 1:
        return spmm(g, x, out, row_scale=row_scale, n_out_rows=n_out_rows, accumulate=accumulate, col_scale=col_scale)
    blocks = g.__dict__.get("_col_blocks")
    if blocks is None or len(blocks) != nb:
        blocks = g._col_blocks = make_col_blocks(g, nb)
    if out is None:
        out = torch.empty(g.n_rows if n_out_rows is None else n_out_rows, F, dtype=torch.float32, device=x.device)
    prof, PROFILE = PROFILE, None
    try:
        if prof is not None:
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record(torch.cuda.current_stream(x.device))
        for i, (gb, c0, c1) in enumerate(blocks):
            spmm(gb, x[c0:c1], out, row_scale=row_scale, accumulate=accumulate or i > 0,
                 col_scale=None if col_scale is None else col_scale[c0:c1])
        if prof is not None:
            ev1.record(torch.cuda.current_stream(x.device))
            alg = 8 * (g.n_rows + 1) + 4 * g.nnz + _table_bytes(x, F) + 4 * F * out.shape[0]
            prof.append((ev0, ev1, alg, g.nnz, F, g.nnz))
    finally:
        PROFILE = prof
    return out


class CompactedCols:
    """Per-epoch compaction of a column-mapped matrix (``bns_graph_compact_cols``): the sampled entries of every
    chunk, already mapped to rows of X, moved to the front of the chunk's own index range."""

    def __init__(self, g: DeviceGraph, with_weights: bool = False, with_positions: bool = False):
        self.g = g
        dev = g.device
        self.cidx = torch.empty(max(g.nnz, 1), dtype=torch.int32, device=dev)
        self.cw = torch.empty(max(g.nnz, 1), dtype=torch.float32, device=dev) if with_weights else None
        # GAT: where each live entry sits in the CSR (its attention is kept at the original positions)
        self.cpos = torch.empty(max(g.nnz, 1), dtype=torch.int32, device=dev) if with_positions else None
        self.chunk_cnt = torch.zeros(max(g.n_chunks, 1), dtype=torch.int32, device=dev)

    def refresh(self, col_map: torch.Tensor, n_direct: int = 0, col_scale: Optional[torch.Tensor] = None) -> None:
        _req(col_map, torch.int32, "col_map")
        if (col_scale is None) != (self.cw is None):
            raise _lib.BnsError("CompactedCols: col_scale must be given exactly when it was built with_weights")
        with torch.cuda.device(self.g.device):
            check(lib.bns_graph_compact_cols(self.g._h, col_map.data_ptr(), n_direct, _ptr(col_scale), self.cidx.data_ptr(),
                                             _ptr(self.cw), _ptr(self.cpos), self.chunk_cnt.data_ptr(), _stream_ptr()),
                  "bns_graph_compact_cols")


def spmm_compact(c: CompactedCols, x: torch.Tensor, out: torch.Tensor, *, row_scale: Optional[torch.Tensor] = None,
                 accumulate: bool = False, slab: int = 0, live_nnz: Optional[int] = None,
                 weights: Optional[torch.Tensor] = None, head: int = 0) -> torch.Tensor:
    """``bns_spmm_compact_f32``: the SpMM over the compacted (sampled) entries only.  ``weights`` ``[nnz, heads]`` at
    the COMPACTED positions (GAT's dropped attention, column ``head``) replaces the compaction's own per-entry weights.
    A bf16 ``x`` takes ``bns_spmm_compact_bf16``, an ``Fp8Rows`` ``x`` ``bns_spmm_compact_fp8``."""
    g = c.g
    kind, xp, ldx, xs = _table(x)
    _req(out, torch.float32, "out")
    if out.stride(1) != 1 or out.shape[1] != x.shape[1]:
        raise _lib.BnsError("x / out must be row-major [*, F]")
    F = x.shape[1]
    ws = g.workspace(F)
    prof = PROFILE
    if prof is not None:
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record(torch.cuda.current_stream(x.device))
    with torch.cuda.device(x.device):
        cw_ptr, cw_ld = (_ptr(c.cw), 1) if weights is None else (weights.data_ptr() + 4 * head, weights.stride(0))
        name = "bns_spmm_compact_" + kind
        xargs = (xp, xs, ldx) if kind == "fp8" else (xp, ldx)
        check(getattr(lib, name)(g._h, c.cidx.data_ptr(), cw_ptr, cw_ld, c.chunk_cnt.data_ptr(), *xargs,
                                 F, out.data_ptr(), out.stride(0), _ptr(row_scale), x.shape[0], slab,
                                 1 if accumulate else 0, _ptr(ws), 0 if ws is None else ws.numel(), _stream_ptr()), name)
    if prof is not None:
        ev1.record(torch.cuda.current_stream(x.device))
        live = int(g.nnz * min(1.0, x.shape[0] / max(g.n_cols, 1))) if live_nnz is None else live_nnz
        # algorithmic bytes of the SAMPLED product: its live entries, the rows of X it can reference, the output rows
        alg = 8 * (g.n_rows + 1) + 4 * live + _table_bytes(x, F) + 4 * F * out.shape[0]
        prof.append((ev0, ev1, alg, live, F, live))
    return out


def spmm_weighted(g: DeviceGraph, x: torch.Tensor, out: torch.Tensor, weights: torch.Tensor, head: int = 0, *,
                  through_perm: bool = False, row_map: Optional[torch.Tensor] = None, accumulate: bool = False) -> torch.Tensor:
    """``bns_spmm_weighted_f32``: ``out[orow(r)] (+)= sum_k w_k x[c_k]`` with ``w_k = weights[pos(k), head]`` where
    ``pos(k) = k``, or -- ``through_perm``, for a transpose -- the position of entry ``k`` in the graph it was made from
    (``weights`` is ``[nnz, heads]`` in THAT graph's entry order: GAT's attention)."""
    _req(x, torch.float32, "x")
    _req(out, torch.float32, "out")
    _req(weights, torch.float32, "weights")
    if x.stride(1) != 1 or out.stride(1) != 1 or weights.dim() != 2 or weights.stride(1) != 1:
        raise _lib.BnsError("spmm_weighted: x / out must have unit column stride, weights must be [nnz, heads]")
    F = x.shape[1]
    ws = g.workspace(F)
    with torch.cuda.device(x.device):
        check(lib.bns_spmm_weighted_f32(g._h, x.data_ptr(), x.stride(0), F, out.data_ptr(), out.stride(0),
                                        weights.data_ptr() + 4 * head, weights.stride(0), 1 if through_perm else 0,
                                        _ptr(row_map), x.shape[0], 1 if accumulate else 0, _ptr(ws),
                                        0 if ws is None else ws.numel(), _stream_ptr()), "bns_spmm_weighted_f32")
    return out


def sddmm_dot(g: DeviceGraph, a: torch.Tensor, b: torch.Tensor, *, row_map=None, col_map=None, n_direct: int = 0,
              out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``out[k] = <a[arow(r)], b[xrow(c_k)]>`` for every entry ``k`` (``bns_sddmm_dot_f32``)."""
    _req(a, torch.float32, "a")
    _req(b, torch.float32, "b")
    F = a.shape[1]
    if out is None:
        out = torch.zeros(g.nnz, dtype=torch.float32, device=a.device)
    with torch.cuda.device(a.device):
        check(lib.bns_sddmm_dot_f32(g._h, a.data_ptr(), a.stride(0), b.data_ptr(), b.stride(0), F, _ptr(row_map),
                                    _ptr(col_map), n_direct, out.data_ptr(), out.stride(0) if out.dim() else 1,
                                    _stream_ptr()), "bns_sddmm_dot_f32")
    return out


class AggregateSum(torch.autograd.Function):
    """``Y = rs * (A @ (cs * X))`` on a static ``DeviceGraph`` ``A [n_dst, n_src]`` and its transpose in backward.

    The full-graph (single partition / evaluation) form of module/layer.py:35-38, 88-91: ``rs`` is ``1/in_deg``
    (GraphSAGE) or ``1/sqrt(in_deg)`` (GCN), ``cs`` is ``1/sqrt(out_deg)`` (GCN) or ``None``.
    """

    @staticmethod
    def forward(ctx, x, g: DeviceGraph, row_scale, col_scale):
        ctx.g, ctx.rs, ctx.cs = g, row_scale, col_scale
        x = x.contiguous() if col_scale is None else x * col_scale.unsqueeze(1)   # scale once per row, not per edge
        return spmm(g, x, row_scale=row_scale)

    @staticmethod
    def backward(ctx, dy):
        gt = ctx.g.transpose()
        dy = dy.contiguous() if ctx.rs is None else dy * ctx.rs.unsqueeze(1)
        dx = spmm(gt, dy, row_scale=ctx.cs)
        return dx, None, None, None


def gather_div(h: torch.Tensor, idx: torch.Tensor, div: float, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``out[i] = h[idx[i]] / div`` (helper/feature_buffer.py:117).  A bf16 ``out`` (``--comm-dtype bf16``) receives the
    f32 quotient rounded to nearest even (``bns_gather_div_bf16``); an ``Fp8Rows`` ``out`` (``--comm-dtype fp8``) the
    fp8 rows of the f32 quotients (``bns_gather_div_fp8``, ``cvt_rows_fp8``'s rule)."""
    _req(h, torch.float32, "h")
    _req(idx, torch.int64, "idx")
    k, F = idx.numel(), h.shape[1]
    if out is None:
        out = torch.empty(k, F, dtype=torch.float32, device=h.device)
    if isinstance(out, Fp8Rows):
        _table(out, "out")
        with torch.cuda.device(h.device):
            check(lib.bns_gather_div_fp8(h.data_ptr(), h.stride(0), F, idx.data_ptr(), k, float(div), out.codes.data_ptr(),
                                         out.codes.stride(0), out.scale.data_ptr(), _stream_ptr()), "bns_gather_div_fp8")
        return out
    fn = "bns_gather_div_bf16" if out.dtype == torch.bfloat16 else "bns_gather_div_f32"
    if fn == "bns_gather_div_f32":
        _req(out, torch.float32, "out")
    with torch.cuda.device(h.device):
        check(getattr(lib, fn)(h.data_ptr(), h.stride(0), F, idx.data_ptr(), k, float(div), out.data_ptr(),
                               out.stride(0), _stream_ptr()), fn)
    return out


def scatter_add_div(g: torch.Tensor, idx: torch.Tensor, src: torch.Tensor, div: float) -> torch.Tensor:
    """``g[idx[i]] += src[i] / div`` in place (helper/feature_buffer.py:129).  A bf16 ``src`` (``--comm-dtype bf16``)
    is widened exactly before the f32 division and sum (``bns_scatter_add_div_bf16``), an ``Fp8Rows`` ``src``
    (``--comm-dtype fp8``) dequantized exactly (``bns_scatter_add_div_fp8``)."""
    _req(g, torch.float32, "g")
    if isinstance(src, Fp8Rows):
        _table(src, "src")
        _req(idx, torch.int64, "idx")
        with torch.cuda.device(g.device):
            check(lib.bns_scatter_add_div_fp8(g.data_ptr(), g.stride(0), g.shape[1], idx.data_ptr(), idx.numel(),
                                              float(div), src.codes.data_ptr(), src.codes.stride(0), src.scale.data_ptr(),
                                              _stream_ptr()), "bns_scatter_add_div_fp8")
        return g
    fn = "bns_scatter_add_div_bf16" if src.dtype == torch.bfloat16 else "bns_scatter_add_div_f32"
    if fn == "bns_scatter_add_div_f32":
        _req(src, torch.float32, "src")
    _req(idx, torch.int64, "idx")
    with torch.cuda.device(g.device):
        check(getattr(lib, fn)(g.data_ptr(), g.stride(0), g.shape[1], idx.data_ptr(), idx.numel(), float(div),
                               src.data_ptr(), src.stride(0), _stream_ptr()), fn)
    return g


def copy_rows(src: torch.Tensor, dst: torch.Tensor, n_rows: int) -> None:
    with torch.cuda.device(src.device):
        check(lib.bns_copy_rows_f32(src.data_ptr(), src.stride(0), dst.data_ptr(), dst.stride(0), n_rows,
                                    src.shape[1], _stream_ptr()), "bns_copy_rows_f32")


def cvt_rows_bf16(src: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``bns_cvt_rows_f32_bf16``: ``src`` rounded to bf16 (nearest even), into ``out`` or a new ``[rows, F]`` matrix whose
    row stride is a multiple of 8 elements (16 bytes: what the bf16 SpMM gathers)."""
    _req(src, torch.float32, "src")
    if src.dim() != 2 or src.stride(1) != 1:
        raise _lib.BnsError("src must be a row-major 2-D tensor")
    n, F = src.shape
    if out is None:
        out = torch.empty(n, (F + 7) // 8 * 8, dtype=torch.bfloat16, device=src.device)[:, :F]
    _req(out, torch.bfloat16, "out")
    if out.shape != src.shape or out.stride(1) != 1:
        raise _lib.BnsError("out must be row-major with the shape of src")
    with torch.cuda.device(src.device):
        check(lib.bns_cvt_rows_f32_bf16(src.data_ptr(), src.stride(0), out.data_ptr(), out.stride(0), n, F, _stream_ptr()),
              "bns_cvt_rows_f32_bf16")
    return out


def cvt_rows_fp8(src: torch.Tensor, out: Optional[Fp8Rows] = None) -> Fp8Rows:
    """``bns_cvt_rows_f32_fp8``: ``src`` as an fp8 table, into ``out`` or a new ``Fp8Rows`` whose code rows are 16-byte
    aligned.  Per row: scale ``2^e`` with ``e`` the smallest integer >= -126 such that ``max|x| * 2^-e <= 448`` (1 for
    a row of zeros), codes ``x * 2^-e`` rounded to nearest even e4m3; a row holding NaN or +-Inf gets scale NaN and
    zero codes.  ``F`` must be a multiple of 16."""
    _req(src, torch.float32, "src")
    if src.dim() != 2 or src.stride(1) != 1:
        raise _lib.BnsError("src must be a row-major 2-D tensor")
    n, F = src.shape
    if out is None:
        out = Fp8Rows(torch.empty(n, (F + 15) // 16 * 16, dtype=torch.float8_e4m3fn, device=src.device)[:, :F],
                      torch.empty(n, dtype=torch.float32, device=src.device))
    _table(out, "out")
    if out.shape != src.shape:
        raise _lib.BnsError("out must have the shape of src")
    with torch.cuda.device(src.device):
        check(lib.bns_cvt_rows_f32_fp8(src.data_ptr(), src.stride(0), out.codes.data_ptr(), out.codes.stride(0),
                                       out.scale.data_ptr(), n, F, _stream_ptr()), "bns_cvt_rows_f32_fp8")
    return out


def _fp8_rows_like(n: int, F: int, device) -> Fp8Rows:
    """An uninitialised ``Fp8Rows`` of ``n`` rows of ``F`` codes, each code row 16-byte aligned."""
    return Fp8Rows(torch.empty(n, (F + 15) // 16 * 16, dtype=torch.float8_e4m3fn, device=device)[:, :F],
                   torch.empty(n, dtype=torch.float32, device=device))


def cvt_rows_fp8_any(src: torch.Tensor) -> Fp8Rows:
    """``bns_cvt_rows_f32_fp8_any``: ``cvt_rows_fp8`` (the same rule, bit for bit) for rows of any width ``F % 4 == 0``
    -- the GEMM operands of ``--dense-dtype fp8`` (K = 1204 or 44).  ``src``: 16-byte aligned, row stride a multiple
    of 4."""
    _req(src, torch.float32, "src")
    if src.dim() != 2 or src.stride(1) != 1:
        raise _lib.BnsError("src must be a row-major 2-D tensor")
    n, F = src.shape
    out = _fp8_rows_like(n, F, src.device)
    with torch.cuda.device(src.device):
        check(lib.bns_cvt_rows_f32_fp8_any(src.data_ptr(), src.stride(0), out.codes.data_ptr(), out.codes.stride(0),
                                           out.scale.data_ptr(), n, F, _stream_ptr()), "bns_cvt_rows_f32_fp8_any")
    return out


def cvt_rows_f32(src: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``bns_cvt_rows_bf16_f32``: bf16 rows widened to f32 (exact), into ``out`` or a new ``[rows, F]`` matrix.  An
    ``Fp8Rows`` ``src`` (``bns_cvt_rows_fp8_f32``) gives its codes times their scales (exact)."""
    fp8 = isinstance(src, Fp8Rows)
    if fp8:
        _table(src, "src")
    else:
        _req(src, torch.bfloat16, "src")
        if src.dim() != 2 or src.stride(1) != 1:
            raise _lib.BnsError("src must be a row-major 2-D tensor")
    n, F = src.shape
    if out is None:
        out = torch.empty(n, F, dtype=torch.float32, device=src.device)
    _req(out, torch.float32, "out")
    if out.shape != src.shape or out.stride(1) != 1:
        raise _lib.BnsError("out must be row-major with the shape of src")
    if fp8:
        with torch.cuda.device(src.device):
            check(lib.bns_cvt_rows_fp8_f32(src.codes.data_ptr(), src.codes.stride(0), src.scale.data_ptr(), out.data_ptr(),
                                           out.stride(0), n, F, _stream_ptr()), "bns_cvt_rows_fp8_f32")
        return out
    with torch.cuda.device(src.device):
        check(lib.bns_cvt_rows_bf16_f32(src.data_ptr(), src.stride(0), out.data_ptr(), out.stride(0), n, F, _stream_ptr()),
              "bns_cvt_rows_bf16_f32")
    return out


class BoundarySampler:
    """All peers' boundary samples in one call (``bns_sample_boundary``; replaces train.py:225-236)."""

    def __init__(self, boundary, send_size, device):
        segs = [(j, b) for j, b in enumerate(boundary) if b is not None]
        self.peers = [j for j, _ in segs]
        self.sizes = [int(send_size[j]) for j in self.peers]
        lens = [int(b.numel()) for _, b in segs]
        self.B, self.K = sum(lens), sum(self.sizes)
        self.device = device
        if segs:
            self.cat = torch.cat([b.to(device=device, dtype=torch.int64) for _, b in segs]).contiguous()
        else:
            self.cat = torch.empty(0, dtype=torch.int64, device=device)
        self.seg_begin = torch.tensor([0] + list(torch.tensor(lens).cumsum(0).tolist()) if lens else [0],
                                      dtype=torch.int64, device=device)
        self.out_begin_host = [0]
        for s in self.sizes:
            self.out_begin_host.append(self.out_begin_host[-1] + s)
        self.out_begin = torch.tensor(self.out_begin_host, dtype=torch.int64, device=device)
        self.ws = torch.empty(max(lib.bns_sample_workspace_bytes(self.B), 16), dtype=torch.uint8, device=device)
        self.world = len(boundary)

    def sample(self, seed: int, offset: int, offset_dev: Optional[torch.Tensor] = None):
        """Returns ``(selected_cat, [per-peer views or None])``.  ``offset_dev`` (int64 ``[1]`` on the device) is added
        to ``offset`` inside the kernel -- used when the epoch is replayed from a CUDA graph."""
        sel = torch.empty(self.K, dtype=torch.int64, device=self.device)
        if self.K:
            with torch.cuda.device(self.device):
                check(lib.bns_sample_boundary(self.cat.data_ptr(), self.seg_begin.data_ptr(), self.out_begin.data_ptr(),
                                              len(self.peers), self.B, self.K, seed & (2**64 - 1), offset & (2**64 - 1),
                                              _ptr(offset_dev), sel.data_ptr(), self.ws.data_ptr(), self.ws.numel(),
                                              _stream_ptr()), "bns_sample_boundary")
        views = [None] * self.world
        for i, j in enumerate(self.peers):
            views[j] = sel[self.out_begin_host[i]:self.out_begin_host[i + 1]]
        return sel, views


def fill_i32(t: torch.Tensor, value: int) -> None:
    _req(t, torch.int32, "t")
    with torch.cuda.device(t.device):
        check(lib.bns_fill_i32(t.data_ptr(), t.numel(), value, _stream_ptr()), "bns_fill_i32")


def halo_slot_update(pos: torch.Tensor, one_hops: torch.Tensor, n_in: int, slab_offset: int, slot: torch.Tensor) -> None:
    """``slot[pos[one_hops[k]] - n_in] = slab_offset + k`` (replaces train.py:268-275)."""
    _req(pos, torch.int64, "pos")
    _req(one_hops, torch.int64, "one_hops")
    _req(slot, torch.int32, "slot")
    with torch.cuda.device(slot.device):
        check(lib.bns_halo_slot_update(pos.data_ptr(), one_hops.data_ptr(), one_hops.numel(), n_in, slab_offset,
                                       slot.data_ptr(), _stream_ptr()), "bns_halo_slot_update")


def stamp_globaltimer(dst: torch.Tensor, stream: Optional[torch.cuda.Stream] = None) -> None:
    """Store the GPU's ``%globaltimer`` (nanoseconds) into the one-element int64 view ``dst`` on ``stream`` (default:
    the current stream) -- when the stream reaches this point, also inside a captured CUDA graph."""
    _req(dst, torch.int64, "dst")
    if dst.numel() != 1:
        raise _lib.BnsError(f"dst must be one element, got {dst.numel()}")
    s = stream if stream is not None else torch.cuda.current_stream(dst.device)
    with torch.cuda.device(dst.device):
        check(lib.bns_stamp_globaltimer(dst.data_ptr(), s.cuda_stream), "bns_stamp_globaltimer")


# ---- fused LayerNorm -> ReLU -> dropout --------------------------------------------------------------------------
# Philox stream of the dropout masks: (seed, offset [+ *offset_dev]); train.train_epoch sets it once per epoch
# (offset = epoch index; under CUDA-graph replay the epoch index comes from the device counter).
class _ThreadLocalRng:
    """dict-like, one instance per thread: ranks that live as threads of one process (tests, smoke, 1-GPU emulation)
    each set their own (seed, offset) in train.train_epoch and must not see each other's."""
    _DEFAULT = {"seed": 0, "offset": 0, "offset_dev": None}

    def __init__(self):
        import threading
        self._tls = threading.local()

    def _d(self):
        d = getattr(self._tls, "d", None)
        if d is None:
            d = self._tls.d = dict(self._DEFAULT)
        return d

    def __getitem__(self, k):
        return self._d()[k]

    def __setitem__(self, k, v):
        self._d()[k] = v

    def update(self, **kw):
        self._d().update(kw)


RNG = _ThreadLocalRng()
_LN_WS: Dict[tuple, torch.Tensor] = {}


class LnReluDropout(torch.autograd.Function):
    """``dropout_p(relu(layer_norm(x)))`` in one pass each way (``bns_ln_relu_dropout_{fwd,bwd}_f32``)."""

    @staticmethod
    def forward(ctx, x, gamma, beta, eps: float, p: float, seed: int, grad_slots=None, out=None):
        """``grad_slots = (dgamma, dbeta)``: destinations of the parameter gradients (slots of fused.ParamArena); the
        backward then writes them there and returns None for gamma / beta.  ``out``: where to write the result (the head
        rows of the next layer's concat buffer, ``Buffer.input_slot``: saves the copy of helper/feature_buffer.py:85-91)."""
        ctx.grad_slots = grad_slots
        x = x.contiguous()
        n, F = x.shape
        y = torch.empty_like(x) if out is None else out
        mean = torch.empty(n, dtype=torch.float32, device=x.device)
        rstd = torch.empty(n, dtype=torch.float32, device=x.device)
        off, off_dev = RNG["offset"], RNG["offset_dev"]
        with torch.cuda.device(x.device):
            check(lib.bns_ln_relu_dropout_fwd_f32(x.data_ptr(), x.stride(0), n, F, gamma.data_ptr(), beta.data_ptr(),
                                                  eps, p, seed & (2**64 - 1), off & (2**64 - 1), _ptr(off_dev),
                                                  y.data_ptr(), y.stride(0), mean.data_ptr(), rstd.data_ptr(),
                                                  _stream_ptr()), "bns_ln_relu_dropout_fwd_f32")
        ctx.save_for_backward(x, gamma, beta, mean, rstd)
        ctx.cfg = (eps, p, seed, off, off_dev)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, gamma, beta, mean, rstd = ctx.saved_tensors
        eps, p, seed, off, off_dev = ctx.cfg
        dy = dy.contiguous()
        n, F = x.shape
        dx = torch.empty_like(x)
        if ctx.grad_slots is not None:
            dgamma, dbeta = ctx.grad_slots
        else:
            dgamma, dbeta = torch.empty_like(gamma), torch.empty_like(beta)
        # per (device, width, stream): ranks that live as threads of one process (tests, smoke) run their backward
        # passes concurrently on their own streams and must not share the partial-sum scratch
        key = (x.device, F, torch.cuda.current_stream(x.device).cuda_stream)
        ws = _LN_WS.get(key)
        if ws is None:
            ws = _LN_WS[key] = torch.empty(lib.bns_ln_bwd_workspace_bytes(F), dtype=torch.uint8, device=x.device)
        with torch.cuda.device(x.device):
            check(lib.bns_ln_relu_dropout_bwd_f32(dy.data_ptr(), dy.stride(0), x.data_ptr(), x.stride(0), n, F,
                                                  gamma.data_ptr(), beta.data_ptr(), mean.data_ptr(), rstd.data_ptr(),
                                                  eps, p, seed & (2**64 - 1), off & (2**64 - 1), _ptr(off_dev),
                                                  dx.data_ptr(), dx.stride(0), dgamma.data_ptr(), dbeta.data_ptr(),
                                                  ws.data_ptr(), ws.numel(), _stream_ptr()), "bns_ln_relu_dropout_bwd_f32")
        if ctx.grad_slots is not None:
            return dx, None, None, None, None, None, None, None
        return dx, dgamma, dbeta, None, None, None, None, None


def ln_relu_dropout_supported(x: torch.Tensor, F: int) -> bool:
    return x.is_cuda and x.dtype == torch.float32 and x.dim() == 2 and F % 4 == 0 and F <= 1024


# ---- the multilevel partitioner (data/multilevel.py): thin wrappers over the bns_part_* entry points ----

def part_edges(indptr: torch.Tensor, idx: torch.Tensor, w: Optional[torch.Tensor], n_out_rows: int, mode: int,
               drop_loops: bool, row_map: Optional[torch.Tensor] = None, col_map: Optional[torch.Tensor] = None):
    """``bns_part_edges``: the merged (row_map[r], col_map[c]) CSR of a CSR; mode 0 as is, 1 transposed, 2 both.
    Returns (indptr int64, idx int32, w int32), trimmed to the merged entry count.  Synchronises."""
    _req(indptr, torch.int64, "indptr")
    _req(idx, torch.int32, "idx")
    for t, name in ((w, "w"), (row_map, "row_map"), (col_map, "col_map")):
        if t is not None:
            _req(t, torch.int32, name)
    nnz = idx.numel()
    cap = 2 * nnz if mode == 2 else nnz
    dev = indptr.device
    out_indptr = torch.empty(n_out_rows + 1, dtype=torch.int64, device=dev)
    out_idx = torch.empty(max(cap, 1), dtype=torch.int32, device=dev)
    out_w = torch.empty(max(cap, 1), dtype=torch.int32, device=dev)
    ws = torch.empty(max(int(lib.bns_part_edges_workspace_bytes(cap)), 1), dtype=torch.uint8, device=dev)
    n_out = ctypes.c_int64()
    check(lib.bns_part_edges(indptr.numel() - 1, nnz, indptr.data_ptr(), _ptr(idx) if nnz else None, _ptr(w),
                             _ptr(row_map), _ptr(col_map), mode, 1 if drop_loops else 0, n_out_rows,
                             out_indptr.data_ptr(), out_idx.data_ptr(), out_w.data_ptr(), ctypes.byref(n_out),
                             ws.data_ptr(), ws.numel(), _stream_ptr()), "bns_part_edges")
    m = n_out.value
    if m == 0:
        return out_indptr, out_idx[:0], out_w[:0]           # views of one element: their data pointers are not NULL
    return out_indptr, out_idx[:m].clone(), out_w[:m].clone()


def part_conn(indptr: torch.Tensor, idx: torch.Tensor, w: Optional[torch.Tensor], part: torch.Tensor, n_parts: int, *,
              table: bool = True, occ: bool = False, quality: bool = False):
    """``bns_part_conn``: (conn int32 [n, P] or None, occ int64 [n] bit sets or None, quality int64 [2] (cut, vol) or None)."""
    _req(part, torch.int32, "part")
    n, dev = part.numel(), part.device
    conn = torch.empty(n, n_parts, dtype=torch.int32, device=dev) if table else None
    o = torch.empty(n, dtype=torch.int64, device=dev) if occ else None
    q = torch.empty(2, dtype=torch.int64, device=dev) if quality else None
    check(lib.bns_part_conn(n, indptr.data_ptr(), idx.data_ptr(), _ptr(w), part.data_ptr(), n_parts, _ptr(conn), _ptr(o),
                            _ptr(q), _stream_ptr()), "bns_part_conn")
    return conn, o, q


def part_gains(objective: str, part: torch.Tensor, conn: torch.Tensor, n_parts: int, allowed: int, *,
               in_graph=None, occ: Optional[torch.Tensor] = None):
    """``bns_part_gains``: each node's best allowed target part (-1: none) and its exact gain (int64).  ``objective``
    "cut": conn of the undirected weighted graph; "vol": conn / occ of the out-CSR and ``in_graph`` = (indptr, idx, w)
    the in-CSR with multiplicities."""
    _req(part, torch.int32, "part")
    _req(conn, torch.int32, "conn")
    n, dev = part.numel(), part.device
    target = torch.empty(n, dtype=torch.int32, device=dev)
    gain = torch.empty(n, dtype=torch.int64, device=dev)
    ip, ix, iw = in_graph if in_graph is not None else (None, None, None)
    check(lib.bns_part_gains(1 if objective == "vol" else 0, n, n_parts, _ptr(ip), _ptr(ix), _ptr(iw), part.data_ptr(),
                             conn.data_ptr(), _ptr(occ), allowed & 0xFFFFFFFFFFFFFFFF, target.data_ptr(),
                             gain.data_ptr(), _stream_ptr()), "bns_part_gains")
    return target, gain


def part_cluster(rating, label: torch.Tensor, nw: Optional[torch.Tensor], cw: torch.Tensor, cap: int, seed: int, *,
                 ew: Optional[torch.Tensor] = None, ce: Optional[torch.Tensor] = None, ecap: int = 0):
    """``bns_part_cluster``: one size-constrained label-propagation proposal per node (target -1: stay).  With ``ew``
    (int64 in-edge weight per node), ``ce`` (the clusters' in-edge weights) and ``ecap``: ``bns_part_cluster_edges``,
    which also keeps every proposed cluster's in-edge weight within ``ecap``."""
    _req(label, torch.int32, "label")
    _req(cw, torch.int64, "cw")
    ip, cid, wt = rating
    n, dev = label.numel(), label.device
    target = torch.empty(n, dtype=torch.int32, device=dev)
    gain = torch.empty(n, dtype=torch.int64, device=dev)
    if ew is None:
        check(lib.bns_part_cluster(n, ip.data_ptr(), cid.data_ptr(), wt.data_ptr(), label.data_ptr(), _ptr(nw),
                                   cw.data_ptr(), int(cap), seed & 0xFFFFFFFFFFFFFFFF, target.data_ptr(),
                                   gain.data_ptr(), _stream_ptr()), "bns_part_cluster")
        return target, gain
    _req(ew, torch.int64, "ew")
    _req(ce, torch.int64, "ce")
    check(lib.bns_part_cluster_edges(n, ip.data_ptr(), cid.data_ptr(), wt.data_ptr(), label.data_ptr(), _ptr(nw),
                                     cw.data_ptr(), int(cap), ew.data_ptr(), ce.data_ptr(), int(ecap),
                                     seed & 0xFFFFFFFFFFFFFFFF, target.data_ptr(), gain.data_ptr(), _stream_ptr()),
          "bns_part_cluster_edges")
    return target, gain


def part_weights(label: torch.Tensor, nw: Optional[torch.Tensor], n_labels: int) -> torch.Tensor:
    """``bns_part_weights``: int64 [n_labels] sums of the node weights per label.  int32 or int64 weights (the latter
    through ``bns_part_weights_i64``: in-edge weights, whose coarse sums pass 2^31)."""
    _req(label, torch.int32, "label")
    out = torch.empty(n_labels, dtype=torch.int64, device=label.device)
    if nw is not None and nw.dtype == torch.int64:
        _req(nw, torch.int64, "nw")
        check(lib.bns_part_weights_i64(label.numel(), label.data_ptr(), nw.data_ptr(), n_labels, out.data_ptr(),
                                       _stream_ptr()), "bns_part_weights_i64")
        return out
    check(lib.bns_part_weights(label.numel(), label.data_ptr(), _ptr(nw), n_labels, out.data_ptr(), _stream_ptr()),
          "bns_part_weights")
    return out
