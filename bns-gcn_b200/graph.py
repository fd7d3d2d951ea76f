"""Graph handles passed to the layers in place of DGL graphs.

``PartitionGraph`` is what ``train.construct_graph`` returns: the reference rebuilds a bipartite ``_U -> _V``
``dgl.heterograph`` every epoch (train.py:256-281); here the structure is static -- ``a_in`` (inner -> inner) and
``a_out`` (halo -> inner), each with its transpose, all built once -- and an epoch only rewrites ``slot``:
``slot[h]`` = row of halo node ``h`` in this epoch's receive slab (U-numbering minus ``n_in``), or -1 when the
owner did not sample it.  Callers see the same surface the layers use: ``num_nodes('_V')``.

``FullGraphHandle`` is the homogeneous graph of the evaluation branch (module/layer.py:39-45, 93-102).
"""
from __future__ import annotations

from typing import Dict, Optional

import torch

from . import ops


class PartitionGraph:
    def __init__(self, n_in: int, n_halo: int, a_in: ops.DeviceGraph, a_out: Optional[ops.DeviceGraph], device):
        self.n_in, self.n_halo = n_in, n_halo
        self.a_in, self.a_out = a_in, a_out
        self.a_in_t = a_in.transpose()
        self.a_out_t = a_out.transpose() if a_out is not None else None
        self.device = device
        self.slot = torch.full((max(n_halo, 1),), -1, dtype=torch.int32, device=device)
        self.n_u = n_in
        self._recip: Dict[int, torch.Tensor] = {}
        # per-epoch compaction of a_out to the sampled halo columns (ops.CompactedCols), refreshed by construct_graph
        self.compact: Optional[ops.CompactedCols] = None
        self.halo_col_scale: Optional[torch.Tensor] = None      # GCN: 1/sqrt(out_deg) of the halo nodes (static)
        self.want_positions = False                             # GAT: the compaction also records CSR positions
        # --agg-dtype bf16 / fp8: the fused layers' wide aggregation passes gather bf16 copies, or fp8 tables
        # (ops.Fp8Rows), of their source rows (fused._gather_table); at most one of the two is set
        self.agg_bf16 = False
        self.agg_fp8 = False

    def refresh_compaction(self) -> None:
        """Call after every change of ``slot`` (train.construct_graph does)."""
        if self.a_out is None or self.a_out.nnz == 0:
            return
        if self.compact is None:
            self.compact = ops.CompactedCols(self.a_out, with_weights=self.halo_col_scale is not None,
                                             with_positions=self.want_positions)
        self.compact.refresh(self.slot, 0, self.halo_col_scale)

    def num_nodes(self, ntype: str = '_V') -> int:
        return self.n_in if ntype == '_V' else self.n_u

    def num_edges(self) -> int:
        return self.a_in.nnz + (self.a_out.nnz if self.a_out is not None else 0)

    def recip(self, t: torch.Tensor) -> torch.Tensor:
        """``1 / t`` as f32, cached per source tensor (degree / norm vectors are static)."""
        # keyed on the tensor OBJECT (kept alive here, so its id cannot be recycled) and its in-place version counter:
        # a freed-and-reallocated buffer at the same address, or a norm updated in place, never returns a stale value
        key = id(t)
        hit = self._recip.get(key)
        if hit is None or hit[0] is not t or hit[1] != t._version:
            hit = (t, t._version, (1.0 / t.to(torch.float32)).contiguous())
            self._recip[key] = hit
        return hit[2]


class FullGraphHandle:
    def __init__(self, a: ops.DeviceGraph, in_deg: torch.Tensor, out_deg: torch.Tensor):
        self.a = a
        self._in, self._out = in_deg, out_deg

    def num_nodes(self, ntype: str = '_V') -> int:
        return self.a.n_rows

    def in_degrees(self):
        return self._in

    def out_degrees(self):
        return self._out

    def has_zero_in_degree(self) -> bool:
        """Whether some node has no in-edge (checked once: it synchronises with the device)."""
        if getattr(self, "_zero_in", None) is None:
            self._zero_in = bool((self._in == 0).any())
        return self._zero_in


class PartitionEvalGraph:
    """This rank's partition with EVERY halo node present: the graph of the partition-parallel evaluation
    (``evaluate.ParallelEvaluator``).  Every inner node holds all its in-edges and full-graph degrees, so with the whole
    boundary exchanged (sampling ratio 1) the forward over the inner rows equals the whole-graph forward (SURVEY §4).

    ``a_in`` (inner -> inner) and ``blocks[j]``: the columns of ``a_out`` owned by peer ``j`` (the halo is sorted by
    global id, so each owner's columns are one contiguous range, ``halo_begin[j]`` onwards), renumbered from 0.
    ``peer_rows(h)`` exchanges one peer at a time -- send ``h[boundary[right]]``, receive the left peer's rows -- so a
    layer's extra memory is one peer's rows, not the whole halo.  Every rank must walk ``peer_rows`` in step: it is
    collective.

    The blocks are cut from ``a_out`` at the first evaluation, not when the handle is made, so training before it runs
    at its own peak; they stay for the later evaluations: ``a_out``'s column ids once more (4 bytes per halo entry) and
    one row-offset array per peer (8 bytes per inner node and peer)."""

    EXCHANGE_TAG = 3000

    def __init__(self, a_in: ops.DeviceGraph, a_out: Optional[ops.DeviceGraph], halo_counts, boundary, in_deg: torch.Tensor,
                 out_deg: torch.Tensor, comm):
        self.a_in, self.n_in = a_in, a_in.n_rows
        self.comm, self.rank, self.size = comm, comm.rank, comm.size
        self.boundary = boundary
        self.halo_count = [0 if c is None else int(c) for c in halo_counts]
        self.halo_begin, tot = [], 0
        for c in self.halo_count:
            self.halo_begin.append(tot)
            tot += c
        self.n_halo = tot
        self._in, self._out = in_deg, out_deg               # full-graph degrees: [inner], [inner | halo]
        dev = in_deg.device
        # the peers in the order of the exchange steps (a ring, as precompute_streaming): a fixed summation order
        self.order = [(self.rank - i + self.size) % self.size for i in range(1, self.size)]
        self._a_out = a_out
        self._blocks: Optional[Dict[int, ops.DeviceGraph]] = None
        # decided over ALL ranks: a layer that refuses such a graph must refuse it on every rank, or the others hang
        zero = torch.tensor([float(bool((in_deg == 0).any()))], dtype=torch.float32, device=dev)
        comm.all_reduce_sum(zero)
        self._zero_in = bool(zero.item() > 0)

    @property
    def blocks(self) -> Dict[int, ops.DeviceGraph]:
        """``blocks[j]``: the entries of ``a_out`` whose column peer ``j`` owns, columns renumbered from 0."""
        if self._blocks is None:
            a_out, n_in, dev = self._a_out, self.n_in, self._in.device
            blocks = {}
            if a_out is not None and a_out.nnz:
                ip, ix = a_out.csr()
                rows = torch.repeat_interleave(torch.arange(n_in, dtype=torch.int32, device=dev), ip[1:] - ip[:-1])
                del ip
            for j in self.order:
                b0, cnt = self.halo_begin[j], self.halo_count[j]
                ipb = torch.zeros(n_in + 1, dtype=torch.int64, device=dev)
                if a_out is not None and a_out.nnz:
                    m = (ix >= b0) & (ix < b0 + cnt)
                    ipb[1:] = torch.cumsum(torch.bincount(rows[m], minlength=n_in), 0)
                    idx = ix[m] - b0
                    del m
                else:
                    idx = torch.empty(0, dtype=torch.int32, device=dev)
                blocks[j] = ops.DeviceGraph.from_csr(ipb, idx, cnt)
                del ipb, idx
            self._blocks = blocks
        return self._blocks

    def num_nodes(self, ntype: str = '_V') -> int:
        return self.n_in

    def in_degrees(self):
        return self._in

    def out_degrees(self):
        return self._out

    def has_zero_in_degree(self) -> bool:
        """Whether some node of the whole graph has no in-edge (the same answer on every rank)."""
        return self._zero_in

    def peer_rows(self, h: torch.Tensor):
        """Yields ``(j, blocks[j], rows of h of j's nodes that are my halo)`` for each peer ``j`` in ``order``, one
        exchange per step (``h``: this rank's inner rows)."""
        dev, blocks = h.device, self.blocks
        for i, left in enumerate(self.order, start=1):
            right = (self.rank + i) % self.size
            send, recv = [None] * self.size, [None] * self.size
            send[right] = h[self.boundary[right]]
            recv[left] = torch.empty(self.halo_count[left], h.shape[1], dtype=h.dtype, device=dev)
            self.comm.alltoall(send, recv, tag=self.EXCHANGE_TAG + i)
            yield left, blocks[left], recv[left]
            del send, recv

    def aggregate(self, x: torch.Tensor, rs: torch.Tensor, cs: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``rs * (A_in (cs_in * x) + sum_j A_j (cs_j * x_j))`` over the inner rows: the whole-graph ``AggregateSum``
        restricted to them (``cs`` over ``[inner | halo]``, ``x`` the inner rows; the halo rows arrive peer by peer)."""
        n_in = self.n_in
        x = x.contiguous()
        # the column scale rides in the gather (no scaled copy of x or of a peer's rows)
        y = ops.spmm_auto(self.a_in, x, row_scale=rs, col_scale=None if cs is None else cs[:n_in])
        for j, blk, xr in self.peer_rows(x):
            if blk.nnz == 0:
                continue
            b0 = n_in + self.halo_begin[j]
            ops.spmm(blk, xr, y, row_scale=rs, col_scale=None if cs is None else cs[b0:b0 + self.halo_count[j]],
                     accumulate=True)
        return y


def halo_aggregate(g: PartitionGraph, x_halo: torch.Tensor, y: torch.Tensor, rs, cs_halo) -> None:
    """``y += rs * A_out[:, sampled] (cs_halo * x_halo)``.  With the epoch's compaction (the default) the kernel walks
    the sampled entries only; without it (a graph whose slot map was set by hand) every halo entry is looked up."""
    c = g.compact
    if c is not None and (c.cw is not None) == (cs_halo is not None):
        ops.spmm_compact(c, x_halo, y, row_scale=rs, accumulate=True)
    else:
        ops.spmm(g.a_out, x_halo, y, row_scale=rs, col_scale=cs_halo, col_map=g.slot, n_direct=0, accumulate=True)


class PartitionAggregate(torch.autograd.Function):
    """K1 + K2 (+ K1b in backward) on a ``PartitionGraph``:

        Y = rs * ( A_in (cs_in * H_U[:n_in])  +  A_out[:, sampled] (cs_halo * H_U[n_in:]) )

    The inner-edge pass only needs the local rows, so it is issued first; the halo pass waits for the exchange
    (``ready`` event recorded by ``Buffer.update(..., overlap=True)``) -- that is the comm/compute overlap.
    """

    @staticmethod
    def forward(ctx, h_u, g: PartitionGraph, rs, cs_in, cs_halo, ready):
        ctx.g, ctx.rs, ctx.cs_in, ctx.cs_halo = g, rs, cs_in, cs_halo
        ctx.n_u = h_u.shape[0]
        h_u = h_u.contiguous()
        # a per-source scale is applied ONCE per row here, not once per edge inside the gather (each source row is
        # gathered ~degree times; the fused col_scale path costs an extra scalar gather per edge)
        x_in = h_u[:g.n_in] if cs_in is None else h_u[:g.n_in] * cs_in.unsqueeze(1)
        y = ops.spmm_auto(g.a_in, x_in, row_scale=rs)
        if ready is not None:
            torch.cuda.current_stream(h_u.device).wait_event(ready)
        if g.a_out is not None and ctx.n_u > g.n_in:
            halo_aggregate(g, h_u[g.n_in:], y, rs, cs_halo)
        return y

    @staticmethod
    def backward(ctx, dy):
        g = ctx.g
        dy = dy.contiguous() if ctx.rs is None else dy * ctx.rs.unsqueeze(1)      # pre-scale once (see forward)
        du = torch.empty(ctx.n_u, dy.shape[1], dtype=torch.float32, device=dy.device)
        if ctx.n_u > g.n_in:
            tail = du[g.n_in:]
            tail.zero_()
            if g.a_out_t is not None:
                ops.spmm(g.a_out_t, dy, tail, row_scale=ctx.cs_halo, row_map=g.slot)
        ops.spmm_auto(g.a_in_t, dy, du[:g.n_in], row_scale=ctx.cs_in)
        return du, None, None, None, None, None


_PROJ_WS = {}


class GatProjection(torch.autograd.Function):
    """``el = <ft_src, attn_l>``, ``er = <ft_dst, attn_r>`` per head (the two ``(feat * attn).sum(-1)`` of
    ``dgl.nn.GATConv``) on ``bns_gat_proj_f32``; the backward (``bns_gat_proj_bwd_f32``) makes ``d ft = s (x) attn`` and
    the deterministic ``d attn = sum_r s_r ft_r`` in one pass over ``ft`` each."""

    @staticmethod
    def forward(ctx, ft_src, ft_dst, attn_l, attn_r, H: int, Fo: int):
        from ._lib import check, lib
        ft_src, ft_dst = ft_src.contiguous(), ft_dst.contiguous()
        al, ar = attn_l.reshape(-1).contiguous(), attn_r.reshape(-1).contiguous()
        dev = ft_src.device
        el = torch.empty(ft_src.shape[0], H, dtype=torch.float32, device=dev)
        er = torch.empty(ft_dst.shape[0], H, dtype=torch.float32, device=dev)
        st = torch.cuda.current_stream(dev).cuda_stream
        with torch.cuda.device(dev):
            check(lib.bns_gat_proj_f32(ft_src.data_ptr(), ft_src.stride(0), ft_src.shape[0], H, Fo, al.data_ptr(), el.data_ptr(),
                                       st), "bns_gat_proj_f32")
            check(lib.bns_gat_proj_f32(ft_dst.data_ptr(), ft_dst.stride(0), ft_dst.shape[0], H, Fo, ar.data_ptr(), er.data_ptr(),
                                       st), "bns_gat_proj_f32")
        ctx.save_for_backward(ft_src, ft_dst, al, ar)
        ctx.cfg = (H, Fo, attn_l.shape)
        return el, er

    @staticmethod
    def backward(ctx, d_el, d_er):
        from ._lib import check, lib
        ft_src, ft_dst, al, ar = ctx.saved_tensors
        H, Fo, shape = ctx.cfg
        dev = ft_src.device
        st = torch.cuda.current_stream(dev).cuda_stream
        key = (dev, H * Fo, st)
        ws = _PROJ_WS.get(key)
        if ws is None:
            ws = _PROJ_WS[key] = torch.empty(lib.bns_colsum_workspace_bytes(H * Fo), dtype=torch.uint8, device=dev)
        outs = []
        with torch.cuda.device(dev):
            for ft, a, s in ((ft_src, al, d_el), (ft_dst, ar, d_er)):
                s = s.contiguous()
                d_ft = torch.empty_like(ft)
                d_a = torch.empty_like(a)
                check(lib.bns_gat_proj_bwd_f32(ft.data_ptr(), ft.stride(0), ft.shape[0], H, Fo, a.data_ptr(), s.data_ptr(),
                                               d_ft.data_ptr(), d_ft.stride(0), 0, d_a.data_ptr(), ws.data_ptr(), ws.numel(),
                                               st), "bns_gat_proj_bwd_f32")
                outs.append((d_ft, d_a.view(shape)))
        return outs[0][0], outs[1][0], outs[0][1], outs[1][1], None, None


class GatAttention(torch.autograd.Function):
    """The attention of ``dgl.nn.GATConv`` for all heads:

        rst_v = sum_u attn_drop(edge_softmax(leaky_relu(el_u + er_v)))_uv * ft_u

    over the inner entries and this epoch's sampled halo entries (the partition graph's compaction with positions).
    ``ft [n_u, H * Fo]``, ``el [n_u, H]``, ``er [n_in, H]`` -> ``[n_in, H * Fo]``; gradients for all three.

    Stages (include/bnsgcn.h): ``bns_gat_scores_f32`` (scalars: probabilities + dropped attention per entry) ->
    ``bns_spmm_weighted_f32`` / ``bns_spmm_compact_f32`` per head; backward ``bns_sddmm_dot_f32`` ->
    ``bns_gat_softmax_bwd_f32`` -> ``bns_gat_colsum_f32`` -> ``bns_spmm_weighted_f32`` on the transposes."""

    @staticmethod
    def forward(ctx, ft, el, er, g: PartitionGraph, H: int, Fo: int, slope: float, p: float, seed: int):
        from ._lib import check, lib
        ft, el, er = ft.contiguous(), el.contiguous(), er.contiguous()
        n_in, dev = g.n_in, ft.device
        c = g.compact if (g.a_out is not None and ft.shape[0] > n_in) else None
        if c is None and g.a_out is not None and g.a_out.nnz and ft.shape[0] > n_in:
            raise RuntimeError("GatAttention: halo rows were passed but the partition graph has no compaction "
                               "(refresh_compaction)")
        if c is not None and c.cpos is None:
            raise RuntimeError("GatAttention: the partition graph was compacted without positions (want_positions)")
        rst = torch.empty(n_in, H * Fo, dtype=torch.float32, device=dev)
        p_in = torch.empty(max(g.a_in.nnz, 1), H, dtype=torch.float32, device=dev)
        p_out = torch.empty(max(g.a_out.nnz, 1), H, dtype=torch.float32, device=dev) if c is not None else None
        w_in = torch.empty_like(p_in) if p > 0 else None
        w_out = torch.empty_like(p_out) if p > 0 and p_out is not None else None
        wc = torch.empty_like(p_out) if p_out is not None else None              # halo attention, compacted positions
        off, off_dev = ops.RNG["offset"], ops.RNG["offset_dev"]
        head = (g.a_in._h, None if c is None else g.a_out._h, None if c is None else c.cidx.data_ptr(),
                None if c is None else c.chunk_cnt.data_ptr(), None if c is None else c.cpos.data_ptr(), n_in)
        tail = (H, el.data_ptr(), er.data_ptr(), float(slope), float(p), seed & (2 ** 64 - 1), off & (2 ** 64 - 1),
                ops._ptr(off_dev))
        st = torch.cuda.current_stream(dev).cuda_stream
        with torch.cuda.device(dev):
            check(lib.bns_gat_scores_f32(*head, *tail, p_in.data_ptr(), ops._ptr(p_out), ops._ptr(w_in), ops._ptr(w_out),
                                         ops._ptr(wc), st), "bns_gat_scores_f32")
        for h in range(H):
            cols = slice(h * Fo, (h + 1) * Fo)
            ops.spmm_weighted(g.a_in, ft[:n_in, cols], rst[:, cols], p_in if w_in is None else w_in, h)
            if c is not None:
                ops.spmm_compact(c, ft[n_in:, cols], rst[:, cols], accumulate=True, weights=wc, head=h)
        ctx.g, ctx.c, ctx.head, ctx.tail, ctx.cfg = g, c, head, tail, (H, Fo)
        saved = [ft, el, er, p_in] + ([p_out] if p_out is not None else [])
        if w_in is not None:
            saved += [w_in] + ([w_out] if w_out is not None else [])
        ctx.n_w = 0 if w_in is None else (2 if w_out is not None else 1)
        ctx.save_for_backward(*saved)
        return rst

    @staticmethod
    def backward(ctx, d_rst):
        from ._lib import check, lib
        g, c = ctx.g, ctx.c
        H, Fo = ctx.cfg
        ft, el, er, p_in, *rest = ctx.saved_tensors
        p_out = rest.pop(0) if c is not None else None
        d_rst = d_rst.contiguous()
        dev, n_in, n_u = ft.device, g.n_in, ft.shape[0]
        de_in = torch.empty_like(p_in)
        de_out = torch.empty_like(p_out) if p_out is not None else None
        d_er = torch.empty(n_in, H, dtype=torch.float32, device=dev)
        st = torch.cuda.current_stream(dev).cuda_stream
        w_in, w_out = p_in, p_out
        if ctx.n_w:
            w_in = rest.pop(0)
            w_out = rest.pop(0) if ctx.n_w == 2 else None
        for h in range(H):                                     # d a'_uv = <d rst_v, ft_u> (0 for an unsampled halo node)
            cols = slice(h * Fo, (h + 1) * Fo)
            ops.sddmm_dot(g.a_in, d_rst[:, cols], ft[:n_in, cols], out=de_in[:, h])
            if c is not None:
                ops.sddmm_dot(g.a_out, d_rst[:, cols], ft[n_in:, cols], col_map=g.slot, n_direct=0, out=de_out[:, h])
        with torch.cuda.device(dev):
            check(lib.bns_gat_softmax_bwd_f32(*ctx.head, *ctx.tail, p_in.data_ptr(), ops._ptr(p_out), de_in.data_ptr(),
                                              ops._ptr(de_out), d_er.data_ptr(), st), "bns_gat_softmax_bwd_f32")
        with torch.cuda.device(dev):
            d_el = torch.empty(n_u, H, dtype=torch.float32, device=dev)
            check(lib.bns_gat_colsum_f32(g.a_in_t._h, de_in.data_ptr(), H, None, 0, d_el.data_ptr(), st),
                  "bns_gat_colsum_f32")
            if c is not None:
                check(lib.bns_gat_colsum_f32(g.a_out_t._h, de_out.data_ptr(), H, g.slot.data_ptr(), n_in, d_el.data_ptr(),
                                             st), "bns_gat_colsum_f32")
        d_ft = torch.empty(n_u, H * Fo, dtype=torch.float32, device=dev)
        for h in range(H):
            cols = slice(h * Fo, (h + 1) * Fo)
            ops.spmm_weighted(g.a_in_t, d_rst[:, cols], d_ft[:n_in, cols], w_in, h, through_perm=True)
            if c is not None:
                ops.spmm_weighted(g.a_out_t, d_rst[:, cols], d_ft[n_in:, cols], w_out, h, through_perm=True,
                                  row_map=g.slot)
        return d_ft, d_el, d_er, None, None, None, None, None, None


GAT_MAX_HEADS, GAT_MAX_WIDTH = 8, 1024


def gat_padded_width(Fo: int) -> int:
    """The per-head width rounded up to a multiple of 4 (16-byte lanes)."""
    return (Fo + 3) // 4 * 4


def gat_unsupported(H: int, Fo: int) -> Optional[str]:
    """``None`` when the GAT kernels (``bns_gat_proj_f32``, ``bns_gat_scores_f32``, ``bns_gat_infer_f32``) take ``H``
    heads of width ``Fo`` padded to a multiple of 4, else the limit that is exceeded."""
    if not 1 <= H <= GAT_MAX_HEADS:
        return f"heads = {H} is outside 1..{GAT_MAX_HEADS}"
    if Fo < 1 or H * gat_padded_width(Fo) > GAT_MAX_WIDTH:
        return (f"heads * padded per-head width = {H} * {gat_padded_width(Fo)} exceeds {GAT_MAX_WIDTH}"
                if Fo >= 1 else f"per-head width {Fo} < 1")
    return None


def gat_infer(a: ops.DeviceGraph, ft: torch.Tensor, el: torch.Tensor, er: torch.Tensor, H: int, Fp: int, slope: float,
              bias: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The evaluation forward of ``dgl.nn.GATConv``'s attention on a homogeneous graph ``a`` (``bns_gat_infer_f32``):

        rst[v, h, :] = sum_{u -> v} softmax_u(leaky_relu(el[u, h] + er[v, h], slope)) * ft[u, h, :] + bias[h, :]

    ``ft [a.n_cols, H * Fp]`` (head-major, ``Fp`` a multiple of 4, pad columns zero), ``el [a.n_cols, H]``,
    ``er [a.n_rows, H]``, ``bias [H * Fp]`` or None -> ``[a.n_rows, H * Fp]``.  No dropout, no gradient."""
    from ._lib import BnsError, check, lib
    why = gat_unsupported(H, Fp)
    if why is not None or Fp % 4:
        raise BnsError(f"gat_infer: {why or f'padded width {Fp} is not a multiple of 4'}")
    for t, name in ((ft, "ft"), (el, "el"), (er, "er")) + (((bias, "bias"),) if bias is not None else ()):
        ops._req(t, torch.float32, name)
        if t.device != a.device:
            raise BnsError(f"gat_infer: {name} is on {t.device}, the graph on {a.device}")
    if ft.dim() != 2 or tuple(ft.shape) != (a.n_cols, H * Fp) or ft.stride(1) != 1:
        raise BnsError(f"gat_infer: ft must be [{a.n_cols}, {H * Fp}] with unit column stride, got {tuple(ft.shape)}")
    if tuple(el.shape) != (a.n_cols, H) or tuple(er.shape) != (a.n_rows, H):
        raise BnsError(f"gat_infer: el / er must be [{a.n_cols}, {H}] / [{a.n_rows}, {H}], got {tuple(el.shape)} / "
                       f"{tuple(er.shape)}")
    if bias is not None and tuple(bias.shape) != (H * Fp,):
        raise BnsError(f"gat_infer: bias must be [{H * Fp}], got {tuple(bias.shape)}")
    el, er = el.contiguous(), er.contiguous()
    bias = bias.contiguous() if bias is not None else None
    rst = torch.empty(a.n_rows, H * Fp, dtype=torch.float32, device=a.device)
    with torch.cuda.device(a.device):
        check(lib.bns_gat_infer_f32(a._h, ft.data_ptr(), ft.stride(0), H, Fp, el.data_ptr(), er.data_ptr(), float(slope),
                                    ops._ptr(bias), rst.data_ptr(), rst.stride(0),
                                    torch.cuda.current_stream(a.device).cuda_stream), "bns_gat_infer_f32")
    return rst


def gat_infer_block(a: ops.DeviceGraph, ft: Optional[torch.Tensor], el: Optional[torch.Tensor], er: torch.Tensor, H: int,
                    Fp: int, slope: float, m: torch.Tensor, l: torch.Tensor, acc: torch.Tensor, first: bool, last: bool,
                    bias: Optional[torch.Tensor] = None, rst: Optional[torch.Tensor] = None) -> None:
    """One column block of ``gat_infer`` (``bns_gat_infer_block_f32``): the rows' online-softmax state ``m``, ``l``
    ``[a.n_rows, H]`` and ``acc [a.n_rows, H * Fp]`` is carried from the previous block (``first``: from empty);
    ``last`` writes ``acc / l + bias`` to ``rst`` (which may be ``acc`` itself, same rows and stride).  ``ft [a.n_cols, H * Fp]`` / ``el
    [a.n_cols, H]`` are this block's source rows (may be None when the block has no entries), ``er`` the rows' own."""
    from ._lib import BnsError, check, lib
    why = gat_unsupported(H, Fp)
    if why is not None or Fp % 4:
        raise BnsError(f"gat_infer_block: {why or f'padded width {Fp} is not a multiple of 4'}")
    if a.nnz and (ft is None or el is None):
        raise BnsError("gat_infer_block: a block with entries needs ft and el")
    if last and rst is None:
        raise BnsError("gat_infer_block: the last block needs rst")
    HF = H * Fp
    for t, name, shape in ((ft, "ft", (a.n_cols, HF)), (el, "el", (a.n_cols, H)), (er, "er", (a.n_rows, H)),
                           (m, "m", (a.n_rows, H)), (l, "l", (a.n_rows, H)), (acc, "acc", (a.n_rows, HF)),
                           (bias, "bias", (HF,)), (rst, "rst", (a.n_rows, HF))):
        if t is None:
            continue
        ops._req(t, torch.float32, name)
        if t.device != a.device:
            raise BnsError(f"gat_infer_block: {name} is on {t.device}, the graph on {a.device}")
        if tuple(t.shape) != shape or t.stride(-1) != 1 or (t.dim() == 2 and name in ("el", "er", "m", "l")
                                                               and not t.is_contiguous()):
            raise BnsError(f"gat_infer_block: {name} must be {list(shape)} with unit column stride, got "
                           f"{tuple(t.shape)}")
    with torch.cuda.device(a.device):
        check(lib.bns_gat_infer_block_f32(a._h, ops._ptr(ft), ft.stride(0) if ft is not None else HF, H, Fp, ops._ptr(el),
                                          er.data_ptr(), float(slope), m.data_ptr(), l.data_ptr(), acc.data_ptr(),
                                          acc.stride(0), 1 if first else 0, 1 if last else 0, ops._ptr(bias),
                                          ops._ptr(rst), rst.stride(0) if rst is not None else HF,
                                          torch.cuda.current_stream(a.device).cuda_stream), "bns_gat_infer_block_f32")


_GATV2_WS = {}


class Gatv2Attention(torch.autograd.Function):
    """The attention of ``dgl.nn.GATv2Conv`` (``share_weights=False``) for all heads:

        s_uv = sum_f attn[h, f] * leaky_relu(z_src[u, h, f] + z_dst[v, h, f])
        rst_v = sum_u attn_drop(edge_softmax(s))_uv * z_src[u]

    over the inner entries and this epoch's sampled halo entries, as ``GatAttention``.  ``zs [n_u, H * Fp]``,
    ``zd [n_in, H * Fp]``, ``attn [1, H, Fp]`` (per-head widths padded to ``Fp``, pad columns zero) -> ``[n_in, H * Fp]``;
    gradients for all three.

    Stages (include/bnsgcn.h, ABI 13): ``bns_gatv2_scores_f32`` (F-wide scores -> probabilities + dropped attention per
    entry) -> ``bns_spmm_weighted_f32`` / ``bns_spmm_compact_f32`` per head; backward ``bns_sddmm_dot_f32`` ->
    ``bns_gatv2_softmax_bwd_f32`` (d s, d z_dst, d attn) -> ``bns_spmm_weighted_f32`` on the transposes +
    ``bns_gatv2_colsum_f32`` (d z_src)."""

    @staticmethod
    def forward(ctx, zs, zd, attn, g: PartitionGraph, H: int, Fp: int, slope: float, p: float, seed: int):
        from ._lib import check, lib
        zs, zd = zs.contiguous(), zd.contiguous()
        av = attn.reshape(-1).contiguous()
        n_in, dev = g.n_in, zs.device
        c = g.compact if (g.a_out is not None and zs.shape[0] > n_in) else None
        if c is None and g.a_out is not None and g.a_out.nnz and zs.shape[0] > n_in:
            raise RuntimeError("Gatv2Attention: halo rows were passed but the partition graph has no compaction "
                               "(refresh_compaction)")
        if c is not None and c.cpos is None:
            raise RuntimeError("Gatv2Attention: the partition graph was compacted without positions (want_positions)")
        rst = torch.empty(n_in, H * Fp, dtype=torch.float32, device=dev)
        p_in = torch.empty(max(g.a_in.nnz, 1), H, dtype=torch.float32, device=dev)
        p_out = torch.empty(max(g.a_out.nnz, 1), H, dtype=torch.float32, device=dev) if c is not None else None
        w_in = torch.empty_like(p_in) if p > 0 else None
        w_out = torch.empty_like(p_out) if p > 0 and p_out is not None else None
        wc = torch.empty_like(p_out) if p_out is not None else None
        off, off_dev = ops.RNG["offset"], ops.RNG["offset_dev"]
        head = (g.a_in._h, None if c is None else g.a_out._h, None if c is None else c.cidx.data_ptr(),
                None if c is None else c.chunk_cnt.data_ptr(), None if c is None else c.cpos.data_ptr(), n_in, H, Fp)
        tail = (zs.data_ptr(), zs.stride(0), zd.data_ptr(), zd.stride(0), av.data_ptr(), float(slope), float(p),
                seed & (2 ** 64 - 1), off & (2 ** 64 - 1), ops._ptr(off_dev))
        st = torch.cuda.current_stream(dev).cuda_stream
        with torch.cuda.device(dev):
            check(lib.bns_gatv2_scores_f32(*head, *tail, p_in.data_ptr(), ops._ptr(p_out), ops._ptr(w_in),
                                           ops._ptr(w_out), ops._ptr(wc), st), "bns_gatv2_scores_f32")
        for h in range(H):
            cols = slice(h * Fp, (h + 1) * Fp)
            ops.spmm_weighted(g.a_in, zs[:n_in, cols], rst[:, cols], p_in if w_in is None else w_in, h)
            if c is not None:
                ops.spmm_compact(c, zs[n_in:, cols], rst[:, cols], accumulate=True, weights=wc, head=h)
        ctx.g, ctx.c, ctx.head, ctx.tail, ctx.cfg = g, c, head, tail, (H, Fp, slope, attn.shape)
        saved = [zs, zd, av, p_in] + ([p_out] if p_out is not None else [])
        if w_in is not None:
            saved += [w_in] + ([w_out] if w_out is not None else [])
        ctx.n_w = 0 if w_in is None else (2 if w_out is not None else 1)
        ctx.save_for_backward(*saved)
        return rst

    @staticmethod
    def backward(ctx, d_rst):
        from ._lib import check, lib
        g, c = ctx.g, ctx.c
        H, Fp, slope, shape = ctx.cfg
        zs, zd, av, p_in, *rest = ctx.saved_tensors
        p_out = rest.pop(0) if c is not None else None
        d_rst = d_rst.contiguous()
        dev, n_in, n_u = zs.device, g.n_in, zs.shape[0]
        de_in = torch.empty_like(p_in)
        de_out = torch.empty_like(p_out) if p_out is not None else None
        w_in, w_out = p_in, p_out
        if ctx.n_w:
            w_in = rest.pop(0)
            w_out = rest.pop(0) if ctx.n_w == 2 else None
        for h in range(H):                                     # d a'_uv = <d rst_v, z_src[u]>
            cols = slice(h * Fp, (h + 1) * Fp)
            ops.sddmm_dot(g.a_in, d_rst[:, cols], zs[:n_in, cols], out=de_in[:, h])
            if c is not None:
                ops.sddmm_dot(g.a_out, d_rst[:, cols], zs[n_in:, cols], col_map=g.slot, n_direct=0, out=de_out[:, h])
        d_zd = torch.empty(n_in, H * Fp, dtype=torch.float32, device=dev)
        d_attn = torch.empty(H * Fp, dtype=torch.float32, device=dev)
        st = torch.cuda.current_stream(dev).cuda_stream
        with torch.cuda.device(dev):                           # the workspace's size follows this device's SM count
            need = lib.bns_gatv2_bwd_workspace_bytes(n_in, H, Fp)
            key = (dev, need, st)
            ws = _GATV2_WS.get(key)
            if ws is None:
                ws = _GATV2_WS[key] = torch.empty(max(need, 16), dtype=torch.uint8, device=dev)
            check(lib.bns_gatv2_softmax_bwd_f32(*ctx.head, *ctx.tail, p_in.data_ptr(), ops._ptr(p_out), de_in.data_ptr(),
                                                ops._ptr(de_out), d_zd.data_ptr(), d_zd.stride(0), d_attn.data_ptr(),
                                                ws.data_ptr(), ws.numel(), st), "bns_gatv2_softmax_bwd_f32")
        d_zs = torch.empty(n_u, H * Fp, dtype=torch.float32, device=dev)
        for h in range(H):                                     # A'^T d rst
            cols = slice(h * Fp, (h + 1) * Fp)
            ops.spmm_weighted(g.a_in_t, d_rst[:, cols], d_zs[:n_in, cols], w_in, h, through_perm=True)
            if c is not None:
                ops.spmm_weighted(g.a_out_t, d_rst[:, cols], d_zs[n_in:, cols], w_out, h, through_perm=True,
                                  row_map=g.slot)
        zargs = (zs.data_ptr(), zs.stride(0), zd.data_ptr(), zd.stride(0), av.data_ptr(), float(slope))
        with torch.cuda.device(dev):                           # + the score's share of d z_src
            check(lib.bns_gatv2_colsum_f32(g.a_in_t._h, de_in.data_ptr(), H, Fp, *zargs, None, 0, d_zs.data_ptr(),
                                           d_zs.stride(0), st), "bns_gatv2_colsum_f32")
            if c is not None:
                check(lib.bns_gatv2_colsum_f32(g.a_out_t._h, de_out.data_ptr(), H, Fp, *zargs, g.slot.data_ptr(), n_in,
                                               d_zs.data_ptr(), d_zs.stride(0), st), "bns_gatv2_colsum_f32")
        return d_zs, d_zd, d_attn.view(shape), None, None, None, None, None, None


def _gatv2_check(who: str, a: ops.DeviceGraph, H: int, Fp: int, tensors) -> None:
    """Refuses, before any launch, what the GATv2 inference kernels do not take: ``tensors`` are ``(t, name, shape)``
    with ``t`` None to skip."""
    from ._lib import BnsError
    why = gat_unsupported(H, Fp)
    if why is not None or Fp % 4:
        raise BnsError(f"{who}: {why or f'padded width {Fp} is not a multiple of 4'}")
    for t, name, shape in tensors:
        if t is None:
            continue
        ops._req(t, torch.float32, name)
        if t.device != a.device:
            raise BnsError(f"{who}: {name} is on {t.device}, the graph on {a.device}")
        if tuple(t.shape) != tuple(shape) or t.stride(-1) != 1 or (t.dim() == 2 and name in ("m", "l")
                                                                   and not t.is_contiguous()):
            raise BnsError(f"{who}: {name} must be {list(shape)} with unit column stride, got {tuple(t.shape)}")


def gatv2_infer(a: ops.DeviceGraph, zs: torch.Tensor, zd: torch.Tensor, attn: torch.Tensor, H: int, Fp: int,
                slope: float) -> torch.Tensor:
    """The evaluation forward of ``dgl.nn.GATv2Conv``'s attention on a homogeneous graph ``a`` (``bns_gatv2_infer_f32``):

        rst[v] = sum_{u -> v} softmax_u(sum_f attn[h, f] leaky_relu(zs[u, h, f] + zd[v, h, f])) * zs[u, h, :]

    ``zs [a.n_cols, H * Fp]``, ``zd [a.n_rows, H * Fp]`` (head-major, ``Fp`` a multiple of 4, pad columns zero),
    ``attn`` with ``H * Fp`` elements -> ``[a.n_rows, H * Fp]``.  No dropout, no gradient."""
    from ._lib import check, lib
    HF = H * Fp
    av = attn.reshape(-1).contiguous()
    _gatv2_check("gatv2_infer", a, H, Fp, ((zs, "zs", (a.n_cols, HF)), (zd, "zd", (a.n_rows, HF)), (av, "attn", (HF,))))
    rst = torch.empty(a.n_rows, HF, dtype=torch.float32, device=a.device)
    with torch.cuda.device(a.device):
        check(lib.bns_gatv2_infer_f32(a._h, zs.data_ptr(), zs.stride(0), zd.data_ptr(), zd.stride(0), av.data_ptr(), H, Fp,
                                      float(slope), rst.data_ptr(), rst.stride(0),
                                      torch.cuda.current_stream(a.device).cuda_stream), "bns_gatv2_infer_f32")
    return rst


def gatv2_infer_block(a: ops.DeviceGraph, zs: Optional[torch.Tensor], zd: torch.Tensor, attn: torch.Tensor, H: int,
                      Fp: int, slope: float, m: torch.Tensor, l: torch.Tensor, acc: torch.Tensor, first: bool,
                      last: bool, rst: Optional[torch.Tensor] = None) -> None:
    """One column block of ``gatv2_infer`` (``bns_gatv2_infer_block_f32``), the online-softmax state ``m``, ``l``
    ``[a.n_rows, H]`` and ``acc [a.n_rows, H * Fp]`` carried as in ``gat_infer_block``; ``last`` writes ``acc / l`` to
    ``rst`` (may be ``acc``).  ``zs [a.n_cols, H * Fp]`` are this block's source rows (None when it has no entries)."""
    from ._lib import BnsError, check, lib
    HF = H * Fp
    if a.nnz and zs is None:
        raise BnsError("gatv2_infer_block: a block with entries needs zs")
    if last and rst is None:
        raise BnsError("gatv2_infer_block: the last block needs rst")
    av = attn.reshape(-1).contiguous()
    _gatv2_check("gatv2_infer_block", a, H, Fp, ((zs, "zs", (a.n_cols, HF)), (zd, "zd", (a.n_rows, HF)),
                                                 (av, "attn", (HF,)), (m, "m", (a.n_rows, H)), (l, "l", (a.n_rows, H)),
                                                 (acc, "acc", (a.n_rows, HF)), (rst, "rst", (a.n_rows, HF))))
    with torch.cuda.device(a.device):
        check(lib.bns_gatv2_infer_block_f32(a._h, ops._ptr(zs), zs.stride(0) if zs is not None else HF, zd.data_ptr(),
                                            zd.stride(0), av.data_ptr(), H, Fp, float(slope), m.data_ptr(), l.data_ptr(),
                                            acc.data_ptr(), acc.stride(0), 1 if first else 0, 1 if last else 0,
                                            ops._ptr(rst), rst.stride(0) if rst is not None else HF,
                                            torch.cuda.current_stream(a.device).cuda_stream),
              "bns_gatv2_infer_block_f32")


SAGE_MAX_WIDTH = 1024


class SageMax(torch.autograd.Function):
    """The max-pooling aggregation of ``dgl.nn.SAGEConv(in, out, 'pool')`` after its ``fc_pool``:

        z = relu(y),   m[v, f] = max over the inner entries and this epoch's sampled halo entries u -> v of z[u, f]

    (0 for a row without entries).  ``y [n_u, Fp]`` (``Fp`` a multiple of 4, at most 1024) -> ``m [n_in, Fp]``.  The
    forward (``bns_sage_max_f32``) records each column's winner, the first entry in walk order whose z is the max, at
    its CSR position (the partition graph's compaction with positions, so a multi-edge is credited once); the backward
    (``bns_sage_max_bwd_f32`` on the static transposes) sends ``d m`` to the winners only, times ``relu'(y)``."""

    @staticmethod
    def forward(ctx, y, g: PartitionGraph):
        from ._lib import check, lib
        n_in, dev, Fp = g.n_in, y.device, y.shape[1]
        z = torch.relu(y).contiguous()
        c = g.compact if (g.a_out is not None and z.shape[0] > n_in) else None
        if c is None and g.a_out is not None and g.a_out.nnz and z.shape[0] > n_in:
            raise RuntimeError("SageMax: halo rows were passed but the partition graph has no compaction "
                               "(refresh_compaction)")
        if c is not None and c.cpos is None:
            raise RuntimeError("SageMax: the partition graph was compacted without positions (want_positions)")
        m = torch.empty(n_in, Fp, dtype=torch.float32, device=dev)
        win = torch.empty(n_in, Fp, dtype=torch.int32, device=dev)
        st = torch.cuda.current_stream(dev).cuda_stream
        with torch.cuda.device(dev):
            check(lib.bns_sage_max_f32(g.a_in._h, None if c is None else g.a_out._h,
                                       None if c is None else c.cidx.data_ptr(),
                                       None if c is None else c.chunk_cnt.data_ptr(),
                                       None if c is None else c.cpos.data_ptr(), n_in, Fp, z.data_ptr(), z.stride(0),
                                       m.data_ptr(), win.data_ptr(), st), "bns_sage_max_f32")
        ctx.g, ctx.halo = g, c is not None
        ctx.save_for_backward(z, win)
        return m

    @staticmethod
    def backward(ctx, dm):
        from ._lib import check, lib
        g = ctx.g
        z, win = ctx.saved_tensors
        dm = dm.contiguous()
        dev, n_in, Fp = z.device, g.n_in, z.shape[1]
        dy = torch.empty_like(z)
        if not ctx.halo and z.shape[0] > n_in:
            dy[n_in:].zero_()                                  # halo rows without halo entries
        st = torch.cuda.current_stream(dev).cuda_stream
        with torch.cuda.device(dev):
            check(lib.bns_sage_max_bwd_f32(g.a_in_t._h, 0, None, 0, Fp, win.data_ptr(), dm.data_ptr(), z.data_ptr(),
                                           z.stride(0), dy.data_ptr(), st), "bns_sage_max_bwd_f32")
            if ctx.halo:
                check(lib.bns_sage_max_bwd_f32(g.a_out_t._h, g.a_in.nnz, g.slot.data_ptr(), n_in, Fp, win.data_ptr(),
                                               dm.data_ptr(), z.data_ptr(), z.stride(0), dy.data_ptr(), st),
                      "bns_sage_max_bwd_f32")
        return dy, None


def _sage_check(who: str, a: ops.DeviceGraph, tensors) -> None:
    """Refuses, before any launch, what the max kernels do not take: ``tensors`` are ``(t, name, shape, dtype)`` with
    ``t`` None to skip."""
    from ._lib import BnsError
    for t, name, shape, dtype in tensors:
        if t is None:
            continue
        ops._req(t, dtype, name)
        if t.device != a.device:
            raise BnsError(f"{who}: {name} is on {t.device}, the graph on {a.device}")
        if tuple(t.shape) != tuple(shape) or not t.is_contiguous():
            raise BnsError(f"{who}: {name} must be a contiguous {list(shape)}, got {tuple(t.shape)}")
        if t.dim() == 2 and (t.shape[1] % 4 or t.shape[1] > SAGE_MAX_WIDTH):
            raise BnsError(f"{who}: width {t.shape[1]} is not a multiple of 4 up to {SAGE_MAX_WIDTH}")


def sage_max_infer(a: ops.DeviceGraph, z: torch.Tensor) -> torch.Tensor:
    """The evaluation forward of the max-pooling aggregation on a homogeneous graph ``a`` (``bns_sage_max_infer_f32``):
    ``m[v] = max over u -> v of z[u]`` per column, 0 for a row without entries.  ``z [a.n_cols, Fp]`` -> ``[a.n_rows,
    Fp]``.  No gradient."""
    from ._lib import check, lib
    Fp = z.shape[1] if z.dim() == 2 else -1
    _sage_check("sage_max_infer", a, ((z, "z", (a.n_cols, Fp), torch.float32),))
    out = torch.empty(a.n_rows, Fp, dtype=torch.float32, device=a.device)
    with torch.cuda.device(a.device):
        check(lib.bns_sage_max_infer_f32(a._h, Fp, z.data_ptr(), z.stride(0), out.data_ptr(),
                                         torch.cuda.current_stream(a.device).cuda_stream), "bns_sage_max_infer_f32")
    return out


def sage_max_infer_block(a: ops.DeviceGraph, z: Optional[torch.Tensor], m: torch.Tensor, seen: torch.Tensor,
                         first: bool, last: bool, out: Optional[torch.Tensor] = None) -> None:
    """One column block of ``sage_max_infer`` (``bns_sage_max_infer_block_f32``): the rows' running max ``m [a.n_rows,
    Fp]`` and ``seen [a.n_rows]`` (int32) are carried from the previous block (``first``: from empty); ``last`` writes
    the max, or 0 for a row that had no entry in any block, to ``out`` (may be ``m``).  ``z [a.n_cols, Fp]``: this
    block's source rows (None when it has no entries)."""
    from ._lib import BnsError, check, lib
    Fp = m.shape[1] if m.dim() == 2 else -1
    if a.nnz and z is None:
        raise BnsError("sage_max_infer_block: a block with entries needs z")
    if last and out is None:
        raise BnsError("sage_max_infer_block: the last block needs out")
    _sage_check("sage_max_infer_block", a, ((z, "z", (a.n_cols, Fp), torch.float32),
                                            (m, "m", (a.n_rows, Fp), torch.float32),
                                            (seen, "seen", (a.n_rows,), torch.int32),
                                            (out, "out", (a.n_rows, Fp), torch.float32)))
    with torch.cuda.device(a.device):
        check(lib.bns_sage_max_infer_block_f32(a._h, Fp, ops._ptr(z), z.stride(0) if z is not None else Fp, m.data_ptr(),
                                               seen.data_ptr(), 1 if first else 0, 1 if last else 0, ops._ptr(out),
                                               torch.cuda.current_stream(a.device).cuda_stream),
              "bns_sage_max_infer_block_f32")


class TconvAttention(torch.autograd.Function):
    """The scaled dot-product attention of the graph transformer layer (``torch_geometric.nn.TransformerConv``) for all
    heads:

        s_uv = scale * <q_v, k_u>,   rst_v = sum_u attn_drop(edge_softmax(s))_uv * v_u

    over the inner entries and this epoch's sampled halo entries, as ``Gatv2Attention``.  ``q [n_in, H * Fp]`` and
    ``kv [n_u, 2 * H * Fp]``, the key rows in its first ``H * Fp`` columns and the value rows in the rest (per-head
    widths padded to ``Fp``, pad columns zero) -> ``[n_in, H * Fp]``; gradients for both.

    Stages (include/bnsgcn.h, ABI 15): ``bns_tconv_scores_f32`` (scores -> probabilities + dropped attention per entry)
    -> ``bns_spmm_weighted_f32`` / ``bns_spmm_compact_f32`` per head on the value columns; backward
    ``bns_sddmm_dot_f32`` -> ``bns_tconv_softmax_bwd_f32`` (d s, d q) -> ``bns_spmm_weighted_f32`` on the transposes
    (d v with the attention, d k with d s)."""

    @staticmethod
    def forward(ctx, q, kv, g: PartitionGraph, H: int, Fp: int, scale: float, p: float, seed: int):
        from ._lib import check, lib
        q, kv = q.contiguous(), kv.contiguous()
        HF = H * Fp
        n_in, dev = g.n_in, kv.device
        if q.shape != (n_in, HF) or kv.dim() != 2 or kv.shape[1] != 2 * HF:
            raise RuntimeError(f"TconvAttention: q must be [{n_in}, {HF}] and kv [*, {2 * HF}], got {tuple(q.shape)} "
                               f"and {tuple(kv.shape)}")
        c = g.compact if (g.a_out is not None and kv.shape[0] > n_in) else None
        if c is None and g.a_out is not None and g.a_out.nnz and kv.shape[0] > n_in:
            raise RuntimeError("TconvAttention: halo rows were passed but the partition graph has no compaction "
                               "(refresh_compaction)")
        if c is not None and c.cpos is None:
            raise RuntimeError("TconvAttention: the partition graph was compacted without positions (want_positions)")
        rst = torch.empty(n_in, HF, dtype=torch.float32, device=dev)
        p_in = torch.empty(max(g.a_in.nnz, 1), H, dtype=torch.float32, device=dev)
        p_out = torch.empty(max(g.a_out.nnz, 1), H, dtype=torch.float32, device=dev) if c is not None else None
        w_in = torch.empty_like(p_in) if p > 0 else None
        w_out = torch.empty_like(p_out) if p > 0 and p_out is not None else None
        wc = torch.empty_like(p_out) if p_out is not None else None
        off, off_dev = ops.RNG["offset"], ops.RNG["offset_dev"]
        head = (g.a_in._h, None if c is None else g.a_out._h, None if c is None else c.cidx.data_ptr(),
                None if c is None else c.chunk_cnt.data_ptr(), None if c is None else c.cpos.data_ptr(), n_in, H, Fp)
        tail = (q.data_ptr(), q.stride(0), kv.data_ptr(), kv.stride(0), float(scale), float(p), seed & (2 ** 64 - 1),
                off & (2 ** 64 - 1), ops._ptr(off_dev))
        st = torch.cuda.current_stream(dev).cuda_stream
        with torch.cuda.device(dev):
            check(lib.bns_tconv_scores_f32(*head, *tail, p_in.data_ptr(), ops._ptr(p_out), ops._ptr(w_in),
                                           ops._ptr(w_out), ops._ptr(wc), st), "bns_tconv_scores_f32")
        for h in range(H):
            cols, vcols = slice(h * Fp, (h + 1) * Fp), slice(HF + h * Fp, HF + (h + 1) * Fp)
            ops.spmm_weighted(g.a_in, kv[:n_in, vcols], rst[:, cols], p_in if w_in is None else w_in, h)
            if c is not None:
                ops.spmm_compact(c, kv[n_in:, vcols], rst[:, cols], accumulate=True, weights=wc, head=h)
        ctx.g, ctx.c, ctx.head, ctx.tail, ctx.cfg = g, c, head, tail, (H, Fp)
        saved = [q, kv, p_in] + ([p_out] if p_out is not None else [])
        if w_in is not None:
            saved += [w_in] + ([w_out] if w_out is not None else [])
        ctx.n_w = 0 if w_in is None else (2 if w_out is not None else 1)
        ctx.save_for_backward(*saved)
        return rst

    @staticmethod
    def backward(ctx, d_rst):
        from ._lib import check, lib
        g, c = ctx.g, ctx.c
        H, Fp = ctx.cfg
        HF = H * Fp
        q, kv, p_in, *rest = ctx.saved_tensors
        p_out = rest.pop(0) if c is not None else None
        d_rst = d_rst.contiguous()
        dev, n_in, n_u = kv.device, g.n_in, kv.shape[0]
        de_in = torch.empty_like(p_in)
        de_out = torch.empty_like(p_out) if p_out is not None else None
        w_in, w_out = p_in, p_out
        if ctx.n_w:
            w_in = rest.pop(0)
            w_out = rest.pop(0) if ctx.n_w == 2 else None
        for h in range(H):                                     # d a'_uv = <d rst_v, v_u>
            cols, vcols = slice(h * Fp, (h + 1) * Fp), slice(HF + h * Fp, HF + (h + 1) * Fp)
            ops.sddmm_dot(g.a_in, d_rst[:, cols], kv[:n_in, vcols], out=de_in[:, h])
            if c is not None:
                ops.sddmm_dot(g.a_out, d_rst[:, cols], kv[n_in:, vcols], col_map=g.slot, n_direct=0, out=de_out[:, h])
        d_q = torch.empty(n_in, HF, dtype=torch.float32, device=dev)
        st = torch.cuda.current_stream(dev).cuda_stream
        with torch.cuda.device(dev):                           # d s in place of d a', and d q
            check(lib.bns_tconv_softmax_bwd_f32(*ctx.head, *ctx.tail, p_in.data_ptr(), ops._ptr(p_out), de_in.data_ptr(),
                                                ops._ptr(de_out), d_q.data_ptr(), d_q.stride(0), st),
                  "bns_tconv_softmax_bwd_f32")
        d_kv = torch.empty(n_u, 2 * HF, dtype=torch.float32, device=dev)
        for h in range(H):                                     # d v = A'^T d rst, d k = dS^T q
            cols, vcols = slice(h * Fp, (h + 1) * Fp), slice(HF + h * Fp, HF + (h + 1) * Fp)
            ops.spmm_weighted(g.a_in_t, d_rst[:, cols], d_kv[:n_in, vcols], w_in, h, through_perm=True)
            ops.spmm_weighted(g.a_in_t, q[:, cols], d_kv[:n_in, cols], de_in, h, through_perm=True)
            if c is not None:
                ops.spmm_weighted(g.a_out_t, d_rst[:, cols], d_kv[n_in:, vcols], w_out, h, through_perm=True,
                                  row_map=g.slot)
                ops.spmm_weighted(g.a_out_t, q[:, cols], d_kv[n_in:, cols], de_out, h, through_perm=True,
                                  row_map=g.slot)
        return d_q, d_kv, None, None, None, None, None, None


def _tconv_ptrs(kv: Optional[torch.Tensor], HF: int):
    """``(k, ldk, v, ldv)`` arguments for the two halves of a ``[n, 2 * HF]`` key / value table (None: no table)."""
    if kv is None:
        return None, 2 * HF, None, 2 * HF
    return kv.data_ptr(), kv.stride(0), kv.data_ptr() + 4 * HF, kv.stride(0)


def tconv_infer(a: ops.DeviceGraph, q: torch.Tensor, kv: torch.Tensor, H: int, Fp: int, scale: float) -> torch.Tensor:
    """The evaluation forward of the graph transformer layer's attention on a homogeneous graph ``a``
    (``bns_tconv_infer_f32``):

        rst[v] = sum_{u -> v} softmax_u(scale * <q[v, h], k[u, h]>) * v[u, h]

    ``q [a.n_rows, H * Fp]``, ``kv [a.n_cols, 2 * H * Fp]`` (key columns, then value columns; head-major, ``Fp`` a
    multiple of 4, pad columns zero) -> ``[a.n_rows, H * Fp]``.  No dropout, no gradient."""
    from ._lib import check, lib
    HF = H * Fp
    _gatv2_check("tconv_infer", a, H, Fp, ((q, "q", (a.n_rows, HF)), (kv, "kv", (a.n_cols, 2 * HF))))
    rst = torch.empty(a.n_rows, HF, dtype=torch.float32, device=a.device)
    with torch.cuda.device(a.device):
        check(lib.bns_tconv_infer_f32(a._h, q.data_ptr(), q.stride(0), *_tconv_ptrs(kv, HF), H, Fp, float(scale),
                                      rst.data_ptr(), rst.stride(0), torch.cuda.current_stream(a.device).cuda_stream),
              "bns_tconv_infer_f32")
    return rst


def tconv_infer_block(a: ops.DeviceGraph, q: torch.Tensor, kv: Optional[torch.Tensor], H: int, Fp: int, scale: float,
                      m: torch.Tensor, l: torch.Tensor, acc: torch.Tensor, first: bool, last: bool,
                      rst: Optional[torch.Tensor] = None) -> None:
    """One column block of ``tconv_infer`` (``bns_tconv_infer_block_f32``), the online-softmax state ``m``, ``l``
    ``[a.n_rows, H]`` and ``acc [a.n_rows, H * Fp]`` carried as in ``gatv2_infer_block``; ``last`` writes ``acc / l`` to
    ``rst`` (may be ``acc``).  ``kv [a.n_cols, 2 * H * Fp]`` are this block's source rows (None when it has no
    entries)."""
    from ._lib import BnsError, check, lib
    HF = H * Fp
    if a.nnz and kv is None:
        raise BnsError("tconv_infer_block: a block with entries needs kv")
    if last and rst is None:
        raise BnsError("tconv_infer_block: the last block needs rst")
    _gatv2_check("tconv_infer_block", a, H, Fp, ((q, "q", (a.n_rows, HF)), (kv, "kv", (a.n_cols, 2 * HF)),
                                                 (m, "m", (a.n_rows, H)), (l, "l", (a.n_rows, H)),
                                                 (acc, "acc", (a.n_rows, HF)), (rst, "rst", (a.n_rows, HF))))
    with torch.cuda.device(a.device):
        check(lib.bns_tconv_infer_block_f32(a._h, q.data_ptr(), q.stride(0), *_tconv_ptrs(kv, HF), H, Fp, float(scale),
                                            m.data_ptr(), l.data_ptr(), acc.data_ptr(), acc.stride(0),
                                            1 if first else 0, 1 if last else 0, ops._ptr(rst),
                                            rst.stride(0) if rst is not None else HF,
                                            torch.cuda.current_stream(a.device).cuda_stream),
              "bns_tconv_infer_block_f32")
