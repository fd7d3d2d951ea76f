"""Host restatements (numpy, on the CPU) of the sampled boundary exchange: the halo compaction of
``bns_graph_compact_cols``, the per-epoch maps of ``bns_epoch_maps_update``, the feature rows ``Buffer.update`` moves
and the gradient scatter of its backward.

All of it is exact: integer bookkeeping, copies, one float32 division per element (``np.float32(x) / np.float32(ratio)``
rounds like ``__fdiv_rn``) and float32 adds in a fixed order, so the tests compare bit for bit."""
import numpy as np


def chunks(indptr, chunk_nnz):
    """``(chunk_row, chunk_start, chunk_end)`` of ``bns_graph_create``: row ``r`` is ``max(1, ceil(deg / chunk_nnz))``
    chunks of at most ``chunk_nnz`` entries, an empty row one empty chunk."""
    indptr = np.asarray(indptr, dtype=np.int64)
    deg = indptr[1:] - indptr[:-1]
    n = np.maximum(1, (deg + chunk_nnz - 1) // chunk_nnz)
    row = np.repeat(np.arange(deg.size, dtype=np.int64), n)
    first = np.cumsum(n) - n
    start = indptr[:-1][row] + (np.arange(int(n.sum()), dtype=np.int64) - np.repeat(first, n)) * chunk_nnz
    end = np.minimum(start + chunk_nnz, indptr[1:][row])
    return row, start, end


def compact_cols(indptr, indices, chunk_nnz, col_map, col_scale=None):
    """``bns_graph_compact_cols`` with ``n_direct = 0``: the live entries (``col_map[c] >= 0``) of every chunk, in CSR
    order, written to the front of the chunk's own index range.  Returns ``(chunk_cnt, dest, cidx, cw, cpos)``: entry
    ``i`` of the last four says what the kernel stores at ``dest[i]``; nothing else of cidx / cw / cpos is defined."""
    indices = np.asarray(indices, dtype=np.int64)
    _, start, end = chunks(indptr, chunk_nnz)
    mapped = np.asarray(col_map)[indices]
    live = mapped >= 0
    before = np.concatenate([[0], np.cumsum(live)])             # live entries before position k
    cnt = (before[end] - before[start]).astype(np.int32)
    entry_chunk = np.repeat(np.arange(start.size), end - start)  # the chunks tile [0, nnz) in order
    k = np.nonzero(live)[0]
    dest = start[entry_chunk[k]] + before[k] - before[start[entry_chunk[k]]]
    cw = None if col_scale is None else np.asarray(col_scale, dtype=np.float32)[indices[k]]
    return cnt, dest, mapped[k].astype(np.int32), cw, k.astype(np.int32)


def epoch_maps(n_in, n_halo, pos, hops, sel):
    """``bns_epoch_maps_update`` over the peers in ascending order (lists ``pos``, ``hops``, ``sel`` of equal length):
    ``slot[pos_j[hops_j[k]] - n_in]`` = the position of that entry in the concatenation of all ``hops_j``,
    ``inv_j[sel_j[t]] = t``, every other entry -1."""
    slot = np.full(n_halo, -1, dtype=np.int32)
    inv = []
    at = 0
    for p, h, s in zip(pos, hops, sel):
        h = np.asarray(h, dtype=np.int64)
        slot[np.asarray(p)[h] - n_in] = at + np.arange(h.size, dtype=np.int32)
        at += h.size
        v = np.full(n_in, -1, dtype=np.int32)
        v[np.asarray(s, dtype=np.int64)] = np.arange(len(s), dtype=np.int32)
        inv.append(v)
    return slot, inv


def send_rows(H, sel, ratio):
    """The rows one peer receives: ``H[sel] / float32(ratio)`` (K3, ``bns_gather_div_f32`` / ``p2p_put_all``)."""
    return np.asarray(H, dtype=np.float32)[np.asarray(sel, dtype=np.int64)] / np.float32(ratio)


def scatter_ring(G, rank, size, sel, recv, ratio):
    """The gradient return trip on rank ``rank``: ``G[sel[left]] += recv[left] / float32(ratio[left])`` for
    ``left = (rank - i) % size``, ``i = 1 .. size-1`` (the reference's ring order), one peer after the other in float32.
    A peer's ``sel`` has no repeats, so each step is one vector add."""
    out = np.array(G, dtype=np.float32, copy=True)
    for i in range(1, size):
        left = (rank - i) % size
        s = np.asarray(sel[left], dtype=np.int64)
        if s.size:
            out[s] = out[s] + np.asarray(recv[left], dtype=np.float32) / np.float32(ratio[left])
    return out
