"""Multilevel k-way graph partitioner on the GPU: ``--partition-method multilevel``.

The METIS scheme (coarsen -> initial partition -> uncoarsen with refinement) over the kernels of ``csrc/partition.cuh``;
this file is the level loop, with torch tensors on the device as workspace.

1. The undirected weighted graph: ``w(u, v)`` = the number of directed edges between u and v, loops dropped, node
   weights 1.  Also the directed out-CSR (and, for ``vol``, the in-CSR), with multiplicities, for the exact objective.
2. Coarsening: size-constrained label propagation.  Every round each (coin-selected) node proposes the neighbouring
   cluster it is most heavily connected to that still has room under the weight cap; proposals are admitted per
   target cluster by (gain, id) under the cluster's remaining capacity.  The clusters are contracted (edge and node
   weights summed).  It stops at about ``30 P`` nodes or when a level shrinks the graph by less than 10 %.
3. Initial partition of the coarsest graph on the host: seeded greedy graph growing trials, the best balanced one.
   Up to ``RESTARTS`` initial partitions are uncoarsened and refined independently, and the one with the lowest exact
   objective is kept.  A coarsest graph too large for growing (``GROWING_MAX_ENTRIES``) is cut into weight-balanced
   blocks of a reverse Cuthill-McKee order instead.  Graphs without community structure (Chung-Lu) stop coarsening
   early; there the flat stand-in's partition (``metis``: reverse Cuthill-McKee blocks refined by balanced label
   propagation) is refined at the finest level as one more candidate, so the result is never worse than it.
4. Uncoarsening: project, then balance-respecting refinement rounds -- the connection table, each node's best target
   by exact gain, moves admitted per target (and per source) under the size bounds, a round that does not improve the
   exact objective rolled back -- on the weighted edge cut at the coarse levels and on ``--partition-obj`` at the
   finest, then a rebalancing pass.

``balance="edges"`` (``--partition-balance edges``) carries a second node weight through every stage: the in-edge count
(loops included; int64, coarse sums pass 2^31).  Clusters stay under an in-edge cap of ``IMBALANCE * E / P`` as well as
the node cap, the initial partition and every admitted move keep each part under the in-edge bound
(``partition.in_edge_bound``), rebalancing drives a part over it back under (then, at the finest level, node swaps
that keep every node count: ``partition.shed_in_edges``), and only candidates within both bounds count; the stand-in's
edge-balanced partition is the last resort.

Everything is integer, ties go by id or a seeded hash, and the only atomics are integer sums: the result is a pure
function of (graph, P, objective, balance, seed).  The output is the owner of every node, int64 ``[N]``, as
``assign_parts``.
"""
from __future__ import annotations

import heapq
import time
from typing import Dict, List, NamedTuple, Optional, Tuple

import numpy as np
import torch

from .synthetic import FullGraph

MAX_PARTS = 64          # occupancy bit sets are one 64-bit word per node
IMBALANCE = 0.03        # METIS's default: every part within [0.97 N / P, 1.03 N / P + 1]
COARSE_NODES_PER_PART = 30
CLUSTER_ROUNDS = 12
REFINE_ROUNDS = 64
REFINE_PATIENCE = 8     # rolled-back rounds in a row that end a level
GROWING_MAX_ENTRIES = 400_000   # larger coarsest graphs (nodes + entries) get block_partition, not greedy growing
INITIAL_TRIALS = 32     # greedy-growing trials per initial partition (fewer on a large coarsest graph)
RESTARTS = 8            # initial partitions uncoarsened and refined independently; the best exact objective is kept


class Csr(NamedTuple):
    indptr: torch.Tensor      # int64 [n + 1]
    idx: torch.Tensor         # int32 [nnz]
    w: torch.Tensor           # int32 [nnz]

    @property
    def n(self) -> int:
        return self.indptr.numel() - 1

    @property
    def nnz(self) -> int:
        return self.idx.numel()


def size_bounds(n: int, n_parts: int, imbalance: float = IMBALANCE) -> Tuple[int, int]:
    """Every part's size must lie in [lo, hi]; no part may be empty."""
    return max(int((1.0 - imbalance) * n / n_parts), 1), int((1.0 + imbalance) * n / n_parts) + 1


def resolve_device(device) -> torch.device:
    """The CUDA device to run on: ``None`` is the current one.  A CPU device is refused."""
    if device is None:
        if not torch.cuda.is_available():
            raise ValueError("--partition-method multilevel runs on a CUDA device and none is available; on the CPU "
                             "use --partition-method metis (the stand-in) or random")
        return torch.device("cuda", torch.cuda.current_device())
    dev = torch.device(device)
    if dev.type != "cuda":
        raise ValueError(f"--partition-method multilevel runs on a CUDA device, not {dev}; on the CPU use "
                         "--partition-method metis (the stand-in) or random")
    return dev


def check_parts(n_nodes: int, n_parts: int) -> None:
    if not 2 <= n_parts <= MAX_PARTS:
        raise ValueError(f"--partition-method multilevel takes 2 <= n_partitions <= {MAX_PARTS} (or 1), "
                         f"got {n_parts}")
    if n_parts > n_nodes:
        raise ValueError(f"--partition-method multilevel needs n_partitions <= the node count ({n_nodes}), "
                         f"got {n_parts}")
    if n_nodes >= 2 ** 31 - 1:
        raise ValueError(f"--partition-method multilevel needs node ids that fit int32, the graph has {n_nodes} nodes")


def _coin(n: int, salt: int, dev) -> torch.Tensor:
    """A seeded pseudo-random half of the nodes (integer hash of (node, salt))."""
    x = (torch.arange(n, dtype=torch.int64, device=dev) * 2654435761 + (salt % 1000003) * 97 + 12345) & 0xFFFFFFFF
    x = (((x >> 16) ^ x) * 0x45D9F3B) & 0xFFFFFFFF
    x = (((x >> 16) ^ x) * 0x45D9F3B) & 0xFFFFFFFF
    return (((x >> 16) ^ x) & 1) == 1


def _seg_cumsum(w: torch.Tensor, key: torch.Tensor) -> torch.Tensor:
    """Inclusive running sum of ``w`` within each run of equal (sorted) ``key``."""
    cs = torch.cumsum(w, 0)
    first = torch.searchsorted(key, key)
    prev = torch.where(first > 0, cs[(first - 1).clamp(min=0)], torch.zeros_like(cs))
    return cs - prev


def _order(nodes: torch.Tensor, gain: torch.Tensor, key: torch.Tensor) -> torch.Tensor:
    """Permutation sorting by (key, gain descending, node id)."""
    o = torch.sort(nodes, stable=True)[1]
    o = o[torch.sort(-gain[o], stable=True)[1]]
    return o[torch.sort(key[o], stable=True)[1]]


def admit(nodes: torch.Tensor, to: torch.Tensor, gain: torch.Tensor, wt: torch.Tensor, frm: torch.Tensor,
          sizes: torch.Tensor, hi: int, lo: Optional[int] = None, need_in: Optional[torch.Tensor] = None,
          need_out: Optional[torch.Tensor] = None, ewt: Optional[torch.Tensor] = None,
          esizes: Optional[torch.Tensor] = None, ehi: Optional[int] = None,
          need_eout: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """The moves ``nodes[i] -> to[i]`` that are admitted: per target, the best by (gain, id) whose summed weight keeps it
    at or below ``hi`` (and, with ``need_in``, until the target's need is met); then per source, the best that keep it at
    or above ``lo`` (and, with ``need_out``, until the source's excess is gone).  Moves into a part are not counted
    against its floor, nor moves out of it against its cap, so the bounds hold whatever subset is applied.
    With ``ewt`` / ``esizes`` / ``ehi`` (in-edge weights of the movers and the parts, and the in-edge cap), a target must
    also stay at or below ``ehi`` by the same running sum; with ``need_eout`` a source keeps moving out until its node
    excess or its in-edge excess is gone."""
    edges = ewt is not None
    if nodes.numel():
        o = _order(nodes, gain, to)
        nodes, to, gain, wt, frm = nodes[o], to[o], gain[o], wt[o], frm[o]
        cum = _seg_cumsum(wt, to)
        ok = sizes[to] + cum <= hi
        if need_in is not None:
            ok &= cum - wt < need_in[to]
        if edges:
            ewt = ewt[o]
            ok &= esizes[to] + _seg_cumsum(ewt, to) <= ehi
            ewt = ewt[ok]
        nodes, to, gain, wt, frm = nodes[ok], to[ok], gain[ok], wt[ok], frm[ok]
    if nodes.numel() and (lo is not None or need_out is not None or need_eout is not None):
        o = _order(nodes, gain, frm)
        nodes, to, gain, wt, frm = nodes[o], to[o], gain[o], wt[o], frm[o]
        cum = _seg_cumsum(wt, frm)
        ok = torch.ones_like(cum, dtype=torch.bool)
        if lo is not None:
            ok &= sizes[frm] - cum >= lo
        if need_eout is not None:
            ewt = ewt[o]
            want = _seg_cumsum(ewt, frm) - ewt < need_eout[frm]
            ok &= want | (cum - wt < need_out[frm]) if need_out is not None else want
        elif need_out is not None:
            ok &= cum - wt < need_out[frm]
        nodes, to = nodes[ok], to[ok]
    return nodes, to


# ---- coarsening ----------------------------------------------------------------------------------------------------

def cluster(g: Csr, nw: Optional[torch.Tensor], cap: int, seed: int, rounds: int = 0,
            ew: Optional[torch.Tensor] = None, ecap: int = 0) -> torch.Tensor:
    """Size-constrained label propagation: int32 cluster label of every node (a node id), every cluster's weight <= cap
    (each node starts alone, so the cap holds as long as cap >= the heaviest node).  With ``ew`` (int64 in-edge weight
    per node), every cluster a node joins also stays within the in-edge cap ``ecap``."""
    from .. import ops
    n, dev = g.n, g.indptr.device
    label = torch.arange(n, dtype=torch.int32, device=dev)
    wl = nw.to(torch.int64) if nw is not None else torch.ones(n, dtype=torch.int64, device=dev)
    for r in range(rounds or CLUSTER_ROUNDS):
        rating = ops.part_edges(g.indptr, g.idx, g.w, n, 0, False, col_map=label)
        cw = ops.part_weights(label, nw, n)
        step_seed = seed * 1000003 + r * 7919 + 1
        if ew is None:
            tgt, gain = ops.part_cluster(rating, label, nw, cw, cap, step_seed)
            two = {}
        else:
            ce = ops.part_weights(label, ew, n)
            tgt, gain = ops.part_cluster(rating, label, nw, cw, cap, step_seed, ew=ew, ce=ce, ecap=ecap)
            two = {"esizes": ce, "ehi": ecap}
        cand = torch.nonzero(tgt >= 0, as_tuple=True)[0]
        if cand.numel() == 0:
            break
        if two:
            two["ewt"] = ew[cand]
        movers, to = admit(cand, tgt[cand].long(), gain[cand], wl[cand], label[cand].long(), cw, cap, **two)
        if movers.numel() == 0:
            break
        label[movers] = to.to(torch.int32)
    return label


def compact(label: torch.Tensor) -> Tuple[torch.Tensor, int]:
    """Renumber the labels 0 .. n_clusters - 1 in order of the label ids."""
    used = torch.zeros(label.numel(), dtype=torch.int64, device=label.device)
    used[label.long()] = 1
    new = torch.cumsum(used, 0) - 1
    return new[label.long()].to(torch.int32), int(used.sum())


def contract(g: Csr, nw: Optional[torch.Tensor], cmap: torch.Tensor, nc: int, ew: Optional[torch.Tensor] = None):
    """The coarse graph: edge weights between clusters summed, intra-cluster edges dropped; node weights summed.
    Returns (coarse graph, int32 node weights), and with ``ew`` the int64 summed in-edge weights as a third value."""
    from .. import ops
    cg = Csr(*ops.part_edges(g.indptr, g.idx, g.w, nc, 0, True, row_map=cmap, col_map=cmap))
    cnw = ops.part_weights(cmap, nw, nc).to(torch.int32)
    if ew is None:
        return cg, cnw
    return cg, cnw, ops.part_weights(cmap, ew, nc)


# ---- initial partition (host) ----------------------------------------------------------------------------------------

def initial_partition(indptr: np.ndarray, idx: np.ndarray, w: np.ndarray, nw: np.ndarray, n_parts: int, lo: int,
                      hi: int, seed: int, trials: int = 8, ew: Optional[np.ndarray] = None,
                      ehi: int = 0) -> np.ndarray:
    """Greedy graph growing on a small weighted graph: parts 0 .. P-2 are grown one at a time from a seeded random
    node, always adding the unassigned node with the largest weight into the part minus weight out of it (ties: lower
    id) that keeps it within
    ``hi``, until it reaches its share of the remaining weight; the last part takes the rest.  The best of ``trials``
    seeded trials by (bound violation, weighted cut) is returned (int64 [n]).  With ``ew`` (in-edge weights), a part
    also stays within ``ehi`` and grows until it holds its share of the remaining in-edges too, and the violation
    counts the in-edges above ``ehi``."""
    n = int(nw.shape[0])
    indptr, idx, w, nw = (np.asarray(a, dtype=np.int64) for a in (indptr, idx, w, nw))
    if ew is not None:
        ew = np.asarray(ew, dtype=np.int64)
    rows = np.repeat(np.arange(n), np.diff(indptr))
    wdeg = np.bincount(rows, weights=w, minlength=n).astype(np.int64)
    best, best_key = None, None
    for t in range(trials):
        rng = np.random.default_rng([seed, t, 104729])
        order = rng.permutation(n)
        nxt = 0
        part = np.full(n, -1, dtype=np.int64)
        remaining = int(nw.sum())
        eremaining = int(ew.sum()) if ew is not None else 0
        for p in range(n_parts - 1):
            share = remaining // (n_parts - p)
            eshare = eremaining // (n_parts - p)
            conn = np.zeros(n, dtype=np.int64)
            blocked = np.zeros(n, dtype=bool)
            heap: List[Tuple[int, int]] = []
            pw = pe = 0
            while pw < share or (ew is not None and pe < eshare):
                v = -1
                while heap:
                    g, u = heapq.heappop(heap)
                    if part[u] < 0 and not blocked[u] and -g == 2 * conn[u] - wdeg[u]:
                        v = u
                        break
                if v < 0:                                   # no frontier: a new seed
                    while nxt < n and (part[order[nxt]] >= 0 or blocked[order[nxt]]):
                        nxt += 1
                    if nxt == n:
                        break
                    v = int(order[nxt])
                if pw > 0 and (pw + nw[v] > hi or (ew is not None and pe + ew[v] > ehi)):
                    blocked[v] = True
                    continue
                part[v] = p
                pw += int(nw[v])
                if ew is not None:
                    pe += int(ew[v])
                for k in range(indptr[v], indptr[v + 1]):
                    u = int(idx[k])
                    if part[u] < 0:
                        conn[u] += w[k]
                        heapq.heappush(heap, (-int(2 * conn[u] - wdeg[u]), u))
            nxt = 0
            remaining -= pw
            eremaining -= pe
        part[part < 0] = n_parts - 1
        sizes = np.bincount(part, weights=nw, minlength=n_parts).astype(np.int64)
        viol = int(np.maximum(sizes - hi, 0).sum() + np.maximum(lo - sizes, 0).sum())
        if ew is not None:
            esizes = np.bincount(part, weights=ew, minlength=n_parts).astype(np.int64)
            viol += int(np.maximum(esizes - ehi, 0).sum())
        cut = int(w[part[rows] != part[idx]].sum())
        key = (viol, cut)
        if best_key is None or key < best_key:
            best, best_key = part, key
    return best


def cut_blocks(nw: np.ndarray, ew: np.ndarray, n_parts: int, lo: int, hi: int, ehi: int) -> Optional[np.ndarray]:
    """Cut a sequence of nodes (weights ``nw``, in-edge weights ``ew``, in order) into ``n_parts`` consecutive blocks,
    each of node weight in ``[lo, hi]`` and in-edge weight at most ``ehi``: the block id of every position (int64), or
    None when this order admits no such cut.  Every block ends at the admissible position nearest to where the running
    node weight reaches its equal share (ties: the earlier), among those from which the rest can still be cut."""
    nw, ew = np.asarray(nw, dtype=np.int64), np.asarray(ew, dtype=np.int64)
    n, P = int(nw.shape[0]), n_parts
    cn = np.concatenate([[0], np.cumsum(nw)])
    ce = np.concatenate([[0], np.cumsum(ew)])
    # a block starting at position s may end at e in [e_lo[s], e_hi[s]]
    e_lo = np.searchsorted(cn, cn + lo, side="left")
    e_hi = np.minimum(np.searchsorted(cn, cn + hi, side="right"), np.searchsorted(ce, ce + ehi, side="right")) - 1
    e_lo = np.maximum(e_lo, np.arange(n + 1) + 1)
    # reach[p][s]: blocks p .. P-1 can cover positions s .. n-1
    reach = np.zeros((P + 1, n + 1), dtype=bool)
    reach[P, n] = True
    for p in range(P - 1, -1, -1):
        cnt = np.concatenate([[0], np.cumsum(reach[p + 1])])
        a, b = np.minimum(e_lo, n + 1), np.clip(e_hi + 1, 0, n + 1)
        reach[p] = (a < b) & (cnt[b] - cnt[np.minimum(a, b)] > 0)
    if not reach[0, 0]:
        return None
    out = np.empty(n, dtype=np.int64)
    s, total = 0, int(cn[-1])
    for p in range(P):
        lo_e, hi_e = int(e_lo[s]), int(e_hi[s])
        ends = lo_e + np.nonzero(reach[p + 1, lo_e:hi_e + 1])[0]
        t = int(np.searchsorted(cn, (p + 1) * total / P, side="left"))
        e = int(ends[np.argmin(np.abs(ends - t))])
        out[s:e] = p
        s = e
    return out


def block_partition(indptr: np.ndarray, idx: np.ndarray, nw: np.ndarray, n_parts: int, ew: Optional[np.ndarray] = None,
                    lo: int = 0, hi: int = 0, ehi: int = 0) -> np.ndarray:
    """A reverse Cuthill-McKee order of the graph cut into P blocks of (about) equal weight (int64 [n]).  With ``ew``
    (in-edge weights), the blocks are cut within the node bounds ``[lo, hi]`` and the in-edge bound ``ehi``
    (``partition.cut_blocks``) when that order admits it; otherwise into equal weight, left to rebalancing."""
    import scipy.sparse as sp
    from scipy.sparse.csgraph import reverse_cuthill_mckee
    n = int(nw.shape[0])
    a = sp.csr_matrix((np.ones(idx.shape[0], dtype=np.int8), idx, indptr), shape=(n, n))
    order = np.asarray(reverse_cuthill_mckee(a, symmetric_mode=True), dtype=np.int64)
    w = np.asarray(nw, dtype=np.int64)[order]
    part = np.empty(n, dtype=np.int64)
    if ew is not None:
        blocks = cut_blocks(w, np.asarray(ew, dtype=np.int64)[order], n_parts, lo, hi, ehi)
        if blocks is not None:
            part[order] = blocks
            return part
    before = np.cumsum(w) - w
    part[order] = np.minimum(before * n_parts // max(int(w.sum()), 1), n_parts - 1)
    return part


# ---- refinement ----------------------------------------------------------------------------------------------------

class _Level:
    """One level's graph and what its objective needs."""

    def __init__(self, g: Csr, nw: Optional[torch.Tensor], n_parts: int, objective: str,
                 out_g: Optional[Csr] = None, in_g: Optional[Csr] = None, ew: Optional[torch.Tensor] = None,
                 ehi: int = 0):
        self.g, self.nw, self.P, self.objective = g, nw, n_parts, objective
        self.out_g, self.in_g = out_g, in_g
        self.ew, self.ehi = ew, ehi            # --partition-balance edges: in-edge weights and the in-edge bound
        n = g.n
        self.wl = nw.to(torch.int64) if nw is not None else torch.ones(n, dtype=torch.int64, device=g.indptr.device)

    def table(self, part: torch.Tensor):
        """(conn, occ, score): the gain tables of ``part`` and its exact objective."""
        from .. import ops
        if self.objective == "vol":
            conn, occ, q = ops.part_conn(*self.out_g, part, self.P, occ=True, quality=True)
            return conn, occ, int(q[1])
        conn, _, q = ops.part_conn(*self.g, part, self.P, quality=True)
        return conn, None, int(q[0])

    def gains(self, part, conn, occ, allowed: int):
        from .. import ops
        return ops.part_gains(self.objective, part, conn, self.P, allowed, in_graph=self.in_g, occ=occ)

    def sizes(self, part):
        from .. import ops
        return ops.part_weights(part, self.nw, self.P)

    def esizes(self, part):
        from .. import ops
        return ops.part_weights(part, self.ew, self.P)

    def edge_args(self, part, cand, esizes=None):
        """admit's in-edge keywords for the movers ``cand`` (none without in-edge weights)."""
        if self.ew is None:
            return {}
        return {"ewt": self.ew[cand], "esizes": self.esizes(part) if esizes is None else esizes, "ehi": self.ehi}


def refine(lv: _Level, part: torch.Tensor, lo: int, hi: int, seed: int, rounds: int = 0) -> torch.Tensor:
    """Balance-respecting rounds of moves with positive exact gain (a seeded half of the candidates per round); a round
    whose exact objective is not lower is rolled back, REFINE_PATIENCE in a row end the level.  Never returns a worse part."""
    n, dev, P = part.numel(), part.device, lv.P
    conn, occ, best = lv.table(part)
    sizes = lv.sizes(part)
    every = (1 << P) - 1
    failed = 0
    for r in range(rounds or REFINE_ROUNDS):
        tgt, gain = lv.gains(part, conn, occ, every)
        cand = torch.nonzero((tgt >= 0) & (gain > 0) & _coin(n, seed * 31 + r, dev), as_tuple=True)[0]
        if cand.numel() == 0:
            if not bool(((tgt >= 0) & (gain > 0)).any()):
                break
            failed += 1
            if failed >= REFINE_PATIENCE:
                break
            continue
        movers, to = admit(cand, tgt[cand].long(), gain[cand], lv.wl[cand], part[cand].long(), sizes, hi, lo,
                           **lv.edge_args(part, cand))
        trial = part.clone()
        trial[movers] = to.to(torch.int32)
        if movers.numel() == 0:
            failed += 1
            if failed >= REFINE_PATIENCE:
                break
            continue
        c2, o2, s2 = lv.table(trial)
        if s2 < best:
            part, conn, occ, best, failed = trial, c2, o2, s2, 0
            sizes = lv.sizes(part)
        else:
            failed += 1
            if failed >= REFINE_PATIENCE:
                break
    return part


def rebalance(lv: _Level, part: torch.Tensor, lo: int, hi: int, max_passes: int = 0) -> torch.Tensor:
    """Moves the lowest-loss nodes out of the parts above ``hi`` (into parts with room), then into the parts below
    ``lo`` (from parts above it), until the bounds hold or no admissible move is left.  With unit node weights (the
    finest level) the bounds always end up holding.  With in-edge weights, a part above the in-edge bound is over
    too: nodes leave it (keeping it at or above ``lo``) into parts with room for both, until both excesses are gone."""
    P, edges = lv.P, lv.ew is not None
    for _ in range(max_passes or 4 * P + 8):
        sizes = lv.sizes(part)
        s = sizes.cpu()
        over, under = s > hi, s < lo
        if edges:
            esizes = lv.esizes(part)
            es = esizes.cpu()
            over |= es > lv.ehi
        if not bool(over.any()) and not bool(under.any()):
            break
        conn, occ, _ = lv.table(part)
        if bool(over.any()):
            if edges:
                allowed = sum(1 << p for p in range(P) if s[p] < hi and es[p] < lv.ehi)
            else:
                allowed = sum(1 << p for p in range(P) if s[p] < hi)
            if allowed == 0:
                break
            tgt, gain = lv.gains(part, conn, occ, allowed)
            src_over = over.to(part.device)[part.long()]
            cand = torch.nonzero(src_over & (tgt >= 0), as_tuple=True)[0]
            if edges:
                movers, to = admit(cand, tgt[cand].long(), gain[cand], lv.wl[cand], part[cand].long(), sizes, hi, lo,
                                   need_out=(sizes - hi).clamp(min=0), need_eout=(esizes - lv.ehi).clamp(min=0),
                                   **lv.edge_args(part, cand, esizes))
            else:
                movers, to = admit(cand, tgt[cand].long(), gain[cand], lv.wl[cand], part[cand].long(), sizes, hi,
                                   need_out=(sizes - hi).clamp(min=0))
        else:
            allowed = sum(1 << p for p in range(P) if s[p] < lo)
            tgt, gain = lv.gains(part, conn, occ, allowed)
            cand = torch.nonzero((tgt >= 0) & (sizes[part.long()] > lo), as_tuple=True)[0]
            movers, to = admit(cand, tgt[cand].long(), gain[cand], lv.wl[cand], part[cand].long(), sizes, hi, lo,
                               need_in=(lo - sizes).clamp(min=0), **lv.edge_args(part, cand, esizes if edges else None))
        if movers.numel() == 0:
            break
        part = part.clone()
        part[movers] = to.to(torch.int32)
    return part


# ---- the whole scheme ------------------------------------------------------------------------------------------------

def multilevel_partition(fg: FullGraph, n_parts: int, objective: str = "vol", seed: int = 0,
                         device=None, balance: str = "nodes") -> Tuple[torch.Tensor, Dict[str, object]]:
    """Owner of every node (int64 ``[N]``, on the host) and a report: ``levels`` = [(nodes, undirected entries)] from
    the finest graph to the coarsest, the final exact ``cut`` / ``vol`` / ``min_size`` / ``max_size`` /
    ``min_in_edges`` / ``max_in_edges``, and ``seconds`` per stage (build, coarsen, initial, uncoarsen).
    ``balance="edges"`` also bounds every part's in-edges by ``partition.in_edge_bound``."""
    from .partition import check_balance, in_edge_bound
    if objective not in ("cut", "vol"):
        raise ValueError(f"--partition-obj must be cut or vol, got {objective!r}")
    check_balance(balance)
    N, P = fg.n_nodes, n_parts
    if P == 1:
        return torch.zeros(N, dtype=torch.int64), {"levels": [], "cut": 0, "vol": 0, "min_size": N, "max_size": N,
                                                   "min_in_edges": fg.n_edges, "max_in_edges": fg.n_edges}
    check_parts(N, P)
    dev = resolve_device(device)
    lo, hi = size_bounds(N, P)
    ehi = in_edge_bound(fg.in_degrees(), P) if balance == "edges" else None
    with torch.cuda.device(dev):
        part, info = _multilevel(fg, P, objective, seed, dev, lo, hi, ehi)
        # every device tensor of the run is gone with _multilevel's frame: hand the cached blocks back, so that a process
        # that only partitions (main.py partitions in its parent before it spawns the ranks) holds no workspace while
        # the ranks train
        torch.cuda.empty_cache()
    if not lo <= info["min_size"] <= info["max_size"] <= hi:
        raise RuntimeError(f"multilevel partition out of its size bounds [{lo}, {hi}]: part sizes "
                           f"{info['min_size']} .. {info['max_size']}")
    if ehi is not None and info["max_in_edges"] > ehi:
        raise RuntimeError(f"multilevel partition out of its in-edge bound {ehi} = int(1.03 E / P) + d_max: part "
                           f"{info['max_in_edges_part']} owns {info['max_in_edges']} in-edges")
    return part, info


def _multilevel(fg: FullGraph, P: int, objective: str, seed: int, dev, lo: int, hi: int, ehi: Optional[int]):
    """The scheme itself, on the current device; every device tensor it makes dies with its frame.  ``ehi``: the
    in-edge bound under ``--partition-balance edges``, None under ``nodes``."""
    from .. import ops
    N = fg.n_nodes
    seconds: Dict[str, float] = {}
    clock = [time.perf_counter()]

    def lap(stage: str) -> None:                       # host clock around synchronised work
        torch.cuda.synchronize(dev)
        now = time.perf_counter()
        seconds[stage] = round(now - clock[0], 4)
        clock[0] = now

    indptr = fg.indptr.to(dev, torch.int64)
    src = fg.src.to(dev, torch.int32)
    g0 = Csr(*ops.part_edges(indptr, src, None, N, 2, True))
    out_g = Csr(*ops.part_edges(indptr, src, None, N, 1, True))
    in_g = Csr(*ops.part_edges(indptr, src, None, N, 0, True)) if objective == "vol" else None
    edges = ehi is not None
    ew0 = (indptr[1:] - indptr[:-1]).contiguous() if edges else None    # in-edges per node, loops included
    del indptr, src
    lap("build")
    # coarsening
    graphs: List[Tuple[Csr, Optional[torch.Tensor], Optional[torch.Tensor]]] = [(g0, None, ew0)]
    maps: List[torch.Tensor] = []
    cap = max(1, int(IMBALANCE * N / P))
    ecap = max(1, int(IMBALANCE * fg.n_edges / P))
    stalled = False                         # coarsening stopped before the coarsest graph got small
    while graphs[-1][0].n > COARSE_NODES_PER_PART * P and len(graphs) < 48:
        g, nw, ew = graphs[-1]
        cmap, nc = compact(cluster(g, nw, cap, seed + 17 * len(graphs), ew=ew, ecap=ecap))
        if nc >= g.n:
            stalled = True
            break
        if edges:
            graphs.append(contract(g, nw, cmap, nc, ew))
        else:
            graphs.append(contract(g, nw, cmap, nc) + (None,))
        maps.append(cmap)
        if nc > 0.9 * g.n:
            stalled = nc > COARSE_NODES_PER_PART * P
            break
    lap("coarsen")
    # initial partitions of the coarsest graph (on the host), each projected and refined down to the finest level
    gc, nwc, ewc = graphs[-1]
    nw_host = nwc.cpu().numpy() if nwc is not None else np.ones(gc.n, dtype=np.int64)
    ew_host = ewc.cpu().numpy() if edges else None
    size = gc.n + gc.nnz + 1
    starts: List[Tuple[int, torch.Tensor]] = []
    if size <= GROWING_MAX_ENTRIES:         # the host work is bounded: trials x restarts x size
        trials = max(1, min(INITIAL_TRIALS, 2 * GROWING_MAX_ENTRIES // size))
        for r in range(max(1, min(RESTARTS, 4 * GROWING_MAX_ENTRIES // (size * trials)))):
            if edges:
                init = initial_partition(gc.indptr.cpu().numpy(), gc.idx.cpu().numpy(), gc.w.cpu().numpy(), nw_host,
                                         P, lo, hi, seed * RESTARTS + r, trials, ew_host, ehi)
            else:
                init = initial_partition(gc.indptr.cpu().numpy(), gc.idx.cpu().numpy(), gc.w.cpu().numpy(), nw_host,
                                         P, lo, hi, seed * RESTARTS + r, trials)
            starts.append((len(graphs) - 1, torch.from_numpy(init).to(dev, torch.int32)))
    elif edges:
        init = block_partition(gc.indptr.cpu().numpy(), gc.idx.cpu().numpy(), nw_host, P, ew_host, lo, hi, ehi)
        starts.append((len(graphs) - 1, torch.from_numpy(init).to(dev, torch.int32)))
    else:
        init = block_partition(gc.indptr.cpu().numpy(), gc.idx.cpu().numpy(), nw_host, P)
        starts.append((len(graphs) - 1, torch.from_numpy(init).to(dev, torch.int32)))
    balance = "edges" if edges else "nodes"

    def stand_in() -> Tuple[int, torch.Tensor]:
        from .partition import assign_parts
        return 0, assign_parts(fg, P, "metis", seed, objective, dev, balance).to(dev, torch.int32)

    if stalled:     # no hierarchy worth the name: the flat stand-in's partition, refined below, is one more candidate
        starts.append(stand_in())
    lap("initial")

    def in_bounds(part) -> bool:
        s = ops.part_weights(part, None, P).cpu()
        if not (int(s.min()) >= lo and int(s.max()) <= hi):
            return False
        return not edges or int(ops.part_weights(part, ew0, P).max()) <= ehi

    # uncoarsening; the candidate with the lowest exact objective is kept (ties: the earlier one); under edges only
    # candidates within both bounds count, and the stand-in's edge-balanced partition is the last resort
    best, best_score = None, None
    k = 0
    while k < len(starts):
        top, part = starts[k]
        for lvl in range(top, -1, -1):
            g, nw, ew = graphs[lvl]
            if lvl < top:
                part = part[maps[lvl].long()]
            lv = _Level(g, nw, P, "cut", ew=ew, ehi=ehi or 0)
            part = rebalance(lv, part, lo, hi)
            if top > 0 or objective == "cut":      # a flat start is refined on the requested objective alone
                part = refine(lv, part, lo, hi, seed * 131 + 7 * k + lvl)
            if lvl == 0 and objective == "vol":    # the finest level: the edge cut first, then the exact volume
                lv = _Level(g, nw, P, "vol", out_g, in_g, ew=ew, ehi=ehi or 0)
                part = refine(lv, part, lo, hi, seed * 131 + 7 * k + 977)
            part = rebalance(lv, part, lo, hi)
        if edges and not in_bounds(part):
            # a part at its node floor cannot shed in-edges by moves: swap its hubs for the lightest part's leaves,
            # which keeps every node count, then refine under both caps again
            from .partition import shed_in_edges
            try:
                part = shed_in_edges(part.long().cpu(), fg.in_degrees(), P, ehi, "multilevel").to(dev, torch.int32)
                part = refine(lv, part, lo, hi, seed * 131 + 7 * k + 1977)
            except RuntimeError:
                pass                                # left out of bounds: this candidate does not count
        _, _, q = ops.part_conn(*out_g, part, P, table=False, quality=True)
        score = int(q[0 if objective == "cut" else 1])
        if (not edges or in_bounds(part)) and (best_score is None or score < best_score):
            best, best_score = part, score
        k += 1
        if k == len(starts) and best is None and edges and not stalled:
            stalled = True
            starts.append(stand_in())
    part = best if best is not None else part
    lap("uncoarsen")
    _, _, q = ops.part_conn(*out_g, part, P, table=False, quality=True)
    sizes = ops.part_weights(part, None, P).cpu()
    esizes = torch.zeros(P, dtype=torch.int64).index_add_(0, part.long().cpu(), fg.in_degrees())
    info = {"levels": [(gg.n, gg.nnz) for gg, _, _ in graphs], "cut": int(q[0]), "vol": int(q[1]),
            "min_size": int(sizes.min()), "max_size": int(sizes.max()), "min_in_edges": int(esizes.min()),
            "max_in_edges": int(esizes.max()), "max_in_edges_part": int(esizes.argmax()), "candidates": len(starts),
            "seconds": seconds}
    return part.to(torch.int64).cpu(), info
