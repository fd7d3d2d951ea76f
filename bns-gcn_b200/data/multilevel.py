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

Everything is integer, ties go by id or a seeded hash, and the only atomics are integer sums: the result is a pure
function of (graph, P, objective, seed).  The output is the owner of every node, int64 ``[N]``, as ``assign_parts``.
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
          need_out: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """The moves ``nodes[i] -> to[i]`` that are admitted: per target, the best by (gain, id) whose summed weight keeps it
    at or below ``hi`` (and, with ``need_in``, until the target's need is met); then per source, the best that keep it at
    or above ``lo`` (and, with ``need_out``, until the source's excess is gone).  Moves into a part are not counted
    against its floor, nor moves out of it against its cap, so the bounds hold whatever subset is applied."""
    if nodes.numel():
        o = _order(nodes, gain, to)
        nodes, to, gain, wt, frm = nodes[o], to[o], gain[o], wt[o], frm[o]
        cum = _seg_cumsum(wt, to)
        ok = sizes[to] + cum <= hi
        if need_in is not None:
            ok &= cum - wt < need_in[to]
        nodes, to, gain, wt, frm = nodes[ok], to[ok], gain[ok], wt[ok], frm[ok]
    if nodes.numel() and (lo is not None or need_out is not None):
        o = _order(nodes, gain, frm)
        nodes, to, gain, wt, frm = nodes[o], to[o], gain[o], wt[o], frm[o]
        cum = _seg_cumsum(wt, frm)
        ok = torch.ones_like(cum, dtype=torch.bool)
        if lo is not None:
            ok &= sizes[frm] - cum >= lo
        if need_out is not None:
            ok &= cum - wt < need_out[frm]
        nodes, to = nodes[ok], to[ok]
    return nodes, to


# ---- coarsening ----------------------------------------------------------------------------------------------------

def cluster(g: Csr, nw: Optional[torch.Tensor], cap: int, seed: int, rounds: int = 0) -> torch.Tensor:
    """Size-constrained label propagation: int32 cluster label of every node (a node id), every cluster's weight <= cap
    (each node starts alone, so the cap holds as long as cap >= the heaviest node)."""
    from .. import ops
    n, dev = g.n, g.indptr.device
    label = torch.arange(n, dtype=torch.int32, device=dev)
    wl = nw.to(torch.int64) if nw is not None else torch.ones(n, dtype=torch.int64, device=dev)
    for r in range(rounds or CLUSTER_ROUNDS):
        rating = ops.part_edges(g.indptr, g.idx, g.w, n, 0, False, col_map=label)
        cw = ops.part_weights(label, nw, n)
        tgt, gain = ops.part_cluster(rating, label, nw, cw, cap, seed * 1000003 + r * 7919 + 1)
        cand = torch.nonzero(tgt >= 0, as_tuple=True)[0]
        if cand.numel() == 0:
            break
        movers, to = admit(cand, tgt[cand].long(), gain[cand], wl[cand], label[cand].long(), cw, cap)
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


def contract(g: Csr, nw: Optional[torch.Tensor], cmap: torch.Tensor, nc: int) -> Tuple[Csr, torch.Tensor]:
    """The coarse graph: edge weights between clusters summed, intra-cluster edges dropped; node weights summed."""
    from .. import ops
    cg = Csr(*ops.part_edges(g.indptr, g.idx, g.w, nc, 0, True, row_map=cmap, col_map=cmap))
    return cg, ops.part_weights(cmap, nw, nc).to(torch.int32)


# ---- initial partition (host) ----------------------------------------------------------------------------------------

def initial_partition(indptr: np.ndarray, idx: np.ndarray, w: np.ndarray, nw: np.ndarray, n_parts: int, lo: int,
                      hi: int, seed: int, trials: int = 8) -> np.ndarray:
    """Greedy graph growing on a small weighted graph: parts 0 .. P-2 are grown one at a time from a seeded random
    node, always adding the unassigned node with the largest weight into the part minus weight out of it (ties: lower
    id) that keeps it within
    ``hi``, until it reaches its share of the remaining weight; the last part takes the rest.  The best of ``trials``
    seeded trials by (bound violation, weighted cut) is returned (int64 [n])."""
    n = int(nw.shape[0])
    indptr, idx, w, nw = (np.asarray(a, dtype=np.int64) for a in (indptr, idx, w, nw))
    rows = np.repeat(np.arange(n), np.diff(indptr))
    wdeg = np.bincount(rows, weights=w, minlength=n).astype(np.int64)
    best, best_key = None, None
    for t in range(trials):
        rng = np.random.default_rng([seed, t, 104729])
        order = rng.permutation(n)
        nxt = 0
        part = np.full(n, -1, dtype=np.int64)
        remaining = int(nw.sum())
        for p in range(n_parts - 1):
            share = remaining // (n_parts - p)
            conn = np.zeros(n, dtype=np.int64)
            blocked = np.zeros(n, dtype=bool)
            heap: List[Tuple[int, int]] = []
            pw = 0
            while pw < share:
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
                if pw > 0 and pw + nw[v] > hi:
                    blocked[v] = True
                    continue
                part[v] = p
                pw += int(nw[v])
                for k in range(indptr[v], indptr[v + 1]):
                    u = int(idx[k])
                    if part[u] < 0:
                        conn[u] += w[k]
                        heapq.heappush(heap, (-int(2 * conn[u] - wdeg[u]), u))
            nxt = 0
            remaining -= pw
        part[part < 0] = n_parts - 1
        sizes = np.bincount(part, weights=nw, minlength=n_parts).astype(np.int64)
        viol = int(np.maximum(sizes - hi, 0).sum() + np.maximum(lo - sizes, 0).sum())
        cut = int(w[part[rows] != part[idx]].sum())
        key = (viol, cut)
        if best_key is None or key < best_key:
            best, best_key = part, key
    return best


def block_partition(indptr: np.ndarray, idx: np.ndarray, nw: np.ndarray, n_parts: int) -> np.ndarray:
    """A reverse Cuthill-McKee order of the graph cut into P blocks of (about) equal weight (int64 [n])."""
    import scipy.sparse as sp
    from scipy.sparse.csgraph import reverse_cuthill_mckee
    n = int(nw.shape[0])
    a = sp.csr_matrix((np.ones(idx.shape[0], dtype=np.int8), idx, indptr), shape=(n, n))
    order = np.asarray(reverse_cuthill_mckee(a, symmetric_mode=True), dtype=np.int64)
    w = np.asarray(nw, dtype=np.int64)[order]
    before = np.cumsum(w) - w
    part = np.empty(n, dtype=np.int64)
    part[order] = np.minimum(before * n_parts // max(int(w.sum()), 1), n_parts - 1)
    return part


# ---- refinement ----------------------------------------------------------------------------------------------------

class _Level:
    """One level's graph and what its objective needs."""

    def __init__(self, g: Csr, nw: Optional[torch.Tensor], n_parts: int, objective: str,
                 out_g: Optional[Csr] = None, in_g: Optional[Csr] = None):
        self.g, self.nw, self.P, self.objective = g, nw, n_parts, objective
        self.out_g, self.in_g = out_g, in_g
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
        movers, to = admit(cand, tgt[cand].long(), gain[cand], lv.wl[cand], part[cand].long(), sizes, hi, lo)
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
    finest level) the bounds always end up holding."""
    P = lv.P
    for _ in range(max_passes or 4 * P + 8):
        sizes = lv.sizes(part)
        s = sizes.cpu()
        over, under = s > hi, s < lo
        if not bool(over.any()) and not bool(under.any()):
            break
        conn, occ, _ = lv.table(part)
        if bool(over.any()):
            allowed = sum(1 << p for p in range(P) if s[p] < hi)
            if allowed == 0:
                break
            tgt, gain = lv.gains(part, conn, occ, allowed)
            src_over = over.to(part.device)[part.long()]
            cand = torch.nonzero(src_over & (tgt >= 0), as_tuple=True)[0]
            movers, to = admit(cand, tgt[cand].long(), gain[cand], lv.wl[cand], part[cand].long(), sizes, hi,
                               need_out=(sizes - hi).clamp(min=0))
        else:
            allowed = sum(1 << p for p in range(P) if s[p] < lo)
            tgt, gain = lv.gains(part, conn, occ, allowed)
            cand = torch.nonzero((tgt >= 0) & (sizes[part.long()] > lo), as_tuple=True)[0]
            movers, to = admit(cand, tgt[cand].long(), gain[cand], lv.wl[cand], part[cand].long(), sizes, hi, lo,
                               need_in=(lo - sizes).clamp(min=0))
        if movers.numel() == 0:
            break
        part = part.clone()
        part[movers] = to.to(torch.int32)
    return part


# ---- the whole scheme ------------------------------------------------------------------------------------------------

def multilevel_partition(fg: FullGraph, n_parts: int, objective: str = "vol", seed: int = 0,
                         device=None) -> Tuple[torch.Tensor, Dict[str, object]]:
    """Owner of every node (int64 ``[N]``, on the host) and a report: ``levels`` = [(nodes, undirected entries)] from
    the finest graph to the coarsest, the final exact ``cut`` / ``vol`` / ``min_size`` / ``max_size``, and ``seconds``
    per stage (build, coarsen, initial, uncoarsen)."""
    if objective not in ("cut", "vol"):
        raise ValueError(f"--partition-obj must be cut or vol, got {objective!r}")
    N, P = fg.n_nodes, n_parts
    if P == 1:
        return torch.zeros(N, dtype=torch.int64), {"levels": [], "cut": 0, "vol": 0, "min_size": N, "max_size": N}
    check_parts(N, P)
    dev = resolve_device(device)
    lo, hi = size_bounds(N, P)
    with torch.cuda.device(dev):
        part, info = _multilevel(fg, P, objective, seed, dev, lo, hi)
        # every device tensor of the run is gone with _multilevel's frame: hand the cached blocks back, so that a process
        # that only partitions (main.py partitions in its parent before it spawns the ranks) holds no workspace while
        # the ranks train
        torch.cuda.empty_cache()
    if not lo <= info["min_size"] <= info["max_size"] <= hi:
        raise RuntimeError(f"multilevel partition out of its size bounds [{lo}, {hi}]: part sizes "
                           f"{info['min_size']} .. {info['max_size']}")
    return part, info


def _multilevel(fg: FullGraph, P: int, objective: str, seed: int, dev, lo: int, hi: int):
    """The scheme itself, on the current device; every device tensor it makes dies with its frame."""
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
    del indptr, src
    lap("build")
    # coarsening
    graphs: List[Tuple[Csr, Optional[torch.Tensor]]] = [(g0, None)]
    maps: List[torch.Tensor] = []
    cap = max(1, int(IMBALANCE * N / P))
    stalled = False                         # coarsening stopped before the coarsest graph got small
    while graphs[-1][0].n > COARSE_NODES_PER_PART * P and len(graphs) < 48:
        g, nw = graphs[-1]
        cmap, nc = compact(cluster(g, nw, cap, seed + 17 * len(graphs)))
        if nc >= g.n:
            stalled = True
            break
        graphs.append(contract(g, nw, cmap, nc))
        maps.append(cmap)
        if nc > 0.9 * g.n:
            stalled = nc > COARSE_NODES_PER_PART * P
            break
    lap("coarsen")
    # initial partitions of the coarsest graph (on the host), each projected and refined down to the finest level
    gc, nwc = graphs[-1]
    nw_host = nwc.cpu().numpy() if nwc is not None else np.ones(gc.n, dtype=np.int64)
    size = gc.n + gc.nnz + 1
    starts: List[Tuple[int, torch.Tensor]] = []
    if size <= GROWING_MAX_ENTRIES:         # the host work is bounded: trials x restarts x size
        trials = max(1, min(INITIAL_TRIALS, 2 * GROWING_MAX_ENTRIES // size))
        for r in range(max(1, min(RESTARTS, 4 * GROWING_MAX_ENTRIES // (size * trials)))):
            init = initial_partition(gc.indptr.cpu().numpy(), gc.idx.cpu().numpy(), gc.w.cpu().numpy(), nw_host,
                                     P, lo, hi, seed * RESTARTS + r, trials)
            starts.append((len(graphs) - 1, torch.from_numpy(init).to(dev, torch.int32)))
    else:
        init = block_partition(gc.indptr.cpu().numpy(), gc.idx.cpu().numpy(), nw_host, P)
        starts.append((len(graphs) - 1, torch.from_numpy(init).to(dev, torch.int32)))
    if stalled:     # no hierarchy worth the name: the flat stand-in's partition, refined below, is one more candidate
        from .partition import assign_parts
        starts.append((0, assign_parts(fg, P, "metis", seed, objective, dev).to(dev, torch.int32)))
    lap("initial")
    # uncoarsening; the candidate with the lowest exact objective is kept (ties: the earlier one)
    best, best_score = None, None
    for k, (top, part) in enumerate(starts):
        for lvl in range(top, -1, -1):
            g, nw = graphs[lvl]
            if lvl < top:
                part = part[maps[lvl].long()]
            lv = _Level(g, nw, P, "cut")
            part = rebalance(lv, part, lo, hi)
            if top > 0 or objective == "cut":      # a flat start is refined on the requested objective alone
                part = refine(lv, part, lo, hi, seed * 131 + 7 * k + lvl)
            if lvl == 0 and objective == "vol":    # the finest level: the edge cut first, then the exact volume
                lv = _Level(g, nw, P, "vol", out_g, in_g)
                part = refine(lv, part, lo, hi, seed * 131 + 7 * k + 977)
            part = rebalance(lv, part, lo, hi)
        _, _, q = ops.part_conn(*out_g, part, P, table=False, quality=True)
        score = int(q[0 if objective == "cut" else 1])
        if best_score is None or score < best_score:
            best, best_score = part, score
    part = best
    lap("uncoarsen")
    _, _, q = ops.part_conn(*out_g, part, P, table=False, quality=True)
    sizes = ops.part_weights(part, None, P).cpu()
    info = {"levels": [(gg.n, gg.nnz) for gg, _ in graphs], "cut": int(q[0]), "vol": int(q[1]),
            "min_size": int(sizes.min()), "max_size": int(sizes.max()), "candidates": len(starts),
            "seconds": seconds}
    return part.to(torch.int64).cpu(), info
