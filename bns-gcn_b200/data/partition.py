"""Vertex partitioner that emits the data contract of the reference's partition loader.

The reference calls ``dgl.distributed.partition_graph`` / ``load_partition``
(``helper/utils.py:73-140``); DGL and METIS are not available here, so this file
produces, per rank, exactly what ``load_partition`` returns and ``train.run``
relies on (SURVEY.md §3.2):

* node ids are relabelled so that partition ``i`` owns the contiguous global range
  ``[ranges[i], ranges[i+1])``  (``gpb.partid2nids``, used at ``train.py:97-101`` and
  ``utils.py:167-168``);
* the local graph holds **all in-edges of the inner nodes**; inner nodes have local ids
  ``[0, n_in)``, the 1-hop halo nodes follow (``train.py:85-86`` depends on this);
* ``node_dict['_ID']`` (global id), ``['part_id']`` (owner) and ``['inner_node']`` have one entry
  per local node; ``feat/label/in_deg/out_deg/train_mask(/val_mask/test_mask)`` one entry per
  inner node; degrees are those of the *full* graph (``utils.py:92-93``);
* ``meta`` = ``n_feat, n_class, n_train`` with the global train count (``utils.py:97-98``).

``--partition-method random`` is the reference's own option (``helper/parser.py:37``).
``metis`` is served by a stand-in: a reverse Cuthill-McKee order cut into equal blocks, then refined by balanced
label propagation (``refine_label_propagation``) on the objective ``--partition-obj`` names (``cut``: edges between
parts; ``vol``: communication volume = halo nodes summed over the parts, the reference's default, parser.py:35-36).
It is structure-aware and never worse than its starting point, but it is not a multilevel partitioner: expect METIS to
cut fewer edges on real graphs.  ``multilevel`` is one, on the GPU (``data/multilevel.py``).  The contract is the same.

``--partition-balance`` picks what every method balances.  ``nodes`` (the default): each part's node count lies in
``[max(int(0.97 N / P), 1), int(1.03 N / P) + 1]``.  ``edges``: those node bounds, and each part's in-edge count (the
directed edges whose destination it owns, loops included: the nnz of its ``a_in`` plus ``a_out`` rows) is at most
``in_edge_bound`` = ``int(1.03 E / P)`` plus the largest in-degree, the slack of one indivisible node.  A rank's
aggregation work is its in-edges, so on power-law graphs a node-balanced part can carry twice the mean rank's work.
"""
from __future__ import annotations

import dataclasses
from typing import Dict, List, Optional

import numpy as np
import torch

from .synthetic import FullGraph

NID = "_ID"   # the key DGL uses for ``dgl.NID``
BALANCES = ("nodes", "edges")
IMBALANCE = 0.03


def in_edge_bound(in_edges: torch.Tensor, n_parts: int, imbalance: float = IMBALANCE) -> int:
    """``--partition-balance edges``: the most in-edges a part may own, ``int((1 + imbalance) E / P)`` plus the largest
    in-degree (``in_edges``: every node's in-edge count, loops included)."""
    if in_edges.numel() == 0:
        return 0
    return int((1.0 + imbalance) * int(in_edges.sum()) / n_parts) + int(in_edges.max())


def check_balance(balance: str) -> None:
    if balance not in BALANCES:
        raise ValueError(f"--partition-balance must be one of {', '.join(BALANCES)}, got {balance!r}")


def check_bounds(fg: FullGraph, part: torch.Tensor, n_parts: int, method: str, balance: str) -> None:
    """Raise unless every part of ``part`` is within the node bounds and, with ``edges``, the in-edge bound; the
    message names the bound and the first part outside it."""
    n = fg.n_nodes
    lo, hi = max(int((1.0 - IMBALANCE) * n / n_parts), 1), int((1.0 + IMBALANCE) * n / n_parts) + 1
    part = part.cpu()
    sizes = torch.bincount(part, minlength=n_parts)
    bad = torch.nonzero((sizes < lo) | (sizes > hi), as_tuple=True)[0]
    if bad.numel():
        p = int(bad[0])
        raise RuntimeError(f"--partition-method {method} --partition-balance {balance}: part {p} has {int(sizes[p])} "
                           f"nodes, outside the node bounds [{lo}, {hi}]")
    if balance == "edges":
        deg = fg.in_degrees()
        ehi = in_edge_bound(deg, n_parts)
        esizes = torch.zeros(n_parts, dtype=torch.int64).index_add_(0, part, deg)
        bad = torch.nonzero(esizes > ehi, as_tuple=True)[0]
        if bad.numel():
            p = int(bad[0])
            raise RuntimeError(f"--partition-method {method} --partition-balance edges: part {p} owns "
                               f"{int(esizes[p])} in-edges, above the in-edge bound {ehi} = int(1.03 E / P) + d_max")


@dataclasses.dataclass
class GraphPartitionBook:
    """Stand-in for DGL's ``gpb``: only ``partid2nids`` is used by the path (``train.py:97-98``)."""
    ranges: torch.Tensor   # int64 [P+1]

    def partid2nids(self, i: int) -> torch.Tensor:
        return torch.arange(int(self.ranges[i]), int(self.ranges[i + 1]), dtype=torch.int64)

    def num_partitions(self) -> int:
        return int(self.ranges.numel() - 1)


@dataclasses.dataclass
class LocalGraph:
    """The ``subg`` of ``load_partition``: in-edges of inner nodes, CSR by (inner) destination.

    ``indices`` are local source ids: ``< n_in`` inner, ``>= n_in`` halo.
    """
    n_in: int
    n_halo: int
    indptr: torch.Tensor    # int64 [n_in+1]
    indices: torch.Tensor   # int64 [E_local]

    def num_nodes(self) -> int:
        return self.n_in + self.n_halo

    def num_edges(self) -> int:
        return int(self.indices.numel())


@dataclasses.dataclass
class Partition:
    rank: int
    n_parts: int
    graph: LocalGraph
    node_dict: Dict[str, torch.Tensor]
    gpb: GraphPartitionBook
    meta: Dict[str, int]


def shed_in_edges(part: torch.Tensor, in_edges: torch.Tensor, n_parts: int, bound: int, method: str) -> torch.Tensor:
    """Bring every part's in-edges within ``bound`` without changing any part's node count: while a part is above it,
    its highest in-degree nodes are swapped, one for one, with the lowest in-degree nodes of the part with the fewest
    in-edges (ties: the lower id), as few pairs as bring the heavy part down to the mean ``E / P`` or the light part up
    to it.  Raises, naming the bound and the part, when a swap can no longer help."""
    part = part.clone()
    target = -(-int(in_edges.sum()) // n_parts)
    for _ in range(4 * n_parts + 8):
        esizes = torch.zeros(n_parts, dtype=torch.int64).index_add_(0, part, in_edges)
        a = int(torch.argmax(esizes))
        if int(esizes[a]) <= bound:
            return part
        b = int(torch.argmin(esizes))
        want = min(int(esizes[a]) - target, target - int(esizes[b]))
        heavy = torch.nonzero(part == a, as_tuple=True)[0]
        light = torch.nonzero(part == b, as_tuple=True)[0]
        heavy = heavy[torch.sort(-in_edges[heavy], stable=True)[1]]
        light = light[torch.sort(in_edges[light], stable=True)[1]]
        k = min(heavy.numel(), light.numel())
        net = torch.cumsum(in_edges[heavy[:k]] - in_edges[light[:k]], 0)
        reach = torch.nonzero(net >= want, as_tuple=True)[0]
        m = int(reach[0]) + 1 if reach.numel() else int(torch.argmax(net)) + 1 if k else 0
        if m == 0 or int(net[m - 1]) <= 0:
            break
        part[heavy[:m]], part[light[:m]] = b, a
    esizes = torch.zeros(n_parts, dtype=torch.int64).index_add_(0, part, in_edges)
    a = int(torch.argmax(esizes))
    raise RuntimeError(f"--partition-method {method} --partition-balance edges: part {a} owns {int(esizes[a])} "
                       f"in-edges, above the in-edge bound {bound} = int(1.03 E / P) + d_max, and no swap of nodes "
                       "lowers it")


def partition_quality(fg: FullGraph, part: torch.Tensor, n_parts: int, device=None) -> Dict[str, float]:
    """``cut``: directed non-loop edges whose ends have different owners; ``vol``: communication volume =
    sum over parts of their halo size (distinct (source node, destination part) pairs across parts); sizes; the fewest
    and most in-edges a part owns (directed edges by the owner of their destination, loops included)."""
    dev = torch.device(device) if device is not None else torch.device("cpu")
    part = part.to(dev)
    src, dst = fg.src.to(dev), fg.dst().to(dev)
    ps, pd = part[src], part[dst]
    cross = ps != pd
    cut = int(cross.sum())
    vol = int(torch.unique(src[cross] * n_parts + pd[cross]).numel())
    sizes = torch.bincount(part, minlength=n_parts)
    in_edges = torch.bincount(pd, minlength=n_parts)
    return {"cut": cut, "vol": vol, "edges": int((src != dst).sum()), "max_size": int(sizes.max()),
            "min_size": int(sizes.min()), "min_in_edges": int(in_edges.min()), "max_in_edges": int(in_edges.max())}


def refine_label_propagation(fg: FullGraph, part: torch.Tensor, n_parts: int, objective: str = "vol",
                             rounds: int = 24, imbalance: float = 0.03, seed: int = 0, device=None,
                             in_edge_cap: Optional[int] = None) -> torch.Tensor:
    """Balanced label propagation: every round each node looks at the owners of its neighbours, the nodes that would
    gain most by joining the majority owner move -- as many as the target part has room for under the size cap
    ``(1 + imbalance) N / P`` (and the source part above the floor ``(1 - imbalance) N / P``), and only a random half of
    them per round (simultaneous moves of neighbours can undo
    each other).  With ``in_edge_cap``, a move is also admitted only while its target part's in-edges (loops included)
    stay within the cap, counted the same way as the room.  A round that does not improve ``objective`` ("cut" |
    "vol") is rolled back (three in a row end the refinement), so the result is never worse than the input.  Pure torch (sorting / unique / scatter): runs on
    ``device``."""
    dev = torch.device(device) if device is not None else torch.device("cpu")
    n, P = fg.n_nodes, n_parts
    if P == 1 or fg.n_edges == 0:
        return part
    gen = torch.Generator().manual_seed(seed + 104729)
    src_all, dst_all = fg.src.to(dev), fg.dst().to(dev)
    keep = src_all != dst_all
    src, dst = src_all[keep], dst_all[keep]
    part = part.to(dev).clone()
    cap = int((1.0 + imbalance) * n / P) + 1
    floor = max(int((1.0 - imbalance) * n / P), 1)
    deg = fg.in_degrees().to(dev) if in_edge_cap is not None else None

    def score(p):
        ps, pd = p[src], p[dst]
        cross = ps != pd
        if objective == "cut":
            return int(cross.sum())
        return int(torch.unique(src[cross] * P + pd[cross]).numel())

    best = score(part)
    failed = 0
    for _ in range(rounds):
        key = dst * P + part[src]                                   # (node, owner of an in-neighbour)
        uk, cnt = torch.unique(key, return_counts=True)
        node, lab = uk // P, uk % P
        cur = torch.zeros(n, dtype=cnt.dtype, device=dev)
        own = lab == part[node]
        cur[node[own]] = cnt[own]
        top = torch.zeros(n, dtype=cnt.dtype, device=dev).scatter_reduce(0, node, cnt, "amax", include_self=True)
        is_top = cnt == top[node]
        target = torch.full((n,), P, dtype=torch.int64, device=dev).scatter_reduce(
            0, node[is_top], lab[is_top], "amin", include_self=True)  # smallest majority owner
        gain = top - cur
        cand = torch.nonzero((gain > 0) & (target < P) & (target != part), as_tuple=True)[0]
        if cand.numel() == 0:
            break
        half = torch.rand(cand.numel(), generator=gen).to(dev) < 0.5
        cand = cand[half] if int(half.sum()) > 0 else cand
        # per target part: the best `room` candidates by gain
        order = torch.argsort(target[cand] * (int(gain.max()) + 1) + (int(gain.max()) - gain[cand]))
        cand = cand[order]
        tgt = target[cand]
        sizes = torch.bincount(part, minlength=P)
        room = (cap - sizes).clamp(min=0)
        first = torch.searchsorted(tgt, torch.arange(P, device=dev))
        rank = torch.arange(cand.numel(), device=dev) - first[tgt]
        ok = rank < room[tgt]
        if deg is not None:                                          # and the target's in-edges under their cap
            esizes = torch.zeros(P, dtype=torch.int64, device=dev).index_add_(0, part, deg)
            cs = torch.cumsum(deg[cand], 0)
            before = torch.where(first > 0, cs[(first - 1).clamp(min=0)], torch.zeros_like(first))
            ok &= esizes[tgt] + cs - before[tgt] <= in_edge_cap
        movers, to = cand[ok], tgt[ok]
        if movers.numel():                                           # nor may a part shrink below the floor
            frm = part[movers]
            o2 = torch.argsort(frm, stable=True)                     # keeps the gain order inside each source part
            movers, to, frm = movers[o2], to[o2], frm[o2]
            first2 = torch.searchsorted(frm, torch.arange(P, device=dev))
            rank2 = torch.arange(movers.numel(), device=dev) - first2[frm]
            ok2 = rank2 < (sizes - floor).clamp(min=0)[frm]
            movers, to = movers[ok2], to[ok2]
        if movers.numel() == 0:
            break
        trial = part.clone()
        trial[movers] = to
        sc = score(trial)
        if sc >= best:                                               # roll back: keep the previous assignment and
            failed += 1                                              # try another random half
            if failed >= 3:
                break
            continue
        part, best, failed = trial, sc, 0
    return part.cpu()


def assign_parts(fg: FullGraph, n_parts: int, method: str, seed: int, objective: str = "vol", device=None,
                 balance: str = "nodes") -> torch.Tensor:
    """Owner of every node, int64 ``[N]``: ``random`` balanced to ±1 node, ``metis`` (stand-in) and ``multilevel`` (the
    GPU partitioner; ``device`` None = the current CUDA device) within 3 %.  ``balance="edges"``: every method keeps
    each part within the node bounds and the in-edge bound (``in_edge_bound``), or raises naming the bound and part."""
    check_balance(balance)
    n = fg.n_nodes
    if n_parts == 1:
        return torch.zeros(n, dtype=torch.int64)
    if method == "random":
        gen = torch.Generator().manual_seed(seed + 7919)
        order = torch.randperm(n, generator=gen)
    elif method == "multilevel":                      # the GPU partitioner (data/multilevel.py)
        from .multilevel import multilevel_partition
        return multilevel_partition(fg, n_parts, objective, seed, device, balance)[0]
    elif method == "metis":
        import scipy.sparse as sp
        from scipy.sparse.csgraph import reverse_cuthill_mckee
        a = sp.csr_matrix((np.ones(fg.n_edges, dtype=np.int8), fg.src.numpy(), fg.indptr.numpy()), shape=(n, n))
        order = torch.from_numpy(np.ascontiguousarray(reverse_cuthill_mckee(a, symmetric_mode=True)).astype(np.int64))
    else:
        raise ValueError(f"unknown partition method {method!r}")
    part = torch.empty(n, dtype=torch.int64)
    part[order] = (torch.arange(n, dtype=torch.int64) * n_parts) // n
    ehi = None
    if balance == "edges":                            # the same blocks with their in-edges evened out by swaps
        deg = fg.in_degrees()
        ehi = in_edge_bound(deg, n_parts)
        part = shed_in_edges(part, deg, n_parts, ehi, method)
    if method == "metis":
        part = refine_label_propagation(fg, part, n_parts, objective=objective, seed=seed, device=device,
                                        in_edge_cap=ehi)
    if balance == "edges":
        check_bounds(fg, part, n_parts, method, balance)
    return part


def relabel(fg: FullGraph, part: torch.Tensor, n_parts: int, device: Optional[torch.device] = None):
    """Renumber nodes so every partition is a contiguous id range (what DGL's partitioner does)."""
    if device is None:
        device = torch.device("cuda") if torch.cuda.is_available() else torch.device("cpu")
    n = fg.n_nodes
    order = torch.argsort(part, stable=True)              # new id -> old id
    new_id = torch.empty(n, dtype=torch.int64)
    new_id[order] = torch.arange(n, dtype=torch.int64)
    counts = torch.bincount(part, minlength=n_parts)
    ranges = torch.zeros(n_parts + 1, dtype=torch.int64)
    ranges[1:] = torch.cumsum(counts, 0)
    nid = new_id.to(device)
    dst = nid[fg.dst().to(device)]
    src = nid[fg.src.to(device)]
    perm = torch.argsort(dst * n + src)
    dst, src = dst[perm], src[perm]
    indptr = torch.zeros(n + 1, dtype=torch.int64, device=device)
    indptr[1:] = torch.cumsum(torch.bincount(dst, minlength=n), 0)
    g = FullGraph(n, indptr.cpu(), src.cpu(), fg.feat[order], fg.label[order], fg.train_mask[order],
                  fg.val_mask[order], fg.test_mask[order], fg.n_class)
    return g, ranges


def induced_subgraph(fg: FullGraph, mask: torch.Tensor) -> FullGraph:
    """``g.subgraph(mask)`` (``utils.py:77`` inductive setting): keep edges with both ends in ``mask``."""
    n = fg.n_nodes
    keep = torch.nonzero(mask, as_tuple=True)[0]
    new_id = torch.full((n,), -1, dtype=torch.int64)
    new_id[keep] = torch.arange(keep.numel(), dtype=torch.int64)
    dst = new_id[fg.dst()]
    src = new_id[fg.src]
    ok = (dst >= 0) & (src >= 0)
    dst, src = dst[ok], src[ok]                            # order (dst, src) is preserved
    m = keep.numel()
    indptr = torch.zeros(m + 1, dtype=torch.int64)
    indptr[1:] = torch.cumsum(torch.bincount(dst, minlength=m), 0)
    return FullGraph(m, indptr, src, fg.feat[keep], fg.label[keep], fg.train_mask[keep],
                     fg.val_mask[keep], fg.test_mask[keep], fg.n_class)


def extract_partition(g: FullGraph, ranges: torch.Tensor, rank: int, inductive: bool = False,
                      in_deg: Optional[torch.Tensor] = None, out_deg: Optional[torch.Tensor] = None) -> Partition:
    """Cut rank ``rank``'s piece out of a relabelled graph (``load_partition``, ``utils.py:101-140``)."""
    n_parts = int(ranges.numel() - 1)
    start, end = int(ranges[rank]), int(ranges[rank + 1])
    n_in = end - start
    e0, e1 = int(g.indptr[start]), int(g.indptr[end])
    src = g.src[e0:e1]
    inner = (src >= start) & (src < end)
    halo = torch.unique(src[~inner])                       # sorted global ids
    local = torch.where(inner, src - start, n_in + torch.searchsorted(halo, src))
    indptr = (g.indptr[start:end + 1] - e0).clone()
    if in_deg is None:
        in_deg = g.in_degrees()
    if out_deg is None:
        out_deg = g.out_degrees()
    gid = torch.cat([torch.arange(start, end, dtype=torch.int64), halo])
    part_id = torch.searchsorted(ranges, gid, right=True) - 1
    inner_node = torch.zeros(gid.numel(), dtype=torch.bool)
    inner_node[:n_in] = True
    nd = {
        NID: gid,
        "part_id": part_id,
        "inner_node": inner_node,
        "feat": g.feat[start:end].clone(),
        "label": g.label[start:end].clone(),
        "in_deg": in_deg[start:end].clone(),
        "out_deg": out_deg[start:end].clone(),
        "train_mask": g.train_mask[start:end].clone(),
    }
    if not inductive:
        nd["val_mask"] = g.val_mask[start:end].clone()
        nd["test_mask"] = g.test_mask[start:end].clone()
    meta = {"n_feat": g.n_feat, "n_class": g.n_class, "n_train": int(g.train_mask.sum())}
    return Partition(rank, n_parts, LocalGraph(n_in, int(halo.numel()), indptr, local.contiguous()), nd,
                     GraphPartitionBook(ranges.clone()), meta)


def partition_graph(fg: FullGraph, n_parts: int, method: str = "random", seed: int = 0,
                    inductive: bool = False, ranks: Optional[List[int]] = None,
                    device: Optional[torch.device] = None, objective: str = "vol",
                    balance: str = "nodes") -> List[Partition]:
    """``graph_partition`` + ``load_partition`` in one call; returns the pieces for ``ranks`` (default all).
    ``objective``: ``--partition-obj`` (``vol`` | ``cut``), used by ``metis`` (the stand-in) and ``multilevel``.
    ``balance``: ``--partition-balance`` (``nodes`` | ``edges``), for every method; under ``inductive`` the bounds are
    those of the train-node subgraph."""
    if inductive:
        fg = induced_subgraph(fg, fg.train_mask)
    part = assign_parts(fg, n_parts, method, seed, objective, device, balance)
    g, ranges = relabel(fg, part, n_parts, device)
    in_deg, out_deg = g.in_degrees(), g.out_degrees()
    if ranks is None:
        ranks = list(range(n_parts))
    return [extract_partition(g, ranges, r, inductive, in_deg, out_deg) for r in ranks]
