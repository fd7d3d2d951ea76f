"""Seeded synthetic graphs with the shapes BASELINE.json names.

Replaces ``helper/utils.py:37-70`` (``load_data``) of the reference, which pulls
Reddit / Yelp / ogbn-* through DGL and OGB (neither installable here, no
network).  What is kept is the *contract* of ``load_data``:

* a simple directed graph without multi-edges whose self-loops were removed and
  re-added exactly once per node (``utils.py:68-69``),
* ``feat`` f32 ``[N, n_feat]``, ``label`` int64 ``[N]`` (or f32 multi-label
  ``[N, n_class]``), boolean ``train/val/test`` masks,
* ``in_deg`` / ``out_deg`` of the *full* graph after the self-loops
  (``utils.py:92-93``).

All randomness comes from one CPU ``torch.Generator`` so that the same seed gives
the same graph whether the heavy sorting below runs on the CPU or on a GPU.
"""
from __future__ import annotations

import dataclasses
from typing import Optional

import torch


@dataclasses.dataclass
class FullGraph:
    """CSR by destination: in-neighbours of ``v`` are ``src[indptr[v]:indptr[v+1]]`` (sorted)."""
    n_nodes: int
    indptr: torch.Tensor      # int64 [N+1]
    src: torch.Tensor         # int64 [E]  (sorted inside each row)
    feat: torch.Tensor        # f32 [N, n_feat]
    label: torch.Tensor       # int64 [N] or f32 [N, n_class]
    train_mask: torch.Tensor  # bool [N]
    val_mask: torch.Tensor
    test_mask: torch.Tensor
    n_class: int

    @property
    def n_edges(self) -> int:
        return int(self.src.numel())

    @property
    def n_feat(self) -> int:
        return int(self.feat.shape[1])

    def in_degrees(self) -> torch.Tensor:
        return self.indptr[1:] - self.indptr[:-1]

    def out_degrees(self) -> torch.Tensor:
        return torch.bincount(self.src, minlength=self.n_nodes)

    def dst(self) -> torch.Tensor:
        return torch.repeat_interleave(torch.arange(self.n_nodes, dtype=torch.int64), self.in_degrees())


# name -> (N, directed edge target incl. self loops, n_feat, n_class, train fraction, multilabel, degree law)
SHAPES = {
    # BASELINE.json configs[0]
    "synthetic-10k": dict(n=10_000, e=100_000, n_feat=64, n_class=8, train=0.6, multilabel=False, law="uniform"),
    # configs[1]: Reddit: 232,965 nodes, 114,615,892 edges, 602 feats, 41 classes, 153,431 train nodes
    "reddit": dict(n=232_965, e=114_615_892, n_feat=602, n_class=41, train=153_431 / 232_965, multilabel=False,
                   law="powerlaw"),
    # configs[2]: ogbn-products
    "ogbn-products": dict(n=2_449_029, e=123_718_280, n_feat=100, n_class=47, train=0.08, multilabel=False,
                          law="powerlaw"),
    # configs[3]: Yelp (multi-label)
    "yelp": dict(n=716_847, e=13_954_819, n_feat=300, n_class=100, train=0.75, multilabel=True, law="powerlaw"),
    # configs[4]: ogbn-papers100M: 111,059,956 nodes, 1,615,685,872 edges, 128 feats, 172 classes.  Never built as one
    # graph (57 GB of features): every rank generates ITS piece on its GPU, see make_local_partition
    # (val / test: ogbn-papers100M's split, 125,265 / 214,338 nodes; read by make_local_partition only)
    "papers100m": dict(n=111_059_956, e=1_615_685_872, n_feat=128, n_class=172, train=0.011, multilabel=False,
                       law="powerlaw", val=0.0011, test=0.0019),
    # small shapes used by tests / smoke
    "tiny": dict(n=600, e=6_000, n_feat=16, n_class=5, train=0.5, multilabel=False, law="powerlaw"),
    "tiny-ml": dict(n=500, e=5_000, n_feat=12, n_class=6, train=0.6, multilabel=True, law="powerlaw"),
    "small": dict(n=6_000, e=240_000, n_feat=32, n_class=7, train=0.6, multilabel=False, law="powerlaw"),
}


def _endpoint_weights(n: int, law: str, avg_deg: float, max_deg_target: Optional[float]) -> torch.Tensor:
    """Expected-degree sequence of the Chung-Lu model (f64, sums to 1)."""
    if law == "uniform":
        w = torch.ones(n, dtype=torch.float64)
    elif law == "powerlaw":
        # shifted power law  w_i ∝ (i + i0)^(-2/3)  (degree exponent 2.5).  i0 caps the largest
        # expected degree near ``max_deg_target`` (Reddit: max degree 21,657 at average 492).
        alpha = 2.0 / 3.0
        i = torch.arange(1, n + 1, dtype=torch.float64)
        if max_deg_target is None:
            max_deg_target = 44.0 * avg_deg
        lo, hi = 0.0, float(n)
        for _ in range(60):                       # bisection on i0
            mid = 0.5 * (lo + hi)
            w = (i + mid) ** (-alpha)
            top = avg_deg * n * (w[0] / w.sum())
            if top > max_deg_target:
                lo = mid
            else:
                hi = mid
        w = (i + hi) ** (-alpha)
    else:
        raise ValueError(f"unknown degree law {law!r}")
    return w / w.sum()


def chung_lu_edges(n: int, n_directed_edges: int, law: str, gen: torch.Generator,
                   device: torch.device, oversample: float = 1.0):
    """Symmetric simple graph + one self loop per node, as CSR by destination.

    Draw ``M`` undirected pairs with both endpoints ∝ w (Chung-Lu), drop self pairs,
    de-duplicate, mirror, then add the self loops (``utils.py:68-69``).
    """
    target_undirected = max((n_directed_edges - n) // 2, 0)
    m = int(target_undirected * oversample)
    avg_deg = n_directed_edges / n
    w = _endpoint_weights(n, law, avg_deg, None)
    cdf = torch.cumsum(w, 0)
    cdf[-1] = 1.0
    perm = torch.randperm(n, generator=gen)        # decorrelate node id from degree
    keys = []
    chunk = 16_000_000
    cdf_d = cdf.to(device)
    perm_d = perm.to(device)
    done = 0
    while done < m:
        c = min(chunk, m - done)
        r = torch.rand(2, c, generator=gen, dtype=torch.float64).to(device)
        ends = torch.searchsorted(cdf_d, r).clamp_(max=n - 1)
        a, b = perm_d[ends[0]], perm_d[ends[1]]
        keep = a != b
        a, b = a[keep], b[keep]
        lo, hi = torch.minimum(a, b), torch.maximum(a, b)
        keys.append(torch.unique(lo * n + hi))
        done += c
    key = torch.unique(torch.cat(keys)) if keys else torch.empty(0, dtype=torch.int64, device=device)
    del keys
    lo, hi = key // n, key % n
    del key
    loops = torch.arange(n, dtype=torch.int64, device=device)
    dst = torch.cat([lo, hi, loops])
    src = torch.cat([hi, lo, loops])
    del lo, hi
    order = torch.argsort(dst * n + src)
    dst, src = dst[order], src[order]
    del order
    indptr = torch.zeros(n + 1, dtype=torch.int64, device=device)
    indptr[1:] = torch.cumsum(torch.bincount(dst, minlength=n), 0)
    return indptr.cpu(), src.cpu()


def make_graph(name: str, seed: int = 0, device: Optional[torch.device] = None,
               with_feat: bool = True, **override) -> FullGraph:
    """Build one of the named shapes.  ``override`` may replace any entry of ``SHAPES[name]``."""
    spec = dict(SHAPES[name])
    spec.update(override)
    if device is None:
        device = torch.device("cuda") if torch.cuda.is_available() else torch.device("cpu")
    gen = torch.Generator().manual_seed(seed)
    n = spec["n"]
    # hub-hub pairs are drawn repeatedly and collapse under de-duplication: oversample a little
    oversample = {"powerlaw": 1.015, "uniform": 1.0}[spec["law"]]
    indptr, src = chung_lu_edges(n, spec["e"], spec["law"], gen, device, oversample)
    fgen = torch.Generator().manual_seed(seed + 1)
    n_feat, n_class = spec["n_feat"], spec["n_class"]
    if with_feat:
        feat = torch.randn(n, n_feat, generator=fgen, dtype=torch.float32)
    else:
        feat = torch.empty(n, 0, dtype=torch.float32)
    if spec["multilabel"]:
        label = (torch.rand(n, n_class, generator=fgen) < 0.1).float()
    else:
        label = torch.randint(0, n_class, (n,), generator=fgen, dtype=torch.int64)
    r = torch.rand(n, generator=fgen)
    n_train = int(round(spec["train"] * n))
    order = torch.argsort(r)
    train_mask = torch.zeros(n, dtype=torch.bool)
    train_mask[order[:n_train]] = True
    rest = order[n_train:]
    val_mask = torch.zeros(n, dtype=torch.bool)
    val_mask[rest[: rest.numel() // 3]] = True
    test_mask = ~(train_mask | val_mask)
    return FullGraph(n, indptr, src, feat, label, train_mask, val_mask, test_mask, n_class)


# ---- per-rank generation (graphs that do not fit one host) -------------------------------------------------------
def _weights_on_device(n: int, avg_deg: float, device) -> torch.Tensor:
    """``_endpoint_weights(n, "powerlaw", ...)`` computed on ``device`` (f64, sums to 1, descending in the index)."""
    alpha = 2.0 / 3.0
    i = torch.arange(1, n + 1, dtype=torch.float64, device=device)
    lo, hi = 0.0, float(n)
    for _ in range(40):
        mid = 0.5 * (lo + hi)
        w = (i + mid) ** (-alpha)
        top = avg_deg * n * float(w[0] / w.sum())
        lo, hi = (mid, hi) if top > 44.0 * avg_deg else (lo, mid)
    w = (i + hi) ** (-alpha)
    return w / w.sum()


def make_local_partition(name: str, rank: int, world: int, seed: int = 0, device: Optional[torch.device] = None,
                         scale: float = 1.0):
    """Rank ``rank``'s partition of shape ``name`` under ``--partition-method random``, generated ON THE DEVICE without
    ever building the full graph (helper/utils.py:37-140 loads, partitions and re-loads the whole dataset on one host;
    the papers100M shape does not fit one).  Same contract as ``partition.extract_partition``.

    Model: directed Chung-Lu in-edges.  Rank r owns the contiguous id range ``[N r / P, N (r+1) / P)``; node u's
    expected degree is ``w[(A u + B) mod N]`` with A coprime to N -- ids are decorrelated from degrees, i.e. a contiguous
    range is a uniformly random set of nodes (the random partition).  It draws ``E / P`` (destination in its range,
    source anywhere) pairs, both ends proportional to w, removes duplicates, adds one self loop per node
    (utils.py:68-69).  ``in_deg`` is exact (every in-edge of an inner node is local); ``out_deg`` is set to ``in_deg``
    (the graph is symmetric in expectation; the true value would need a global count -- GraphSAGE does not use it).
    ``scale`` shrinks node and edge counts together (same average degree)."""
    from .partition import NID, GraphPartitionBook, LocalGraph, Partition
    spec = dict(SHAPES[name])
    if device is None:
        device = torch.device("cuda") if torch.cuda.is_available() else torch.device("cpu")
    n, e = max(int(spec["n"] * scale), world * 4), max(int(spec["e"] * scale), world * 8)
    ranges = torch.tensor([(n * i) // world for i in range(world + 1)], dtype=torch.int64)
    start, end = int(ranges[rank]), int(ranges[rank + 1])
    n_in = end - start
    w = _weights_on_device(n, e / n, device)
    cdf = torch.cumsum(w, 0)
    cdf[-1] = 1.0
    # the bijection id -> weight rank, and back
    import math
    A = 2_654_435_761 % n
    while math.gcd(A, n) != 1:
        A += 1
    B, A_inv = (7919 * (seed + 1)) % n, pow(A, -1, n)
    own = torch.arange(start, end, dtype=torch.int64, device=device)

    def to_rank(u):                                   # (A u + B) mod n without overflowing int64: A, u < 2^31 for n < 2^31
        return (u * A + B) % n

    def from_rank(k):
        return ((k - B) % n) * A_inv % n

    gen = torch.Generator(device=device).manual_seed(seed * 1_000_003 + rank)
    cdf_own = torch.cumsum(w[to_rank(own)], 0)
    total_own = float(cdf_own[-1])
    m = e // world
    keys = [own * n + own]                            # the self loops, as (dst, src) keys
    chunk = 32_000_000
    done = 0
    while done < m:
        c = min(chunk, m - done)
        r = torch.rand(2, c, generator=gen, dtype=torch.float64, device=device)
        dst = own[torch.searchsorted(cdf_own, r[0] * total_own).clamp_(max=n_in - 1)]
        src = from_rank(torch.searchsorted(cdf, r[1]).clamp_(max=n - 1))
        keys.append(torch.unique(dst * n + src))
        done += c
    key = torch.unique(torch.cat(keys))               # sorted by (dst, src)
    del keys
    dst, src = key // n, key % n
    del key
    indptr = torch.zeros(n_in + 1, dtype=torch.int64, device=device)
    indptr[1:] = torch.cumsum(torch.bincount(dst - start, minlength=n_in), 0)
    inner = (src >= start) & (src < end)
    halo = torch.unique(src[~inner])                  # sorted global ids
    local = torch.where(inner, src - start, n_in + torch.searchsorted(halo, src))
    gid = torch.cat([own, halo])
    part_id = torch.searchsorted(ranges.to(device), gid, right=True) - 1
    inner_node = torch.zeros(gid.numel(), dtype=torch.bool, device=device)
    inner_node[:n_in] = True
    in_deg = indptr[1:] - indptr[:-1]
    fgen = torch.Generator(device=device).manual_seed(seed * 1_000_003 + 7 + rank)
    n_feat, n_class = spec["n_feat"], spec["n_class"]
    feat = torch.randn(n_in, n_feat, generator=fgen, dtype=torch.float32, device=device)
    if spec["multilabel"]:
        label = (torch.rand(n_in, n_class, generator=fgen, device=device) < 0.1).float()
    else:
        label = torch.randint(0, n_class, (n_in,), generator=fgen, dtype=torch.int64, device=device)
    train_mask = torch.rand(n_in, generator=fgen, device=device) < spec["train"]
    # val / test from a generator of their own, so that every tensor above stays what it was without them; disjoint
    # from train_mask and from each other, at the shape's fractions of all nodes (default: make_graph's 1/3 : 2/3 split
    # of the rest)
    rest = 1.0 - spec["train"]
    p_val, p_test = spec.get("val", rest / 3) / rest, spec.get("test", 2 * rest / 3) / rest
    u = torch.rand(n_in, generator=torch.Generator(device=device).manual_seed(seed * 1_000_003 + 11 + rank),
                   device=device)
    val_mask = ~train_mask & (u < p_val)
    test_mask = ~train_mask & (u >= p_val) & (u < p_val + p_test)
    nd = {NID: gid, "part_id": part_id, "inner_node": inner_node, "feat": feat, "label": label, "in_deg": in_deg,
          "out_deg": in_deg.clone(), "train_mask": train_mask, "val_mask": val_mask, "test_mask": test_mask}
    meta = {"n_feat": n_feat, "n_class": n_class, "n_train": max(int(round(spec["train"] * n)), 1)}
    return Partition(rank, world, LocalGraph(n_in, int(halo.numel()), indptr, local.contiguous()), nd,
                     GraphPartitionBook(ranges.clone()), meta)
