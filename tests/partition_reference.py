"""Host restatement of the multilevel partitioner's kernels (csrc/partition.cuh), for the tests: plain torch on the CPU,
one definition per entry point, written for clarity rather than speed."""
import torch

M64 = (1 << 64) - 1


def edges(indptr, idx, w, n_out, mode, drop_loops, row_map=None, col_map=None):
    """bns_part_edges: (indptr int64, idx int32, w int32) of the merged, mapped, oriented entries."""
    indptr, idx = indptr.cpu().long(), idx.cpu().long()
    n = indptr.numel() - 1
    rows = torch.repeat_interleave(torch.arange(n), indptr[1:] - indptr[:-1])
    R = row_map.cpu().long()[rows] if row_map is not None else rows
    C = col_map.cpu().long()[idx] if col_map is not None else idx
    wt = w.cpu().long() if w is not None else torch.ones(idx.numel(), dtype=torch.int64)
    if mode == 0:
        a, b = R, C
    elif mode == 1:
        a, b = C, R
    else:
        a, b, wt = torch.cat([R, C]), torch.cat([C, R]), torch.cat([wt, wt])
    if drop_loops:
        keep = a != b
        a, b, wt = a[keep], b[keep], wt[keep]
    key = a * (1 << 32) + b
    uk, inv = torch.unique(key, return_inverse=True)
    sums = torch.zeros(uk.numel(), dtype=torch.int64).scatter_add_(0, inv, wt)
    out = torch.zeros(n_out + 1, dtype=torch.int64)
    out[1:] = torch.cumsum(torch.bincount(uk >> 32, minlength=n_out), 0)
    return out, (uk & 0xFFFFFFFF).int(), sums.int()


def conn(indptr, idx, w, part, P):
    """bns_part_conn: (conn int32 [n, P], occ int64 [n], (cut, vol))."""
    indptr, idx, part = indptr.cpu().long(), idx.cpu().long(), part.cpu().long()
    n = part.numel()
    rows = torch.repeat_interleave(torch.arange(n), indptr[1:] - indptr[:-1])
    wt = w.cpu().long() if w is not None else torch.ones(idx.numel(), dtype=torch.int64)
    c = torch.zeros(n * P, dtype=torch.int64).scatter_add_(0, rows * P + part[idx], wt).view(n, P)
    bits = (c > 0).long() << torch.arange(P)
    occ = torch.tensor([int(x) for x in bits.sum(1).tolist()], dtype=torch.int64) if n else torch.zeros(0, dtype=torch.int64)
    other = torch.ones(n, P, dtype=torch.bool)
    other[torch.arange(n), part] = False
    return c.int(), occ, (int(c[other].sum()), int((c[other] > 0).sum()))


def best_target(g, part, allowed=None):
    """bns_part_gains' choice from a full gain table [n, P]: the largest gain over the allowed parts != own (bit b of
    ``allowed``, None = all), ties to the lowest; target -1 and gain 0 where no such part exists."""
    part = part.cpu().long()
    n, P = g.shape
    mask = torch.ones(n, P, dtype=torch.bool)
    mask[torch.arange(n), part] = False
    if allowed is not None:
        mask &= torch.tensor([(int(allowed) >> b) & 1 == 1 for b in range(P)])[None, :]
    gm = torch.where(mask, g, torch.full_like(g, -(1 << 62)))
    best = gm.max(1).values
    tgt = (gm == best[:, None]).int().argmax(1).int()
    none = ~mask.any(1)
    return torch.where(none, -1, tgt).int(), torch.where(none, 0, best)


def cut_gains(indptr, idx, w, part, P, nodes):
    """The edge-cut gain of moving v alone to b, [len(nodes), P] int64, from the definition: the sum over v's row of
    w(u, v) ([part u = b] - [part u = a]), a = part v (0 at b = a)."""
    indptr, idx, part = indptr.cpu().long(), idx.cpu().long(), part.cpu().long()
    wt = w.cpu().long() if w is not None else torch.ones(idx.numel(), dtype=torch.int64)
    out = torch.zeros(len(nodes), P, dtype=torch.int64)
    for i, v in enumerate(nodes):
        s, e = int(indptr[v]), int(indptr[v + 1])
        a = int(part[v])
        pu, wu = part[idx[s:e]], wt[s:e]
        for b in range(P):
            if b != a:
                out[i, b] = int((wu * ((pu == b).long() - (pu == a).long())).sum())
    return out


def vol_gains(out_csr, in_csr, part, P, nodes):
    """The communication-volume gain of moving v alone to b, [len(nodes), P] int64, by recomputing the terms that can
    change: v's own (its out-neighbour parts other than its own) and each in-neighbour u's, from u's per-part out-edge
    counts with v's m(u, v) edges taken out of a and put into b.  ``out_csr`` / ``in_csr``: the merged out- and in-CSRs
    with multiplicities, loops dropped (bns_part_edges modes 1 and 0)."""
    part = part.cpu().long()
    cnt = conn(*out_csr, part, P)[0].long()                 # cnt[u][p]: u's out-edges into part p
    ip, ix = in_csr[0].cpu().long(), in_csr[1].cpu().long()
    iw = in_csr[2].cpu().long() if in_csr[2] is not None else torch.ones(ix.numel(), dtype=torch.int64)
    ar = torch.arange(P)

    def term(c, own):                                       # parts in c's support other than own, per row
        return ((c > 0) & (ar[None, :] != own[:, None])).sum(1)

    out = torch.zeros(len(nodes), P, dtype=torch.int64)
    for i, v in enumerate(nodes):
        a = int(part[v])
        s, e = int(ip[v]), int(ip[v + 1])
        u, m = ix[s:e], iw[s:e]
        cu, pu = cnt[u], part[u]
        before = int(term(cnt[v][None], part[v][None]).sum()) + int(term(cu, pu).sum())
        for b in range(P):
            if b == a:
                continue
            c2 = cu.clone()
            c2[:, a] -= m
            c2[:, b] += m
            after = int(term(cnt[v][None], torch.tensor([b])).sum()) + int(term(c2, pu).sum())
            out[i, b] = before - after
    return out


def part_hash(x):
    x = int(x) & M64
    x ^= x >> 33
    x = (x * 0xFF51AFD7ED558CCD) & M64
    x ^= x >> 33
    x = (x * 0xC4CEB9FE1A85EC53) & M64
    x ^= x >> 33
    return x & 0xFFFFFFFF


def cluster_step(rating, label, nw, cw, cap, seed):
    """bns_part_cluster, node by node."""
    ip, cid, wt = (t.cpu().long() for t in rating)
    label, cw = label.cpu().long(), cw.cpu().long()
    n = label.numel()
    nwl = nw.cpu().long() if nw is not None else torch.ones(n, dtype=torch.int64)
    tgt, gain = torch.full((n,), -1, dtype=torch.int32), torch.zeros(n, dtype=torch.int64)
    for v in range(n):
        if not part_hash(seed ^ ((v * 0x9E3779B97F4A7C15) & M64)) & 1:
            continue
        cur, best = 0, None
        for k in range(int(ip[v]), int(ip[v + 1])):
            c, w = int(cid[k]), int(wt[k])
            if c == int(label[v]):
                cur = w
                continue
            if int(cw[c]) + int(nwl[v]) > cap:
                continue
            key = (-w, part_hash(seed + c), c)
            if best is None or key < best:
                best = key
        if best is not None and -best[0] > cur:
            tgt[v], gain[v] = best[2], -best[0] - cur
    return tgt, gain


def admit(nodes, to, gain, wt, frm, sizes, hi, lo=None, need_in=None, need_out=None):
    """multilevel.admit, move by move: the admitted (node, target) pairs, sorted.  Per target, in (gain descending, id
    ascending) order, a move is kept while the target's size plus the running weight of every candidate so far (kept or
    not) is at most ``hi`` and, with ``need_in``, the weight before it is below the target's need; then the same per
    source over the kept moves, with the floor ``lo`` and ``need_out``."""
    L = [dict(v=int(nodes[i]), t=int(to[i]), g=int(gain[i]), w=int(wt[i]), f=int(frm[i])) for i in range(len(nodes))]
    sizes = [int(s) for s in sizes]
    kept, run = [], {}
    for x in sorted(L, key=lambda x: (x["t"], -x["g"], x["v"])):
        before = run.get(x["t"], 0)
        run[x["t"]] = before + x["w"]
        if sizes[x["t"]] + run[x["t"]] <= hi and (need_in is None or before < int(need_in[x["t"]])):
            kept.append(x)
    if lo is not None or need_out is not None:
        L, kept, run = kept, [], {}
        for x in sorted(L, key=lambda x: (x["f"], -x["g"], x["v"])):
            before = run.get(x["f"], 0)
            run[x["f"]] = before + x["w"]
            if (lo is None or sizes[x["f"]] - run[x["f"]] >= lo) and (need_out is None or before < int(need_out[x["f"]])):
                kept.append(x)
    return sorted((x["v"], x["t"]) for x in kept)


def directed_objective(src, dst, part, P):
    """(cut, vol) of partition_quality, from the directed edge list."""
    part = part.cpu().long()
    src, dst = src.cpu().long(), dst.cpu().long()
    cross = part[src] != part[dst]
    return int(cross.sum()), int(torch.unique(src[cross] * P + part[dst][cross]).numel())


def random_graph(n, m, seed, symmetric=False, multi=True, isolated=0):
    """A seeded directed graph in the FullGraph layout (CSR by destination, one self loop per node), with multi-edges
    unless ``multi`` is False, and ``isolated`` nodes at the end that only have their loop."""
    g = torch.Generator().manual_seed(seed)
    k = n - isolated
    a = torch.randint(0, k, (m,), generator=g)
    b = torch.randint(0, k, (m,), generator=g)
    if symmetric:
        a, b = torch.cat([a, b]), torch.cat([b, a])
    if not multi:
        key = torch.unique(a * n + b)
        a, b = key // n, key % n
    src, dst = torch.cat([a, torch.arange(n)]), torch.cat([b, torch.arange(n)])
    return graph_from_edges(n, src, dst)


def graph_from_edges(n, src, dst):
    from bns_gcn_b200.data import FullGraph
    o = torch.argsort(dst * n + src, stable=True)
    src, dst = src[o], dst[o]
    indptr = torch.zeros(n + 1, dtype=torch.int64)
    indptr[1:] = torch.cumsum(torch.bincount(dst, minlength=n), 0)
    z = torch.zeros(n, dtype=torch.bool)
    return FullGraph(n, indptr, src, torch.zeros(n, 1), torch.zeros(n, dtype=torch.int64), z, z, z, 2)


def star_plus_components(n_leaves=50, n_comp=3, comp_size=20, seed=0):
    """A star (node 0 at the centre, both directions) next to ``n_comp`` disconnected random components."""
    g = torch.Generator().manual_seed(seed)
    dst = [torch.zeros(n_leaves, dtype=torch.int64), torch.arange(1, n_leaves + 1)]
    src = [torch.arange(1, n_leaves + 1), torch.zeros(n_leaves, dtype=torch.int64)]
    base = n_leaves + 1
    for _ in range(n_comp):
        a = torch.randint(0, comp_size, (comp_size * 3,), generator=g) + base
        b = torch.randint(0, comp_size, (comp_size * 3,), generator=g) + base
        src.append(a)
        dst.append(b)
        base += comp_size
    n = base
    src = torch.cat(src + [torch.arange(n)])
    dst = torch.cat(dst + [torch.arange(n)])
    return graph_from_edges(n, src, dst)


def grid_graph(side):
    """The side x side four-neighbour grid, both directions, one loop per node."""
    i = torch.arange(side * side)
    r, c = i // side, i % side
    right, down = i[c < side - 1], i[r < side - 1]
    a = torch.cat([right, right + 1, down, down + side, i])
    b = torch.cat([right + 1, right, down + side, down, i])
    return graph_from_edges(side * side, a, b)


def equal_planted_blocks(n, n_blocks, deg_in, deg_out, seed=0):
    """A symmetric planted partition with ``n_blocks`` blocks of equal size (n / n_blocks, rounded), so that the planted
    grouping lies inside the partitioner's size bounds at any block count: ``deg_in`` / 2 edges per node drawn inside its
    block, ``deg_out`` / 2 anywhere, duplicates and loops merged away, then one loop per node.  Returns the graph and
    the planted grouping (int64 [n])."""
    g = torch.Generator().manual_seed(seed)
    blk = (torch.arange(n) % n_blocks)[torch.randperm(n, generator=g)]
    order = torch.argsort(blk, stable=True)
    sizes = torch.bincount(blk, minlength=n_blocks)
    starts = torch.cumsum(sizes, 0) - sizes
    m_in, m_out = n * deg_in // 2, n * deg_out // 2
    u = torch.randint(0, n, (m_in,), generator=g)
    v = order[starts[blk[u]] + (torch.rand(m_in, generator=g) * sizes[blk[u]]).long().clamp(max=sizes[blk[u]] - 1)]
    a = torch.cat([u, torch.randint(0, n, (m_out,), generator=g)])
    b = torch.cat([v, torch.randint(0, n, (m_out,), generator=g)])
    keep = a != b
    lo, hi = torch.minimum(a[keep], b[keep]), torch.maximum(a[keep], b[keep])
    key = torch.unique(lo * n + hi)
    lo, hi = key // n, key % n
    return graph_from_edges(n, torch.cat([lo, hi, torch.arange(n)]), torch.cat([hi, lo, torch.arange(n)])), blk


def degree_corrected_blocks(n, n_blocks, avg_deg, mix, seed=0, alpha=2.5):
    """A degree-corrected block model: ``n_blocks`` equal communities, power-law expected degrees (exponent alpha) with
    mean ``avg_deg``, a share ``mix`` of the edge ends leaving their community; symmetric, loops added.  Returns the
    graph and the planted grouping (int64 [n])."""
    g = torch.Generator().manual_seed(seed)
    blk = torch.arange(n) % n_blocks
    blk = blk[torch.randperm(n, generator=g)]
    u = torch.rand(n, generator=g, dtype=torch.float64)
    theta = (1 - u) ** (-1.0 / (alpha - 1))
    theta = theta / theta.mean()
    m = n * avg_deg // 2
    a = torch.multinomial(theta, m, replacement=True, generator=g)
    inside = torch.rand(m, generator=g) >= mix
    order = torch.argsort(blk, stable=True)
    sizes = torch.bincount(blk, minlength=n_blocks)
    starts = torch.cumsum(sizes, 0) - sizes
    # the other end: inside the community by theta (sampled per block), or anywhere by theta
    b = torch.multinomial(theta, m, replacement=True, generator=g)
    in_idx = torch.nonzero(inside, as_tuple=True)[0]
    for k in range(n_blocks):
        sel = in_idx[blk[a[in_idx]] == k]
        if sel.numel() == 0:
            continue
        members = order[starts[k]:starts[k] + sizes[k]]
        b[sel] = members[torch.multinomial(theta[members], sel.numel(), replacement=True, generator=g)]
    keep = a != b
    a, b = a[keep], b[keep]
    src = torch.cat([a, b, torch.arange(n)])
    dst = torch.cat([b, a, torch.arange(n)])
    return graph_from_edges(n, src, dst), blk
