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


def best_target(g, part):
    """bns_part_gains' choice from a full gain table [n, P]: the largest gain over the parts != own, ties to the lowest."""
    part = part.cpu().long()
    n, P = g.shape
    mask = torch.ones(n, P, dtype=torch.bool)
    mask[torch.arange(n), part] = False
    gm = torch.where(mask, g, torch.full_like(g, -(1 << 62)))
    best = gm.max(1).values
    return (gm == best[:, None]).int().argmax(1).int(), best


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
