// partition.cuh -- the device work of the multilevel partitioner (--partition-method multilevel), included by bnsgcn.cu.
//
// The level loop lives in data/multilevel.py; these are its hot loops.  Everything is integer: weights, gains and the
// objective are exact, and every atomic is an integer sum, so no result depends on the order the atomics land in.
//   part_expand_kernel   CSR entries -> 64-bit (row, col) keys through optional node maps (mapped loops dropped on
//                        request), with int32 weights; then cub radix sort + ReduceByKey sum equal keys:
//                        the undirected weighted graph, the directed in / out CSRs with multiplicities, the contracted
//                        coarse graph and the (node, neighbouring cluster) rating lists all come out of this one pass
//   part_csr_kernel      unique keys -> column ids; part_rows_kernel: row offsets by lower bound
//   part_conn_kernel     conn[v][p] = sum of w(v, u) over the row's u in part p, one warp per row, the row's table in
//                        shared memory; optionally the occupancy bits of the row and the exact cut / vol (int64)
//   part_gain_kernel     each node's best target among the allowed parts and its exact gain: the weighted edge cut
//                        from conn, or the communication volume from the out-edge counts of the in-neighbours
//   part_cluster_kernel  size-constrained label propagation: each node's heaviest neighbouring cluster with room
//                        (kEdges: room under the node-weight cap and under the int64 in-edge cap, --partition-balance
//                        edges)
//   part_weight_kernel   integer weight sums per label (part sizes, cluster weights; int32 node weights or int64
//                        in-edge weights)
// Rows are walked by one warp per node: the longest rows of the Reddit shape hold about 19 k entries.

namespace {

constexpr int kPartMaxParts = 64;

__device__ __forceinline__ uint32_t part_hash(uint64_t x) {
    x ^= x >> 33;
    x *= 0xff51afd7ed558ccdull;
    x ^= x >> 33;
    x *= 0xc4ceb9fe1a85ec53ull;
    x ^= x >> 33;
    return (uint32_t)x;
}

// entry k of row r -> key (R << 32 | C) and its weight.  mode 0: (R, C); 1: (C, R); 2: both, the second copy at m + k.
// A dropped entry gets the key n_out_rows << 32, which sorts after every kept key.
__global__ void part_expand_kernel(const int64_t *__restrict__ indptr, int64_t n_rows, const int32_t *__restrict__ idx,
                                   const int32_t *__restrict__ w, const int32_t *__restrict__ row_map,
                                   const int32_t *__restrict__ col_map, int mode, int drop_loops, int64_t m,
                                   int64_t n_out_rows, uint64_t *__restrict__ keys, int32_t *__restrict__ vals) {
    const int64_t r = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (r >= n_rows) return;
    const uint64_t R = (uint64_t)(row_map ? row_map[r] : (int32_t)r);
    const uint64_t drop = (uint64_t)n_out_rows << 32;
    for (int64_t k = indptr[r] + lane; k < indptr[r + 1]; k += 32) {
        const int32_t c = idx[k];
        const uint64_t C = (uint64_t)(col_map ? col_map[c] : c);
        const bool loop = drop_loops && R == C;
        const int32_t wk = w ? w[k] : 1;
        if (mode != 1) {
            keys[k] = loop ? drop : (R << 32 | C);
            vals[k] = wk;
        }
        if (mode != 0) {
            const int64_t o = mode == 2 ? m + k : k;
            keys[o] = loop ? drop : (C << 32 | R);
            vals[o] = wk;
        }
    }
}

__global__ void part_csr_kernel(const uint64_t *__restrict__ keys, const int64_t *__restrict__ n_runs,
                                int32_t *__restrict__ out_idx) {
    const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (j < *n_runs) out_idx[j] = (int32_t)(keys[j] & 0xffffffffull);
}

__global__ void part_rows_kernel(const uint64_t *__restrict__ keys, const int64_t *__restrict__ n_runs,
                                 int64_t n_out_rows, int64_t *__restrict__ out_indptr) {
    const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (r > n_out_rows) return;
    const uint64_t want = (uint64_t)r << 32;   // r == n_out_rows: the dropped entries start there
    int64_t lo = 0, hi = *n_runs;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (keys[mid] < want) lo = mid + 1; else hi = mid;
    }
    out_indptr[r] = lo;
}

struct PartAddI32 {
    __device__ __forceinline__ int32_t operator()(int32_t a, int32_t b) const { return a + b; }
};

// one region of the bns_part_edges workspace, 256-byte aligned
inline size_t part_align(size_t b) { return (b + 255) & ~(size_t)255; }

struct PartEdgesWs {
    uint64_t *k0 = nullptr, *k1 = nullptr;
    int32_t *v0 = nullptr, *v1 = nullptr;
    int64_t *runs = nullptr;
    void *tmp = nullptr;
    size_t tmp_bytes = 0, total = 0;
};

// carve (base != NULL) or size (base == NULL) the workspace for n entries
int part_edges_ws(int64_t n, char *base, PartEdgesWs *w) {
    const int ni = (int)n;
    size_t sort_bytes = 0, red_bytes = 0;
    BNS_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (const uint64_t *)nullptr, (uint64_t *)nullptr,
                                             (const int32_t *)nullptr, (int32_t *)nullptr, ni, 0, 64));
    BNS_CUDA(cub::DeviceReduce::ReduceByKey(nullptr, red_bytes, (const uint64_t *)nullptr, (uint64_t *)nullptr,
                                            (const int32_t *)nullptr, (int32_t *)nullptr, (int64_t *)nullptr,
                                            PartAddI32(), ni));
    const size_t nk = part_align((size_t)(n + 1) * 8), nv = part_align((size_t)(n + 1) * 4);
    w->tmp_bytes = part_align(sort_bytes > red_bytes ? sort_bytes : red_bytes);
    size_t off = 0;
    auto take = [&](size_t b) { char *p = base ? base + off : nullptr; off += b; return p; };
    w->k0 = reinterpret_cast<uint64_t *>(take(nk));
    w->k1 = reinterpret_cast<uint64_t *>(take(nk));
    w->v0 = reinterpret_cast<int32_t *>(take(nv));
    w->v1 = reinterpret_cast<int32_t *>(take(nv));
    w->runs = reinterpret_cast<int64_t *>(take(256));
    w->tmp = take(w->tmp_bytes);
    w->total = off;
    return BNS_OK;
}

template <bool kOcc, bool kQuality>
__global__ void __launch_bounds__(kThreads) part_conn_kernel(int64_t n, const int64_t *__restrict__ indptr,
                                                             const int32_t *__restrict__ idx,
                                                             const int32_t *__restrict__ w,
                                                             const int32_t *__restrict__ part, int P,
                                                             int32_t *__restrict__ conn, uint64_t *__restrict__ occ,
                                                             unsigned long long *__restrict__ quality) {
    __shared__ int32_t tab[kWarps][kPartMaxParts];
    __shared__ unsigned long long red[2][kWarps];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t v = blockIdx.x * (int64_t)kWarps + warp;
    unsigned long long cut = 0, vol = 0;
    if (v < n) {
        tab[warp][lane] = 0;
        tab[warp][lane + 32] = 0;
        __syncwarp();
        for (int64_t k = indptr[v] + lane; k < indptr[v + 1]; k += 32) atomicAdd(&tab[warp][part[idx[k]]], w ? w[k] : 1);
        __syncwarp();
        const int32_t c0 = tab[warp][lane], c1 = tab[warp][lane + 32];
        if (conn) {
            int32_t *row = conn + v * P;
            if (lane < P) row[lane] = c0;
            if (lane + 32 < P) row[lane + 32] = c1;
        }
        if (kOcc) {
            const unsigned lo = __ballot_sync(0xffffffffu, c0 > 0), hi = __ballot_sync(0xffffffffu, c1 > 0);
            if (lane == 0) occ[v] = (uint64_t)lo | (uint64_t)hi << 32;
        }
        if (kQuality) {
            const int pv = part[v];
            if (lane != pv) { cut += (unsigned long long)c0; vol += c0 > 0; }
            if (lane + 32 != pv) { cut += (unsigned long long)c1; vol += c1 > 0; }
        }
    }
    if (kQuality) {
        for (int o = 16; o; o >>= 1) {
            cut += __shfl_xor_sync(0xffffffffu, cut, o);
            vol += __shfl_xor_sync(0xffffffffu, vol, o);
        }
        if (lane == 0) { red[0][warp] = cut; red[1][warp] = vol; }
        __syncthreads();
        if (threadIdx.x == 0) {
            unsigned long long c = 0, s = 0;
            for (int i = 0; i < kWarps; ++i) { c += red[0][i]; s += red[1][i]; }
            if (c) atomicAdd(quality, c);
            if (s) atomicAdd(quality + 1, s);
        }
    }
}

// the best (gain, then lowest part id) over the warp; target -1 when no allowed part differs from the node's own
__device__ __forceinline__ void part_warp_best(long long &g, int &b) {
    for (int o = 16; o; o >>= 1) {
        const long long g2 = __shfl_xor_sync(0xffffffffu, g, o);
        const int b2 = __shfl_xor_sync(0xffffffffu, b, o);
        if (b2 >= 0 && (b < 0 || g2 > g || (g2 == g && b2 < b))) { g = g2; b = b2; }
    }
}

// kVol == false: gain(v, b) = conn[v][b] - conn[v][a] (a = part[v]) on the weighted undirected graph.
// kVol == true: the exact change of the communication volume when v alone moves from a to b.  conn / occ are the out-edge
// counts per part and their occupancy bits; the CSR is the in-CSR with multiplicities m(u, v), loops dropped.
//   gain(b) = [b in S_v] - [a in S_v] - D + C[b] + R,   S_v = occ[v], D = #in-neighbours u,
//   C[b] = #u with b in occ[u] or b == part[u],   R = #u with cnt_u(a) == m(u, v) and a != part[u]
template <bool kVol>
__global__ void __launch_bounds__(kThreads) part_gain_kernel(int64_t n, int P, const int64_t *__restrict__ indptr,
                                                             const int32_t *__restrict__ idx,
                                                             const int32_t *__restrict__ w,
                                                             const int32_t *__restrict__ part,
                                                             const int32_t *__restrict__ conn,
                                                             const uint64_t *__restrict__ occ, uint64_t allowed,
                                                             int32_t *__restrict__ target, int64_t *__restrict__ gain) {
    __shared__ int32_t cnt[kWarps][kPartMaxParts];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t v = blockIdx.x * (int64_t)kWarps + warp;
    if (v >= n) return;
    const int a = part[v];
    const int32_t *row = conn + v * P;
    long long base = 0;
    if (kVol) {
        cnt[warp][lane] = 0;
        cnt[warp][lane + 32] = 0;
        __syncwarp();
        long long d = 0, r = 0;
        for (int64_t k = indptr[v] + lane; k < indptr[v + 1]; k += 32) {
            const int32_t u = idx[k];
            const int pu = part[u];
            uint64_t bits = occ[u] | (1ull << pu);
            while (bits) {
                const int b = __ffsll((long long)bits) - 1;
                bits &= bits - 1;
                atomicAdd(&cnt[warp][b], 1);
            }
            d += 1;
            r += (a != pu && conn[(int64_t)u * P + a] == (w ? w[k] : 1));
        }
        for (int o = 16; o; o >>= 1) {
            d += __shfl_xor_sync(0xffffffffu, d, o);
            r += __shfl_xor_sync(0xffffffffu, r, o);
        }
        __syncwarp();
        base = r - d - (long long)((occ[v] >> a) & 1);
    } else {
        base = -(long long)row[a];
    }
    long long best = 0;
    int bt = -1;
    for (int b = lane; b < P; b += 32) {
        if (b == a || !((allowed >> b) & 1)) continue;
        const long long g = kVol ? base + (long long)((occ[v] >> b) & 1) + cnt[warp][b] : base + row[b];
        if (bt < 0 || g > best) { best = g; bt = b; }   // b ascends within a lane: ties keep the lower id
    }
    part_warp_best(best, bt);
    if (lane == 0) {
        target[v] = bt;
        gain[v] = bt < 0 ? 0 : best;
    }
}

// One label-propagation step.  The rating CSR lists, for node v, (cluster c, total weight of v's edges into c), sorted
// by c.  A node whose coin (hash of node and seed) comes up odd proposes the heaviest neighbouring cluster other than
// its own that still has room for it (cw[c] + nw[v] <= cap and, with kEdges, ce[c] + ew[v] <= ecap; ties: the lower
// seeded hash, then the lower id), if that weight beats its connection to its own cluster.  Otherwise target = -1.
// The in-edge arguments come last, so that kEdges == false reads its parameters where the one-cap kernel did.
template <bool kEdges>
__global__ void __launch_bounds__(kThreads) part_cluster_kernel(int64_t n, const int64_t *__restrict__ indptr,
                                                                const int32_t *__restrict__ cid,
                                                                const int32_t *__restrict__ cw_edge,
                                                                const int32_t *__restrict__ label,
                                                                const int32_t *__restrict__ nw,
                                                                const int64_t *__restrict__ cw, int64_t cap,
                                                                uint64_t seed, int32_t *__restrict__ target,
                                                                int64_t *__restrict__ gain,
                                                                const int64_t *__restrict__ ew,
                                                                const int64_t *__restrict__ ce, int64_t ecap) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t v = blockIdx.x * (int64_t)kWarps + warp;
    if (v >= n) return;
    const bool active = part_hash(seed ^ ((uint64_t)v * 0x9e3779b97f4a7c15ull)) & 1u;
    if (!active) {
        if (lane == 0) { target[v] = -1; gain[v] = 0; }
        return;
    }
    const int32_t own = label[v];
    const int64_t wv = nw ? nw[v] : 1;
    const int64_t ev = kEdges ? ew[v] : 0;
    long long cur = 0, best = -1;
    uint32_t best_h = 0;
    int bc = -1;
    for (int64_t k = indptr[v] + lane; k < indptr[v + 1]; k += 32) {
        const int32_t c = cid[k];
        const long long wt = cw_edge[k];
        if (c == own) { cur = wt; continue; }
        if (cw[c] + wv > cap) continue;
        if (kEdges && ce[c] + ev > ecap) continue;
        const uint32_t h = part_hash(seed + (uint64_t)c);
        if (bc < 0 || wt > best || (wt == best && (h < best_h || (h == best_h && c < bc)))) {
            best = wt; best_h = h; bc = c;
        }
    }
    for (int o = 16; o; o >>= 1) {
        cur += __shfl_xor_sync(0xffffffffu, cur, o);      // one lane holds it, the others 0
        const long long b2 = __shfl_xor_sync(0xffffffffu, best, o);
        const uint32_t h2 = __shfl_xor_sync(0xffffffffu, best_h, o);
        const int c2 = __shfl_xor_sync(0xffffffffu, bc, o);
        if (c2 >= 0 && (bc < 0 || b2 > best || (b2 == best && (h2 < best_h || (h2 == best_h && c2 < bc))))) {
            best = b2; best_h = h2; bc = c2;
        }
    }
    if (lane == 0) {
        const bool move = bc >= 0 && best > cur;
        target[v] = move ? bc : -1;
        gain[v] = move ? best - cur : 0;
    }
}

template <typename W>
__global__ void part_weight_kernel(int64_t n, const int32_t *__restrict__ label, const W *__restrict__ nw,
                                   unsigned long long *__restrict__ out) {
    const int64_t v = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (v < n) atomicAdd(out + label[v], (unsigned long long)(nw ? nw[v] : 1));
}

inline unsigned part_warp_grid(int64_t n) { return (unsigned)((n + kWarps - 1) / kWarps); }
inline unsigned part_grid(int64_t n) { return (unsigned)((n + kThreads - 1) / kThreads); }

bool part_graph_ok(int64_t n, const int64_t *indptr, const int32_t *idx) {
    return n >= 0 && n < INT32_MAX && (n == 0 || (indptr && idx));
}

}  // namespace

extern "C" size_t bns_part_edges_workspace_bytes(int64_t n_entries) {
    if (n_entries < 0 || n_entries >= INT32_MAX) return 0;
    PartEdgesWs w;
    if (part_edges_ws(n_entries, nullptr, &w) != BNS_OK) return 0;
    return w.total;
}

extern "C" int bns_part_edges(int64_t n_rows, int64_t nnz, const int64_t *indptr, const int32_t *idx, const int32_t *w,
                              const int32_t *row_map, const int32_t *col_map, int32_t mode, int32_t drop_loops,
                              int64_t n_out_rows, int64_t *out_indptr, int32_t *out_idx, int32_t *out_w,
                              int64_t *out_nnz, void *ws, size_t ws_bytes, void *stream) {
    BNS_REQUIRE(mode >= 0 && mode <= 2, "bns_part_edges: mode %d is not 0, 1 or 2", (int)mode);
    BNS_REQUIRE(nnz >= 0 && n_out_rows >= 0 && n_out_rows < INT32_MAX, "bns_part_edges: bad size");
    BNS_REQUIRE(n_rows >= 0 && n_rows < INT32_MAX && indptr && (nnz == 0 || idx), "bns_part_edges: bad input graph");
    BNS_REQUIRE(row_map || mode == 1 || n_rows <= n_out_rows,
                "bns_part_edges: %lld input rows, no row map, but only %lld output rows", (long long)n_rows,
                (long long)n_out_rows);
    const int64_t M = mode == 2 ? 2 * nnz : nnz;
    BNS_REQUIRE(M < INT32_MAX, "bns_part_edges: %lld entries, more than 2^31-1", (long long)M);
    BNS_REQUIRE(out_indptr && out_nnz && (M == 0 || (out_idx && out_w)), "bns_part_edges: NULL output");
    BNS_REQUIRE(ws || M == 0, "bns_part_edges: NULL workspace");
    PartEdgesWs p;
    int rc = part_edges_ws(M, reinterpret_cast<char *>(ws), &p);
    if (rc != BNS_OK) return rc;
    if (ws_bytes < p.total) return fail(BNS_E_WORKSPACE, "bns_part_edges: workspace %zu bytes < %zu needed", ws_bytes,
                                        p.total);
    cudaStream_t st = as_stream(stream);
    if (M == 0) {
        BNS_CUDA(cudaMemsetAsync(out_indptr, 0, (size_t)(n_out_rows + 1) * sizeof(int64_t), st));
        *out_nnz = 0;
        return BNS_OK;
    }
    part_expand_kernel<<<(unsigned)((n_rows * 32 + kThreads - 1) / kThreads), kThreads, 0, st>>>(
        indptr, n_rows, idx, w, row_map, col_map, mode, drop_loops, nnz, n_out_rows, p.k0, p.v0);
    ++g_launches;
    int end_bit = 33;
    while (end_bit < 64 && ((uint64_t)1 << (end_bit - 32)) <= (uint64_t)n_out_rows) ++end_bit;
    size_t tb = p.tmp_bytes;
    BNS_CUDA(cub::DeviceRadixSort::SortPairs(p.tmp, tb, p.k0, p.k1, p.v0, p.v1, (int)M, 0, end_bit, st));
    tb = p.tmp_bytes;
    BNS_CUDA(cub::DeviceReduce::ReduceByKey(p.tmp, tb, p.k1, p.k0, p.v1, out_w, p.runs, PartAddI32(), (int)M, st));
    part_csr_kernel<<<part_grid(M), kThreads, 0, st>>>(p.k0, p.runs, out_idx);
    part_rows_kernel<<<part_grid(n_out_rows + 1), kThreads, 0, st>>>(p.k0, p.runs, n_out_rows, out_indptr);
    g_launches += 2;
    BNS_CUDA(cudaGetLastError());
    BNS_CUDA(cudaMemcpyAsync(out_nnz, out_indptr + n_out_rows, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    BNS_CUDA(cudaStreamSynchronize(st));
    return BNS_OK;
}

extern "C" int bns_part_conn(int64_t n, const int64_t *indptr, const int32_t *idx, const int32_t *w, const int32_t *part,
                             int32_t P, int32_t *conn, uint64_t *occ, int64_t *quality, void *stream) {
    BNS_REQUIRE(part_graph_ok(n, indptr, idx), "bns_part_conn: bad graph");
    BNS_REQUIRE(P >= 1 && P <= kPartMaxParts, "bns_part_conn: %d parts, outside [1, 64]", (int)P);
    BNS_REQUIRE(n == 0 || part, "bns_part_conn: NULL part");
    BNS_REQUIRE(conn || occ || quality, "bns_part_conn: nothing to compute");
    cudaStream_t st = as_stream(stream);
    if (quality) BNS_CUDA(cudaMemsetAsync(quality, 0, 2 * sizeof(int64_t), st));
    if (n == 0) return BNS_OK;
    unsigned long long *q = reinterpret_cast<unsigned long long *>(quality);
    const unsigned grid = part_warp_grid(n);
    if (occ && quality)
        part_conn_kernel<true, true><<<grid, kThreads, 0, st>>>(n, indptr, idx, w, part, P, conn, occ, q);
    else if (occ)
        part_conn_kernel<true, false><<<grid, kThreads, 0, st>>>(n, indptr, idx, w, part, P, conn, occ, q);
    else if (quality)
        part_conn_kernel<false, true><<<grid, kThreads, 0, st>>>(n, indptr, idx, w, part, P, conn, occ, q);
    else
        part_conn_kernel<false, false><<<grid, kThreads, 0, st>>>(n, indptr, idx, w, part, P, conn, occ, q);
    ++g_launches;
    BNS_CUDA(cudaGetLastError());
    return BNS_OK;
}

extern "C" int bns_part_gains(int32_t objective, int64_t n, int32_t P, const int64_t *indptr, const int32_t *idx,
                              const int32_t *w, const int32_t *part, const int32_t *conn, const uint64_t *occ,
                              uint64_t allowed, int32_t *target, int64_t *gain, void *stream) {
    BNS_REQUIRE(objective == 0 || objective == 1, "bns_part_gains: objective %d is not 0 (cut) or 1 (vol)",
                (int)objective);
    BNS_REQUIRE(n >= 0 && n < INT32_MAX, "bns_part_gains: bad node count");
    BNS_REQUIRE(P >= 2 && P <= kPartMaxParts, "bns_part_gains: %d parts, outside [2, 64]", (int)P);
    BNS_REQUIRE(n == 0 || (part && conn && target && gain), "bns_part_gains: NULL argument");
    BNS_REQUIRE(objective == 0 || n == 0 || (occ && indptr && idx), "bns_part_gains: vol needs the in-CSR and occ");
    if (n == 0) return BNS_OK;
    cudaStream_t st = as_stream(stream);
    if (objective == 1)
        part_gain_kernel<true><<<part_warp_grid(n), kThreads, 0, st>>>(n, P, indptr, idx, w, part, conn, occ, allowed,
                                                                        target, gain);
    else
        part_gain_kernel<false><<<part_warp_grid(n), kThreads, 0, st>>>(n, P, indptr, idx, w, part, conn, occ, allowed,
                                                                         target, gain);
    ++g_launches;
    BNS_CUDA(cudaGetLastError());
    return BNS_OK;
}

extern "C" int bns_part_cluster(int64_t n, const int64_t *indptr, const int32_t *cid, const int32_t *cw_edge,
                                const int32_t *label, const int32_t *nw, const int64_t *cw, int64_t cap, uint64_t seed,
                                int32_t *target, int64_t *gain, void *stream) {
    BNS_REQUIRE(part_graph_ok(n, indptr, cid), "bns_part_cluster: bad rating graph");
    BNS_REQUIRE(n == 0 || (cw_edge && label && cw && target && gain), "bns_part_cluster: NULL argument");
    BNS_REQUIRE(cap >= 1, "bns_part_cluster: cap %lld < 1", (long long)cap);
    if (n == 0) return BNS_OK;
    part_cluster_kernel<false><<<part_warp_grid(n), kThreads, 0, as_stream(stream)>>>(
        n, indptr, cid, cw_edge, label, nw, cw, cap, seed, target, gain, nullptr, nullptr, 0);
    ++g_launches;
    BNS_CUDA(cudaGetLastError());
    return BNS_OK;
}

extern "C" int bns_part_cluster_edges(int64_t n, const int64_t *indptr, const int32_t *cid, const int32_t *cw_edge,
                                      const int32_t *label, const int32_t *nw, const int64_t *cw, int64_t cap,
                                      const int64_t *ew, const int64_t *ce, int64_t ecap, uint64_t seed,
                                      int32_t *target, int64_t *gain, void *stream) {
    BNS_REQUIRE(part_graph_ok(n, indptr, cid), "bns_part_cluster_edges: bad rating graph");
    BNS_REQUIRE(n == 0 || (cw_edge && label && cw && ew && ce && target && gain), "bns_part_cluster_edges: NULL argument");
    BNS_REQUIRE(cap >= 1 && ecap >= 1, "bns_part_cluster_edges: cap %lld or in-edge cap %lld < 1", (long long)cap,
                (long long)ecap);
    if (n == 0) return BNS_OK;
    part_cluster_kernel<true><<<part_warp_grid(n), kThreads, 0, as_stream(stream)>>>(
        n, indptr, cid, cw_edge, label, nw, cw, cap, seed, target, gain, ew, ce, ecap);
    ++g_launches;
    BNS_CUDA(cudaGetLastError());
    return BNS_OK;
}

template <typename W>
static int part_weights(const char *what, int64_t n, const int32_t *label, const W *nw, int64_t n_labels, int64_t *out,
                 void *stream) {
    BNS_REQUIRE(n >= 0 && n < INT32_MAX && n_labels >= 1 && n_labels < INT32_MAX, "%s: bad size", what);
    BNS_REQUIRE(out && (n == 0 || label), "%s: NULL argument", what);
    cudaStream_t st = as_stream(stream);
    BNS_CUDA(cudaMemsetAsync(out, 0, (size_t)n_labels * sizeof(int64_t), st));
    if (n == 0) return BNS_OK;
    part_weight_kernel<W><<<part_grid(n), kThreads, 0, st>>>(n, label, nw, reinterpret_cast<unsigned long long *>(out));
    ++g_launches;
    BNS_CUDA(cudaGetLastError());
    return BNS_OK;
}

extern "C" int bns_part_weights(int64_t n, const int32_t *label, const int32_t *nw, int64_t n_labels, int64_t *out,
                                void *stream) {
    return part_weights("bns_part_weights", n, label, nw, n_labels, out, stream);
}

extern "C" int bns_part_weights_i64(int64_t n, const int32_t *label, const int64_t *nw, int64_t n_labels, int64_t *out,
                                    void *stream) {
    return part_weights("bns_part_weights_i64", n, label, nw, n_labels, out, stream);
}
