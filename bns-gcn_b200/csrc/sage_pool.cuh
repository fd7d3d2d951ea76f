// sage_pool.cuh -- GraphSAGE's max-pooling aggregator (SAGEConv(in, out, 'pool')) as kernels (included by bnsgcn.cu after
// gatv2.cuh, whose row walk gatv2_walk_row and 16-byte row loads gatv2_load_row it shares, with gat.cuh's GatGraph,
// gat_fill and gat_grid).  Per destination row v and column f
//
//   m[v, f] = max over the entries u -> v of z[u, f]     (0 for a row without entries; z = relu(fc_pool(x)) >= 0)
//
// The training forward also records the WINNER of each (v, f): the position of the first entry, in walk order, whose z
// equals the maximum (a strict > keeps the first).  The walk order is a_in's CSR order, then the sampled halo entries in
// a_out's order; positions are a_in positions, and nnz_in + a_out position for halo entries, so a source that occupies
// two entries of a row (a multi-edge) is credited once.  The backward adds d m[v, f] to the winner only.
//
//   sage_max_kernel            one warp per destination row (inner entries, then the sampled halo entries chunk by
//                              chunk), lane l owning the float4 column groups l, l + 32, ... (NV of them), U gathered
//                              z rows in flight: m and win
//   sage_max_bwd_kernel        one warp per source row of a static transpose, entries in its order through its
//                              permutation: d y[u] = relu'(z[u]) * sum of d m[v, f] over the entries whose position is
//                              win[v, f] (no float atomics, so repeats are bit-identical)
//   sage_max_infer_kernel      the evaluation forward on a homogeneous graph, no winner; BLOCK carries the running max
//                              and a "seen an entry" flag between column blocks (partition-parallel evaluation)
//
// A max involves no rounding and, with -0 stored as +0, does not depend on the order of the entries: the single pass
// and any split into blocks give the same bits.
namespace {

constexpr int kSageMaxWidth = 1024;

template <int NV> struct SageUnroll { static constexpr int value = NV <= 4 ? 4 : 2; };

// x > m takes x: the first of equal values stays (the winner rule); NaN never wins
__device__ __forceinline__ void sage_take(float x, int32_t p, float &m, int32_t &w) {
    if (x > m) { m = x; w = p; }
}

// sm_90a: 48 / 78 / 128 / 168 registers for NV = 1 / 2 / 4 / 8, no spills (DESIGN §3)
template <int NV>
__global__ void __launch_bounds__(kThreads) sage_max_kernel(GatGraph g, int64_t nnz_in, int32_t F, const float *z,
                                                            int64_t ldz, float *m_out, int32_t *win_out) {
    constexpr int U = SageUnroll<NV>::value;
    __shared__ int32_t s_u[kWarps][32];
    __shared__ int32_t s_p[kWarps][32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int64_t warps_total = (int64_t)gridDim.x * kWarps;
    for (int64_t v = (int64_t)blockIdx.x * kWarps + w; v < g.n_rows; v += warps_total) {
        float4 m[NV];
        int4 wi[NV];
#pragma unroll
        for (int t = 0; t < NV; ++t) {
            m[t] = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
            wi[t] = make_int4(-1, -1, -1, -1);
        }
        gatv2_walk_row(g, v, lane, [&](bool valid, int32_t u, int64_t pos, bool halo, int64_t, int n) {
            s_u[w][lane] = u;
            s_p[w][lane] = valid ? (int32_t)(halo ? nnz_in + pos : pos) : -1;
            __syncwarp();
            for (int jj = 0; jj < n; jj += U) {
                float4 x[U][NV];
#pragma unroll
                for (int q = 0; q < U; ++q)
                    if (jj + q < n) gatv2_load_row<NV>(z + (int64_t)s_u[w][jj + q] * ldz, lane, F, x[q]);
#pragma unroll
                for (int q = 0; q < U; ++q) {
                    if (jj + q < n) {
                        const int32_t p = s_p[w][jj + q];
#pragma unroll
                        for (int t = 0; t < NV; ++t) {
                            sage_take(x[q][t].x, p, m[t].x, wi[t].x); sage_take(x[q][t].y, p, m[t].y, wi[t].y);
                            sage_take(x[q][t].z, p, m[t].z, wi[t].z); sage_take(x[q][t].w, p, m[t].w, wi[t].w);
                        }
                    }
                }
            }
            __syncwarp();                                 // s_u / s_p are rewritten by the next block
        });
#pragma unroll
        for (int t = 0; t < NV; ++t) {
            const int c = (lane + 32 * t) * 4;
            if (c < F) {
                // no winner: a row without entries (z is finite, so any entry wins over -inf)
                const float4 y = m[t];
                *reinterpret_cast<float4 *>(m_out + v * F + c) =
                    make_float4(wi[t].x >= 0 ? y.x + 0.f : 0.f, wi[t].y >= 0 ? y.y + 0.f : 0.f,
                                wi[t].z >= 0 ? y.z + 0.f : 0.f, wi[t].w >= 0 ? y.w + 0.f : 0.f);
                *reinterpret_cast<int4 *>(win_out + v * F + c) = wi[t];
            }
        }
    }
}

// d_y[out_base + orow(r)] = relu'(z[...]) * sum over the entries k of row r of the transpose gT, in gT's order, of
// d m[idx[k], f] where win[idx[k], f] == pos_base + perm[k]
template <int NV>
__global__ void __launch_bounds__(kThreads) sage_max_bwd_kernel(const int64_t *__restrict__ indptr,
                                                                const int32_t *__restrict__ idx,
                                                                const int32_t *__restrict__ perm, int64_t n_rows,
                                                                int64_t pos_base, const int32_t *__restrict__ row_map,
                                                                int64_t out_base, int32_t F,
                                                                const int32_t *__restrict__ win,
                                                                const float *__restrict__ dm,
                                                                const float *__restrict__ z, int64_t ldz, float *dy) {
    constexpr int U = SageUnroll<NV>::value;
    __shared__ int32_t s_v[kWarps][32];
    __shared__ int32_t s_p[kWarps][32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int64_t warps_total = (int64_t)gridDim.x * kWarps;
    for (int64_t r = (int64_t)blockIdx.x * kWarps + w; r < n_rows; r += warps_total) {
        int64_t u = out_base + r;
        if (row_map) {
            const int32_t mrow = row_map[r];
            if (mrow < 0) continue;                       // not sampled this epoch: no row of d_y
            u = out_base + mrow;
        }
        const int64_t b = indptr[r], e = indptr[r + 1];
        float4 acc[NV];
#pragma unroll
        for (int t = 0; t < NV; ++t) acc[t] = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int64_t k0 = b; k0 < e; k0 += 32) {
            const int64_t k = k0 + lane;
            const int n = (int)(e - k0 < 32 ? e - k0 : 32);
            if (k < e) {
                s_v[w][lane] = idx[k];
                s_p[w][lane] = (int32_t)(pos_base + perm[k]);
            }
            __syncwarp();
            for (int jj = 0; jj < n; jj += U) {
                int4 wv[U][NV];
#pragma unroll
                for (int q = 0; q < U; ++q) {
                    if (jj + q < n) {
                        const int32_t *wr = win + (int64_t)s_v[w][jj + q] * F;
#pragma unroll
                        for (int t = 0; t < NV; ++t) {
                            const int c = (lane + 32 * t) * 4;
                            wv[q][t] = c < F ? __ldg(reinterpret_cast<const int4 *>(wr + c)) : make_int4(-1, -1, -1, -1);
                        }
                    }
                }
#pragma unroll
                for (int q = 0; q < U; ++q) {
                    if (jj + q < n) {
                        const int32_t p = s_p[w][jj + q];
                        const float *dr = dm + (int64_t)s_v[w][jj + q] * F;
#pragma unroll
                        for (int t = 0; t < NV; ++t) {
                            const bool hx = wv[q][t].x == p, hy = wv[q][t].y == p;
                            const bool hz = wv[q][t].z == p, hw = wv[q][t].w == p;
                            if (hx | hy | hz | hw) {              // d m is read only where this entry won
                                const float4 d = __ldg(reinterpret_cast<const float4 *>(dr + (lane + 32 * t) * 4));
                                if (hx) acc[t].x += d.x;
                                if (hy) acc[t].y += d.y;
                                if (hz) acc[t].z += d.z;
                                if (hw) acc[t].w += d.w;
                            }
                        }
                    }
                }
            }
            __syncwarp();
        }
        float4 zr[NV];
        gatv2_load_row<NV>(z + u * ldz, lane, F, zr);
        float *o = dy + u * F;
#pragma unroll
        for (int t = 0; t < NV; ++t) {
            const int c = (lane + 32 * t) * 4;
            if (c < F)
                *reinterpret_cast<float4 *>(o + c) =
                    make_float4(zr[t].x > 0.f ? acc[t].x : 0.f, zr[t].y > 0.f ? acc[t].y : 0.f,
                                zr[t].z > 0.f ? acc[t].z : 0.f, zr[t].w > 0.f ? acc[t].w : 0.f);
        }
    }
}

struct SageInferArgs {
    const int64_t *indptr; const int32_t *indices; int64_t n_rows;
    const float *z; int64_t ldz;                          // [n_cols, F]
    int32_t F;
    float *out;                                           // [n_rows, F]
};

struct SageInferBlockArgs : SageInferArgs {
    float *sm; int32_t *seen;                             // running max [n_rows, F], seen an entry [n_rows]
    int32_t first, last;
};

// BLOCK: the row's entries arrive as several matrices over different column sets, one launch each; a launch that is
// not `first` reloads (sm, seen), one that is not `last` stores them back, `last` writes the max (0 if never seen); a
// row without entries in a middle launch keeps its state untouched
template <int NV, bool BLOCK = false>
__global__ void __launch_bounds__(kThreads)
sage_max_infer_kernel(typename std::conditional<BLOCK, SageInferBlockArgs, SageInferArgs>::type a) {
    constexpr int U = SageUnroll<NV>::value;
    __shared__ int32_t s_u[kWarps][32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int64_t warps_total = (int64_t)gridDim.x * kWarps;
    const int F = a.F;
    for (int64_t v = (int64_t)blockIdx.x * kWarps + w; v < a.n_rows; v += warps_total) {
        const int64_t b = a.indptr[v], e = a.indptr[v + 1];
        float4 m[NV];
#pragma unroll
        for (int t = 0; t < NV; ++t) m[t] = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
        bool seen = b < e;
        if constexpr (BLOCK) {
            if (b == e && !a.first && !a.last) continue;
            if (!a.first) {
                seen = seen || a.seen[v] != 0;
                const float *sr = a.sm + v * F;
#pragma unroll
                for (int t = 0; t < NV; ++t) {
                    const int c = (lane + 32 * t) * 4;
                    if (c < F) m[t] = *reinterpret_cast<const float4 *>(sr + c);
                }
            }
        }
        for (int64_t k0 = b; k0 < e; k0 += 32) {
            const int n = (int)(e - k0 < 32 ? e - k0 : 32);
            if (lane < n) s_u[w][lane] = __ldg(a.indices + k0 + lane);
            __syncwarp();
            for (int jj = 0; jj < n; jj += U) {
                float4 x[U][NV];
#pragma unroll
                for (int q = 0; q < U; ++q)
                    if (jj + q < n) gatv2_load_row<NV>(a.z + (int64_t)s_u[w][jj + q] * a.ldz, lane, F, x[q]);
#pragma unroll
                for (int q = 0; q < U; ++q) {
                    if (jj + q < n) {
#pragma unroll
                        for (int t = 0; t < NV; ++t) {
                            m[t].x = x[q][t].x > m[t].x ? x[q][t].x : m[t].x;
                            m[t].y = x[q][t].y > m[t].y ? x[q][t].y : m[t].y;
                            m[t].z = x[q][t].z > m[t].z ? x[q][t].z : m[t].z;
                            m[t].w = x[q][t].w > m[t].w ? x[q][t].w : m[t].w;
                        }
                    }
                }
            }
            __syncwarp();
        }
        if constexpr (BLOCK) {
            if (!a.last) {
                if (lane == 0) a.seen[v] = seen ? 1 : 0;
                float *sr = a.sm + v * F;
#pragma unroll
                for (int t = 0; t < NV; ++t) {
                    const int c = (lane + 32 * t) * 4;
                    if (c < F) *reinterpret_cast<float4 *>(sr + c) = m[t];
                }
                continue;
            }
        }
        float *o = a.out + v * F;
#pragma unroll
        for (int t = 0; t < NV; ++t) {
            const int c = (lane + 32 * t) * 4;
            if (c < F)
                *reinterpret_cast<float4 *>(o + c) =
                    seen ? make_float4(m[t].x + 0.f, m[t].y + 0.f, m[t].z + 0.f, m[t].w + 0.f)
                         : make_float4(0.f, 0.f, 0.f, 0.f);
        }
    }
}

inline int sage_nv(int32_t F) {
    const int nv = (F + 127) / 128;
    return nv <= 1 ? 1 : (nv == 2 ? 2 : (nv <= 4 ? 4 : 8));
}

#define BNS_SAGE_DISPATCH(NVV, LAUNCH) \
    switch (NVV) {                     \
    case 1: { constexpr int NV = 1; LAUNCH; } break; \
    case 2: { constexpr int NV = 2; LAUNCH; } break; \
    case 4: { constexpr int NV = 4; LAUNCH; } break; \
    default: { constexpr int NV = 8; LAUNCH; } break; \
    }

inline bool sage_width_ok(int32_t F) { return F > 0 && F % 4 == 0 && F <= kSageMaxWidth; }

}  // namespace

extern "C" int bns_sage_max_f32(const bns_graph_t *a_in, const bns_graph_t *a_out, const int32_t *cidx,
                                const int32_t *chunk_cnt, const int32_t *cpos, int64_t x_halo_base, int32_t F,
                                const float *z, int64_t ldz, float *m, int32_t *win, void *stream) {
    GatArgs ga{};
    int rc = gat_fill(ga, a_in, a_out, cidx, chunk_cnt, cpos, x_halo_base, "bns_sage_max_f32");
    if (rc) return rc;
    BNS_REQUIRE(sage_width_ok(F), "bns_sage_max_f32: need a width %% 4 == 0 in 4..%d (got %d)", kSageMaxWidth, F);
    const int64_t nnz_out = ga.g.cidx ? a_out->nnz : 0;
    BNS_REQUIRE(a_in->nnz + nnz_out <= INT32_MAX, "bns_sage_max_f32: nnz_in + nnz_out = %lld does not fit int32 positions",
                (long long)(a_in->nnz + nnz_out));
    if (ga.g.n_rows == 0) return BNS_OK;
    BNS_REQUIRE(z && m && win, "bns_sage_max_f32: NULL pointer");
    BNS_REQUIRE(ldz % 4 == 0 && ldz >= F && gatv2_aligned(z) && gatv2_aligned(m) && gatv2_aligned(win),
                "bns_sage_max_f32: 16-byte aligned rows required");
    const unsigned grid = gat_grid(ga.g.n_rows);
    cudaStream_t st = as_stream(stream);
    BNS_SAGE_DISPATCH(sage_nv(F), (sage_max_kernel<NV><<<grid, kThreads, 0, st>>>(ga.g, a_in->nnz, F, z, ldz, m, win)));
    ++g_launches;
    BNS_CUDA(cudaGetLastError());
    return BNS_OK;
}

extern "C" int bns_sage_max_bwd_f32(const bns_graph_t *gT, int64_t pos_base, const int32_t *row_map, int64_t out_base,
                                    int32_t F, const int32_t *win, const float *dm, const float *z, int64_t ldz,
                                    float *dy, void *stream) {
    BNS_REQUIRE(gT && gT->perm, "bns_sage_max_bwd_f32: needs a graph made by bns_graph_transpose");
    BNS_REQUIRE(sage_width_ok(F), "bns_sage_max_bwd_f32: need a width %% 4 == 0 in 4..%d (got %d)", kSageMaxWidth, F);
    BNS_REQUIRE(pos_base >= 0 && pos_base + gT->nnz <= INT32_MAX,
                "bns_sage_max_bwd_f32: positions %lld + %lld do not fit int32", (long long)pos_base, (long long)gT->nnz);
    BNS_REQUIRE(out_base >= 0, "bns_sage_max_bwd_f32: negative out_base");
    if (gT->n_rows == 0) return BNS_OK;
    BNS_REQUIRE(z && dy && (gT->nnz == 0 || (win && dm)), "bns_sage_max_bwd_f32: NULL pointer");
    BNS_REQUIRE(ldz % 4 == 0 && ldz >= F && gatv2_aligned(z) && gatv2_aligned(dy) && gatv2_aligned(win) &&
                    gatv2_aligned(dm), "bns_sage_max_bwd_f32: 16-byte aligned rows required");
    const unsigned grid = gat_grid(gT->n_rows);
    cudaStream_t st = as_stream(stream);
    BNS_SAGE_DISPATCH(sage_nv(F),
                      (sage_max_bwd_kernel<NV><<<grid, kThreads, 0, st>>>(gT->indptr, gT->indices, gT->perm, gT->n_rows,
                                                                          pos_base, row_map, out_base, F, win, dm, z,
                                                                          ldz, dy)));
    ++g_launches;
    BNS_CUDA(cudaGetLastError());
    return BNS_OK;
}

extern "C" int bns_sage_max_infer_f32(const bns_graph_t *g, int32_t F, const float *z, int64_t ldz, float *out,
                                      void *stream) {
    BNS_REQUIRE(g, "bns_sage_max_infer_f32: NULL graph");
    BNS_REQUIRE(sage_width_ok(F), "bns_sage_max_infer_f32: need a width %% 4 == 0 in 4..%d (got %d)", kSageMaxWidth, F);
    if (g->n_rows == 0) return BNS_OK;
    BNS_REQUIRE(out && (g->nnz == 0 || z), "bns_sage_max_infer_f32: NULL pointer");
    BNS_REQUIRE(ldz % 4 == 0 && ldz >= F && gatv2_aligned(z) && gatv2_aligned(out),
                "bns_sage_max_infer_f32: 16-byte aligned rows required");
    SageInferArgs a{};
    a.indptr = g->indptr; a.indices = g->indices; a.n_rows = g->n_rows; a.z = z; a.ldz = ldz; a.F = F; a.out = out;
    const unsigned grid = gat_grid(g->n_rows);
    cudaStream_t st = as_stream(stream);
    BNS_SAGE_DISPATCH(sage_nv(F), (sage_max_infer_kernel<NV><<<grid, kThreads, 0, st>>>(a)));
    ++g_launches;
    BNS_CUDA(cudaGetLastError());
    return BNS_OK;
}

extern "C" int bns_sage_max_infer_block_f32(const bns_graph_t *g, int32_t F, const float *z, int64_t ldz, float *m,
                                            int32_t *seen, int first, int last, float *out, void *stream) {
    BNS_REQUIRE(g, "bns_sage_max_infer_block_f32: NULL graph");
    BNS_REQUIRE(sage_width_ok(F), "bns_sage_max_infer_block_f32: need a width %% 4 == 0 in 4..%d (got %d)",
                kSageMaxWidth, F);
    if (g->n_rows == 0) return BNS_OK;
    BNS_REQUIRE(m && seen && (g->nnz == 0 || z) && (!last || out), "bns_sage_max_infer_block_f32: NULL pointer");
    BNS_REQUIRE(ldz % 4 == 0 && ldz >= F && gatv2_aligned(z) && gatv2_aligned(m) && gatv2_aligned(out),
                "bns_sage_max_infer_block_f32: 16-byte aligned rows required");
    SageInferBlockArgs a{};
    a.indptr = g->indptr; a.indices = g->indices; a.n_rows = g->n_rows; a.z = z; a.ldz = ldz; a.F = F; a.out = out;
    a.sm = m; a.seen = seen; a.first = first ? 1 : 0; a.last = last ? 1 : 0;
    const unsigned grid = gat_grid(g->n_rows);
    cudaStream_t st = as_stream(stream);
    BNS_SAGE_DISPATCH(sage_nv(F), (sage_max_infer_kernel<NV, true><<<grid, kThreads, 0, st>>>(a)));
    ++g_launches;
    BNS_CUDA(cudaGetLastError());
    return BNS_OK;
}

#undef BNS_SAGE_DISPATCH
