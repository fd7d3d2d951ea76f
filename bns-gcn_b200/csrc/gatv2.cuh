// gatv2.cuh -- GATv2Conv's dynamic attention as kernels (included by bnsgcn.cu after gat.cuh, whose GatGraph, gat_keep,
// gat_fill and gat_grid it shares).  Per entry u -> v and head h the score is F-wide:
//
//   s_uv = sum_f attn[h, f] * leaky_relu(z_src[u, h, f] + z_dst[v, h, f])
//   a = attn_drop(edge_softmax(s)),   rst_v = sum_u a_uv z_src[u]
//
// Every kernel here holds a row of z in a warp, lane l owning the float4 column groups l, l + 32, ... (NV of them, so
// heads * padded width <= 128 NV), gathers z_src rows U at a time and reduces the per-head partial dots across the warp
// in a fixed shuffle tree: two launches on the same inputs give bit-identical results.
//
//   gatv2_scores_kernel       one warp per destination row (inner entries, then this epoch's sampled halo entries chunk
//                             by chunk): the scores, an online max / sum per lane, then P and the dropped a' per entry
//                             (a' of the halo entries also at their compacted positions), as gat_scores_kernel writes them
//   (rst = A' z_src is bns_spmm_weighted_f32 + bns_spmm_compact_f32; d a' = <d rst_v, z_src[u]> is bns_sddmm_dot_f32)
//   gatv2_softmax_bwd_kernel  one warp per destination row: d a' -> d s = P (d P - sum_u P d P) per entry (in place),
//                             d z_dst[v] = sum_u d s_uv attn * lrelu'(z_src[u] + z_dst[v]) and a per-warp partial of
//                             d attn = sum d s_uv lrelu(z_src[u] + z_dst[v]), reduced by colsum_final_kernel
//   gatv2_colsum_kernel       one warp per source row of a static transpose, entries through its permutation:
//                             d z_src[u] += sum_v d s_uv attn * lrelu'(z_src[u] + z_dst[v]) (on top of A'^T d rst)
//   gatv2_infer_kernel        the evaluation forward, one pass per row gathering each z_src row once, nothing stored per
//                             entry; BLOCK carries the softmax state between column blocks as gat_infer_kernel does
namespace {

struct Gatv2Args {
    GatGraph g;
    int32_t H, Fp;
    const float *zs, *zd, *attn;                           // [n_u, H*Fp], [n_rows, H*Fp], [H*Fp]
    int64_t ldzs, ldzd;
    float slope, p_drop, keep_scale;
    uint64_t seed, offset; const uint64_t *offset_dev;
    float *P_in, *P_out;                                   // [nnz, H] at the ORIGINAL entry positions
    float *dE_in, *dE_out, *d_zd; int64_t ldd;             // backward
    float4 *partial;                                       // backward: [warps, H*Fp / 4] partial sums of d attn
};

// entries of a 32-entry block whose z_src row gathers are in flight together
template <int NV> struct Gatv2Unroll { static constexpr int value = NV <= 2 ? 4 : (NV == 4 ? 2 : 1); };

// head of each float4 column group of this lane (-1 past the row)
template <int NV> __device__ __forceinline__ void gatv2_heads(int lane, int F, int Fp, int (&hd)[NV]) {
#pragma unroll
    for (int t = 0; t < NV; ++t) {
        const int c = (lane + 32 * t) * 4;
        hd[t] = c < F ? c / Fp : -1;
    }
}

template <int NV> __device__ __forceinline__ void gatv2_load_row(const float *row, int lane, int F, float4 (&x)[NV]) {
#pragma unroll
    for (int t = 0; t < NV; ++t) {
        const int c = (lane + 32 * t) * 4;
        x[t] = c < F ? __ldg(reinterpret_cast<const float4 *>(row + c)) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
}

// per head, the warp-reduced sum of the lanes' partials part[t] of head hd[t]
template <int NV> __device__ __forceinline__ void gatv2_head_sums(const float (&part)[NV], const int (&hd)[NV], int H,
                                                                  float (&s)[kGatMaxHeads]) {
#pragma unroll
    for (int h = 0; h < kGatMaxHeads; ++h) {
        float v = 0.f;
#pragma unroll
        for (int t = 0; t < NV; ++t) v += hd[t] == h ? part[t] : 0.f;
        s[h] = h < H ? warp_sum(v) : 0.f;
    }
}

// the value of head hd of a per-head register array, without a runtime index into it
__device__ __forceinline__ float gatv2_pick(const float (&v)[kGatMaxHeads], int hd) {
    float r = 0.f;
#pragma unroll
    for (int h = 0; h < kGatMaxHeads; ++h) r = hd == h ? v[h] : r;
    return r;
}

// the scores of one gathered z_src row x against the destination row xd: s[h] on every lane
template <int NV> __device__ __forceinline__ void gatv2_score(const float4 (&x)[NV], const float4 (&xd)[NV],
                                                              const float4 (&av)[NV], const int (&hd)[NV], int H,
                                                              float slope, float (&s)[kGatMaxHeads]) {
    float part[NV];
#pragma unroll
    for (int t = 0; t < NV; ++t)
        part[t] = (av[t].x * leaky(x[t].x + xd[t].x, slope) + av[t].y * leaky(x[t].y + xd[t].y, slope)) +
                  (av[t].z * leaky(x[t].z + xd[t].z, slope) + av[t].w * leaky(x[t].w + xd[t].w, slope));
    gatv2_head_sums<NV>(part, hd, H, s);
}

// Walks the entries of row v in warp-uniform blocks of at most 32, one entry per lane:
//   body(valid, u = source row of z_src, pos = position in the original CSR arrays, halo, compacted position, n)
// with n the block's entry count (the lanes below n are valid).
template <class Body>
__device__ __forceinline__ void gatv2_walk_row(const GatGraph &g, int64_t v, int lane, Body body) {
    const int64_t b = g.in_ptr[v], e = g.in_ptr[v + 1];
    for (int64_t k0 = b; k0 < e; k0 += 32) {
        const int64_t k = k0 + lane;
        const bool valid = k < e;
        body(valid, valid ? g.in_idx[k] : 0, k, false, (int64_t)0, (int)(e - k0 < 32 ? e - k0 : 32));
    }
    if (g.cidx) {
        for (int32_t c = g.out_row_chunk[v]; c < g.out_row_chunk[v + 1]; ++c) {
            const int64_t s0 = g.out_chunk_start[c];
            const int32_t cnt = g.chunk_cnt[c];
            for (int32_t j0 = 0; j0 < cnt; j0 += 32) {
                const int32_t j = j0 + lane;
                const bool valid = j < cnt;
                body(valid, valid ? (int32_t)g.x_halo_base + g.cidx[s0 + j] : 0, valid ? (int64_t)g.cpos[s0 + j] : 0,
                     true, s0 + j, cnt - j0 < 32 ? cnt - j0 : 32);
            }
        }
    }
}

// (kThreads, 1): without the minimum ptxas capped NV = 1 at 80 and NV = 4 at 128 registers and spilled; with it, 91 /
// 118 / 138 / 168 registers for NV = 1 / 2 / 4 / 8 and no spills
template <int NV>
__global__ void __launch_bounds__(kThreads, 1) gatv2_scores_kernel(Gatv2Args a, int64_t nnz_in, float *W_in, float *W_out,
                                                               float *Wc) {
    constexpr int U = Gatv2Unroll<NV>::value;
    __shared__ int32_t s_u[kWarps][32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int64_t warps_total = (int64_t)gridDim.x * kWarps;
    const uint64_t offset = a.offset + (a.offset_dev ? *a.offset_dev : 0ull);
    const int H = a.H, F = a.H * a.Fp;
    int hd[NV];
    gatv2_heads<NV>(lane, F, a.Fp, hd);
    float4 av[NV];
    gatv2_load_row<NV>(a.attn, lane, F, av);
    for (int64_t v = (int64_t)blockIdx.x * kWarps + w; v < a.g.n_rows; v += warps_total) {
        float4 xd[NV];
        gatv2_load_row<NV>(a.zd + v * a.ldzd, lane, F, xd);
        float m[kGatMaxHeads], l[kGatMaxHeads];          // this lane's entries: running max and sum of exp
#pragma unroll
        for (int h = 0; h < kGatMaxHeads; ++h) { m[h] = -INFINITY; l[h] = 0.f; }
        // first walk: each lane keeps the scores of its own entry and stores them raw in P
        gatv2_walk_row(a.g, v, lane, [&](bool valid, int32_t u, int64_t pos, bool halo, int64_t, int n) {
            s_u[w][lane] = u;
            __syncwarp();
            float mine[kGatMaxHeads];
#pragma unroll
            for (int h = 0; h < kGatMaxHeads; ++h) mine[h] = 0.f;
            for (int jj = 0; jj < n; jj += U) {
                float4 x[U][NV];
#pragma unroll
                for (int q = 0; q < U; ++q) {
                    if (jj + q < n) gatv2_load_row<NV>(a.zs + (int64_t)s_u[w][jj + q] * a.ldzs, lane, F, x[q]);
                }
#pragma unroll
                for (int q = 0; q < U; ++q) {
                    if (jj + q < n) {
                        float s[kGatMaxHeads];
                        gatv2_score<NV>(x[q], xd, av, hd, H, a.slope, s);
                        if (lane == jj + q) {
#pragma unroll
                            for (int h = 0; h < kGatMaxHeads; ++h) mine[h] = s[h];
                        }
                    }
                }
            }
            if (valid) {
                float *P = (halo ? a.P_out : a.P_in) + pos * H;
#pragma unroll
                for (int h = 0; h < kGatMaxHeads; ++h)
                    if (h < H) {
                        const float sc = mine[h];
                        if (sc > m[h]) { l[h] = l[h] * expf(m[h] - sc) + 1.f; m[h] = sc; }
                        else l[h] += expf(sc - m[h]);
                        P[h] = sc;
                    }
            }
            __syncwarp();                                 // s_u is rewritten by the next block
        });
#pragma unroll
        for (int h = 0; h < kGatMaxHeads; ++h) {
            float mt = m[h];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) mt = fmaxf(mt, __shfl_xor_sync(0xffffffffu, mt, o));
            l[h] = warp_sum(m[h] == -INFINITY ? 0.f : l[h] * expf(m[h] - mt));
            m[h] = mt;
        }
        // second walk (each lane rereads the scores it stored): probabilities and dropped attention
        gatv2_walk_row(a.g, v, lane, [&](bool valid, int32_t, int64_t pos, bool halo, int64_t cp, int) {
            if (!valid) return;
            float *P = (halo ? a.P_out : a.P_in) + pos * H;
            const int64_t gid = halo ? nnz_in + pos : pos;
#pragma unroll
            for (int h = 0; h < kGatMaxHeads; ++h)
                if (h < H) {
                    const float p = expf(P[h] - m[h]) / l[h];
                    float wt = p;
                    if (a.p_drop > 0.f) wt = gat_keep(a.seed, offset, gid, h, a.p_drop) ? p * a.keep_scale : 0.f;
                    P[h] = p;
                    if (a.p_drop > 0.f) (halo ? W_out : W_in)[pos * H + h] = wt;
                    if (halo) Wc[cp * H + h] = wt;
                }
        });
    }
}

// in: dE_in / dE_out hold d a' (the SDDMM <d rst_v, z_src[u]>) at the original positions; out: d s in place, d z_dst,
// and one partial of d attn per warp of the grid (every warp writes its slot, zeros when it had no row)
template <int NV>
__global__ void __launch_bounds__(kThreads) gatv2_softmax_bwd_kernel(Gatv2Args a, int64_t nnz_in) {
    constexpr int U = Gatv2Unroll<NV>::value;
    __shared__ int32_t s_u[kWarps][32];
    __shared__ float s_d[kWarps][32][kGatMaxHeads];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int64_t warps_total = (int64_t)gridDim.x * kWarps;
    const uint64_t offset = a.offset + (a.offset_dev ? *a.offset_dev : 0ull);
    const int H = a.H, F = a.H * a.Fp;
    int hd[NV];
    gatv2_heads<NV>(lane, F, a.Fp, hd);
    float4 av[NV], dat[NV];
    gatv2_load_row<NV>(a.attn, lane, F, av);
#pragma unroll
    for (int t = 0; t < NV; ++t) dat[t] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int64_t v = (int64_t)blockIdx.x * kWarps + w; v < a.g.n_rows; v += warps_total) {
        float rowdot[kGatMaxHeads];
#pragma unroll
        for (int h = 0; h < kGatMaxHeads; ++h) rowdot[h] = 0.f;
        gatv2_walk_row(a.g, v, lane, [&](bool valid, int32_t, int64_t pos, bool halo, int64_t, int) {
            if (!valid) return;
            const float *P = (halo ? a.P_out : a.P_in) + pos * H;
            float *dE = (halo ? a.dE_out : a.dE_in) + pos * H;
            const int64_t gid = halo ? nnz_in + pos : pos;
#pragma unroll
            for (int h = 0; h < kGatMaxHeads; ++h)
                if (h < H) {
                    float ms = 1.f;
                    if (a.p_drop > 0.f) ms = gat_keep(a.seed, offset, gid, h, a.p_drop) ? a.keep_scale : 0.f;
                    const float dp = dE[h] * ms;
                    dE[h] = dp;
                    rowdot[h] += P[h] * dp;
                }
        });
#pragma unroll
        for (int h = 0; h < kGatMaxHeads; ++h) rowdot[h] = warp_sum(rowdot[h]);
        float4 xd[NV], dzd[NV];
        gatv2_load_row<NV>(a.zd + v * a.ldzd, lane, F, xd);
#pragma unroll
        for (int t = 0; t < NV; ++t) dzd[t] = make_float4(0.f, 0.f, 0.f, 0.f);
        gatv2_walk_row(a.g, v, lane, [&](bool valid, int32_t u, int64_t pos, bool halo, int64_t, int n) {
            if (valid) {
                const float *P = (halo ? a.P_out : a.P_in) + pos * H;
                float *dE = (halo ? a.dE_out : a.dE_in) + pos * H;
#pragma unroll
                for (int h = 0; h < kGatMaxHeads; ++h) {
                    float ds = 0.f;
                    if (h < H) {
                        ds = P[h] * (dE[h] - rowdot[h]);
                        dE[h] = ds;
                    }
                    s_d[w][lane][h] = ds;
                }
            }
            s_u[w][lane] = u;
            __syncwarp();
            for (int jj = 0; jj < n; jj += U) {
                float4 x[U][NV];
#pragma unroll
                for (int q = 0; q < U; ++q)
                    if (jj + q < n) gatv2_load_row<NV>(a.zs + (int64_t)s_u[w][jj + q] * a.ldzs, lane, F, x[q]);
#pragma unroll
                for (int q = 0; q < U; ++q) {
                    if (jj + q < n) {
#pragma unroll
                        for (int t = 0; t < NV; ++t) {
                            const float ds = hd[t] >= 0 ? s_d[w][jj + q][hd[t]] : 0.f;
                            const float zx = x[q][t].x + xd[t].x, zy = x[q][t].y + xd[t].y;
                            const float zz = x[q][t].z + xd[t].z, zw = x[q][t].w + xd[t].w;
                            const float gx = zx > 0.f ? ds : ds * a.slope, gy = zy > 0.f ? ds : ds * a.slope;
                            const float gz = zz > 0.f ? ds : ds * a.slope, gw = zw > 0.f ? ds : ds * a.slope;
                            dzd[t].x = fmaf(gx, av[t].x, dzd[t].x); dzd[t].y = fmaf(gy, av[t].y, dzd[t].y);
                            dzd[t].z = fmaf(gz, av[t].z, dzd[t].z); dzd[t].w = fmaf(gw, av[t].w, dzd[t].w);
                            dat[t].x = fmaf(gx, zx, dat[t].x); dat[t].y = fmaf(gy, zy, dat[t].y);
                            dat[t].z = fmaf(gz, zz, dat[t].z); dat[t].w = fmaf(gw, zw, dat[t].w);
                        }
                    }
                }
            }
            __syncwarp();                                 // s_u / s_d are rewritten by the next block
        });
        float *o = a.d_zd + v * a.ldd;
#pragma unroll
        for (int t = 0; t < NV; ++t) {
            const int c = (lane + 32 * t) * 4;
            if (c < F) *reinterpret_cast<float4 *>(o + c) = dzd[t];
        }
    }
    const int64_t gw = (int64_t)blockIdx.x * kWarps + w;
#pragma unroll
    for (int t = 0; t < NV; ++t) {
        const int c = (lane + 32 * t) * 4;
        if (c < F) a.partial[gw * (F / 4) + c / 4] = dat[t];
    }
}

// d_zs[out_base + orow(r)] += sum over the entries k of row r of the transpose gT of
//   d s[perm[k], h] attn * lrelu'(z_src[out_base + orow(r)] + z_dst[indices[k]])
template <int NV>
__global__ void __launch_bounds__(kThreads) gatv2_colsum_kernel(const int64_t *__restrict__ indptr, const int32_t *__restrict__ idx,
                                                               const int32_t *__restrict__ perm, int64_t n_rows,
                                                               const float *__restrict__ dS, int32_t H, int32_t Fp,
                                                               const float *__restrict__ zs, int64_t ldzs,
                                                               const float *__restrict__ zd, int64_t ldzd,
                                                               const float *__restrict__ attn, float slope,
                                                               const int32_t *__restrict__ row_map, int64_t out_base,
                                                               float *d_zs, int64_t ldd) {
    constexpr int U = Gatv2Unroll<NV>::value;
    __shared__ int32_t s_v[kWarps][32];
    __shared__ float s_d[kWarps][32][kGatMaxHeads];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int64_t warps_total = (int64_t)gridDim.x * kWarps;
    const int F = H * Fp;
    int hd[NV];
    gatv2_heads<NV>(lane, F, Fp, hd);
    float4 av[NV];
    gatv2_load_row<NV>(attn, lane, F, av);
    for (int64_t r = (int64_t)blockIdx.x * kWarps + w; r < n_rows; r += warps_total) {
        int64_t u = out_base + r;
        if (row_map) {
            const int32_t mrow = row_map[r];
            if (mrow < 0) continue;
            u = out_base + mrow;
        }
        const int64_t b = indptr[r], e = indptr[r + 1];
        if (b == e) continue;
        float4 xs[NV], acc[NV];
        gatv2_load_row<NV>(zs + u * ldzs, lane, F, xs);
#pragma unroll
        for (int t = 0; t < NV; ++t) acc[t] = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int64_t k0 = b; k0 < e; k0 += 32) {
            const int64_t k = k0 + lane;
            const int n = (int)(e - k0 < 32 ? e - k0 : 32);
            if (k < e) {
                const float *d = dS + (int64_t)perm[k] * H;
                s_v[w][lane] = idx[k];
#pragma unroll
                for (int h = 0; h < kGatMaxHeads; ++h) s_d[w][lane][h] = h < H ? d[h] : 0.f;
            }
            __syncwarp();
            for (int jj = 0; jj < n; jj += U) {
                float4 x[U][NV];
#pragma unroll
                for (int q = 0; q < U; ++q)
                    if (jj + q < n) gatv2_load_row<NV>(zd + (int64_t)s_v[w][jj + q] * ldzd, lane, F, x[q]);
#pragma unroll
                for (int q = 0; q < U; ++q) {
                    if (jj + q < n) {
#pragma unroll
                        for (int t = 0; t < NV; ++t) {
                            const float ds = hd[t] >= 0 ? s_d[w][jj + q][hd[t]] : 0.f;
                            const float zx = x[q][t].x + xs[t].x, zy = x[q][t].y + xs[t].y;
                            const float zz = x[q][t].z + xs[t].z, zw = x[q][t].w + xs[t].w;
                            acc[t].x = fmaf(zx > 0.f ? ds : ds * slope, av[t].x, acc[t].x);
                            acc[t].y = fmaf(zy > 0.f ? ds : ds * slope, av[t].y, acc[t].y);
                            acc[t].z = fmaf(zz > 0.f ? ds : ds * slope, av[t].z, acc[t].z);
                            acc[t].w = fmaf(zw > 0.f ? ds : ds * slope, av[t].w, acc[t].w);
                        }
                    }
                }
            }
            __syncwarp();
        }
        float *o = d_zs + u * ldd;
#pragma unroll
        for (int t = 0; t < NV; ++t) {
            const int c = (lane + 32 * t) * 4;
            if (c < F) {
                float4 y = *reinterpret_cast<float4 *>(o + c);
                y.x += acc[t].x; y.y += acc[t].y; y.z += acc[t].z; y.w += acc[t].w;
                *reinterpret_cast<float4 *>(o + c) = y;
            }
        }
    }
}

// ---- the evaluation forward on a homogeneous graph (no dropout, no backward) ---------------------------------------
// Per row, the entries are taken U at a time: their z_src rows are gathered once, their scores reduced across the
// warp, and the running maximum m, sum of exp l (both warp-uniform) and the accumulator are rescaled by exp(m_old -
// m_new) once per group.  BLOCK = true: the row's entries arrive as several matrices over different column sets, one
// launch each, with m, l [n_rows, H] and acc [n_rows, H * Fp] carried between launches in memory (gat_infer_kernel's
// protocol: a launch that is not `first` reloads the state, one that is not `last` stores it back, `last` writes
// acc / l; a row without entries in a middle launch keeps its state untouched).
struct Gatv2InferArgs {
    const int64_t *indptr; const int32_t *indices; int64_t n_rows;
    const float *zs; int64_t ldzs;                         // [n_cols, H * Fp]
    const float *zd; int64_t ldzd;                         // [n_rows, H * Fp]
    const float *attn; int32_t H, Fp;
    float slope;
    float *rst; int64_t ldr;
};

struct Gatv2InferBlockArgs : Gatv2InferArgs {
    float *sm, *sl, *sacc; int64_t ldacc;
    int32_t first, last;
};

template <int NV, bool BLOCK = false>
__global__ void __launch_bounds__(kThreads)
gatv2_infer_kernel(typename std::conditional<BLOCK, Gatv2InferBlockArgs, Gatv2InferArgs>::type a) {
    constexpr int U = Gatv2Unroll<NV>::value;
    __shared__ int32_t s_u[kWarps][32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int64_t warps_total = (int64_t)gridDim.x * kWarps;
    const int H = a.H, F = a.H * a.Fp;
    int hd[NV];
    gatv2_heads<NV>(lane, F, a.Fp, hd);
    float4 av[NV];
    gatv2_load_row<NV>(a.attn, lane, F, av);
    for (int64_t v = (int64_t)blockIdx.x * kWarps + w; v < a.n_rows; v += warps_total) {
        const int64_t b = a.indptr[v], e = a.indptr[v + 1];
        float m[kGatMaxHeads], l[kGatMaxHeads];
        float4 acc[NV];
#pragma unroll
        for (int h = 0; h < kGatMaxHeads; ++h) { m[h] = -INFINITY; l[h] = 0.f; }
#pragma unroll
        for (int t = 0; t < NV; ++t) acc[t] = make_float4(0.f, 0.f, 0.f, 0.f);
        if constexpr (BLOCK) {
            if (b == e && !a.first && !a.last) continue;
            if (!a.first) {
#pragma unroll
                for (int h = 0; h < kGatMaxHeads; ++h)
                    if (h < H) { m[h] = a.sm[v * H + h]; l[h] = a.sl[v * H + h]; }
                const float *sa = a.sacc + v * a.ldacc;
#pragma unroll
                for (int t = 0; t < NV; ++t) {
                    const int c = (lane + 32 * t) * 4;
                    if (c < F) acc[t] = *reinterpret_cast<const float4 *>(sa + c);
                }
            }
        }
        float4 xd[NV];
        if (b < e) gatv2_load_row<NV>(a.zd + v * a.ldzd, lane, F, xd);
        for (int64_t k0 = b; k0 < e; k0 += 32) {
            const int n = (int)(e - k0 < 32 ? e - k0 : 32);
            if (lane < n) s_u[w][lane] = __ldg(a.indices + k0 + lane);
            __syncwarp();
            for (int jj = 0; jj < n; jj += U) {
                float4 x[U][NV];
                float s[U][kGatMaxHeads];
#pragma unroll
                for (int q = 0; q < U; ++q) {
                    if (jj + q < n) gatv2_load_row<NV>(a.zs + (int64_t)s_u[w][jj + q] * a.ldzs, lane, F, x[q]);
                    else {                                // weight 0 below: keep 0 * x finite
#pragma unroll
                        for (int t = 0; t < NV; ++t) x[q][t] = make_float4(0.f, 0.f, 0.f, 0.f);
                    }
                }
#pragma unroll
                for (int q = 0; q < U; ++q) {
                    if (jj + q < n) gatv2_score<NV>(x[q], xd, av, hd, H, a.slope, s[q]);
                    else {
#pragma unroll
                        for (int h = 0; h < kGatMaxHeads; ++h) s[q][h] = -INFINITY;
                    }
                }
                float f[kGatMaxHeads];
#pragma unroll
                for (int h = 0; h < kGatMaxHeads; ++h) {
                    float mn = m[h];
#pragma unroll
                    for (int q = 0; q < U; ++q) mn = fmaxf(mn, s[q][h]);
                    f[h] = h < H ? expf(m[h] - mn) : 1.f;             // 0 on the first group
                    float ls = l[h] * f[h];
#pragma unroll
                    for (int q = 0; q < U; ++q) {
                        s[q][h] = h < H && jj + q < n ? expf(s[q][h] - mn) : 0.f;     // now the weight
                        ls += s[q][h];
                    }
                    l[h] = ls;
                    m[h] = mn;
                }
#pragma unroll
                for (int t = 0; t < NV; ++t) {
                    const float sf = gatv2_pick(f, hd[t]);
                    float4 y = make_float4(acc[t].x * sf, acc[t].y * sf, acc[t].z * sf, acc[t].w * sf);
#pragma unroll
                    for (int q = 0; q < U; ++q) {
                        const float p = gatv2_pick(s[q], hd[t]);
                        y.x = fmaf(p, x[q][t].x, y.x); y.y = fmaf(p, x[q][t].y, y.y);
                        y.z = fmaf(p, x[q][t].z, y.z); y.w = fmaf(p, x[q][t].w, y.w);
                    }
                    acc[t] = y;
                }
            }
            __syncwarp();
        }
        if constexpr (BLOCK) {
            if (!a.last) {
                if (lane == 0) {
#pragma unroll
                    for (int h = 0; h < kGatMaxHeads; ++h)
                        if (h < H) { a.sm[v * H + h] = m[h]; a.sl[v * H + h] = l[h]; }
                }
                float *sa = a.sacc + v * a.ldacc;
#pragma unroll
                for (int t = 0; t < NV; ++t) {
                    const int c = (lane + 32 * t) * 4;
                    if (c < F) *reinterpret_cast<float4 *>(sa + c) = acc[t];
                }
                continue;
            }
        }
        float *out = a.rst + v * a.ldr;
#pragma unroll
        for (int t = 0; t < NV; ++t) {
            const int c = (lane + 32 * t) * 4;
            if (c < F) {
                const float den = gatv2_pick(l, hd[t]);
                *reinterpret_cast<float4 *>(out + c) =
                    den > 0.f ? make_float4(acc[t].x / den, acc[t].y / den, acc[t].z / den, acc[t].w / den)
                              : make_float4(0.f, 0.f, 0.f, 0.f);        // a row without entries
            }
        }
    }
}

inline int gatv2_nv(int64_t HF) {
    const int nv = (int)((HF + 127) / 128);
    return nv <= 1 ? 1 : (nv == 2 ? 2 : (nv <= 4 ? 4 : 8));
}

#define BNS_GATV2_DISPATCH(NVV, LAUNCH) \
    switch (NVV) {                      \
    case 1: { constexpr int NV = 1; LAUNCH; } break; \
    case 2: { constexpr int NV = 2; LAUNCH; } break; \
    case 4: { constexpr int NV = 4; LAUNCH; } break; \
    default: { constexpr int NV = 8; LAUNCH; } break; \
    }

inline bool gatv2_width_ok(int32_t H, int32_t Fp) {
    return H >= 1 && H <= kGatMaxHeads && Fp > 0 && Fp % 4 == 0 && (int64_t)H * Fp <= 1024;
}

inline bool gatv2_aligned(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

int gatv2_fill(Gatv2Args &a, const bns_graph *a_in, const bns_graph *a_out, const int32_t *cidx, const int32_t *chunk_cnt,
               const int32_t *cpos, int64_t x_halo_base, int32_t H, int32_t Fp, const float *zs, int64_t ldzs,
               const float *zd, int64_t ldzd, const float *attn, float slope, float p_drop, uint64_t seed,
               uint64_t offset, const uint64_t *offset_dev, const char *who) {
    GatArgs ga{};
    int rc = gat_fill(ga, a_in, a_out, cidx, chunk_cnt, cpos, x_halo_base, who);
    if (rc) return rc;
    a.g = ga.g;
    BNS_REQUIRE(gatv2_width_ok(H, Fp), "%s: need 1 <= heads <= 8, padded width %% 4 == 0, heads * padded width <= 1024 "
                "(got %d, %d)", who, H, Fp);
    BNS_REQUIRE(p_drop >= 0.f && p_drop < 1.f, "%s: p must be in [0, 1)", who);
    const int64_t HF = (int64_t)H * Fp;
    if (a.g.n_rows == 0) return BNS_OK;
    BNS_REQUIRE(zs && zd && attn, "%s: NULL pointer", who);
    BNS_REQUIRE(ldzs % 4 == 0 && ldzd % 4 == 0 && ldzs >= HF && ldzd >= HF && gatv2_aligned(zs) && gatv2_aligned(zd) &&
                    gatv2_aligned(attn), "%s: 16-byte aligned rows required", who);
    a.H = H; a.Fp = Fp; a.zs = zs; a.ldzs = ldzs; a.zd = zd; a.ldzd = ldzd; a.attn = attn;
    a.slope = slope; a.p_drop = p_drop; a.keep_scale = 1.f / (1.f - p_drop);
    a.seed = seed; a.offset = offset; a.offset_dev = offset_dev;
    return BNS_OK;
}

}  // namespace

extern "C" int bns_gatv2_scores_f32(const bns_graph_t *a_in, const bns_graph_t *a_out, const int32_t *cidx,
                                    const int32_t *chunk_cnt, const int32_t *cpos, int64_t x_halo_base, int32_t H,
                                    int32_t Fp, const float *zs, int64_t ldzs, const float *zd, int64_t ldzd,
                                    const float *attn, float slope, float p_drop, uint64_t seed, uint64_t offset,
                                    const uint64_t *offset_dev, float *P_in, float *P_out, float *W_in, float *W_out,
                                    float *W_out_compact, void *stream) {
    Gatv2Args a{};
    int rc = gatv2_fill(a, a_in, a_out, cidx, chunk_cnt, cpos, x_halo_base, H, Fp, zs, ldzs, zd, ldzd, attn, slope,
                        p_drop, seed, offset, offset_dev, "bns_gatv2_scores_f32");
    if (rc || a.g.n_rows == 0) return rc;
    BNS_REQUIRE(P_in && (a.g.cidx == nullptr || (P_out && W_out_compact)), "bns_gatv2_scores_f32: NULL pointer");
    BNS_REQUIRE(p_drop == 0.f || (W_in && (a.g.cidx == nullptr || W_out)), "bns_gatv2_scores_f32: dropout needs W_in / W_out");
    a.P_in = P_in; a.P_out = P_out;
    const unsigned grid = gat_grid(a.g.n_rows);
    cudaStream_t st = as_stream(stream);
    BNS_GATV2_DISPATCH(gatv2_nv((int64_t)H * Fp),
                       (gatv2_scores_kernel<NV><<<grid, kThreads, 0, st>>>(a, a_in->nnz, W_in, W_out, W_out_compact)));
    ++g_launches;
    BNS_CUDA(cudaGetLastError());
    return BNS_OK;
}

extern "C" size_t bns_gatv2_bwd_workspace_bytes(int64_t n_rows, int32_t H, int32_t Fp) {
    if (n_rows <= 0 || H <= 0 || Fp <= 0) return 0;
    return (size_t)gat_grid(n_rows) * kWarps * (size_t)H * (size_t)Fp * sizeof(float);
}

extern "C" int bns_gatv2_softmax_bwd_f32(const bns_graph_t *a_in, const bns_graph_t *a_out, const int32_t *cidx,
                                         const int32_t *chunk_cnt, const int32_t *cpos, int64_t x_halo_base, int32_t H,
                                         int32_t Fp, const float *zs, int64_t ldzs, const float *zd, int64_t ldzd,
                                         const float *attn, float slope, float p_drop, uint64_t seed, uint64_t offset,
                                         const uint64_t *offset_dev, const float *P_in, const float *P_out, float *dE_in,
                                         float *dE_out, float *d_zd, int64_t ldd, float *d_attn, void *ws,
                                         size_t ws_bytes, void *stream) {
    Gatv2Args a{};
    int rc = gatv2_fill(a, a_in, a_out, cidx, chunk_cnt, cpos, x_halo_base, H, Fp, zs, ldzs, zd, ldzd, attn, slope,
                        p_drop, seed, offset, offset_dev, "bns_gatv2_softmax_bwd_f32");
    if (rc) return rc;
    BNS_REQUIRE(d_attn && gatv2_aligned(d_attn), "bns_gatv2_softmax_bwd_f32: d_attn must be a 16-byte aligned pointer");
    const int64_t HF = (int64_t)H * Fp;
    cudaStream_t st = as_stream(stream);
    if (a.g.n_rows == 0) {
        BNS_CUDA(cudaMemsetAsync(d_attn, 0, (size_t)HF * sizeof(float), st));
        return BNS_OK;
    }
    BNS_REQUIRE(P_in && dE_in && d_zd && (a.g.cidx == nullptr || (P_out && dE_out)), "bns_gatv2_softmax_bwd_f32: NULL pointer");
    BNS_REQUIRE(ldd % 4 == 0 && ldd >= HF && gatv2_aligned(d_zd), "bns_gatv2_softmax_bwd_f32: 16-byte aligned d_zd rows required");
    const size_t need = bns_gatv2_bwd_workspace_bytes(a.g.n_rows, H, Fp);
    if (!ws || ws_bytes < need || !gatv2_aligned(ws))
        return fail(BNS_E_WORKSPACE, "bns_gatv2_softmax_bwd_f32: workspace %zu bytes < %zu needed", ws_bytes, need);
    a.P_in = const_cast<float *>(P_in); a.P_out = const_cast<float *>(P_out);
    a.dE_in = dE_in; a.dE_out = dE_out; a.d_zd = d_zd; a.ldd = ldd; a.partial = reinterpret_cast<float4 *>(ws);
    const unsigned grid = gat_grid(a.g.n_rows);
    BNS_GATV2_DISPATCH(gatv2_nv(HF), (gatv2_softmax_bwd_kernel<NV><<<grid, kThreads, 0, st>>>(a, a_in->nnz)));
    const int CV = (int)(HF / 4);
    colsum_final_kernel<<<(CV + kWarps - 1) / kWarps, kThreads, 0, st>>>(reinterpret_cast<const float4 *>(ws),
                                                                         (int)(grid * kWarps), CV,
                                                                         reinterpret_cast<float4 *>(d_attn), nullptr);
    g_launches += 2;
    BNS_CUDA(cudaGetLastError());
    return BNS_OK;
}

extern "C" int bns_gatv2_colsum_f32(const bns_graph_t *gT, const float *dS, int32_t H, int32_t Fp, const float *zs,
                                    int64_t ldzs, const float *zd, int64_t ldzd, const float *attn, float slope,
                                    const int32_t *row_map, int64_t out_base, float *d_zs, int64_t ldd, void *stream) {
    BNS_REQUIRE(gT && gT->perm, "bns_gatv2_colsum_f32: needs a graph made by bns_graph_transpose");
    BNS_REQUIRE(gatv2_width_ok(H, Fp), "bns_gatv2_colsum_f32: need 1 <= heads <= 8, padded width %% 4 == 0, heads * "
                "padded width <= 1024 (got %d, %d)", H, Fp);
    if (gT->n_rows == 0 || gT->nnz == 0) return BNS_OK;
    BNS_REQUIRE(dS && zs && zd && attn && d_zs, "bns_gatv2_colsum_f32: NULL pointer");
    const int64_t HF = (int64_t)H * Fp;
    BNS_REQUIRE(ldzs % 4 == 0 && ldzd % 4 == 0 && ldd % 4 == 0 && ldzs >= HF && ldzd >= HF && ldd >= HF &&
                    gatv2_aligned(zs) && gatv2_aligned(zd) && gatv2_aligned(attn) && gatv2_aligned(d_zs),
                "bns_gatv2_colsum_f32: 16-byte aligned rows required");
    const unsigned grid = gat_grid(gT->n_rows);
    cudaStream_t st = as_stream(stream);
    BNS_GATV2_DISPATCH(gatv2_nv(HF),
                       (gatv2_colsum_kernel<NV><<<grid, kThreads, 0, st>>>(gT->indptr, gT->indices, gT->perm, gT->n_rows,
                                                                          dS, H, Fp, zs, ldzs, zd, ldzd, attn, slope,
                                                                          row_map, out_base, d_zs, ldd)));
    ++g_launches;
    BNS_CUDA(cudaGetLastError());
    return BNS_OK;
}

extern "C" int bns_gatv2_infer_f32(const bns_graph_t *g, const float *zs, int64_t ldzs, const float *zd, int64_t ldzd,
                                   const float *attn, int32_t H, int32_t Fp, float slope, float *rst, int64_t ldr,
                                   void *stream) {
    BNS_REQUIRE(g, "bns_gatv2_infer_f32: NULL graph");
    BNS_REQUIRE(gatv2_width_ok(H, Fp), "bns_gatv2_infer_f32: need 1 <= heads <= 8, padded width %% 4 == 0, heads * "
                "padded width <= 1024 (got %d, %d)", H, Fp);
    if (g->n_rows == 0) return BNS_OK;
    BNS_REQUIRE(zs && zd && attn && rst, "bns_gatv2_infer_f32: NULL pointer");
    const int64_t HF = (int64_t)H * Fp;
    BNS_REQUIRE(ldzs % 4 == 0 && ldzd % 4 == 0 && ldr % 4 == 0 && ldzs >= HF && ldzd >= HF && ldr >= HF &&
                    gatv2_aligned(zs) && gatv2_aligned(zd) && gatv2_aligned(attn) && gatv2_aligned(rst),
                "bns_gatv2_infer_f32: 16-byte aligned rows required");
    Gatv2InferArgs a{};
    a.indptr = g->indptr; a.indices = g->indices; a.n_rows = g->n_rows;
    a.zs = zs; a.ldzs = ldzs; a.zd = zd; a.ldzd = ldzd; a.attn = attn; a.H = H; a.Fp = Fp; a.slope = slope;
    a.rst = rst; a.ldr = ldr;
    const unsigned grid = gat_grid(g->n_rows);
    cudaStream_t st = as_stream(stream);
    BNS_GATV2_DISPATCH(gatv2_nv(HF), (gatv2_infer_kernel<NV><<<grid, kThreads, 0, st>>>(a)));
    ++g_launches;
    BNS_CUDA(cudaGetLastError());
    return BNS_OK;
}

extern "C" int bns_gatv2_infer_block_f32(const bns_graph_t *g, const float *zs, int64_t ldzs, const float *zd,
                                         int64_t ldzd, const float *attn, int32_t H, int32_t Fp, float slope, float *m,
                                         float *l, float *acc, int64_t ldacc, int first, int last, float *rst,
                                         int64_t ldr, void *stream) {
    BNS_REQUIRE(g, "bns_gatv2_infer_block_f32: NULL graph");
    BNS_REQUIRE(gatv2_width_ok(H, Fp), "bns_gatv2_infer_block_f32: need 1 <= heads <= 8, padded width %% 4 == 0, heads "
                "* padded width <= 1024 (got %d, %d)", H, Fp);
    if (g->n_rows == 0) return BNS_OK;
    const int64_t HF = (int64_t)H * Fp;
    BNS_REQUIRE(attn && m && l && acc && (g->nnz == 0 || (zs && zd)) && (!last || rst),
                "bns_gatv2_infer_block_f32: NULL pointer");
    BNS_REQUIRE(ldzs % 4 == 0 && ldzd % 4 == 0 && ldr % 4 == 0 && ldacc % 4 == 0 && (g->nnz == 0 || (ldzs >= HF && ldzd >= HF)) &&
                    (!last || ldr >= HF) && ldacc >= HF && gatv2_aligned(zs) && gatv2_aligned(zd) && gatv2_aligned(attn) &&
                    gatv2_aligned(acc) && gatv2_aligned(rst),
                "bns_gatv2_infer_block_f32: 16-byte aligned rows required");
    BNS_REQUIRE(!last || rst != acc || ldr == ldacc, "bns_gatv2_infer_block_f32: rst aliases acc with a different stride");
    Gatv2InferBlockArgs a{};
    a.indptr = g->indptr; a.indices = g->indices; a.n_rows = g->n_rows;
    a.zs = zs; a.ldzs = ldzs; a.zd = zd; a.ldzd = ldzd; a.attn = attn; a.H = H; a.Fp = Fp; a.slope = slope;
    a.rst = rst; a.ldr = ldr;
    a.sm = m; a.sl = l; a.sacc = acc; a.ldacc = ldacc; a.first = first ? 1 : 0; a.last = last ? 1 : 0;
    const unsigned grid = gat_grid(g->n_rows);
    cudaStream_t st = as_stream(stream);
    BNS_GATV2_DISPATCH(gatv2_nv(HF), (gatv2_infer_kernel<NV, true><<<grid, kThreads, 0, st>>>(a)));
    ++g_launches;
    BNS_CUDA(cudaGetLastError());
    return BNS_OK;
}

#undef BNS_GATV2_DISPATCH
