// transformer.cuh -- the graph transformer layer's scaled dot-product attention as kernels (included by bnsgcn.cu after
// gatv2.cuh, whose row walk, column-group layout and per-head warp sums it shares).  Per entry u -> v and head h:
//
//   s_uv = scale * <q[v, h, :], k[u, h, :]>,   a = attn_drop(edge_softmax(s)),   rst_v = sum_u a_uv v[u]
//
// Three tables take part: q (destination rows), k and v (source rows).  Each may be a column view of a wider table
// (row stride ld*): the layer projects k and v with one GEMM into [n_u, 2 * H * Fp], so the evaluation forward reads
// one contiguous row per entry.  A warp holds a row, lane l owning the float4 column groups l, l + 32, ... (NV of
// them); per-head dots are reduced across the warp in a fixed shuffle tree, so two launches give bit-identical results.
//
//   tconv_scores_kernel       one warp per destination row (inner entries, then this epoch's sampled halo entries):
//                             the scores, an online max / sum, then P and the dropped a' per entry as
//                             gatv2_scores_kernel writes them
//   (rst = A' v is bns_spmm_weighted_f32 + bns_spmm_compact_f32; d a' = <d rst_v, v[u]> is bns_sddmm_dot_f32;
//    d v = A'^T d rst and d k = dS^T q are bns_spmm_weighted_f32 on the transposes)
//   tconv_softmax_bwd_kernel  one warp per destination row: d a' -> d s = scale P (g - sum_u P g) per entry (in place,
//                             g = d a' through the dropout mask) and d q[v] = sum_u d s_uv k[u], no atomics
//   tconv_infer_kernel        the evaluation forward, one pass per row gathering each k / v row once; BLOCK carries
//                             the softmax state between column blocks as gatv2_infer_kernel does
namespace {

struct TconvArgs {
    GatGraph g;
    int32_t H, Fp;
    const float *q, *k;                                    // [n_rows, H*Fp], [n_u, H*Fp]
    int64_t ldq, ldk;
    float scale, p_drop, keep_scale;
    uint64_t seed, offset; const uint64_t *offset_dev;
    float *P_in, *P_out;                                   // [nnz, H] at the ORIGINAL entry positions
    float *dE_in, *dE_out, *d_q; int64_t ldd;              // backward
};

// the scaled per-head dots of one gathered k row x against the destination's q row xq: s[h] on every lane
template <int NV> __device__ __forceinline__ void tconv_score(const float4 (&x)[NV], const float4 (&xq)[NV],
                                                              const int (&hd)[NV], int H, float scale,
                                                              float (&s)[kGatMaxHeads]) {
    float part[NV];
#pragma unroll
    for (int t = 0; t < NV; ++t)
        part[t] = fmaf(x[t].x, xq[t].x, x[t].y * xq[t].y) + fmaf(x[t].z, xq[t].z, x[t].w * xq[t].w);
    gatv2_head_sums<NV>(part, hd, H, s);
#pragma unroll
    for (int h = 0; h < kGatMaxHeads; ++h) s[h] *= scale;
}

template <int NV>
__global__ void __launch_bounds__(kThreads, 1) tconv_scores_kernel(TconvArgs a, int64_t nnz_in, float *W_in,
                                                                   float *W_out, float *Wc) {
    constexpr int U = Gatv2Unroll<NV>::value;
    __shared__ int32_t s_u[kWarps][32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int64_t warps_total = (int64_t)gridDim.x * kWarps;
    const uint64_t offset = a.offset + (a.offset_dev ? *a.offset_dev : 0ull);
    const int H = a.H, F = a.H * a.Fp;
    int hd[NV];
    gatv2_heads<NV>(lane, F, a.Fp, hd);
    for (int64_t v = (int64_t)blockIdx.x * kWarps + w; v < a.g.n_rows; v += warps_total) {
        float4 xq[NV];
        gatv2_load_row<NV>(a.q + v * a.ldq, lane, F, xq);
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
                    if (jj + q < n) gatv2_load_row<NV>(a.k + (int64_t)s_u[w][jj + q] * a.ldk, lane, F, x[q]);
                }
#pragma unroll
                for (int q = 0; q < U; ++q) {
                    if (jj + q < n) {
                        float s[kGatMaxHeads];
                        tconv_score<NV>(x[q], xq, hd, H, a.scale, s);
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

// in: dE_in / dE_out hold d a' (the SDDMM <d rst_v, v[u]>) at the original positions; out: d s in place and d q
template <int NV>
__global__ void __launch_bounds__(kThreads, 1) tconv_softmax_bwd_kernel(TconvArgs a, int64_t nnz_in) {
    constexpr int U = Gatv2Unroll<NV>::value;
    __shared__ int32_t s_u[kWarps][32];
    __shared__ float s_d[kWarps][32][kGatMaxHeads];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int64_t warps_total = (int64_t)gridDim.x * kWarps;
    const uint64_t offset = a.offset + (a.offset_dev ? *a.offset_dev : 0ull);
    const int H = a.H, F = a.H * a.Fp;
    int hd[NV];
    gatv2_heads<NV>(lane, F, a.Fp, hd);
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
        float4 dq[NV];
#pragma unroll
        for (int t = 0; t < NV; ++t) dq[t] = make_float4(0.f, 0.f, 0.f, 0.f);
        gatv2_walk_row(a.g, v, lane, [&](bool valid, int32_t u, int64_t pos, bool halo, int64_t, int n) {
            if (valid) {
                const float *P = (halo ? a.P_out : a.P_in) + pos * H;
                float *dE = (halo ? a.dE_out : a.dE_in) + pos * H;
#pragma unroll
                for (int h = 0; h < kGatMaxHeads; ++h) {
                    float ds = 0.f;
                    if (h < H) {
                        ds = a.scale * (P[h] * (dE[h] - rowdot[h]));
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
                    if (jj + q < n) gatv2_load_row<NV>(a.k + (int64_t)s_u[w][jj + q] * a.ldk, lane, F, x[q]);
#pragma unroll
                for (int q = 0; q < U; ++q) {
                    if (jj + q < n) {
#pragma unroll
                        for (int t = 0; t < NV; ++t) {
                            const float ds = hd[t] >= 0 ? s_d[w][jj + q][hd[t]] : 0.f;
                            dq[t].x = fmaf(ds, x[q][t].x, dq[t].x); dq[t].y = fmaf(ds, x[q][t].y, dq[t].y);
                            dq[t].z = fmaf(ds, x[q][t].z, dq[t].z); dq[t].w = fmaf(ds, x[q][t].w, dq[t].w);
                        }
                    }
                }
            }
            __syncwarp();                                 // s_u / s_d are rewritten by the next block
        });
        float *o = a.d_q + v * a.ldd;
#pragma unroll
        for (int t = 0; t < NV; ++t) {
            const int c = (lane + 32 * t) * 4;
            if (c < F) *reinterpret_cast<float4 *>(o + c) = dq[t];
        }
    }
}

// ---- the evaluation forward on a homogeneous graph (no dropout, no backward) ---------------------------------------
// gatv2_infer_kernel's structure: per row the entries are taken U at a time, their k rows gathered and scored, their v
// rows gathered and added with the group's weights; m, l and acc are rescaled by exp(m_old - m_new) once per group.
// BLOCK = true carries m, l [n_rows, H] and acc [n_rows, H * Fp] between launches in memory (gat_infer_kernel's
// protocol: `first` starts from nothing, a launch that is not `last` stores the state back, `last` writes acc / l; a row
// without entries in a middle launch keeps its state untouched).
struct TconvInferArgs {
    const int64_t *indptr; const int32_t *indices; int64_t n_rows;
    const float *q; int64_t ldq;                           // [n_rows, H * Fp]
    const float *k; int64_t ldk;                           // [n_cols, H * Fp]
    const float *v; int64_t ldv;                           // [n_cols, H * Fp]
    int32_t H, Fp;
    float scale;
    float *rst; int64_t ldr;
};

struct TconvInferBlockArgs : TconvInferArgs {
    float *sm, *sl, *sacc; int64_t ldacc;
    int32_t first, last;
};

template <int NV, bool BLOCK = false>
__global__ void __launch_bounds__(kThreads, 1)
tconv_infer_kernel(typename std::conditional<BLOCK, TconvInferBlockArgs, TconvInferArgs>::type a) {
    constexpr int U = Gatv2Unroll<NV>::value;
    __shared__ int32_t s_u[kWarps][32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int64_t warps_total = (int64_t)gridDim.x * kWarps;
    const int H = a.H, F = a.H * a.Fp;
    int hd[NV];
    gatv2_heads<NV>(lane, F, a.Fp, hd);
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
        float4 xq[NV];
        if (b < e) gatv2_load_row<NV>(a.q + v * a.ldq, lane, F, xq);
        for (int64_t k0 = b; k0 < e; k0 += 32) {
            const int n = (int)(e - k0 < 32 ? e - k0 : 32);
            if (lane < n) s_u[w][lane] = __ldg(a.indices + k0 + lane);
            __syncwarp();
            for (int jj = 0; jj < n; jj += U) {
                float4 xk[U][NV], x[U][NV];                  // the group's k rows and v rows, all in flight together
                float s[U][kGatMaxHeads];
#pragma unroll
                for (int q = 0; q < U; ++q) {
                    if (jj + q < n) {
                        const int64_t u = s_u[w][jj + q];
                        gatv2_load_row<NV>(a.k + u * a.ldk, lane, F, xk[q]);
                        gatv2_load_row<NV>(a.v + u * a.ldv, lane, F, x[q]);
                    } else {                              // weight 0 below: keep 0 * x finite
#pragma unroll
                        for (int t = 0; t < NV; ++t) x[q][t] = make_float4(0.f, 0.f, 0.f, 0.f);
                    }
                }
#pragma unroll
                for (int q = 0; q < U; ++q) {
                    if (jj + q < n) tconv_score<NV>(xk[q], xq, hd, H, a.scale, s[q]);
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

#define BNS_TCONV_DISPATCH(NVV, LAUNCH) \
    switch (NVV) {                      \
    case 1: { constexpr int NV = 1; LAUNCH; } break; \
    case 2: { constexpr int NV = 2; LAUNCH; } break; \
    case 4: { constexpr int NV = 4; LAUNCH; } break; \
    default: { constexpr int NV = 8; LAUNCH; } break; \
    }

int tconv_fill(TconvArgs &a, const bns_graph *a_in, const bns_graph *a_out, const int32_t *cidx,
               const int32_t *chunk_cnt, const int32_t *cpos, int64_t x_halo_base, int32_t H, int32_t Fp,
               const float *q, int64_t ldq, const float *k, int64_t ldk, float scale, float p_drop, uint64_t seed,
               uint64_t offset, const uint64_t *offset_dev, const char *who) {
    GatArgs ga{};
    int rc = gat_fill(ga, a_in, a_out, cidx, chunk_cnt, cpos, x_halo_base, who);
    if (rc) return rc;
    a.g = ga.g;
    BNS_REQUIRE(gatv2_width_ok(H, Fp), "%s: need 1 <= heads <= 8, padded width %% 4 == 0, heads * padded width <= 1024 "
                "(got %d, %d)", who, H, Fp);
    BNS_REQUIRE(p_drop >= 0.f && p_drop < 1.f, "%s: p must be in [0, 1)", who);
    BNS_REQUIRE(scale > 0.f && scale < INFINITY, "%s: scale must be finite and positive", who);
    const int64_t HF = (int64_t)H * Fp;
    if (a.g.n_rows == 0) return BNS_OK;
    BNS_REQUIRE(q && k, "%s: NULL pointer", who);
    BNS_REQUIRE(ldq % 4 == 0 && ldk % 4 == 0 && ldq >= HF && ldk >= HF && gatv2_aligned(q) && gatv2_aligned(k),
                "%s: 16-byte aligned rows required", who);
    a.H = H; a.Fp = Fp; a.q = q; a.ldq = ldq; a.k = k; a.ldk = ldk;
    a.scale = scale; a.p_drop = p_drop; a.keep_scale = 1.f / (1.f - p_drop);
    a.seed = seed; a.offset = offset; a.offset_dev = offset_dev;
    return BNS_OK;
}

int tconv_infer_fill(TconvInferArgs &a, const bns_graph *g, const float *q, int64_t ldq, const float *k, int64_t ldk,
                     const float *v, int64_t ldv, int32_t H, int32_t Fp, float scale, float *rst, int64_t ldr,
                     bool need_rst, const char *who) {
    BNS_REQUIRE(g, "%s: NULL graph", who);
    BNS_REQUIRE(gatv2_width_ok(H, Fp), "%s: need 1 <= heads <= 8, padded width %% 4 == 0, heads * padded width <= 1024 "
                "(got %d, %d)", who, H, Fp);
    BNS_REQUIRE(scale > 0.f && scale < INFINITY, "%s: scale must be finite and positive", who);
    const int64_t HF = (int64_t)H * Fp;
    BNS_REQUIRE((g->nnz == 0 || (q && k && v)) && (!need_rst || rst), "%s: NULL pointer", who);
    BNS_REQUIRE(ldq % 4 == 0 && ldk % 4 == 0 && ldv % 4 == 0 && ldr % 4 == 0 &&
                    (g->nnz == 0 || (ldq >= HF && ldk >= HF && ldv >= HF)) && (!need_rst || ldr >= HF) &&
                    gatv2_aligned(q) && gatv2_aligned(k) && gatv2_aligned(v) && gatv2_aligned(rst),
                "%s: 16-byte aligned rows required", who);
    a.indptr = g->indptr; a.indices = g->indices; a.n_rows = g->n_rows;
    a.q = q; a.ldq = ldq; a.k = k; a.ldk = ldk; a.v = v; a.ldv = ldv; a.H = H; a.Fp = Fp; a.scale = scale;
    a.rst = rst; a.ldr = ldr;
    return BNS_OK;
}

}  // namespace

extern "C" int bns_tconv_scores_f32(const bns_graph_t *a_in, const bns_graph_t *a_out, const int32_t *cidx,
                                    const int32_t *chunk_cnt, const int32_t *cpos, int64_t x_halo_base, int32_t H,
                                    int32_t Fp, const float *q, int64_t ldq, const float *k, int64_t ldk, float scale,
                                    float p_drop, uint64_t seed, uint64_t offset, const uint64_t *offset_dev,
                                    float *P_in, float *P_out, float *W_in, float *W_out, float *W_out_compact,
                                    void *stream) {
    TconvArgs a{};
    int rc = tconv_fill(a, a_in, a_out, cidx, chunk_cnt, cpos, x_halo_base, H, Fp, q, ldq, k, ldk, scale, p_drop, seed,
                        offset, offset_dev, "bns_tconv_scores_f32");
    if (rc || a.g.n_rows == 0) return rc;
    BNS_REQUIRE(P_in && (a.g.cidx == nullptr || (P_out && W_out_compact)), "bns_tconv_scores_f32: NULL pointer");
    BNS_REQUIRE(p_drop == 0.f || (W_in && (a.g.cidx == nullptr || W_out)), "bns_tconv_scores_f32: dropout needs W_in / W_out");
    a.P_in = P_in; a.P_out = P_out;
    const unsigned grid = gat_grid(a.g.n_rows);
    cudaStream_t st = as_stream(stream);
    BNS_TCONV_DISPATCH(gatv2_nv((int64_t)H * Fp),
                       (tconv_scores_kernel<NV><<<grid, kThreads, 0, st>>>(a, a_in->nnz, W_in, W_out, W_out_compact)));
    ++g_launches;
    BNS_CUDA(cudaGetLastError());
    return BNS_OK;
}

extern "C" int bns_tconv_softmax_bwd_f32(const bns_graph_t *a_in, const bns_graph_t *a_out, const int32_t *cidx,
                                         const int32_t *chunk_cnt, const int32_t *cpos, int64_t x_halo_base, int32_t H,
                                         int32_t Fp, const float *q, int64_t ldq, const float *k, int64_t ldk,
                                         float scale, float p_drop, uint64_t seed, uint64_t offset,
                                         const uint64_t *offset_dev, const float *P_in, const float *P_out,
                                         float *dE_in, float *dE_out, float *d_q, int64_t ldd, void *stream) {
    TconvArgs a{};
    int rc = tconv_fill(a, a_in, a_out, cidx, chunk_cnt, cpos, x_halo_base, H, Fp, q, ldq, k, ldk, scale, p_drop, seed,
                        offset, offset_dev, "bns_tconv_softmax_bwd_f32");
    if (rc || a.g.n_rows == 0) return rc;
    const int64_t HF = (int64_t)H * Fp;
    BNS_REQUIRE(P_in && dE_in && d_q && (a.g.cidx == nullptr || (P_out && dE_out)), "bns_tconv_softmax_bwd_f32: NULL pointer");
    BNS_REQUIRE(ldd % 4 == 0 && ldd >= HF && gatv2_aligned(d_q), "bns_tconv_softmax_bwd_f32: 16-byte aligned d_q rows required");
    a.P_in = const_cast<float *>(P_in); a.P_out = const_cast<float *>(P_out);
    a.dE_in = dE_in; a.dE_out = dE_out; a.d_q = d_q; a.ldd = ldd;
    const unsigned grid = gat_grid(a.g.n_rows);
    cudaStream_t st = as_stream(stream);
    BNS_TCONV_DISPATCH(gatv2_nv(HF), (tconv_softmax_bwd_kernel<NV><<<grid, kThreads, 0, st>>>(a, a_in->nnz)));
    ++g_launches;
    BNS_CUDA(cudaGetLastError());
    return BNS_OK;
}

extern "C" int bns_tconv_infer_f32(const bns_graph_t *g, const float *q, int64_t ldq, const float *k, int64_t ldk,
                                   const float *v, int64_t ldv, int32_t H, int32_t Fp, float scale, float *rst,
                                   int64_t ldr, void *stream) {
    TconvInferArgs a{};
    int rc = tconv_infer_fill(a, g, q, ldq, k, ldk, v, ldv, H, Fp, scale, rst, ldr, true, "bns_tconv_infer_f32");
    if (rc || g->n_rows == 0) return rc;
    const unsigned grid = gat_grid(g->n_rows);
    cudaStream_t st = as_stream(stream);
    BNS_TCONV_DISPATCH(gatv2_nv((int64_t)H * Fp), (tconv_infer_kernel<NV><<<grid, kThreads, 0, st>>>(a)));
    ++g_launches;
    BNS_CUDA(cudaGetLastError());
    return BNS_OK;
}

extern "C" int bns_tconv_infer_block_f32(const bns_graph_t *g, const float *q, int64_t ldq, const float *k,
                                         int64_t ldk, const float *v, int64_t ldv, int32_t H, int32_t Fp, float scale,
                                         float *m, float *l, float *acc, int64_t ldacc, int first, int last, float *rst,
                                         int64_t ldr, void *stream) {
    TconvInferBlockArgs a{};
    int rc = tconv_infer_fill(a, g, q, ldq, k, ldk, v, ldv, H, Fp, scale, rst, ldr, last != 0,
                              "bns_tconv_infer_block_f32");
    if (rc || g->n_rows == 0) return rc;
    const int64_t HF = (int64_t)H * Fp;
    BNS_REQUIRE(m && l && acc, "bns_tconv_infer_block_f32: NULL pointer");
    BNS_REQUIRE(ldacc % 4 == 0 && ldacc >= HF && gatv2_aligned(acc), "bns_tconv_infer_block_f32: 16-byte aligned rows required");
    BNS_REQUIRE(!last || rst != acc || ldr == ldacc, "bns_tconv_infer_block_f32: rst aliases acc with a different stride");
    a.sm = m; a.sl = l; a.sacc = acc; a.ldacc = ldacc; a.first = first ? 1 : 0; a.last = last ? 1 : 0;
    const unsigned grid = gat_grid(g->n_rows);
    cudaStream_t st = as_stream(stream);
    BNS_TCONV_DISPATCH(gatv2_nv(HF), (tconv_infer_kernel<NV, true><<<grid, kThreads, 0, st>>>(a)));
    ++g_launches;
    BNS_CUDA(cudaGetLastError());
    return BNS_OK;
}

#undef BNS_TCONV_DISPATCH
