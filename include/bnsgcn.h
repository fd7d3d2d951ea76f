/*
 * bnsgcn.h -- C ABI of libbnsgcn.so: the H100 (sm_90a) replacement for the device work the
 * BNS-GCN hot path reaches through DGL / ATen / numpy (SURVEY.md §2.3 K1-K7, §8b).
 *
 * The reference (GATECH-EIC/BNS-GCN, 100 % Python) has no FFI layer of its own: its "operator API"
 * is the set of Python call sites cited beside each entry point below (paths relative to the
 * reference root).  INTEGRATION.md shows the ctypes stub a maintainer would add at each of them.
 *
 * Conventions
 *   - plain C symbols, plain pointers and sizes; no torch / C++ types cross this boundary;
 *   - every pointer marked "device" is a CUDA device pointer owned by the caller (PyTorch owns the
 *     tensors; the library never frees or reallocates caller memory);
 *   - `stream` is a cudaStream_t passed as void*; all work is enqueued on it, nothing synchronises
 *     the host except bns_graph_create / bns_graph_transpose (setup) and where stated;
 *   - return value: 0 = ok, negative = error (BNS_E_*); bns_last_error() gives the message of the
 *     calling thread's most recent failure;
 *   - after *_create the library allocates nothing: scratch space is passed in (`ws`, sized by the
 *     matching *_workspace_bytes query);
 *   - thread-compatible: distinct handles may be used from distinct threads concurrently.
 *   - feature matrices are row-major f32; graph ids int32 on device (train.py:71-73 uses int32
 *     graphs), row offsets int64, exchanged index lists int64 (train.py:233-234, utils.py:171).
 */
#ifndef BNSGCN_H_
#define BNSGCN_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BNS_OK            0
#define BNS_E_INVALID    (-1)   /* bad argument (null pointer, negative size, misaligned leading dim) */
#define BNS_E_CUDA       (-2)   /* a CUDA runtime call failed; message holds cudaGetErrorString */
#define BNS_E_WORKSPACE  (-3)   /* workspace too small */
#define BNS_E_UNSUPPORTED (-4)

#define BNS_ABI_VERSION 15

typedef struct bns_graph bns_graph_t;   /* opaque: a static CSR matrix resident in HBM */
typedef struct bns_p2p   bns_p2p_t;     /* opaque: peer-mapped exchange slabs of one rank */
typedef struct bns_ctx   bns_ctx_t;     /* opaque: one rank's communicator (NCCL) */

int         bns_abi_version(void);
const char *bns_last_error(void);
/* Number of kernels of this library enqueued so far by this process (bench.py reports the delta as gpu_launches). */
uint64_t    bns_launch_count(void);
/* Name, SM count, L2 bytes of the current device (for bench.py's grid / roofline bookkeeping). */
int         bns_device_info(char *name, size_t name_len, int *sm_count, int64_t *l2_bytes, int *cc_major, int *cc_minor);

/* ------------------------------------------------------------------------------------------------
 * Static graphs.  Replaces the per-epoch dgl.heterograph rebuild of train.py:256-281
 * (construct_graph) and DGL's lazy COO->CSR/CSC conversion: a graph is built ONCE, per-epoch
 * sampling only changes the small `col_map` / `row_map` arrays given to bns_spmm_sum_f32.
 *
 * bns_graph_create copies a device CSR (row r's entries are indices[indptr[r] .. indptr[r+1])) and
 * precomputes the nnz-balanced work decomposition (rows are cut into chunks of <= chunk_nnz
 * entries; rows longer than a chunk are combined by a deterministic second pass).
 *   n_rows, n_cols : matrix shape; every index must lie in [0, n_cols)
 *   chunk_nnz      : 0 = library default
 * ----------------------------------------------------------------------------------------------*/
int bns_graph_create(bns_graph_t **out, int64_t n_rows, int64_t n_cols, int64_t nnz,
                     const int64_t *indptr /*device [n_rows+1]*/, const int32_t *indices /*device [nnz]*/,
                     int32_t chunk_nnz, void *stream);
/* CSR of the reversed graph (what autograd needs for K1b, SURVEY §2.3): out[c] lists the rows r with
 * (r, c) in g, ascending.  Built once, on the device (radix sort). */
int bns_graph_transpose(const bns_graph_t *g, bns_graph_t **out, void *stream);
int bns_graph_destroy(bns_graph_t *g);
int bns_graph_info(const bns_graph_t *g, int64_t *n_rows, int64_t *n_cols, int64_t *nnz,
                   int64_t *n_chunks, int64_t *n_split_rows);
/* For a graph made by bns_graph_transpose: perm_out[k] (device [nnz]) = index, in the SOURCE graph's CSR order, of
 * the entry that became entry k of the transpose -- carries per-entry weights across (w_T[k] = w[perm[k]]). */
int bns_graph_copy_perm(const bns_graph_t *gT, int32_t *perm_out, void *stream);
/* Copy the library-owned CSR into caller buffers (device [n_rows+1] / [nnz]); for tests and tools. */
int bns_graph_copy_csr(const bns_graph_t *g, int64_t *indptr_out, int32_t *indices_out, void *stream);

/* ------------------------------------------------------------------------------------------------
 * K1 / K1b / K2: the aggregation.  Replaces
 *     graph['_E'].update_all(fn.copy_u('h','m'), fn.sum('m','h'))        module/layer.py:35-37, 88-90
 *     ... / degs, feat / out_norm, ... / in_norm                         module/layer.py:34, 38, 91
 * and their autograd transposes, with
 *     Y[orow(r), :] = (accumulate ? Y[orow(r), :] : 0)
 *                     + row_scale[r] * sum_{k in row r, xrow(c_k) >= 0} col_scale[c_k] * X[xrow(c_k), :]
 *   xrow(c) = c                       if c <  n_direct
 *           = col_map[c - n_direct]   otherwise (-1 = entry skipped: an unsampled halo node)
 *   orow(r) = r  if row_map == NULL, else row_map[r]  (-1 = row skipped)
 * row_scale / col_scale / row_map / col_map may be NULL (= 1 / identity; col_map == NULL means
 * n_direct = n_cols).  All f32; summation order inside a row is the CSR order (deterministic).
 *   X  [*, F] with leading dimension ldx (floats); Y [*, F] with ldy.
 * The 16-byte vector path needs F % 4 == 0, ldx % 4 == 0, ldy % 4 == 0 and 16-byte aligned X, Y;
 * anything else takes the scalar path (same results).
 * ws: scratch of at least bns_spmm_workspace_bytes(g, F) bytes (0 when no row is split).
 * L2 blocking: the feature dimension is processed in column slabs (256/128/64/32 floats) picked so that
 * x_rows * slab * 4 bytes stays resident in L2 (override: slab_hint, or env BNS_SPMM_SLAB).
 * ----------------------------------------------------------------------------------------------*/
size_t bns_spmm_workspace_bytes(const bns_graph_t *g, int64_t F);
int bns_spmm_sum_f32(const bns_graph_t *g,
                     const float *X, int64_t ldx, int64_t F,
                     float *Y, int64_t ldy,
                     const float *row_scale /*device [n_rows] or NULL*/,
                     const float *col_scale /*device [n_cols] or NULL*/,
                     const float *edge_weight /*device [nnz], CSR order, or NULL: multiplies entry k's source row
                                                (GAT attention, u_mul_e + sum of dgl.nn.GATConv)*/,
                     const int32_t *row_map /*device [n_rows] or NULL*/,
                     const int32_t *col_map /*device [n_cols - n_direct] or NULL*/, int64_t n_direct,
                     int64_t x_rows /*rows of X that can be referenced (0 = n_cols); sizes the L2 blocking*/,
                     int32_t slab_hint /*0 = automatic; 256 | 128 | 64 | 32 forces the column-slab width*/,
                     int accumulate, void *ws, size_t ws_bytes, void *stream);

/* ------------------------------------------------------------------------------------------------
 * K8 helper (dense layers): split n contiguous f32 values into three bf16 arrays with x = b0 + b1 + b2 exact to
 * 24 mantissa bits (round-to-nearest-even at each step).  Six bf16 tensor-core GEMMs b_i * w_j (i + j <= 2) with f32
 * accumulation then reproduce the f32 product to ~2^-23 (module/dense.py, mode "bf16x3").  n % 4 == 0.
 * ----------------------------------------------------------------------------------------------*/
int bns_split_bf16x3_f32(const float *x, int64_t n, void *out0 /*bf16 [n]*/, void *out1, void *out2, void *stream);
/* Same idea with TF32 (module/dense.py "3xtf32"): hi = x rounded to 10 mantissa bits, lo = x - hi (exact);
 * hi*hi + hi*lo + lo*hi in three TF32 tensor-core GEMMs with f32 accumulation is f32-accurate to ~2^-21. */
int bns_split_tf32_f32(const float *x, int64_t n, float *hi, float *lo, void *stream);

/* ------------------------------------------------------------------------------------------------
 * K8: the dense layers themselves.  Replaces, for 2-D f32 operands,
 *     self.linear(feat) / self.linear1(feat) + self.linear2(ah)      module/layer.py:30, 38, 83, 92  (forward)
 * and what autograd runs for them (grad_input = dY W, grad_weight = dY^T X) with hand-written wgmma kernels:
 * .tf32 wgmma.mma_async accumulating in registers, operands staged by TMA (SWIZZLE_128B), and the 3xTF32 operand split
 * (hi = x truncated to tf32, lo = x - hi; hi*hi + hi*lo + lo*hi) done in shared memory inside the pipeline, so the result is
 * f32-accurate (~2^-21 relative per product) while every operand byte crosses HBM/L2 once (csrc/dense_tc.cuh).
 *
 * bns_dense_tn_3xtf32:  C[M, N] = A[M, K] * B[N, K]^T (+ bias[N]) (+ addend[M, N]);  A, B, C row-major with leading
 *   dimensions lda, ldb, ldc (floats).  Forward: A = X, B = weight; `addend` fuses the "+" of
 *   linear1(feat) + linear2(ah) (module/layer.py:92) into the epilogue.  Input gradient: A = dY, B = weight^T (a
 *   contiguous copy).
 * bns_dense_nt_3xtf32:  C[N1, N2] = A[R, N1]^T * B[R, N2]  (contraction over the R rows, split across CTAs and
 *   combined in split order -- deterministic).  Weight gradient: A = dY, B = X.  ws: at least
 *   bns_dense_nt_workspace_bytes(R, N1, N2) bytes.
 * All pointers 16-byte aligned, leading dimensions multiples of 4 (and N2 % 4 == 0); anything else returns
 * BNS_E_INVALID and the caller uses the library GEMM.
 * ----------------------------------------------------------------------------------------------*/
int    bns_dense_tn_3xtf32(const float *A, int64_t lda, const float *B, int64_t ldb, const float *bias /*device [N] or NULL*/,
                           const float *addend /*device [M, N] with leading dimension ldadd, or NULL; may alias C*/, int64_t ldadd,
                           const float *row_scale /*device [M] or NULL: C[r, :] = (A B^T + bias + addend)[r, :] * row_scale[r]
                                                    (the 1/deg pre-scale of the aggregation's backward, module/layer.py:91)*/,
                           float *C, int64_t ldc, int64_t M, int64_t N, int64_t K, void *stream);
size_t bns_dense_nt_workspace_bytes(int64_t R, int64_t N1, int64_t N2);
int    bns_dense_nt_3xtf32(const float *A, int64_t lda, const float *B, int64_t ldb, float *C, int64_t ldc,
                           int64_t R, int64_t N1, int64_t N2, void *ws, size_t ws_bytes, void *stream);
/* Bias gradient of the same layers (autograd's dY.sum(0)): out[c] = sum_r X[r, c], two deterministic passes.
 * cols % 4 == 0, cols <= 1024, ld % 4 == 0, 16-byte aligned; ws >= bns_colsum_workspace_bytes(cols). */
size_t bns_colsum_workspace_bytes(int64_t cols);
int    bns_colsum_f32(const float *X, int64_t ld, int64_t rows, int64_t cols, float *out,
                      float *out2 /*optional second destination (linear1.bias and linear2.bias share dY.sum(0))*/, void *ws,
                      size_t ws_bytes, void *stream);

/* ------------------------------------------------------------------------------------------------
 * K10 (GAT, module/model.py:96-132 via dgl.nn.GATConv): the attention gradient.  For every entry k of row r:
 *     out[k * ldo] = < A[arow(r), :F], B[xrow(c_k), :F] >      (0 when the row or the entry is skipped)
 * arow / xrow as in bns_spmm_sum_f32 (row_map / col_map / n_direct).  F % 4 == 0, F <= 1024, 16-byte aligned rows.
 * With bns_spmm_sum_f32(edge_weight) and the transpose permutation this is all GATConv needs besides elementwise
 * work on per-entry vectors: forward  rst = A_w ft,  backward  d ft = A_w^T d rst,  d w = sddmm(d rst, ft).
 * ----------------------------------------------------------------------------------------------*/
int bns_sddmm_dot_f32(const bns_graph_t *g, const float *A, int64_t lda, const float *B, int64_t ldb, int64_t F,
                      const int32_t *row_map, const int32_t *col_map, int64_t n_direct, float *out, int64_t ldo,
                      void *stream);

/* ------------------------------------------------------------------------------------------------
 * K3 / K4 / K5: boundary pack / concat / scatter.  helper/feature_buffer.py:
 *   :117  send_cpu[right].copy_(send_gpu[self._selected[right]] / self._ratio[right])
 *   :85-91 __feat_concat  (cat([feat, recv_0, ...]))
 *   :129  send_gpu[self._selected[idx]] += recv / self._ratio[idx]
 * out[i, :] = H[idx[i], :] / div        (true division, as the reference)
 * G[idx[i], :] += src[i, :] / div       (idx must not repeat inside one call; calls on one stream
 *                                         are ordered, which is how the reference orders peers)
 * ----------------------------------------------------------------------------------------------*/
int bns_gather_div_f32(const float *H, int64_t ldh, int64_t F, const int64_t *idx /*device [k]*/, int64_t k,
                       float div, float *out, int64_t ldo, void *stream);
int bns_scatter_add_div_f32(float *G, int64_t ldg, int64_t F, const int64_t *idx /*device [k]*/, int64_t k,
                            float div, const float *src, int64_t lds, void *stream);
/* dst[r, :F] = src[r, :F] for r < n_rows (the "inner" block of the concat buffer). */
int bns_copy_rows_f32(const float *src, int64_t lds, float *dst, int64_t ldd, int64_t n_rows, int64_t F, void *stream);

/* ------------------------------------------------------------------------------------------------
 * K6: boundary-node sampling.  Replaces train.py:225-236 (select_node):
 *     idx = np.random.choice(b.shape[0], send_size[i], replace=False);  selected = boundary[i][idx]
 * i.e. a uniformly random ORDERED k-subset per peer.  All peers are drawn by one call:
 *   boundary_cat : the sorted boundary lists of the n_seg peers, concatenated (device, int64 [B])
 *   seg_begin    : device int64 [n_seg+1], boundary list s is boundary_cat[seg_begin[s] .. seg_begin[s+1])
 *   out_begin    : device int64 [n_seg+1], prefix sums of the sample sizes k_s (k_s <= b_s)
 *   selected     : device int64 [K_total], peer s's sample is selected[out_begin[s] .. out_begin[s+1])
 * Element i of boundary_cat gets the key  (s << 56) | r56(i),  r56 = the top 56 bits of
 * Philox4x32-10(counter = (i_lo, i_hi, offset_lo, offset_hi), key = (seed_lo, seed_hi)) words 0,1;
 * a stable radix sort orders each segment by key and the first k_s entries are the sample.
 * Counter-based => reproducible: the oracle replays it bit for bit (oracle/philox.py).
 * ----------------------------------------------------------------------------------------------*/
size_t bns_sample_workspace_bytes(int64_t B);
int bns_sample_boundary(const int64_t *boundary_cat, const int64_t *seg_begin, const int64_t *out_begin,
                        int32_t n_seg, int64_t B, int64_t K_total, uint64_t seed, uint64_t offset,
                        const uint64_t *offset_dev /*device, optional: added to `offset` at run time, so that a
                                                     captured CUDA graph draws a new sample on every replay*/,
                        int64_t *selected, void *ws, size_t ws_bytes, void *stream);

/* ------------------------------------------------------------------------------------------------
 * K7: per-epoch graph "rebuild".  Replaces train.py:256-281 (construct_graph) and 245-253
 * (construct_out_norm): instead of building a new heterograph, record where each sampled halo node's
 * row lives in the receive slab:
 *     slot[pos[one_hops[k]] - n_in] = slab_offset + k        k = 0 .. r-1
 * (`pos` = get_pos() of train.py:90-104: owner-local id -> my local node id, -1 if not my halo).
 * Call bns_fill_i32(slot, n_halo, -1) first, then once per peer.
 * ----------------------------------------------------------------------------------------------*/
int bns_fill_i32(int32_t *dst, int64_t n, int32_t value, void *stream);
int bns_halo_slot_update(const int64_t *pos /*device [part size of the peer]*/, const int64_t *one_hops /*device [r]*/,
                         int64_t r, int64_t n_in, int32_t slab_offset, int32_t *slot /*device [n_halo]*/, void *stream);

/* ------------------------------------------------------------------------------------------------
 * K9 (fused): LayerNorm -> ReLU -> dropout between two layers.  Replaces the three ATen ops of
 * module/model.py:88-91 (`h = self.norm[i](h); h = self.activation(h)`) and :45/:80 of the next iteration
 * (`h = self.dropout(h)`), forward and backward, in one pass each:
 *     y = dropout_p( relu( (x - mean) * rstd * gamma + beta ) )        mean / biased var over the F columns
 * The dropout mask is Philox4x32-10(counter = (row, vector, offset), key = seed) -- regenerated, not stored, in
 * backward; offset_dev (optional, device) is added to offset at run time (CUDA-graph replays).  F % 4 == 0,
 * F <= 1024, 0 <= p < 1, leading dimensions >= F and multiples of 4, x / y / dy / dx / gamma / beta 16-byte
 * aligned (they are read and written as float4).  Backward also returns dgamma / dbeta (column sums, fixed summation order: deterministic);
 * ws: bns_ln_bwd_workspace_bytes(F) bytes.
 * ----------------------------------------------------------------------------------------------*/
size_t bns_ln_bwd_workspace_bytes(int64_t F);
int bns_ln_relu_dropout_fwd_f32(const float *x, int64_t ldx, int64_t n, int64_t F, const float *gamma,
                                const float *beta, float eps, float p, uint64_t seed, uint64_t offset,
                                const uint64_t *offset_dev, float *y, int64_t ldy, float *mean /*[n]*/,
                                float *rstd /*[n]*/, void *stream);
int bns_ln_relu_dropout_bwd_f32(const float *dy, int64_t lddy, const float *x, int64_t ldx, int64_t n, int64_t F,
                                const float *gamma, const float *beta, const float *mean, const float *rstd,
                                float eps, float p, uint64_t seed, uint64_t offset, const uint64_t *offset_dev,
                                float *dx, int64_t lddx, float *dgamma /*[F]*/, float *dbeta /*[F]*/, void *ws,
                                size_t ws_bytes, void *stream);

/* ------------------------------------------------------------------------------------------------
 * C1/C2 fused with K3/K5: the boundary exchange over peer-mapped memory (NVLink 5 / NVSwitch).
 * Replaces Buffer.__gloo_all_to_all / __mpi_all_to_all (helper/feature_buffer.py:101-153): the pack
 * kernel of rank a stores  H[selected_b] / ratio_b  straight into rank b's receive slab, then raises a
 * flag in b's memory; b's stream waits on the flag.  No staging buffer, no host round trip.
 * One bns_p2p_t per rank; slabs are cudaMalloc'd by the library so that they can be exported with
 * cudaIpcGetMemHandle (processes) or shared by pointer (ranks that are threads of one process).
 * ----------------------------------------------------------------------------------------------*/
#define BNS_P2P_HANDLE_BYTES 64
int bns_p2p_create(bns_p2p_t **out, int32_t rank, int32_t world, size_t slab_bytes, int32_t n_flags);
int bns_p2p_destroy(bns_p2p_t *p);
/* base of this rank's slab / flag block (device pointers, valid in this process) */
int bns_p2p_local(const bns_p2p_t *p, void **slab, void **flags, size_t *slab_bytes);
/* IPC export / import (multi-process).  handle_out: BNS_P2P_HANDLE_BYTES bytes for the slab followed by
 * BNS_P2P_HANDLE_BYTES bytes for the flags. */
int bns_p2p_export(const bns_p2p_t *p, void *handle_out /*2*BNS_P2P_HANDLE_BYTES*/);
int bns_p2p_import(bns_p2p_t *p, int32_t peer, const void *handle /*2*BNS_P2P_HANDLE_BYTES*/, size_t peer_slab_bytes);
/* In-process peers (threads): register the peer's pointers directly. */
int bns_p2p_set_peer(bns_p2p_t *p, int32_t peer, void *slab, void *flags, size_t peer_slab_bytes);
/* remote_rows[i, :F] (in peer's slab at byte offset remote_off, leading dim ld_remote floats)
 *     = H[idx[i], :F] / div   for i < k   (idx == NULL: rows i of H, used for the gradient return trip);
 * then, after a system-scope fence, peer.flags[flag_index] = flag_value (release). */
int bns_p2p_put_rows_f32(bns_p2p_t *p, int32_t peer, size_t remote_off, int64_t ld_remote,
                         const float *H, int64_t ldh, int64_t F, const int64_t *idx, int64_t k, float div,
                         int32_t flag_index, uint64_t flag_value,
                         const uint64_t *flag_value_dev /*device, optional: added to flag_value at run time (graph replays)*/,
                         void *stream);
/* Enqueue a wait on `stream` until this rank's flags[flag_index] >= flag_value (acquire).  The spin is bounded
 * (20 s): a peer that never signals traps the kernel (a loud CUDA error) instead of hanging the device. */
int bns_p2p_wait_flag(bns_p2p_t *p, int32_t flag_index, uint64_t flag_value, const uint64_t *flag_value_dev,
                      void *stream);


/* ================================================================================================
 * ABI 2: the rest of the epoch (train.py:385-425) as ONE launch per step instead of one per peer / per parameter /
 * per ATen op.  At 8 partitions the round-1 epoch spent ~59 % of its time in such launches.
 * ================================================================================================*/
#define BNS_MAX_PEERS 16

/* ------------------------------------------------------------------------------------------------
 * K7': slot map of ALL peers + the inverse maps the gradient scatter walks, one memset + one kernel.  Replaces the
 * per-peer loop of train.py:256-281 (construct_graph) done by bns_fill_i32 + bns_halo_slot_update x (P-1):
 *     slot[pos_s[one_hops_cat[k]] - n_in] = k                         k over the concatenated received id lists
 *     inv_s[selected_cat[i]] = i - sel_begin[s]                       i over the concatenated sampled id lists
 * Segments = the peers in ascending order, self skipped.  [fill_base, +fill_bytes) -- the allocation that holds `slot`
 * and every inv_s -- is set to -1 first.
 * ----------------------------------------------------------------------------------------------*/
typedef struct bns_epoch_maps {
    int32_t n_seg;
    int64_t sel_begin[BNS_MAX_PEERS + 1];
    int64_t hop_begin[BNS_MAX_PEERS + 1];
    const int64_t *pos[BNS_MAX_PEERS];      /* device: get_pos() of train.py:90-104 */
    int32_t *inv[BNS_MAX_PEERS];            /* device [n_in] each, may be NULL */
    const int64_t *selected_cat, *one_hops_cat;
    int32_t *slot;                          /* device [n_halo] */
    int64_t n_in;
} bns_epoch_maps;
int bns_epoch_maps_update(const bns_epoch_maps *maps /*host*/, void *fill_base, size_t fill_bytes, void *stream);

/* ------------------------------------------------------------------------------------------------
 * K1 on the SAMPLED halo only.  bns_graph_compact_cols rewrites, once per epoch, the column ids of a column-mapped
 * matrix (A_out with col_map = slot): chunk by chunk, the entries whose column is sampled are moved -- already mapped to
 * rows of X, CSR order kept -- to the front of the chunk's own index range in `cidx`, their number goes to
 * `chunk_cnt`; bns_spmm_compact_f32 then runs the plain kernel over exactly those entries.  Same numbers added in the
 * same order as bns_spmm_sum_f32(col_map): bit-identical results, work proportional to the sample
 * (train.py:256-281 builds the sampled graph per epoch for the same reason).
 * ----------------------------------------------------------------------------------------------*/
int bns_graph_compact_cols(const bns_graph_t *g, const int32_t *col_map, int64_t n_direct,
                           const float *col_scale /*device [n_cols] or NULL: gathered per live entry into cw*/,
                           int32_t *cidx /*device [nnz]*/, float *cw /*device [nnz] or NULL*/,
                           int32_t *cpos /*device [nnz] or NULL: position of each live entry in the CSR (GAT keeps its
                                           per-entry attention at those positions)*/,
                           int32_t *chunk_cnt /*device [n_chunks]*/, void *stream);
int bns_spmm_compact_f32(const bns_graph_t *g, const int32_t *cidx, const float *cw /*per compacted entry, or NULL*/,
                         int64_t cw_ld /*stride of cw in floats (1; heads for GAT's [nnz, heads] attention)*/,
                         const int32_t *chunk_cnt, const float *X, int64_t ldx, int64_t F, float *Y, int64_t ldy,
                         const float *row_scale, int64_t x_rows, int32_t slab_hint, int accumulate, void *ws, size_t ws_bytes,
                         void *stream);

/* ------------------------------------------------------------------------------------------------
 * ABI 4: BF16 gather tables (--agg-dtype bf16).  bns_spmm_sum_bf16 / bns_spmm_compact_bf16 are bns_spmm_sum_f32 /
 * bns_spmm_compact_f32 with X stored as bf16 bit patterns (ldx in elements): every other operand, the accumulation
 * (f32, same entry order) and Y stay f32.  X is read as 16-byte vectors of 8 elements: F % 8 == 0, ldx % 8 == 0,
 * ldy % 4 == 0 and 16-byte aligned X, Y, else BNS_E_INVALID (there is no scalar path).  The column slab is sized from
 * x_rows * slab * 2 bytes; the workspace is the f32 one (bns_spmm_workspace_bytes).
 * bns_cvt_rows_f32_bf16: dst[r, :F] = bf16(src[r, :F]), round to nearest even (NaN stays NaN, subnormals are kept).
 * ----------------------------------------------------------------------------------------------*/
int bns_spmm_sum_bf16(const bns_graph_t *g, const uint16_t *X /*bf16*/, int64_t ldx, int64_t F, float *Y, int64_t ldy,
                      const float *row_scale, const float *col_scale, const float *edge_weight, const int32_t *row_map,
                      const int32_t *col_map, int64_t n_direct, int64_t x_rows, int32_t slab_hint, int accumulate, void *ws,
                      size_t ws_bytes, void *stream);
int bns_spmm_compact_bf16(const bns_graph_t *g, const int32_t *cidx, const float *cw, int64_t cw_ld, const int32_t *chunk_cnt,
                          const uint16_t *X /*bf16*/, int64_t ldx, int64_t F, float *Y, int64_t ldy, const float *row_scale,
                          int64_t x_rows, int32_t slab_hint, int accumulate, void *ws, size_t ws_bytes, void *stream);
int bns_cvt_rows_f32_bf16(const float *src, int64_t lds, uint16_t *dst /*bf16*/, int64_t ldd, int64_t n_rows, int64_t F,
                          void *stream);

/* ------------------------------------------------------------------------------------------------
 * ABI 7: FP8 gather tables (--agg-dtype fp8).  A table is e4m3 codes X [rows, F] (ldx in bytes) plus one f32 power-of-two
 * scale per row, x_scale [rows]; row r stands for x_scale[r] * e4m3(X[r, :]).  bns_spmm_sum_fp8 / bns_spmm_compact_fp8
 * are bns_spmm_sum_f32 / bns_spmm_compact_f32 over such a table: entry k adds w_k * x_scale[xrow(c_k)] * X[xrow(c_k)]
 * (codes widened exactly, f32 FMA, same entry order), where w_k is the f32 column scale / per-entry weight (or 1) and the
 * scale is indexed by the row of X the entry gathers (after col_map / compaction).  X is read as 16-byte vectors of 16
 * codes: F % 16 == 0, ldx % 16 == 0, ldy % 4 == 0 and 16-byte aligned X, Y, else BNS_E_INVALID.  The column slab is
 * sized from x_rows * slab * 1 byte; the workspace is the f32 one (bns_spmm_workspace_bytes).
 * bns_cvt_rows_f32_fp8: with m = max |src[r, :F]|, scale[r] = 2^e for the smallest integer e >= -126 with
 * m * 2^-e <= 448 (1 when m == 0), codes[r, c] = e4m3(src[r, c] * 2^-e) rounded to nearest even (the product is exact
 * and never saturates; subnormal codes are kept).  A row holding NaN or +-Inf gets scale NaN and all-zero codes, so
 * every sum that gathers it is NaN.  Needs F % 16 == 0, ldc % 16 == 0, lds % 4 == 0 and 16-byte aligned src, codes.
 * ----------------------------------------------------------------------------------------------*/
int bns_spmm_sum_fp8(const bns_graph_t *g, const uint8_t *X /*e4m3*/, const float *x_scale, int64_t ldx, int64_t F,
                     float *Y, int64_t ldy, const float *row_scale, const float *col_scale, const float *edge_weight,
                     const int32_t *row_map, const int32_t *col_map, int64_t n_direct, int64_t x_rows, int32_t slab_hint,
                     int accumulate, void *ws, size_t ws_bytes, void *stream);
int bns_spmm_compact_fp8(const bns_graph_t *g, const int32_t *cidx, const float *cw, int64_t cw_ld, const int32_t *chunk_cnt,
                         const uint8_t *X /*e4m3*/, const float *x_scale, int64_t ldx, int64_t F, float *Y, int64_t ldy,
                         const float *row_scale, int64_t x_rows, int32_t slab_hint, int accumulate, void *ws,
                         size_t ws_bytes, void *stream);
int bns_cvt_rows_f32_fp8(const float *src, int64_t lds, uint8_t *codes /*e4m3*/, int64_t ldc, float *scale, int64_t n_rows,
                         int64_t F, void *stream);

/* ------------------------------------------------------------------------------------------------
 * K10 fused: the attention of dgl.nn.GATConv (module/model.py:96-132; DGL 0.9 python/dgl/nn/pytorch/conv/gatconv.py):
 *     e_uv = leaky_relu(el_u + er_v);  p = edge_softmax(e) over each destination's in-entries;  a = attn_drop(p);
 *     rst_v = sum_u a_uv ft_u                     for all `heads` at once.
 * The entries of row v are those of a_in followed by the SAMPLED ones of a_out (cidx / chunk_cnt / cpos from
 * bns_graph_compact_cols with col_map = slot, n_direct = 0; halo source k reads row x_halo_base + k of el / ft).
 *   el [n_u, heads], er [n_in, heads]; heads <= 8.  Dropout: Philox4x32-10(counter = (entry, head), key = seed,
 *   offset [+ *offset_dev]), regenerated in backward.
 * bns_gat_scores_f32, one warp per destination row, scalars only: the probabilities P_in [nnz(a_in), heads] /
 *   P_out [nnz(a_out), heads] and the dropped attention a = p * mask / (1 - q) W_in / W_out, stored at the ORIGINAL
 *   entry positions (P kept for the backward), W_out_compact [nnz(a_out), heads] at the compacted positions -- then
 *   bns_spmm_weighted_f32 / bns_spmm_compact_f32 per head make rst.
 * Backward: bns_sddmm_dot_f32 into dE (d a per entry), bns_gat_softmax_bwd_f32 (dE: d a -> d e in place, d er
 *   [n_in, heads]), bns_gat_colsum_f32 (on a_in_t, then on a_out_t with row_map = slot: d el_u = sum over column u of
 *   d e), and bns_spmm_weighted_f32: d ft = A^T d rst, one head per call, the attention read through the transpose's
 *   permutation.
 * ----------------------------------------------------------------------------------------------*/
int bns_gat_scores_f32(const bns_graph_t *a_in, const bns_graph_t *a_out, const int32_t *cidx, const int32_t *chunk_cnt,
                       const int32_t *cpos, int64_t x_halo_base, int32_t heads, const float *el, const float *er,
                       float negative_slope, float p_drop, uint64_t seed, uint64_t offset, const uint64_t *offset_dev,
                       float *P_in, float *P_out, float *W_in /*NULL when p_drop == 0*/, float *W_out, float *W_out_compact,
                       void *stream);
int bns_gat_softmax_bwd_f32(const bns_graph_t *a_in, const bns_graph_t *a_out, const int32_t *cidx, const int32_t *chunk_cnt,
                            const int32_t *cpos, int64_t x_halo_base, int32_t heads, const float *el, const float *er,
                            float negative_slope, float p_drop, uint64_t seed, uint64_t offset, const uint64_t *offset_dev,
                            const float *P_in, const float *P_out, float *dE_in, float *dE_out, float *d_er, void *stream);
/* el / er of GATConv (module/model.py:102; DGL 0.9 gatconv.py: el = (feat_src * attn_l).sum(-1), er likewise): out[r, h] = <X[r, h*Fo:(h+1)*Fo], attn[h, :]>, and its backward: dX[r, h, :] (+)= s[r, h] * attn[h, :],
 * d_attn[h, :] = sum_r s[r, h] * X[r, h, :] (deterministic).  ws: bns_colsum_workspace_bytes(heads * Fo). */
int bns_gat_proj_f32(const float *X, int64_t ldx, int64_t rows, int32_t heads, int32_t Fo, const float *attn, float *out,
                     void *stream);
int bns_gat_proj_bwd_f32(const float *X, int64_t ldx, int64_t rows, int32_t heads, int32_t Fo, const float *attn,
                         const float *s, float *dX, int64_t lddx, int accumulate, float *d_attn, void *ws, size_t ws_bytes,
                         void *stream);
int bns_gat_colsum_f32(const bns_graph_t *gT, const float *dE, int32_t heads, const int32_t *row_map, int64_t out_base,
                       float *d_el, void *stream);
/* The evaluation forward of GATConv on a homogeneous graph g (CSR by destination; DGL 0.9 gatconv.py with
 * h_src = h_dst, no dropout):
 *     rst[v, h, :] = sum_{u -> v} softmax_u(leaky_relu(el[u, h] + er[v, h])) * ft[u, h, :] + bias[h, :]
 * in ONE pass over each row (online softmax: running maximum and sum rescaled per block of 32 entries), one warp per
 * destination row, nothing stored per entry.  ft [n_cols, heads, Fp] and rst [n_rows, heads, Fp] (rows ldft / ldr
 * floats apart, 16-byte aligned), Fp = the per-head width rounded up to a multiple of 4 with zero pad columns;
 * heads <= 8, heads * Fp <= 1024.  el [n_cols, heads], er [n_rows, heads], bias [heads * Fp] (16-byte aligned) or NULL.
 * A row without entries gets the bias alone.  Deterministic: the summation order is fixed per row. */
int bns_gat_infer_f32(const bns_graph_t *g, const float *ft, int64_t ldft, int32_t heads, int32_t Fp, const float *el,
                      const float *er, float negative_slope, const float *bias, float *rst, int64_t ldr, void *stream);
/* bns_gat_infer_f32 over destination rows whose in-entries come as several matrices with the same rows and different
 * columns (a partition's inner matrix, then one column block per peer's halo rows): one call per block, g / ft / el
 * that block's, er the rows' own.  The online-softmax state is carried between calls, per row and head:
 * m [n_rows, heads] running maximum, l [n_rows, heads] sum of exp, acc [n_rows, heads * Fp] (rows ldacc floats apart,
 * 16-byte aligned) the un-normalised weighted sum.  `first` starts from the empty state (m, l, acc need not be
 * initialised); otherwise the call reloads it and rescales it when the maximum grows.  `last` writes
 * rst = acc / l + bias (rst may be acc itself, with ldr == ldacc; ft / el may be NULL for a block without entries);
 * otherwise the state is
 * stored.  A row without entries in a block keeps its state; a row without entries in any block gets the bias alone.
 * Same limits as bns_gat_infer_f32.  Deterministic for a fixed block order. */
int bns_gat_infer_block_f32(const bns_graph_t *g, const float *ft, int64_t ldft, int32_t heads, int32_t Fp,
                            const float *el, const float *er, float negative_slope, float *m, float *l, float *acc,
                            int64_t ldacc, int first, int last, const float *bias, float *rst, int64_t ldr, void *stream);
int bns_spmm_weighted_f32(const bns_graph_t *g, const float *X, int64_t ldx, int64_t F, float *Y, int64_t ldy,
                          const float *weights, int64_t ldw, int perm_from_transpose, const int32_t *row_map, int64_t x_rows,
                          int accumulate, void *ws, size_t ws_bytes, void *stream);

/* ------------------------------------------------------------------------------------------------
 * C1/C2 + K3/K5 for ALL peers at once (helper/feature_buffer.py:101-129).
 * bns_p2p_put_all_f32: segment s sends rows [row_begin[s], row_begin[s+1]) of the concatenated send list to peer[s]:
 *     remote_s[i, :F] = H[idx_cat[row_begin[s] + i], :F] / div[s]      (idx_cat == NULL: H[src_begin[s] + i, :F])
 * into the peer's slab at byte offset remote_off[s] (a multiple of 4; rows of any F, the 16-byte path is taken when
 * every remote_off is a multiple of 16 and F, ldh, ld_remote are multiples of 4); after the last row of the LAUNCH
 * every peer's flags[flag_index] is set to flag_value (+ *flag_value_dev) with a system-scope release.
 * ticket_index < world + max(n_flags, 16) (n_flags of bns_p2p_create) picks the completion counter; launches that
 * share one must be stream-ordered.
 * bns_p2p_put_ids_i64: the same for the sampled id lists (data_transfer(..., tag=NODE), helper/utils.py:187-213).
 * bns_p2p_wait_all: one kernel that waits for n flags of this rank (bounded spin, 20 s -> trap).
 * bns_scatter_rows_all_f32: G[r, :] += recv_s[inv_s[r], :] / div[s] for every segment s IN ORDER and every row r with
 *     inv_s[r] >= 0 -- the P-1 scatter-adds of :129 in the reference's peer order, race-free in one launch.
 * ----------------------------------------------------------------------------------------------*/
typedef struct bns_put_all {
    int32_t n_seg;
    int64_t row_begin[BNS_MAX_PEERS + 1];
    int32_t peer[BNS_MAX_PEERS];
    uint64_t remote_off[BNS_MAX_PEERS];
    int64_t src_begin[BNS_MAX_PEERS];
    float div[BNS_MAX_PEERS];
} bns_put_all;
int bns_p2p_put_all_f32(bns_p2p_t *p, const bns_put_all *segs /*host*/, int64_t ld_remote, const float *H, int64_t ldh,
                        int64_t F, const int64_t *idx_cat, int32_t flag_index, int32_t ticket_index, uint64_t flag_value,
                        const uint64_t *flag_value_dev, void *stream);
int bns_p2p_put_ids_i64(bns_p2p_t *p, int32_t n_seg, const int64_t *begin /*host [n_seg+1]*/, const int32_t *peers /*host*/,
                        const uint64_t *remote_off /*host*/, const int64_t *ids_cat /*device*/, int32_t flag_index,
                        int32_t ticket_index, uint64_t flag_value, const uint64_t *flag_value_dev, void *stream);
int bns_p2p_wait_all(bns_p2p_t *p, int32_t n, const int32_t *flag_indices /*host*/, uint64_t flag_value,
                     const uint64_t *flag_value_dev, void *stream);
int bns_scatter_rows_all_f32(float *G, int64_t ldg, int64_t n_rows, int64_t F, int32_t n_seg,
                             const int32_t *const *inv /*host array of device pointers*/,
                             const float *const *recv /*host array of device pointers*/, int64_t ld_recv,
                             const float *div /*host*/, void *stream);

/* ------------------------------------------------------------------------------------------------
 * ABI 5: the boundary exchange with a bf16 wire side (--comm-dtype bf16).  Every division stays f32; the sender rounds
 * its quotient once to bf16 (nearest even, NaN stays NaN, subnormals kept: bns_cvt_rows_f32_bf16's rule) and the
 * receiver widens each row exactly before it divides and adds in f32.
 * bns_p2p_put_all_bf16: bns_p2p_put_all_f32 with the remote rows stored as bf16 (ld_remote in bf16 elements); same
 *     segments, flags and tickets.  F, ldh and ld_remote multiples of 8, H 16-byte aligned, every remote_off a multiple
 *     of 16, else BNS_E_INVALID (there is no scalar path).
 * bns_scatter_rows_all_bf16: bns_scatter_rows_all_f32 reading bf16 recv rows (ld_recv in elements), same order and
 *     same per-element arithmetic.  F % 8 == 0, ldg % 4 == 0, ld_recv % 8 == 0, 16-byte aligned G and recv rows.
 * bns_gather_div_bf16 / bns_scatter_add_div_bf16: bns_gather_div_f32 / bns_scatter_add_div_f32 (the staged transport's
 *     pack and scatter) with a bf16 out / src.  F and both leading dimensions multiples of 8, 16-byte aligned matrices.
 * bns_cvt_rows_bf16_f32: dst[r, :F] = (float)src[r, :F], exact.
 * ----------------------------------------------------------------------------------------------*/
int bns_p2p_put_all_bf16(bns_p2p_t *p, const bns_put_all *segs /*host*/, int64_t ld_remote, const float *H, int64_t ldh,
                         int64_t F, const int64_t *idx_cat, int32_t flag_index, int32_t ticket_index, uint64_t flag_value,
                         const uint64_t *flag_value_dev, void *stream);
int bns_scatter_rows_all_bf16(float *G, int64_t ldg, int64_t n_rows, int64_t F, int32_t n_seg,
                              const int32_t *const *inv /*host array of device pointers*/,
                              const uint16_t *const *recv /*host array of device pointers, bf16*/, int64_t ld_recv,
                              const float *div /*host*/, void *stream);
int bns_gather_div_bf16(const float *H, int64_t ldh, int64_t F, const int64_t *idx /*device [k]*/, int64_t k, float div,
                        uint16_t *out /*bf16*/, int64_t ldo, void *stream);
int bns_scatter_add_div_bf16(float *G, int64_t ldg, int64_t F, const int64_t *idx /*device [k]*/, int64_t k, float div,
                             const uint16_t *src /*bf16*/, int64_t lds, void *stream);
int bns_cvt_rows_bf16_f32(const uint16_t *src /*bf16*/, int64_t lds, float *dst, int64_t ldd, int64_t n_rows, int64_t F,
                          void *stream);

/* ------------------------------------------------------------------------------------------------
 * ABI 8: the boundary exchange with an fp8 wire side (--comm-dtype fp8).  Every row that crosses the wire is an ABI 7
 * fp8 row -- e4m3 codes plus one f32 power-of-two scale, by bns_cvt_rows_f32_fp8's rule -- made by the sender from the
 * f32 quotients H / div (m is the max of |H / div|, not of |H|).  The receiver's scatters add (code * scale) / div in
 * f32: the product is exact, so they are the f32 scatters over the dequantized rows, bit for bit.
 * bns_p2p_put_all_fp8: bns_p2p_put_all_f32 with the remote rows stored as fp8 rows, one warp per row: the codes at
 *     remote_off[s] (ld_remote bytes apart, as in bns_put_all) and the scales at scale_off[s] (host [n_seg], one float
 *     per row); same segments, idx_cat / src_begin modes, flags and tickets.  F <= 1024; F, ldh and ld_remote multiples
 *     of 16, H 16-byte aligned, every remote_off a multiple of 16 and every scale_off of 4, both ranges inside the
 *     peer's slab, else BNS_E_INVALID before anything launches.
 * bns_scatter_rows_all_fp8: bns_scatter_rows_all_f32 reading fp8 recv rows (ld_recv in bytes) with their scales
 *     recv_scale[s] (row k of segment s is scaled by recv_scale[s][k]); same order, same division.  F % 16 == 0,
 *     ldg % 4 == 0, ld_recv % 16 == 0, 16-byte aligned G and recv rows, 4-byte aligned scales.
 * bns_gather_div_fp8 / bns_scatter_add_div_fp8: bns_gather_div_f32 / bns_scatter_add_div_f32 (the staged transport's
 *     pack and scatter) with an fp8 out / src and its scales.  The pack: F <= 1024, F, ldh, ldo multiples of 16; the
 *     scatter: F, lds multiples of 16, ldg of 4; 16-byte aligned matrices and 4-byte aligned scales.
 * bns_cvt_rows_fp8_f32: dst[r, :F] = codes[r, :F] * scale[r], exact.  F, ldc multiples of 16, ldd of 4, 16-byte aligned
 *     codes and dst.
 * ----------------------------------------------------------------------------------------------*/
int bns_p2p_put_all_fp8(bns_p2p_t *p, const bns_put_all *segs /*host*/, const uint64_t *scale_off /*host [n_seg]*/,
                        int64_t ld_remote, const float *H, int64_t ldh, int64_t F, const int64_t *idx_cat,
                        int32_t flag_index, int32_t ticket_index, uint64_t flag_value, const uint64_t *flag_value_dev,
                        void *stream);
int bns_scatter_rows_all_fp8(float *G, int64_t ldg, int64_t n_rows, int64_t F, int32_t n_seg,
                             const int32_t *const *inv /*host array of device pointers*/,
                             const uint8_t *const *recv /*host array of device pointers, e4m3*/,
                             const float *const *recv_scale /*host array of device pointers*/, int64_t ld_recv,
                             const float *div /*host*/, void *stream);
int bns_gather_div_fp8(const float *H, int64_t ldh, int64_t F, const int64_t *idx /*device [k]*/, int64_t k, float div,
                       uint8_t *out /*e4m3*/, int64_t ldo, float *out_scale, void *stream);
int bns_scatter_add_div_fp8(float *G, int64_t ldg, int64_t F, const int64_t *idx /*device [k]*/, int64_t k, float div,
                            const uint8_t *src /*e4m3*/, int64_t lds, const float *src_scale, void *stream);
int bns_cvt_rows_fp8_f32(const uint8_t *codes /*e4m3*/, int64_t ldc, const float *scale, float *dst, int64_t ldd,
                         int64_t n_rows, int64_t F, void *stream);

/* ------------------------------------------------------------------------------------------------
 * ABI 6: the dense layers with bf16 tensor-core products (--dense-dtype bf16).  Same operands (f32 in HBM), shapes,
 * alignment rules, epilogue, split-K plan and workspace (bns_dense_nt_workspace_bytes) as bns_dense_tn_3xtf32 /
 * bns_dense_nt_3xtf32, and the same BNS_E_INVALID / BNS_E_WORKSPACE returns.  The kernels round each operand element
 * once to bf16 (nearest even; NaN stays NaN, +-Inf stays +-Inf) in shared memory and accumulate the products in f32:
 * C = bf16(A) bf16(B)^T (+ bias) (+ addend) (* row_scale), the epilogue in f32.  Not f32-accurate: for runs that have
 * opted out of the 1e-4 parity bar.
 * ----------------------------------------------------------------------------------------------*/
int bns_dense_tn_bf16(const float *A, int64_t lda, const float *B, int64_t ldb, const float *bias, const float *addend,
                      int64_t ldadd, const float *row_scale, float *C, int64_t ldc, int64_t M, int64_t N, int64_t K, void *stream);
int bns_dense_nt_bf16(const float *A, int64_t lda, const float *B, int64_t ldb, float *C, int64_t ldc, int64_t R, int64_t N1,
                      int64_t N2, void *ws, size_t ws_bytes, void *stream);

/* ------------------------------------------------------------------------------------------------
 * ABI 9: the dense layers' forward and input-gradient products on fp8 rows (--dense-dtype fp8).  Every operand is an
 * ABI 7 fp8 row: e4m3 codes plus one power-of-two f32 scale per row, by bns_cvt_rows_f32_fp8's rule.
 * bns_dense_tn_fp8: C[m, n] = (sum_k qa[m, k] qb[n, k]) * a_scale[m] * b_scale[n] (+ bias[n]) (+ addend[m, n])
 *     (* row_scale[m]), the epilogue in f32 in that order; addend may alias C.  The e4m3 wgmmas of each 128-code block
 *     start from zero and their sums are added in f32.  A [M, K] and B [N, K] code rows: lda, ldb in bytes, multiples of
 *     16, 16-byte aligned bases; K is any value >= 1 and the bytes between K and lda / ldb are never read.  Scales 4-byte
 *     aligned; bias, addend, C, ldc, ldadd as for bns_dense_tn_bf16, with the same BNS_E_INVALID returns before any
 *     launch.  A NaN scale (a row that held NaN or +-Inf) makes its own output row (a_scale) or column (b_scale) NaN.
 *     The scales are applied as (sum * a_scale[m]) * b_scale[n] in f32, so with extreme scales of opposite exponent
 *     (a row near 1e38 against one near 1e-30) the intermediate can overflow to +-Inf or lose bits to underflow even
 *     where the exact product is representable.
 * bns_cvt_rows_f32_fp8_any: bns_cvt_rows_f32_fp8 for rows of any width F % 4 == 0 (the codes between F and ldc are not
 *     written).  ldc % 16 == 0, lds % 4 == 0, 16-byte aligned src and codes, 4-byte aligned scale.
 * bns_dropout_fp8: bns_dropout_f32 (the same Philox mask, the same kept values bit for bit) that also stores each dropped
 *     row y[r, :F] as an fp8 row (codes with ldc bytes per row, a multiple of 16; scale[r]).  F % 4 == 0, 16-byte aligned
 *     x, y and codes.
 * ----------------------------------------------------------------------------------------------*/
int bns_dense_tn_fp8(const uint8_t *A /*e4m3*/, int64_t lda, const float *a_scale, const uint8_t *B /*e4m3*/, int64_t ldb,
                     const float *b_scale, const float *bias, const float *addend, int64_t ldadd, const float *row_scale,
                     float *C, int64_t ldc, int64_t M, int64_t N, int64_t K, void *stream);
int bns_cvt_rows_f32_fp8_any(const float *src, int64_t lds, uint8_t *codes /*e4m3*/, int64_t ldc, float *scale,
                             int64_t n_rows, int64_t F, void *stream);
int bns_dropout_fp8(const float *x, int64_t ldx, int64_t n, int64_t F, float p, uint64_t seed, uint64_t offset,
                    const uint64_t *offset_dev, float *y, int64_t ldy, uint8_t *codes /*e4m3*/, int64_t ldc, float *scale,
                    void *stream);

/* ------------------------------------------------------------------------------------------------
 * Loss and its gradient in one launch.  Replaces train.py:406-408 for the two losses of train.py:358-361:
 *     loss = CrossEntropyLoss(reduction='sum')(logits[train_mask], labels[train_mask])          (labels != NULL)
 *     loss = BCEWithLogitsLoss(reduction='sum')(logits[train_mask], labels[train_mask])        (labels_f != NULL)
 * dlogits[r, :n_class] = d loss / d logits[r, :] * grad_scale for train rows, 0 for the others and for the pad columns
 * [n_class, n_cols_out).  grad_scale = 1 / n_train folds helper/reducer.py:34 (grad /= n_train) into the source of
 * every gradient.  The loss is summed block by block in a fixed order (deterministic).  ws: bns_xent_workspace_bytes()
 * bytes, zeroed ONCE by the caller.
 * ----------------------------------------------------------------------------------------------*/
size_t bns_xent_workspace_bytes(void);
int bns_xent_f32(const float *logits, int64_t ld, int64_t n_rows, int32_t n_class, const int64_t *labels,
                 const float *labels_f, int64_t ldl, const uint8_t *mask /*device bool [n_rows] or NULL*/, float grad_scale,
                 float *loss_out /*device [1]*/, float *dlogits, int64_t ldd, int32_t n_cols_out, void *ws, size_t ws_bytes,
                 void *stream);

/* ------------------------------------------------------------------------------------------------
 * torch.optim.Adam (train.py:362, :413) over ONE flat parameter arena: every parameter, its gradient and both moments
 * live at the same offsets of four flat buffers, so the step is one launch (torch: ~15 multi-tensor launches).
 *     g += weight_decay * p;  m += (1 - b1) (g - m);  v = b2 v + (1 - b2) g^2;
 *     p -= lr / (1 - b1^t) * m / (sqrt(v) / sqrt(1 - b2^t) + eps),        t = *step_dev + 1
 * bns_derive_refresh (enqueue right after): refreshes the table of derived parameters -- cached W^T for the input
 * gradients, bias sums -- and advances *step_dev.  Entry layout: bns_derive_entry, table in device memory.
 * ----------------------------------------------------------------------------------------------*/
typedef struct bns_derive_entry {
    int32_t op;        /* 0: dst[c * ld_dst + r] = a[r * ld_a + c], r < rows, c < cols;  1: dst[i] = a[i] + b[i], i < rows;
                          2 / 3 (ABI 9): the fp8 rows (bns_cvt_rows_f32_fp8's rule) of x_r[k] = a[r * ld_a + k] (2) or
                          a[k * ld_a + r] (3), r < rows, k < cols: codes of row r at (uint8_t *)dst + r * ld_dst (ld_dst in
                          bytes, a multiple of 16), the rows' scales right after the codes, at (uint8_t *)dst + rows * ld_dst;
                          cols % 4 == 0, and for op 2 16-byte aligned rows of a */
    int32_t rows, cols, ld_a, ld_dst, pad_;
    const float *a, *b;
    float *dst;
} bns_derive_entry;
size_t bns_derive_entry_bytes(void);
int bns_adam_step_f32(float *param, const float *grad, float *exp_avg, float *exp_avg_sq, int64_t n, float lr, float beta1,
                      float beta2, float eps, float weight_decay, const int64_t *step_dev, void *stream);
int bns_derive_refresh(const void *table_dev, int32_t n_entries, int64_t *step_dev, void *stream);

/* ------------------------------------------------------------------------------------------------
 * SyncBatchNorm (--norm batch; module/sync_bn.py:7-56): batch statistics over every partition.
 * Forward:  bns_bn_colsums_f32(mode 0) -> [sum x | sum x^2] per column; the caller all-reduces the packed [2F] vector;
 *           bns_bn_apply_f32: mean = S1 / n, var = (S2 - mean S1) / n (n = whole_size, the global TRAIN count:
 *           sync_bn.py:19-20 with model.py:39), y = (x - mean) / sqrt(var + eps) * weight + bias, running statistics
 *           moved by `momentum`, mean / rstd kept for the backward.
 * Backward: bns_bn_colsums_f32(mode 1) -> [sum dy | sum dy x_hat]; packed all-reduce; these ARE d bias / d weight;
 *           bns_bn_bwd_f32: dx = (weight / n) / std * (n dy - d bias - x_hat d weight)        (sync_bn.py:51-54).
 * Two collectives per layer and step instead of four, three passes over the activations instead of ~12.
 * F % 4 == 0, F <= 1024, 16-byte aligned rows.
 * ----------------------------------------------------------------------------------------------*/
size_t bns_bn_workspace_bytes(int64_t F);
int bns_bn_colsums_f32(int mode, const float *A, int64_t lda, const float *X, int64_t ldx, int64_t rows, int64_t F,
                       const float *mean, const float *rstd, float *out /*device [2F]*/, void *ws, size_t ws_bytes, void *stream);
int bns_bn_apply_f32(const float *x, int64_t ldx, int64_t rows, int64_t F, const float *sums /*device [2F]*/, float whole_size,
                     float eps, const float *weight, const float *bias, float momentum, float *running_mean /*or NULL*/,
                     float *running_var, float *y, int64_t ldy, float *mean_out /*[F]*/, float *rstd_out /*[F]*/, void *stream);
int bns_bn_bwd_f32(const float *dy, int64_t lddy, const float *x, int64_t ldx, int64_t rows, int64_t F, const float *mean,
                   const float *rstd, const float *weight, const float *sums /*device [2F]*/, float whole_size, float *dx,
                   int64_t lddx, void *stream);

/* ------------------------------------------------------------------------------------------------
 * Collectives (SURVEY 8b).  One context per rank / GPU; NCCL underneath, resolved at run time (dlopen).
 * Bootstrap: rank 0 calls bns_comm_unique_id and hands the BNS_COMM_ID_BYTES bytes to the other ranks by any
 * out-of-band means (the reference rendezvouses over TCP, train.py:459-468); every rank then calls bns_ctx_create.
 *   bns_allreduce_sum_f32   helper/reducer.py:28-49: the weight gradients, as ONE flat bucket, in place
 *   bns_alltoallv_i64       helper/utils.py:187-213 data_transfer(..., tag=NODE): the sampled id lists
 *   bns_alltoallv_f32       helper/feature_buffer.py:101-153: boundary rows, staged transport (the peer-mapped transport
 *                           -- bns_p2p_* -- needs no collective at all)
 * counts / offsets: host arrays [world], in rows of `width` elements; the entry of the own rank is ignored.
 * ----------------------------------------------------------------------------------------------*/
#define BNS_COMM_ID_BYTES 128
int bns_comm_unique_id(void *id_out /*host, BNS_COMM_ID_BYTES*/);
int bns_ctx_create(bns_ctx_t **out, int32_t rank, int32_t world, const void *unique_id /*host, BNS_COMM_ID_BYTES*/);
int bns_ctx_destroy(bns_ctx_t *c);
int bns_allreduce_sum_f32(bns_ctx_t *c, float *buf /*device*/, int64_t n, void *stream);
int bns_alltoallv_f32(bns_ctx_t *c, const float *send, const int64_t *send_counts, const int64_t *send_offsets, float *recv,
                      const int64_t *recv_counts, const int64_t *recv_offsets, int64_t width, void *stream);
int bns_alltoallv_i64(bns_ctx_t *c, const int64_t *send, const int64_t *send_counts, const int64_t *send_offsets,
                      int64_t *recv, const int64_t *recv_counts, const int64_t *recv_offsets, void *stream);
/* the same for per-peer buffers that are separate allocations (host arrays [world] of device pointers / byte counts) */
int bns_alltoallv_bytes(bns_ctx_t *c, const void *const *send_ptrs, const int64_t *send_bytes, void *const *recv_ptrs,
                        const int64_t *recv_bytes, void *stream);

/* y = dropout_p(x) with the Philox mask of bns_ln_relu_dropout_fwd_f32 (counter = (row, vector, offset), key = seed):
 * module/model.py:80 for the layer-0 input; nothing but y is stored. */
int bns_dropout_f32(const float *x, int64_t ldx, int64_t n, int64_t F, float p, uint64_t seed, uint64_t offset,
                    const uint64_t *offset_dev, float *y, int64_t ldy, void *stream);
/* y[r, :] = x[r, :] * row_scale[r] + bias[:]      (row_scale / bias may be NULL: 1 / 0) */
int bns_scale_rows_f32(const float *x, int64_t ldx, int64_t n, int64_t F, const float *row_scale, const float *bias, float *y,
                       int64_t ldy, void *stream);

/* ------------------------------------------------------------------------------------------------
 * ABI 10: the multilevel graph partitioner (--partition-method multilevel; data/multilevel.py runs the level loop).
 * The reference partitions with METIS through dgl.distributed.partition_graph (helper/utils.py:94).  Graphs here are
 * CSRs: indptr int64 [n+1], column ids int32, optional int32 weights (NULL = 1 each).  Every result is integer and
 * independent of the order atomics land in, so two calls give bit-identical output.  Malformed arguments return
 * BNS_E_INVALID before any launch.
 * bns_part_edges: the entries (r, c, w) of the input, mapped to (row_map[r], col_map[c]) (NULL maps = identity), emitted
 *     as (R, C) (mode 0), (C, R) (mode 1) or both (mode 2); with drop_loops, entries with R == C are dropped; equal
 *     (R, C) are merged with their weights summed.  Output: a CSR with n_out_rows rows, columns ascending within a
 *     row, capacity nnz (modes 0, 1) or 2 nnz (mode 2) entries; *out_nnz (host) = its entry count.  Every R must be
 *     < n_out_rows (without a row map, modes 0 and 2 refuse n_rows > n_out_rows), and the summed weights must stay
 *     < 2^31.  One radix sort of 64-bit keys and a reduce-by-key.
 *     Synchronises the stream.  ws: bns_part_edges_workspace_bytes(nnz or 2 nnz).
 * bns_part_conn: conn[v * P + p] (device int32 [n, P], or NULL) = sum of the weights of row v's entries whose column u
 *     has part[u] == p; occ[v] (device [n], or NULL) = the bits p with conn[v][p] > 0; quality (device int64 [2], or
 *     NULL) = { sum over v of conn[v][p] for p != part[v],  number of (v, p) with p != part[v] and conn[v][p] > 0 }:
 *     on the out-CSR with multiplicities, the directed edge cut and the communication volume of partition_quality.
 *     1 <= P <= 64.
 * bns_part_gains: target[v] = the allowed part b != part[v] (bit b of `allowed`) with the largest gain, ties to the
 *     lowest b, or -1; gain[v] its gain = objective before - objective after the move of v alone.  objective 0 (cut):
 *     conn is the table of an undirected weighted graph, gain = conn[v][b] - conn[v][part[v]].  objective 1 (vol):
 *     conn / occ are those of the out-CSR with multiplicities and (indptr, idx, w) the in-CSR with multiplicities, loops
 *     dropped (bns_part_edges modes 1 and 0).  2 <= P <= 64.
 * bns_part_cluster: one size-constrained label-propagation step.  (indptr, cid, cw_edge): per node v, the clusters of its
 *     neighbours with the summed edge weight into each (bns_part_edges with col_map = label), cw: cluster weights.
 *     target[v] = the heaviest neighbouring cluster c != label[v] with cw[c] + nw[v] <= cap, when it beats v's weight
 *     into its own cluster (gain[v] = the difference), else -1.  Only the nodes whose coin (a hash of v and seed) is odd
 *     propose.  nw NULL = 1 each.
 * bns_part_weights: out[l] (device int64 [n_labels]) = sum of nw[v] (NULL = 1) over v with label[v] == l.
 * ----------------------------------------------------------------------------------------------*/
size_t bns_part_edges_workspace_bytes(int64_t n_entries);
int bns_part_edges(int64_t n_rows, int64_t nnz, const int64_t *indptr, const int32_t *idx, const int32_t *w,
                   const int32_t *row_map, const int32_t *col_map, int32_t mode, int32_t drop_loops, int64_t n_out_rows,
                   int64_t *out_indptr, int32_t *out_idx, int32_t *out_w, int64_t *out_nnz /*host*/, void *ws,
                   size_t ws_bytes, void *stream);
int bns_part_conn(int64_t n, const int64_t *indptr, const int32_t *idx, const int32_t *w, const int32_t *part, int32_t P,
                  int32_t *conn, uint64_t *occ, int64_t *quality, void *stream);
int bns_part_gains(int32_t objective, int64_t n, int32_t P, const int64_t *indptr, const int32_t *idx, const int32_t *w,
                   const int32_t *part, const int32_t *conn, const uint64_t *occ, uint64_t allowed, int32_t *target,
                   int64_t *gain, void *stream);
int bns_part_cluster(int64_t n, const int64_t *indptr, const int32_t *cid, const int32_t *cw_edge, const int32_t *label,
                     const int32_t *nw, const int64_t *cw, int64_t cap, uint64_t seed, int32_t *target, int64_t *gain,
                     void *stream);
int bns_part_weights(int64_t n, const int32_t *label, const int32_t *nw, int64_t n_labels, int64_t *out, void *stream);

/* ------------------------------------------------------------------------------------------------
 * ABI 11: edge-balanced partitions (--partition-balance edges): a second node weight, the in-edge count (int64, since
 * coarse sums pass 2^31), carried through the multilevel partitioner's coarsening.
 * bns_part_cluster_edges: bns_part_cluster with a second cap: a cluster c is a candidate only while cw[c] + nw[v] <= cap
 *     and ce[c] + ew[v] <= ecap (ew: device int64 [n] in-edge weight of each node; ce: the clusters' summed in-edge
 *     weights, bns_part_weights_i64 of ew).  Everything else, coin and tie breaks included, is bns_part_cluster's.
 * bns_part_weights_i64: bns_part_weights over int64 weights nw (NULL = 1 each).
 * ----------------------------------------------------------------------------------------------*/
int bns_part_cluster_edges(int64_t n, const int64_t *indptr, const int32_t *cid, const int32_t *cw_edge,
                           const int32_t *label, const int32_t *nw, const int64_t *cw, int64_t cap, const int64_t *ew,
                           const int64_t *ce, int64_t ecap, uint64_t seed, int32_t *target, int64_t *gain, void *stream);
int bns_part_weights_i64(int64_t n, const int32_t *label, const int64_t *nw, int64_t n_labels, int64_t *out,
                         void *stream);

/* ------------------------------------------------------------------------------------------------
 * ABI 12: interval stamps inside a captured CUDA graph (train.GraphedEpoch(timed=True), the --cuda-graph log line).
 * bns_stamp_globaltimer: one single-thread kernel on `stream` that stores the GPU's %globaltimer (nanoseconds) to dst
 *     (device, 8-byte aligned).  Two stamps on one stream bracket the work enqueued between them, as two CUDA events
 *     would; unlike events they may sit inside a captured graph and are rewritten at the same address by every replay.
 *     Differences are only meaningful between stamps of one GPU.
 * ----------------------------------------------------------------------------------------------*/
int bns_stamp_globaltimer(uint64_t *dst /*device*/, void *stream);

/* ------------------------------------------------------------------------------------------------
 * ABI 13: GATv2Conv's dynamic attention (--model gatv2, csrc/gatv2.cuh).  z_src [n_u, heads * Fp], z_dst [n_in, heads * Fp]
 * and attn [heads * Fp] are head-major with the per-head width padded to Fp (a multiple of 4, pad columns zero), 16-byte
 * aligned rows; 1 <= heads <= 8 and heads * Fp <= 1024.  Per entry u -> v and head h
 *     s_uv = sum_f attn[h, f] * leaky_relu(z_src[u, h, f] + z_dst[v, h, f], slope).
 * bns_gatv2_scores_f32: bns_gat_scores_f32 with these scores: the same graph arguments, P / W / W_out_compact outputs and
 *     dropout mask (one Philox4x32-10 call per entry and 4 heads).  The aggregation A' z_src is bns_spmm_weighted_f32 /
 *     bns_spmm_compact_f32 and d a' is bns_sddmm_dot_f32, as for GAT.
 * bns_gatv2_softmax_bwd_f32: dE holds d a' at the original positions; writes d s = P (d P - sum_u P d P) in place
 *     (d P = d a' * mask / (1 - p)), d_zd [n_in, heads * Fp] (row stride ldd) = sum_u d s_uv attn * lrelu'(z_src[u] +
 *     z_dst[v]) and d_attn [heads * Fp] = sum over entries of d s_uv lrelu(z_src[u] + z_dst[v]) from one partial per warp
 *     summed in a fixed order (ws: bns_gatv2_bwd_workspace_bytes(n_in, heads, Fp) bytes, 16-byte aligned).
 * bns_gatv2_colsum_f32: on a transpose gT (bns_graph_transpose) of a_in, or of a_out with row_map = slot and out_base =
 *     n_in: d_zs[out_base + orow(r)] += sum over the entries k of row r of dS[perm[k], h] attn * lrelu'(z_src[out_base +
 *     orow(r)] + z_dst[gT.indices[k]]) (rows with row_map -1 skipped).  Accumulates onto A'^T d rst.
 * bns_gatv2_infer_f32: the evaluation forward on a homogeneous graph: rst = sum_u softmax_u(s_uv) z_src[u], one pass per
 *     row, nothing stored per entry.  bns_gatv2_infer_block_f32: the same over column blocks, the state m, l [n_rows,
 *     heads] and acc [n_rows, heads * Fp] carried between launches as in bns_gat_infer_block_f32 (no bias).
 * Every kernel sums in an order fixed by the inputs: two launches give bit-identical results.
 * ----------------------------------------------------------------------------------------------*/
int bns_gatv2_scores_f32(const bns_graph_t *a_in, const bns_graph_t *a_out, const int32_t *cidx, const int32_t *chunk_cnt,
                         const int32_t *cpos, int64_t x_halo_base, int32_t heads, int32_t Fp, const float *zs, int64_t ldzs,
                         const float *zd, int64_t ldzd, const float *attn, float slope, float p_drop, uint64_t seed,
                         uint64_t offset, const uint64_t *offset_dev, float *P_in, float *P_out, float *W_in, float *W_out,
                         float *W_out_compact, void *stream);
size_t bns_gatv2_bwd_workspace_bytes(int64_t n_rows, int32_t heads, int32_t Fp);
int bns_gatv2_softmax_bwd_f32(const bns_graph_t *a_in, const bns_graph_t *a_out, const int32_t *cidx,
                              const int32_t *chunk_cnt, const int32_t *cpos, int64_t x_halo_base, int32_t heads, int32_t Fp,
                              const float *zs, int64_t ldzs, const float *zd, int64_t ldzd, const float *attn, float slope,
                              float p_drop, uint64_t seed, uint64_t offset, const uint64_t *offset_dev, const float *P_in,
                              const float *P_out, float *dE_in, float *dE_out, float *d_zd, int64_t ldd, float *d_attn,
                              void *ws, size_t ws_bytes, void *stream);
int bns_gatv2_colsum_f32(const bns_graph_t *gT, const float *dS, int32_t heads, int32_t Fp, const float *zs, int64_t ldzs,
                         const float *zd, int64_t ldzd, const float *attn, float slope, const int32_t *row_map,
                         int64_t out_base, float *d_zs, int64_t ldd, void *stream);
int bns_gatv2_infer_f32(const bns_graph_t *g, const float *zs, int64_t ldzs, const float *zd, int64_t ldzd,
                        const float *attn, int32_t heads, int32_t Fp, float slope, float *rst, int64_t ldr, void *stream);
int bns_gatv2_infer_block_f32(const bns_graph_t *g, const float *zs, int64_t ldzs, const float *zd, int64_t ldzd,
                              const float *attn, int32_t heads, int32_t Fp, float slope, float *m, float *l, float *acc,
                              int64_t ldacc, int first, int last, float *rst, int64_t ldr, void *stream);

/* ------------------------------------------------------------------------------------------------
 * ABI 14: GraphSAGE's max-pooling aggregator (--model graphsage-pool, csrc/sage_pool.cuh).  z [n_u, F] (row stride ldz)
 * holds relu(fc_pool(x)), finite, with F a multiple of 4 and at most 1024 (pad columns zero), 16-byte aligned rows;
 * m, win, dm and d_y are contiguous [rows, F].  Per destination row v and column f, m[v, f] = max over the entries
 * u -> v of z[u, f], 0 for a row without entries; -0 is stored as +0, so m does not depend on the order of the entries.
 * bns_sage_max_f32: over the inner entries (a_in) and this epoch's sampled halo entries (a_out through the compaction
 *     cidx / chunk_cnt / cpos, with positions, as bns_gat_scores_f32): m [n_in, F] and win [n_in, F], the position of
 *     the first entry in that walk order whose z equals the max (a_in position, or nnz_in + a_out position for a halo
 *     entry; -1 for a row without entries).  Refuses nnz_in + nnz_out > INT32_MAX.
 * bns_sage_max_bwd_f32: on a transpose gT (bns_graph_transpose) of a_in with pos_base = 0, or of a_out with pos_base =
 *     nnz_in, row_map = slot and out_base = n_in: d_y[out_base + orow(r)] = (z[...] > 0) * sum over the entries k of
 *     row r, in gT's order, of dm[gT.indices[k], f] where win[gT.indices[k], f] == pos_base + perm[k] (rows with
 *     row_map -1 skipped; a row without a winning entry gets 0).  No float atomics.
 * bns_sage_max_infer_f32: m over every entry of a homogeneous graph, no winner.  bns_sage_max_infer_block_f32: the same
 *     over column blocks, the running max m [n_rows, F] and seen [n_rows] (int32) carried between launches (first: from
 *     empty; a launch that is not last stores them; last writes the max, or 0 for a row never seen, to out, which may
 *     be m).  The result equals the single pass bit for bit for any split of the columns.
 * Two launches on the same inputs give bit-identical results.
 * ----------------------------------------------------------------------------------------------*/
int bns_sage_max_f32(const bns_graph_t *a_in, const bns_graph_t *a_out, const int32_t *cidx, const int32_t *chunk_cnt,
                     const int32_t *cpos, int64_t x_halo_base, int32_t F, const float *z, int64_t ldz, float *m,
                     int32_t *win, void *stream);
int bns_sage_max_bwd_f32(const bns_graph_t *gT, int64_t pos_base, const int32_t *row_map, int64_t out_base, int32_t F,
                         const int32_t *win, const float *dm, const float *z, int64_t ldz, float *d_y, void *stream);
int bns_sage_max_infer_f32(const bns_graph_t *g, int32_t F, const float *z, int64_t ldz, float *out, void *stream);
int bns_sage_max_infer_block_f32(const bns_graph_t *g, int32_t F, const float *z, int64_t ldz, float *m, int32_t *seen,
                                 int first, int last, float *out, void *stream);

/* ------------------------------------------------------------------------------------------------
 * ABI 15: the graph transformer layer's scaled dot-product attention (--model transformer, csrc/transformer.cuh).
 * q [n_in, heads * Fp], k and v [n_u, heads * Fp] are head-major with the per-head width padded to Fp (a multiple of 4,
 * pad columns zero), 16-byte aligned rows with their own row strides (k and v may be the two halves of one
 * [n_u, 2 * heads * Fp] table); 1 <= heads <= 8 and heads * Fp <= 1024; scale finite and positive.  Per entry u -> v
 * and head h
 *     s_uv = scale * <q[v, h, :], k[u, h, :]>.
 * bns_tconv_scores_f32: bns_gatv2_scores_f32 with these scores: the same graph arguments, P / W / W_out_compact outputs
 *     and dropout mask (GAT's Philox stream and entry numbering).  The aggregation A' v is bns_spmm_weighted_f32 /
 *     bns_spmm_compact_f32 and d a' = <d rst_v, v[u]> is bns_sddmm_dot_f32.
 * bns_tconv_softmax_bwd_f32: dE holds d a' at the original positions; writes d s = scale P (g - sum_u P g) in place
 *     (g = d a' * mask / (1 - p)) and d_q [n_in, heads * Fp] (row stride ldd) = sum_u d s_uv k[u], one warp per row, no
 *     atomics.  d k = sum_v d s_uv q[v] and d v = A'^T d rst are bns_spmm_weighted_f32 on the transposes.
 * bns_tconv_infer_f32: the evaluation forward on a homogeneous graph: rst = sum_u softmax_u(s_uv) v[u], one pass per
 *     row, nothing stored per entry.  bns_tconv_infer_block_f32: the same over column blocks, the state m, l [n_rows,
 *     heads] and acc [n_rows, heads * Fp] carried between launches as in bns_gatv2_infer_block_f32.
 * Every kernel sums in an order fixed by the inputs: two launches give bit-identical results.
 * ----------------------------------------------------------------------------------------------*/
int bns_tconv_scores_f32(const bns_graph_t *a_in, const bns_graph_t *a_out, const int32_t *cidx, const int32_t *chunk_cnt,
                         const int32_t *cpos, int64_t x_halo_base, int32_t heads, int32_t Fp, const float *q, int64_t ldq,
                         const float *k, int64_t ldk, float scale, float p_drop, uint64_t seed, uint64_t offset,
                         const uint64_t *offset_dev, float *P_in, float *P_out, float *W_in, float *W_out,
                         float *W_out_compact, void *stream);
int bns_tconv_softmax_bwd_f32(const bns_graph_t *a_in, const bns_graph_t *a_out, const int32_t *cidx,
                              const int32_t *chunk_cnt, const int32_t *cpos, int64_t x_halo_base, int32_t heads, int32_t Fp,
                              const float *q, int64_t ldq, const float *k, int64_t ldk, float scale, float p_drop,
                              uint64_t seed, uint64_t offset, const uint64_t *offset_dev, const float *P_in,
                              const float *P_out, float *dE_in, float *dE_out, float *d_q, int64_t ldd, void *stream);
int bns_tconv_infer_f32(const bns_graph_t *g, const float *q, int64_t ldq, const float *k, int64_t ldk, const float *v,
                        int64_t ldv, int32_t heads, int32_t Fp, float scale, float *rst, int64_t ldr, void *stream);
int bns_tconv_infer_block_f32(const bns_graph_t *g, const float *q, int64_t ldq, const float *k, int64_t ldk,
                              const float *v, int64_t ldv, int32_t heads, int32_t Fp, float scale, float *m, float *l,
                              float *acc, int64_t ldacc, int first, int last, float *rst, int64_t ldr, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* BNSGCN_H_ */
