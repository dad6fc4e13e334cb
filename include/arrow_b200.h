/*
 * arrow_b200.h -- C ABI of libarrow_b200.so: H100 (sm_90a) arrow-decomposed SpMM hot path.
 *
 * The reference (spcl/arrow-matrix) is pure Python and has no FFI of its own; this is the
 * boundary a maintainer binds with ctypes (see INTEGRATION.md) to replace the arithmetic and the
 * data movement of
 *     arrow/arrow_slim_mpi.py:78-244   (_ad_spmm / _ad_spmm_gpu: three CSR x dense products)
 *     arrow/arrow_mpi.py:177-336       (wide layout: row-tile / column-tile products)
 *     arrow/common/sp2cp.py:6-16       (_sp2cp: per-iteration CSR upload -> upload once)
 *     arrow/arrow_dec_mpi.py:404-440   (backward exchange: C_{j-1}[to_prev[r]] += C_j[r])
 *     arrow/arrow_dec_mpi.py:507-550   (forward exchange:  X_j[r] = X_{j-1}[to_prev[r]])
 *
 * Conventions: extern "C", opaque context, int return codes (0 = ok, negative = error, text via
 * arrow_last_error), no exceptions cross the boundary.  The caller owns host memory; the library
 * owns device memory (handles are small non-negative ints, valid for one context).  All work is
 * stream-ordered on the context's stream; arrow_sync() waits for it.  One host thread per context.
 * Dense tiles are row-major [rows x k] of fp32 or fp64 (or int32 labels, or bits); CSR is fp32 or fp64 values with int32 indices
 * on the device.
 * The precision is fixed when a tile is allocated / a block uploaded (ARROW_F32 / ARROW_F64), and every operand of one
 * launch has the same precision.  fp64 covers the one-GPU product (arrow_spmm, arrow_spmm_add, arrow_gather_rows); the
 * multi-GPU entry points (two-part operand, pointer tables, push / reduce, multi-source gather) are fp32 only.
 */
#ifndef ARROW_B200_H
#define ARROW_B200_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct arrow_ctx arrow_ctx;

#define ARROW_ABI_VERSION 15

/* error codes */
#define ARROW_OK              0
#define ARROW_ERR_CUDA       -1
#define ARROW_ERR_ARG        -2
#define ARROW_ERR_HANDLE     -3
#define ARROW_ERR_RANGE      -4   /* index / size exceeds the int32 device layout */
#define ARROW_ERR_NOMEM      -5
#define ARROW_ERR_UNSUPPORTED -6

/* element types of dense tiles and CSR values */
#define ARROW_F32             0
#define ARROW_F64             1
#define ARROW_I32             2   /* dense tiles only: labels / parents of arrow_spmm_sr_witness.  Allocation, free, h2d / d2h
                                     (and the lane copies), copy and arrow_dense_dtype accept it; every arithmetic launch
                                     refuses an int32 operand with ARROW_ERR_ARG */
#define ARROW_B1              3   /* dense tiles only: bits, column c of a row is bit c % 32 of uint32 word c / 32; a row is
                                     one word for k <= 32, else ((k + 31) / 32 rounded up to a multiple of 4) words (16-byte
                                     vectors), and host rows of h2d / d2h have that layout.  Allocation zero-fills (padding bits stay 0 under every
                                     launch), free, h2d / d2h (and the lane copies), copy, ptr, dtype and fill with 0 accept it;
                                     the (or, and) launches below run on it; every other arithmetic or multi-GPU launch refuses a
                                     bit operand with ARROW_ERR_ARG */

/* flags for arrow_spmm / arrow_gather_rows */
#define ARROW_ACCUMULATE      1   /* C += ... instead of C = ...  (reference: `C_i += A_i0 @ X_0`,
                                     arrow_slim_mpi.py:142-144; scatter-add, arrow_dec_mpi.py:437) */

/* SpMM kernel variants (arrow_spmm `variant`); ARROW_VARIANT_AUTO picks per k. */
#define ARROW_VARIANT_AUTO    -1
#define ARROW_VARIANT_DIRECT   0  /* sub-warp per row, broadcast index loads, float4 X gathers          */
#define ARROW_VARIANT_SHFL     1  /* sub-warp per row, coalesced index/value chunk + shuffle broadcast  */
#define ARROW_VARIANT_TMA      2  /* X rows staged into shared memory with cp.async.bulk + mbarrier     */
#define ARROW_VARIANT_TILES    3  /* default: CSR row tiles streamed by cp.async.bulk (TMA) + mbarrier,
                                     two stages; warps only issue X gathers.  Bits 4..7 of `variant`
                                     optionally force the float4-per-lane count (1, 2 or 4), bits 8..9 the
                                     rows a lane group works on at once (1 or 2; 2 needs k <= 32).     */

int  arrow_b200_abi_version(void);

/* ---- context ------------------------------------------------------------------------------- */
/* `stream` is a cudaStream_t to run on (e.g. torch's current stream) or NULL: the context then
 * creates its own non-blocking stream. */
int  arrow_ctx_create(int device, void *stream, arrow_ctx **out);
void arrow_ctx_destroy(arrow_ctx *ctx);
const char *arrow_last_error(const arrow_ctx *ctx);      /* ctx may be NULL: last creation error */
int  arrow_sync(arrow_ctx *ctx);
int  arrow_device_info(arrow_ctx *ctx, int *sm_count, int64_t *free_bytes, int64_t *total_bytes);
int  arrow_set_tuning(arrow_ctx *ctx, int long_row_threshold, int long_row_segment);
/* Tuning knobs.  L2 hint masks of the tile kernel: bit 0 = X gathers evict_last, bit 1 = CSR and C streams
 * evict_first; PLAIN applies to C = A X launches, FUSED to launches with a row map or ARROW_ACCUMULATE. */
#define ARROW_OPT_L2_HINTS_PLAIN 1
#define ARROW_OPT_L2_HINTS_FUSED 2
#define ARROW_OPT_BIG_TILES      3   /* 1 (default): 128-row / 2048-entry CSR tiles may be picked when k <= 32 (see ARROW_OPT_TILE_ROWS) */
#define ARROW_OPT_PREFETCH        5   /* bulk L2 prefetch (cp.async.bulk.prefetch.L2, one request per X row) of a CSR tile's X rows
                                        before its math: bit 0 = plain launches, bit 4 = fused launches (row map / accumulate /
                                        gather-add / dual X / row pointers).  Measured as a loss;
                                        off by default, kept as the A/B switch */
#define ARROW_OPT_SPMM_CTAS_PER_SM 4 /* cap on resident SpMM CTAs per SM (0 = no cap): leaves SM resources to exchange
                                        kernels running on the side lane */
#define ARROW_OPT_ROWS_PER_GROUP  6   /* rows a lane group gathers for at once when k <= 32: 0 (default) = 1, 1, 2 */
#define ARROW_OPT_SPMM_SM_LIMIT   7   /* cap on the SMs a SpMM grid covers (0 = all): concurrent launches on two lanes share the GPU */
#define ARROW_OPT_PUSH_CTAS       8   /* grid of arrow_push_rows (0 = 2 per SM) */
#define ARROW_OPT_SMEM_CARVEOUT  10   /* preferred shared-memory carve-out (percent, -1 = driver default) of the tile kernel: the rest of
                                        the SM's 256 KB L1 / shared array is L1, the landing buffer of the gathers in flight (measurement switch) */
#define ARROW_OPT_FORCE_PREDICATED 11  /* 1: the tile kernel takes its predicated gather path even when every column is valid (measurement switch) */
#define ARROW_OPT_TILE_KERNEL     12   /* 1 (default): plain / row-map / accumulate launches with one row per lane group run the round-1 tile
                                        kernel, 0: the generalised kernel everywhere (A/B switch) */
#define ARROW_OPT_PUSH_INTERLEAVE 13   /* 1 (default): arrow_push_rows walks its destination blocks interleaved (every peer is written to at
                                        every instant); 0: block after block */
#define ARROW_OPT_BARRIER_TIMEOUT_MS 9 /* arrow_peer_barrier gives up after this long (default 30000) and poisons the context */
#define ARROW_OPT_TILE_ROWS      14   /* CSR row tiles the tile kernels walk: 0 (default) = picked per launch from the L2 size (arrow_tile_rows),
                                         16 / 32 / 64 / 128 = that list (128 only where k <= 32 on float32, else 64).  Results are
                                         bit-identical for every value: only the rows in flight change */
int  arrow_set_option(arrow_ctx *ctx, int option, int value);
/* Rows per CSR tile of the tile-kernel launches at feature width k and element type dtype (ARROW_F32 / ARROW_F64) under the
 * context's options and device.  The automatic rule: the largest of 128 (float32, k <= 32, ARROW_OPT_BIG_TILES on) / 64 / 32 / 16
 * rows for which resident CTAs x rows x k x element bytes <= L2 size / 4 (the X rows of the window in flight stay in L2), else 16.
 * arrow_tile_rows_rule evaluates that rule for given values without a context or device (a negative value: bad arguments). */
int  arrow_tile_rows(arrow_ctx *ctx, int k, int dtype, int *rows);
int  arrow_tile_rows_rule(int k, int elem_bytes, int64_t l2_bytes, int resident_ctas, int big_ok);

/* ---- sparse blocks (replaces _sp2cp, sp2cp.py:6-16: uploaded once, resident) ----------------- */
/* indptr has n_rows+1 entries of indptr_bytes (4 or 8) each and may start at any base value
 * (a row slice of a bigger file); indices/data point at the entry indptr[0] refers to.
 * data == NULL means all ones (missing _data.npy, graphio.py:292-298).
 * Rejected with ARROW_ERR_ARG / ARROW_ERR_RANGE (nothing stays allocated): a row pointer that is not a
 * non-decreasing sequence spanning exactly nnz entries, a column index outside [0, n_cols), a block beyond the
 * int32 device layout. */
int  arrow_csr_upload(arrow_ctx *ctx, int64_t n_rows, int64_t n_cols, int64_t nnz,
                      const void *indptr, int indptr_bytes,
                      const void *indices, int indices_bytes,
                      const float *data, int *csr_out);
/* The same with float64 values: the block's launches compute in float64 on float64 tiles. */
int  arrow_csr_upload_f64(arrow_ctx *ctx, int64_t n_rows, int64_t n_cols, int64_t nnz,
                          const void *indptr, int indptr_bytes,
                          const void *indices, int indices_bytes,
                          const double *data, int *csr_out);
/* Refused (ARROW_ERR_ARG) while remapped copies made by arrow_csr_remap_columns still share the block's arrays. */
int  arrow_csr_free(arrow_ctx *ctx, int csr);
int  arrow_csr_info(arrow_ctx *ctx, int csr, int64_t *n_rows, int64_t *n_cols, int64_t *nnz,
                    int64_t *max_row_nnz, int64_t *n_long_rows);
/* New CSR sharing indptr/values (whatever their precision) with `csr`, columns sent through `map` (col' = map[col]; entries
 * whose image is invalid are skipped by the kernels).  This folds the forward permutation gather
 * (arrow_dec_mpi.py:526, 544) into the SpMM's X read.  `map`'s limit must not exceed new_n_cols; the copy must be
 * freed before its source. */
int  arrow_csr_remap_columns(arrow_ctx *ctx, int csr, int map, int64_t new_n_cols, int *csr_out);

/* ---- row maps (to_prev / to_next slices, arrow_dec_mpi.py:737-749) ---------------------------- */
/* int64 host map -> int32 device map; entries < 0 or >= limit (the reference's sentinel
 * 2*width*n_blocks[0] lands here) become -1 = "not routed". */
int  arrow_map_upload(arrow_ctx *ctx, const int64_t *map, int64_t n, int64_t limit, int *map_out);
int  arrow_map_free(arrow_ctx *ctx, int map);
/* out[r] = outer[inner[r]] (invalid if either step is); chains level maps for the fused path. */
int  arrow_map_compose(arrow_ctx *ctx, int inner, int outer, int *map_out);
/* out[q] = r where map[r] == q (injective maps only), size n_out, -1 elsewhere. */
int  arrow_map_invert(arrow_ctx *ctx, int map, int64_t n_out, int *map_out);
int  arrow_map_d2h(arrow_ctx *ctx, int map, int32_t *host, int64_t n);

/* ---- dense tiles (X_i / C_i / X_0 / C_0 of arrow_slim_mpi.py:354-394, concatenated) ----------- */
int  arrow_dense_alloc(arrow_ctx *ctx, int64_t rows, int k, int *buf_out);      /* fp32, zero filled */
int  arrow_dense_alloc_dtype(arrow_ctx *ctx, int64_t rows, int k, int dtype, int *buf_out);   /* ARROW_F32 / F64 / I32 */
int  arrow_dense_dtype(arrow_ctx *ctx, int buf, int *dtype);
int  arrow_dense_free(arrow_ctx *ctx, int buf);
int  arrow_dense_fill(arrow_ctx *ctx, int buf, float value);                    /* converted to the tile's type */
/* host rows are of the tile's element type (float, double or int32_t) */
int  arrow_dense_h2d(arrow_ctx *ctx, int buf, int64_t row0, int64_t rows, const void *host);
int  arrow_dense_d2h(arrow_ctx *ctx, int buf, int64_t row0, int64_t rows, void *host);
/* both tiles have the same element type, else ARROW_ERR_ARG */
int  arrow_dense_copy(arrow_ctx *ctx, int dst, int64_t dst_row0, int src, int64_t src_row0, int64_t rows);
int  arrow_dense_ptr(arrow_ctx *ctx, int buf, void **device_ptr, int64_t *rows, int *k);
/* Wrap fp32 device memory owned by someone else (a torch tensor, an IPC-imported peer tile).  The pointer must be 16-byte
 * aligned when k % 4 == 0 (float4 rows), else 4-byte aligned: ARROW_ERR_ARG otherwise. */
int  arrow_dense_wrap(arrow_ctx *ctx, void *device_ptr, int64_t rows, int k, int *buf_out);
/* Copy lanes: host<->device staging on side streams so that step i's download, step i+1's upload and the
 * compute in between overlap (PCIe is full duplex).  Lane 0 is the context's main stream.  arrow_lane_wait
 * makes `waiting_lane` wait for everything submitted so far on `signalling_lane` (event, no host sync).
 * Replaces the blocking cp.asarray / cp.asnumpy round trips of arrow_slim_mpi.py:186-191, 228-232. */
#define ARROW_LANE_MAIN 0
#define ARROW_LANE_H2D  1
#define ARROW_LANE_D2H  2
#define ARROW_LANE_SIDE 3   /* compute-side lane: exchange kernels overlapping the main lane's SpMM */
#define ARROW_N_LANES   4
int  arrow_dense_h2d_lane(arrow_ctx *ctx, int lane, int buf, int64_t row0, int64_t rows, const void *host);
int  arrow_dense_d2h_lane(arrow_ctx *ctx, int lane, int buf, int64_t row0, int64_t rows, void *host);
int  arrow_lane_wait(arrow_ctx *ctx, int waiting_lane, int signalling_lane);
int  arrow_lane_sync(arrow_ctx *ctx, int lane);
/* Select the lane on which the following arrow_spmm* / arrow_gather_rows[_multi] / arrow_push_rows / arrow_reduce_rows /
 * arrow_peer_barrier / arrow_dense_copy calls are launched (every lane has its own tile scheduler state).  Used to run
 * the exchange chain of the deeper levels beside the level-0 SpMM; a barrier issued on lane L must use flag tiles
 * reserved for lane L. */
int  arrow_set_lane(arrow_ctx *ctx, int lane);
/* Named events for finer ordering between lanes (waiting on a never-recorded event is a no-op). */
#define ARROW_MAX_EVENTS 16
int  arrow_event_record(arrow_ctx *ctx, int event, int lane);
int  arrow_event_wait(arrow_ctx *ctx, int event, int lane);
/* pinned host staging */
int  arrow_host_alloc(size_t bytes, void **ptr);
int  arrow_host_free(void *ptr);
/* Pinned staging memory placed on the NUMA node of `device` (mmap + mbind + first touch + cudaHostRegister); freed with
 * arrow_host_free.  arrow_bind_thread_to_device_numa pins the calling thread to that node's CPUs (node_out = -1 when
 * the topology is unknown: nothing is changed); device < 0 undoes it (every CPU, default memory policy). */
int  arrow_host_alloc_numa(size_t bytes, int device, void **ptr);
int  arrow_bind_thread_to_device_numa(int device, int *node_out, int *n_cpus_out);

/* ---- the hot path ------------------------------------------------------------------------------ */
/* C[out(r), :] (+)= sum_p A[r, col_p] * X[col_p, :]   for every row r of `csr`
 *   out(r) = r, or rowmap[r] when rowmap >= 0 (rows with rowmap[r] == -1 are dropped): the backward
 *   scatter-add of arrow_dec_mpi.py:421-437 folded into the SpMM epilogue.
 * X must have >= n_cols rows; C must cover every out(r); X and C must not alias.
 * The block, X, C (and the addend of arrow_spmm_add) share one element type, else ARROW_ERR_ARG.  An fp64 launch runs
 * with ARROW_VARIANT_AUTO or ARROW_VARIANT_TILES only (any other variant: ARROW_ERR_UNSUPPORTED). */
int  arrow_spmm(arrow_ctx *ctx, int csr, int x_buf, int c_buf, int rowmap, int flags, int variant);

/* C[r, :] = sum_p A[r, col_p] * X[col_p, :] + add[add_map[r], :]   (rows with add_map[r] == -1 get the product only).
 * The backward exchange C_{j-1}[to_prev[r]] += C_j[r] (arrow_dec_mpi.py:437) folded into the RECEIVING level's SpMM as
 * a gather-add: levels are multiplied deepest first, each writes its tile once, nothing is read-modify-written. */
int  arrow_spmm_add(arrow_ctx *ctx, int csr, int x_buf, int c_buf, int add_buf, int add_map, int variant);

/* dst[r, :] (+)= src[map[r], :] for r in [0, map length); rows with map[r] == -1 are left alone; dst and src share
 * one element type (ARROW_ERR_ARG otherwise)
 * (the reference's stale-row behaviour, arrow_dec_mpi.py:544).  Forward exchange with to_prev,
 * backward exchange (as a gather-add) with to_next. */
int  arrow_gather_rows(arrow_ctx *ctx, int dst_buf, int src_buf, int map, int flags);

/* ---- semirings (one GPU) --------------------------------------------------------------------------- */
/* (min, +) / (max, +): ⊗ is the fp32 add (round to nearest, identity 0), ⊕ is fminf / fmaxf (identity +inf / -inf).
 * ARROW_SR_PLUS_TIMES forwards to arrow_spmm / arrow_spmm_add (ARROW_VARIANT_AUTO, either precision) and to the
 * accumulating arrow_gather_rows.  MIN_PLUS / MAX_PLUS validate their operands like arrow_spmm_add: mixed precision,
 * aliasing, bad shapes or an unknown semiring code return ARROW_ERR_ARG, fp64 operands ARROW_ERR_UNSUPPORTED.
 * Each result element is ⊕ over once-rounded terms, so it does not depend on the kernel, the grid or the order. */
#define ARROW_SR_PLUS_TIMES 0
#define ARROW_SR_MIN_PLUS   1
#define ARROW_SR_MAX_PLUS   2
#define ARROW_SR_OR_AND     3   /* the boolean semiring on ARROW_B1 tiles (k <= 8192, else ARROW_ERR_UNSUPPORTED): ⊗ is "the
                                   entry exists" (the block's values, of either precision, are not read), ⊕ is OR.  Every
                                   operand is a bit tile, else ARROW_ERR_ARG; a bit operand with another semiring: ARROW_ERR_ARG.
                                   arrow_gather_rows without ARROW_ACCUMULATE moves bit rows (with it: ARROW_ERR_ARG) */
/* The bottleneck semirings (fp32, validated and refused like MIN_PLUS / MAX_PLUS).  ⊕ and ⊗ are both min or max, so every
 * result element is one of the operands, exactly.  A NaN operand is dropped by ⊕ and ⊗ (a NaN weight passes the feature
 * through), and -0 orders below +0 everywhere. */
#define ARROW_SR_MAX_MIN    4   /* widest paths: ⊕ = max (identity -inf), ⊗ = min (identity +inf) */
#define ARROW_SR_MIN_MAX    5   /* minimax paths: ⊕ = min (identity +inf), ⊗ = max (identity -inf) */
/* C[r] = (⊕_p A[r,p] ⊗ X[col_p]) ⊕ add[add_map[r]]  (add_buf / add_map may be -1; rows with add_map[r] == -1 get the
 * product only; a row without entries, or whose entries are all skipped columns, gets the ⊕ identity) */
int  arrow_spmm_sr(arrow_ctx *ctx, int csr, int x_buf, int c_buf, int add_buf, int add_map, int semiring);
/* dst[r] = dst[r] ⊕ src[map[r]] for map[r] >= 0 (the backward exchange of a semiring step) */
int  arrow_gather_rows_sr(arrow_ctx *ctx, int dst_buf, int src_buf, int map, int semiring);
/* number of rows of two equally shaped tiles (same rows, k and element type) that differ in some element, compared by
 * value (-0 == +0, NaN != NaN; bit tiles over their k columns); synchronises the context's current lane */
int  arrow_dense_count_diff(arrow_ctx *ctx, int a, int b, int64_t *rows_changed);
/* number of rows of two fp32 tiles of one shape that differ in some element's bits (-0 != +0, a NaN equal to the same NaN):
 * the stop test of the bottleneck fixed point, whose order puts -0 below +0; ARROW_ERR_ARG for other types or shapes;
 * synchronises the context's current lane */
int  arrow_dense_count_diff_bits(arrow_ctx *ctx, int a, int b, int64_t *rows_changed);
/* BFS level record of the (or, and) step: dist[r, c] = level for every (r, c < k) whose bit is set in new_buf and clear in
 * old_buf (bit tiles); every other element of dist_buf (ARROW_I32, same rows and k) is left alone.  *n_new = the number of
 * such bits (0: the step reached its fixed point); synchronises the context's current lane. */
int  arrow_bits_mark_new(arrow_ctx *ctx, int new_buf, int old_buf, int dist_buf, int level, int64_t *n_new);

/* ---- direction-optimising BFS (one GPU, (or, and) on bit tiles) ------------------------------------------------------ */
/* Push adjacency: a boolean n_vertices x n_vertices matrix M stored transposed, as CSR without values (row u lists every
 * v with an edge u -> v in ascending order, duplicates kept), built on the device from n_parts blocks.  Entry (r, c) of
 * block csrs[i] with c >= 0 gives the edge m_i(c) -> m_i(r), m_i the row map maps[i] (-1: the identity); edges with an
 * end at -1 and edges with u == v are dropped.  With level 0's block and identity, and each level j >= 1's block with its
 * level-j -> level-0 row map, M is the operator of the fused (or, and) step with the identity: X' = X | M X.  Temporary
 * device memory of 16 bytes per edge is freed before the call returns; the adjacency keeps 4 (n + 1) + 4 m bytes and a
 * frontier record of 8 n bytes.  ARROW_ERR_ARG: a map shorter than its block's rows or columns, a map or an identity
 * block that reaches past n_vertices; ARROW_ERR_RANGE: 2^31 edges or more; ARROW_ERR_UNSUPPORTED: during graph capture.
 * Synchronises. */
int  arrow_adj_build(arrow_ctx *ctx, int n_parts, const int *csrs, const int *maps, int64_t n_vertices, int *adj_out);
int  arrow_adj_free(arrow_ctx *ctx, int adj);
int  arrow_adj_info(arrow_ctx *ctx, int adj, int64_t *n_vertices, int64_t *n_edges);
/* indptr: n_vertices + 1 entries, indices: n_edges entries */
int  arrow_adj_d2h(arrow_ctx *ctx, int adj, int32_t *indptr, int32_t *indices);
/* arrow_bits_mark_new (the same dist and *n_new; new_buf has the adjacency's rows), and in the same pass the frontier
 * record of `adj`: the rows with a bit set in new_buf and clear in old_buf in one of the k columns, tagged with new_buf.
 * *frontier_rows is their number, *frontier_edges the sum of their rows' lengths in the adjacency.  Synchronises. */
int  arrow_bits_mark_frontier(arrow_ctx *ctx, int adj, int new_buf, int old_buf, int dist_buf, int level, int64_t *n_new,
                              int64_t *frontier_rows, int64_t *frontier_edges);
/* out = x, then out[v] |= x[u] for every recorded frontier row u and every v of adj row u (non-returning ORs; zero words
 * are skipped).  x must be the tile of the last arrow_bits_mark_frontier on `adj`.  When X_h = X_{h-1} | M X_{h-1} and the
 * record holds the rows of X_h & ~X_{h-1}, out = X_h | M X_h: the pull step's bits for the frontier's edges.  out may be
 * X_{h-1}'s tile (x alone is read).  ARROW_ERR_ARG: non-bit tiles, no record, x not the recorded tile, out == x, rows
 * other than the adjacency's, out of another shape or k; ARROW_ERR_UNSUPPORTED: k > 8192. */
int  arrow_bits_push_frontier(arrow_ctx *ctx, int adj, int x_buf, int out_buf);
/* In-adjacency of the same M: row v lists every u with an edge u -> v in ascending order, duplicates kept; the edges are
 * arrow_adj_build's (same blocks, maps and dropped edges) and so are the refusals.  It keeps 4 (n + 1) + 4 m bytes and no
 * frontier record; rows of more than 512 entries are also listed as 512-entry segments (16 bytes each) for
 * arrow_bits_parents.  arrow_adj_info, arrow_adj_d2h and arrow_adj_free accept it; every other call taking an adjacency
 * refuses it with ARROW_ERR_ARG.  Synchronises. */
int  arrow_adj_build_in(arrow_ctx *ctx, int n_parts, const int *csrs, const int *maps, int64_t n_vertices, int *adj_out);
/* BFS parents of one level.  For every row v of adj's frontier record (written by arrow_bits_mark_frontier for new_buf
 * against old_buf) and every bit (v, s), s < k, set in new_buf and clear in old_buf: parent[v, s] = the smallest u of
 * in_adj's row v whose bit s is set in old_buf, -1 when there is none.  Every other element of parent_buf is left alone.
 * When new = X_h = X_{h-1} | M X_{h-1} and old = X_{h-1}, that u is the smallest in-neighbour of v one hop closer to s.
 * Exact: the result depends on neither the grid nor the kernel.  edges_scanned (may be NULL; then the call does not
 * synchronise) receives the in-edges gathered.  ARROW_ERR_ARG: non-bit new / old, a parent tile that is not ARROW_I32 of
 * the same rows and k, in_adj not an in-adjacency or adj one, adjacencies of different vertex counts, rows other than
 * theirs, no record in adj or one for another tile, new_buf == old_buf; ARROW_ERR_UNSUPPORTED: k > 8192. */
int  arrow_bits_parents(arrow_ctx *ctx, int in_adj, int adj, int new_buf, int old_buf, int parent_buf, int64_t *edges_scanned);

/* ---- betweenness on bit tiles (one GPU): shortest-path counts and Brandes dependencies over k source columns ---------- */
/* M is taken as a set here: a list entry equal to its predecessor is skipped.  Every sum below runs over a list in
 * ascending order, 512 entries at a time from the row's start: each segment is summed left to right into a partial starting
 * at 0 and the partials are added in segment order.  Lists longer than 512 entries are split across warps at the
 * adjacency's 512-entry segments, their partials kept in a scratch of 8 * k bytes per segment owned by the adjacency.  No
 * floating-point atomics: the results depend on neither the grid nor the launch. */
/* Path counts of one level.  For every row v of adj's frontier record (written by arrow_bits_mark_frontier for new_buf
 * against old_buf) and every bit (v, s), s < k, set in new_buf and clear in old_buf: sigma[v, s] = the sum of sigma[u, s]
 * over the distinct u of in_adj's row v whose bit s is set in old_buf.  Every other element of sigma_buf is left alone.
 * When new = X_h = X_{h-1} | M X_{h-1} and old = X_{h-1} those u are the in-neighbours at level h - 1, so sigma holds the
 * shortest-path counts of level h once it holds those of level h - 1.  edges_scanned (may be NULL; then the call does
 * not synchronise) receives the in-list entries read, once per row and 32-column word with a fresh bit.  ARROW_ERR_ARG:
 * non-bit new / old, a sigma tile that is not ARROW_F64 of the same rows and k, in_adj not an in-adjacency or adj one,
 * adjacencies of different vertex counts, rows other than theirs, no record in adj or one for another tile,
 * new_buf == old_buf; ARROW_ERR_UNSUPPORTED: k > 8192. */
int  arrow_bits_path_counts(arrow_ctx *ctx, int in_adj, int adj, int new_buf, int old_buf, int sigma_buf, int64_t *edges_scanned);
/* Keeps a copy of adj's current frontier record as level `level` of the adjacency's history: level 0 clears the history
 * first, any other level must be the next one (the number of levels kept).  4 bytes per recorded row (one BFS keeps at
 * most n * min(k, levels + 1) rows); the device buffer doubles when it runs out, so it holds up to twice the rows kept (at
 * least 1024), the old and new buffers coexist while it grows (up to three times), and it is kept at its largest size
 * until the adjacency is freed.
 * ARROW_ERR_ARG: an in-adjacency, no record, another level.  Stream-ordered. */
int  arrow_adj_keep_record(arrow_ctx *ctx, int adj, int level);
/* Dependencies of one level, 1 <= level < the levels kept.  For every row u of the history's level `level` and every
 * column s with dist[u, s] == level: delta[u, s] = sigma[u, s] * (the sum of fl((1 + delta[w, s]) / sigma[w, s]) over
 * the distinct w of adj's row u with dist[w, s] == level + 1; 0 when there is none).  Every other element of delta_buf is
 * left alone; run the levels from the deepest down to 1.  edges_scanned (may be NULL; then the call does not synchronise)
 * receives the out-list entries read, once per row and 32-column word holding the level.  ARROW_ERR_ARG: an in-adjacency,
 * a weighted adjacency, dist not ARROW_I32 or sigma / delta not ARROW_F64, shapes other than the adjacency's rows and
 * dist's k, delta aliasing sigma, a level outside the history.  The first call lists the push adjacency's segments
 * (synchronises). */
int  arrow_bits_dependencies(arrow_ctx *ctx, int adj, int level, int dist_buf, int sigma_buf, int delta_buf, int64_t *edges_scanned);
/* out[r, s] = value for every bit (r, s), s < k, set in new_buf and clear in old_buf; out is an ARROW_F64 tile of the
 * same rows and k, its other elements left alone.  ARROW_ERR_ARG: non-bit new / old, another out type or shape. */
int  arrow_bits_fill_f64(arrow_ctx *ctx, int new_buf, int old_buf, int out_buf, double value);
/* out[r, 0] = in[r, 0] + in[r, 1] + ... + in[r, k - 1], summed left to right from 0; in ARROW_F64 [rows x k], out
 * ARROW_F64 [rows x 1].  ARROW_ERR_ARG: other types or shapes, out aliasing in. */
int  arrow_dense_row_sum(arrow_ctx *ctx, int in_buf, int out_buf);

/* ---- direction-optimising shortest and critical paths (one GPU, min-plus / max-plus on fp32 tiles) ---------------------- */
/* The push adjacency of arrow_adj_build carrying each edge's fp32 weight (the entry's value), with the edges u == v kept
 * (a negative self-loop changes a min-plus step); edges with an end at -1 are still dropped.  Duplicates of (u, v) come
 * out in any order.  Temporary device memory of 24 bytes per edge is freed before the call returns; the adjacency keeps
 * 4 (n + 1) + 8 m bytes and the frontier record of 8 n bytes.  Refusals: those of arrow_adj_build, and
 * ARROW_ERR_UNSUPPORTED for a fp64 block.  Synchronises. */
int  arrow_adj_build_weighted(arrow_ctx *ctx, int n_parts, const int *csrs, const int *maps, int64_t n_vertices,
                              int *adj_out);
/* values: n_edges weights, in the order of arrow_adj_d2h's indices; ARROW_ERR_ARG on an adjacency without weights */
int  arrow_adj_values_d2h(arrow_ctx *ctx, int adj, float *values);
/* One pass over two fp32 tiles of the adjacency's rows: *rows_changed counts the rows that differ by value (-0 == +0,
 * NaN != NaN: arrow_dense_count_diff's figure), and the frontier record of `adj`, tagged with new_buf, lists the rows that
 * differ in bits.  *frontier_rows is their number, *frontier_edges the sum of their rows' lengths.  Synchronises. */
int  arrow_sr_mark_frontier(arrow_ctx *ctx, int adj, int new_buf, int old_buf, int64_t *rows_changed, int64_t *frontier_rows,
                            int64_t *frontier_edges);
/* out = canon(x) (fl(0 + x), NaN -> the ⊕ identity: what the identity diagonal contributes to a step), then for every
 * recorded frontier row u and edge u -> v of weight a, t = fl(a + x[u, s]) is folded into out[v, s] with a non-returning
 * min (MIN_PLUS) or max (MAX_PLUS) where it improves on canon(x[v, s]); NaN terms are skipped.  x must be the tile of the
 * last arrow_sr_mark_frontier on `adj`.  When X_h is the step of X_{h-1} (with the identity), X_h <= X_{h-1} in the
 * semiring's order, the record holds the rows where they differ and no weight is -0, out is the step of X_h bit for bit.
 * ARROW_ERR_ARG: non-fp32 tiles, an adjacency without weights, no record, x not the recorded tile, out aliasing x, rows
 * other than the adjacency's, out of another shape or k, an unknown semiring code; ARROW_ERR_UNSUPPORTED: PLUS_TIMES,
 * OR_AND. */
int  arrow_sr_push_frontier(arrow_ctx *ctx, int adj, int x_buf, int out_buf, int semiring);
/* MAX_MIN / MIN_MAX: out = canon(x) = x ⊗ the ⊗ identity (NaN -> that identity, every other value, -0 included, kept),
 * then t = a ⊗ x[u, s] is folded into out[v, s] with a non-returning max (MAX_MIN) or min (MIN_MAX) where it improves on
 * canon(x[v, s]) in the ⊕ order with -0 below +0.  Out is the step of X_h bit for bit under the conditions above, -0
 * weights included. */

/* ---- bottleneck path trees (one GPU, max-min / min-max on fp32 tiles) ------------------------------------------------ */
/* arrow_sr_mark_frontier, and in the same pass steps[r, c] = level for every element where new_buf and old_buf differ in
 * bits; level 0 writes 0 to every element instead.  steps_buf is an ARROW_I32 tile of new_buf's rows and k.  In a
 * fixed-point loop steps then holds T, the level at which every element last changed.  ARROW_ERR_ARG: those of
 * arrow_sr_mark_frontier, another steps type or shape, steps aliasing new or old, a negative level.  Synchronises. */
int  arrow_sr_mark_frontier_steps(arrow_ctx *ctx, int adj, int new_buf, int old_buf, int steps_buf, int level,
                                  int64_t *rows_changed, int64_t *frontier_rows, int64_t *frontier_edges);
/* Parents of a bottleneck fixed point D (dist_buf, fp32) with its step record T (steps_buf, int32), over the loop-free
 * weighted in-adjacency (arrow_adj_build_loopfree, incoming != 0).  parent[v, s] = -1 where T[v, s] == 0 or D[v, s] is the
 * ⊕ identity; otherwise the smallest u of in_adj's row v with an entry of weight a such that a ⊗ D[u, s] == D[v, s] in
 * bits and either D[u, s] is strictly better than D[v, s] in the ⊕ order (-0 below +0) or the two are equal and
 * T[u, s] < T[v, s]; -1 when there is none.  Along every parent edge D strictly improves or T strictly drops, so the
 * parents form a forest whose roots have T == 0 or no parent.  At a fixed point in bits every element with T > 0 that is
 * reached has a parent, except NaN features and the elements the first level gives the ⊗ identity from one through an
 * edge of weight ⊗ identity.  A warp walks a row's ascending in-list for one 32-column
 * word until every element of it has a hit; lists longer than 512 entries are split at the adjacency's segments and folded
 * with an unsigned min into -1, so the result depends on neither the grid nor the order.  *entries_read (may be NULL; then
 * the call does not synchronise) receives the in-list entries read.  ARROW_ERR_ARG: in_adj not the loop-free
 * in-adjacency, dist not fp32, steps or parent not ARROW_I32, shapes other than the adjacency's rows and dist's k, parent
 * aliasing dist or steps, a semiring other than MAX_MIN / MIN_MAX (ARROW_ERR_UNSUPPORTED for the other known codes). */
int  arrow_sr_tree_parents(arrow_ctx *ctx, int in_adj, int dist_buf, int steps_buf, int parent_buf, int semiring,
                           int64_t *entries_read);

/* ---- weighted betweenness (one GPU, min-plus on fp32 tiles): shortest-path counts and Brandes dependencies ------------- */
/* The weighted adjacency of M without the edges u == v: the lists of arrow_adj_build (incoming == 0) or arrow_adj_build_in
 * (incoming != 0), in the same order, each entry carrying its fp32 weight (duplicates of (u, v) in any order).  Lists
 * longer than 512 entries are also listed as 512-entry segments.  The out-adjacency gets the frontier record of
 * arrow_adj_build_weighted and serves every call that takes a weighted push adjacency (as one without self-loops).
 * Memory and refusals: those of arrow_adj_build_weighted.  Synchronises. */
int  arrow_adj_build_loopfree(arrow_ctx *ctx, int n_parts, const int *csrs, const int *maps, int64_t n_vertices, int incoming,
                              int *adj_out);
/* Shortest-path counts over the tight pairs of a min-plus fixed point.  dist (D) and x0 (X0, the features the fixed-point
 * loop started from) are fp32, state int32 and sigma float64 tiles, all [n x k] with n the adjacencies' vertices.  An
 * entry u -> v of weight a is tight in column s when D[u, s] < D[v, s] < +inf and fl(a + D[u, s]) == D[v, s] (a +inf
 * weight or an overflowing sum never reaches an element that is not reached); the pair (u, v) is tight when one of its
 * entries is.  S_s = {v : D[v, s] finite and D[v, s] == X0[v, s]}.  sigma[v, s] = 0 where D[v, s]
 * is not finite, else [v in S_s] + the sum of sigma[u, s] over the distinct tight pairs u -> v, summed over v's in-list in
 * ascending order, 512 entries at a time, the partials added in order (no floating-point atomics).  The tight pairs form
 * a DAG per column: state receives -1 where D is not finite, else -(depth + 2), the depth being the round of Kahn's
 * algorithm that finalised the element; the rows of each round are kept in out_adj's history (4 bytes per row and round
 * with an element at that depth; the buffer doubles and holds up to twice that, plus 4 n bytes).  *rounds (may be NULL)
 * receives the rounds, *entries_read (may be NULL) the list entries read, once per row and 32-column word taking part in
 * a pass.  Temporary device memory of 4 n bytes.  ARROW_ERR_ARG: adjacencies that are not the loop-free in- and
 * out-adjacency of the same vertices, other tile types or shapes, two tiles aliasing; ARROW_ERR_UNSUPPORTED: k > 8192,
 * graph capture.  Synchronises after every round. */
int  arrow_wpaths_counts(arrow_ctx *ctx, int in_adj, int out_adj, int x0_buf, int dist_buf, int state_buf, int sigma_buf,
                         int64_t *rounds, int64_t *entries_read);
/* Dependencies over the rounds kept by the last arrow_wpaths_counts on out_adj with this state tile, from the deepest to
 * round 0: delta[v, s] = 0 for v in S_s, else sigma[v, s] * the sum of fl((1 + delta[w, s]) / sigma[w, s]) over the
 * distinct tight pairs v -> w with sigma[w, s] != 0 (a successor without paths, which a loop cut short by max_steps can
 * leave, adds nothing), summed like the counts over v's out-list, for every element with a finite D; the other
 * elements of delta are left alone.  The tiles are those of arrow_wpaths_counts, unchanged since, and delta a float64 tile
 * of their shape.  *entries_read (may be NULL; then the call does not synchronise) receives the out-list entries read.
 * ARROW_ERR_ARG: those of arrow_wpaths_counts, and no rounds of it kept for the state tile. */
int  arrow_wpaths_dependencies(arrow_ctx *ctx, int out_adj, int x0_buf, int dist_buf, int state_buf, int sigma_buf, int delta_buf,
                               int64_t *entries_read);

/* ---- personalized PageRank (one GPU, plus-times on float32 or float64 tiles) ---------------------------------------------- */
/* Every column reduction below (sigma, the dangling mass m, the residual r) runs in float64 over fixed 512-row chunks from
 * row 0: sequential in ascending rows inside a chunk, the chunk partials then added in ascending chunk order.  No
 * floating-point atomics: the results depend neither on the grid nor on the schedule.  The float64 arithmetic is separately
 * rounded (no contraction). */
/* Out-weights of the operator M of arrow_adj_build's parts, self-loops and duplicates included: w[u] (w_buf, ARROW_F64
 * [n_vertices x 1]) is the float64 sum, from +0 and in (part, entry) order, of the values of the entries whose edge
 * map(c) -> map(r) leaves u (an end at -1: not an edge); inv[u] (inv_buf, the blocks' element type T, [n_vertices x 1]) is
 * fl_T(1 / w[u]) from a float64 divide, 0 where w[u] == 0 (u is dangling).  One pass writes a key per entry, a stable radix
 * sort groups them by source and one thread per vertex sums its run.  *bad_entries receives the edges whose value is
 * negative, NaN or +-inf (-0 is allowed), *dangling the vertices with w == 0, *bad_inverses the other vertices whose
 * inverse is not finite or 0 (each pointer may be NULL).  Temporary device memory of 24 bytes per entry plus the sort's
 * storage is freed before the call returns.  ARROW_ERR_ARG: the refusals of arrow_adj_build, parts of different element
 * types, w / inv of another type or shape; ARROW_ERR_RANGE: 2^31 entries or more; ARROW_ERR_UNSUPPORTED: during graph
 * capture.  Synchronises. */
int  arrow_out_weights(arrow_ctx *ctx, int n_parts, const int *csrs, const int *maps, int64_t n_vertices, int w_buf, int inv_buf,
                       int64_t *bad_entries, int64_t *dangling, int64_t *bad_inverses);
/* A values-only copy of a block (ARROW_F32 or ARROW_F64) whose entry (r, c) of value a holds fl_T(a * scale[map(c)])
 * (map -1: the identity; 0 where the column or its image is -1); scale_buf is a [rows x 1] tile of the block's type that
 * covers every (mapped) column.  Row pointers, indices, long-row lists and tile lists are shared with the source, which
 * may itself be a remapped copy (arrow_csr_remap_columns): arrow_csr_free refuses the source while the copy lives.  The
 * copy owns (nnz + 8) values.  Synchronises. */
int  arrow_csr_scale_columns(arrow_ctx *ctx, int csr, int map, int scale_buf, int *csr_out);
/* The restart of personalized PageRank.  x_buf holds X0 (T [n x k], T float32 or float64), inv_buf the inverse
 * out-weights (T [n x 1], 0 marking the dangling rows), s_buf receives S (T [n x k]), scratch_buf is float64
 * [ceil(n / 512) x 2k] and state_buf float64 [4 x k].  sigma_s = the chunked float64 sum of column s.  A column is bad
 * when it holds a negative, NaN or +-inf value or sigma_s is not a positive finite number; *bad_columns (may be NULL)
 * receives their number, *first_bad_column (may be NULL) the smallest (-1: none) and col_sums (k host doubles, may be
 * NULL) sigma.  When no column is bad, S[v, s] = fl_T(X0[v, s] / sigma_s) (float64 divide) and state row 0 receives m_0,
 * the dangling mass of S; rows 2 and 3 hold sigma and the bad flags.  x_buf is never written.  The grid of this pass and of
 * arrow_pagerank_update follows ARROW_OPT_SPMM_SM_LIMIT and ARROW_OPT_SPMM_CTAS_PER_SM and changes no bit.  ARROW_ERR_ARG:
 * other types or shapes, two tiles aliasing; ARROW_ERR_UNSUPPORTED: graph capture.  Synchronises. */
int  arrow_pagerank_restart(arrow_ctx *ctx, int x_buf, int inv_buf, int s_buf, int scratch_buf, int state_buf, double *col_sums,
                            int64_t *bad_columns, int64_t *first_bad_column);
/* One iterate of personalized PageRank after the step Y = M^ p_t (y_buf): with beta = fl(1 - alpha) and c_s = fl(beta +
 * fl(alpha * m_t[s])), m_t in state row 0, p_{t+1}[v, s] = fl_T(fl(fl(alpha * Y[v, s]) + fl(c_s * S[v, s]))) is written over
 * Y in place.  The same pass sums the chunk partials of m_{t+1} (the dangling mass of p_{t+1}) and of r_{t+1}[s] = the sum
 * of |fl(p_{t+1}[v, s] - p_t[v, s])|; a second kernel adds them in order into state rows 0 and 1 and residuals (k host
 * doubles, may be NULL) receives r_{t+1}.  Traffic: Y, p and S read, p_{t+1} written.  Tiles as arrow_pagerank_restart,
 * p_buf and y_buf T [n x k].  ARROW_ERR_ARG: alpha outside [0, 1) or NaN, other types or shapes, two tiles aliasing;
 * ARROW_ERR_UNSUPPORTED: graph capture.  Synchronises. */
int  arrow_pagerank_update(arrow_ctx *ctx, int y_buf, int p_buf, int s_buf, int inv_buf, int scratch_buf, int state_buf,
                           double alpha, double *residuals);

/* ---- connected components (one GPU, any element type of the blocks) ------------------------------------------------------ */
/* Weakly connected components of the operator of arrow_adj_build's parts: the vertices are 0 .. n_vertices - 1 and every
 * entry (r, c) gives the undirected edge map(c) -- map(r), whatever its value (0, NaN and +-inf included); an end at -1 and
 * u == v give none.  labels_buf (ARROW_I32 [n_vertices x 1]) receives, for every vertex, the smallest vertex of its
 * component; *n_components (may be NULL) the number of v with labels[v] == v; sizes_buf (ARROW_I32 [n_vertices x 1], -1:
 * none) the member count of the component labelled r at row r and 0 at the rows that are not labels.  The answer is unique,
 * so no bit depends on the grid (which follows ARROW_OPT_SPMM_SM_LIMIT and ARROW_OPT_SPMM_CTAS_PER_SM and changes no
 * bit) or on the schedule.  A lock-free union-find over labels_buf itself (DESIGN.md §4): every parent is at most its vertex,
 * a hook CASes the larger root onto the smaller, one pass takes every entry (warps over 256-entry chunks, so a long row is
 * split across warps) and a second sets every label to its root.  No other device memory beyond an 8-byte counter.
 * ARROW_ERR_HANDLE / ARROW_ERR_ARG: the refusals of arrow_adj_build, tiles of another type or shape, sizes aliasing
 * labels; ARROW_ERR_RANGE: n_vertices of 2^31 - 1 or more; ARROW_ERR_UNSUPPORTED: during graph capture.  Synchronises. */
int  arrow_connected_components(arrow_ctx *ctx, int n_parts, const int *csrs, const int *maps, int64_t n_vertices,
                                int labels_buf, int sizes_buf, int64_t *n_components);

/* ---- predecessors of the tropical semirings (one GPU, fp32) ------------------------------------------ */
/* The product of arrow_spmm_sr over (value, label) pairs.  A candidate of row r is an entry p whose column c is valid
 * (not a skipped -1) and differs from the row's own label self(r); its value is fl(A[r,p] + X[c]) and its label c.
 * The witness of an element is the lexicographic ⊕ of its candidates: the better value wins (smaller for MIN_PLUS,
 * larger for MAX_PLUS), equal values (-0 == +0) go to the smaller label; a NaN term never wins; no candidate gives
 * (⊕ identity, -1).  The addend pair (add_val, add_lab)[add_map[r]] is ⊕-ed in where add_map[r] >= 0.  Exact: the
 * result does not depend on the kernel, the grid or the order of the terms.
 *   row_labels: map with self(r) per row (-1: none), or -1: self(r) = r
 *   dist_buf < 0:  pair out, values to val_out (fp32), labels to lab_out (int32)
 *   dist_buf >= 0: parents to lab_out: P[r] = label where D[r] (row r of dist_buf; it may be x_buf) is not the ⊕
 *                  identity and the witness value equals it, else -1; values to val_out when val_out >= 0
 *   add_val / add_lab / add_map: all three or none (-1)
 * Every output has the block's rows and X's k; no output aliases an input or the other output.  ARROW_SR_PLUS_TIMES,
 * MAX_MIN / MIN_MAX (ties are the rule there and this witness makes cycles: arrow_sr_tree_parents) and fp64 operands:
 * ARROW_ERR_UNSUPPORTED; mixed or wrong element types, bad shapes, aliasing, an unknown semiring
 * code: ARROW_ERR_ARG. */
int  arrow_spmm_sr_witness(arrow_ctx *ctx, int csr, int x_buf, int row_labels, int val_out, int lab_out, int add_val,
                           int add_lab, int add_map, int dist_buf, int semiring);

/* Multi-source gather over NVLink peer memory: `map` holds GLOBAL source rows; source s owns global
 * rows [row_bounds[s], row_bounds[s+1]) and src_bufs[s] is its (wrapped / IPC-imported) tile. */
int  arrow_gather_rows_multi(arrow_ctx *ctx, int dst_buf, const int *src_bufs,
                             const int64_t *row_bounds, int n_src, int map, int flags);

/* ---- the fused multi-GPU step ------------------------------------------------------------------- */
/* A pointer table holds one destination per row: tile bufs[which[i]], row row[i] (which[i] < 0: the row is dropped).
 * The tiles may be peer GPUs' memory (arrow_ipc_import): a SpMM with a pointer table delivers every result row
 * straight to the GPU that needs it -- the backward exchange (pack + Alltoallv + scatter-add,
 * arrow_dec_mpi.py:421, 442-475, 437) folded into the epilogue as NVLink stores. */
int  arrow_ptrtable_upload(arrow_ctx *ctx, const int *bufs, int n_bufs, const int32_t *which, const int64_t *row,
                           int64_t n, int *table_out);
int  arrow_ptrtable_free(arrow_ctx *ctx, int table);
/* Generalised product.  Columns < x_split read X[col], columns >= x_split read X2[col - x_split] (x2_buf < 0: X only):
 * the feature operand of a level > 0 is [this GPU's level-0 tile | receive region filled by its peers], never
 * materialised as a tile of its own (forward exchange, arrow_dec_mpi.py:507-550, folded into the column indices).
 * out_table >= 0: row r is written to table[r] (c_buf may be -1); else to C[r].  add_buf / add_map as arrow_spmm_add.
 * An fp64 launch with x2_buf or out_table returns ARROW_ERR_UNSUPPORTED. */
int  arrow_spmm_ex(arrow_ctx *ctx, int csr, int x_buf, int x2_buf, int64_t x_split, int c_buf, int out_table,
                   int add_buf, int add_map, int variant);
/* Push: for item i in [item_bounds[d], item_bounds[d+1]):  dst_bufs[d][i - item_bounds[d]] = src[map[i]].
 * The forward exchange in one pass: local gather, sequential posted stores into each peer's receive region. */
int  arrow_push_rows(arrow_ctx *ctx, const int *dst_bufs, const int64_t *item_bounds, int n_dst, int src_buf, int map);
/* out(r) = sum_s src_bufs[s][r] (source order, deterministic) for r < rows; out(r) = table[r] when out_table >= 0 and the
 * entry is non-null, else dst_buf[r] (dst_buf may be -1: rows without a table entry are skipped).  The reduction of
 * the partial head tiles (Reduce, arrow_slim_mpi.py:116) in one launch, reading the peers over NVLink. */
int  arrow_reduce_rows(arrow_ctx *ctx, int dst_buf, int out_table, const int *src_bufs, int n_src, int64_t rows);

/* ---- CUDA graphs: record a whole step once, replay it with one call ------------------------------ */
/* Between begin and end every launch on the main lane (and on lanes forked from / joined back into it with
 * arrow_lane_wait) is recorded, not executed.  Run the step once un-captured first (lazy allocations). */
int  arrow_graph_begin(arrow_ctx *ctx);
int  arrow_graph_end(arrow_ctx *ctx, int *graph_out);
int  arrow_graph_launch(arrow_ctx *ctx, int graph);
int  arrow_graph_free(arrow_ctx *ctx, int graph);

/* ---- cross-process peer memory (one process per GPU; NVLink P2P through CUDA IPC) -------------- */
/* handle = 64-byte cudaIpcMemHandle_t + 8-byte offset of the tile inside the exported allocation + padding */
#define ARROW_IPC_HANDLE_BYTES 80
int  arrow_ipc_export(arrow_ctx *ctx, int buf, void *handle);
int  arrow_ipc_import(arrow_ctx *ctx, const void *handle, int64_t rows, int k, int *buf_out);
/* Device-side barrier across `world` ranks over peer-mapped flag words (no host sync, no NCCL):
 * flags_buf[s] is rank s's flag tile (>= world words), my slot = rank.  The epoch counter is device resident (one per
 * lane), so the launch can be part of a captured graph.  A barrier that waits longer than ARROW_OPT_BARRIER_TIMEOUT_MS
 * sets a device flag; arrow_sync / arrow_lane_sync then fail and the context refuses further launches. */
int  arrow_peer_barrier(arrow_ctx *ctx, const int *flag_bufs, int rank, int world);

/* ---- timing (CUDA events on the context's stream) ----------------------------------------------- */
#define ARROW_MAX_TIMERS 32
int  arrow_timer_start(arrow_ctx *ctx, int slot);
int  arrow_timer_stop(arrow_ctx *ctx, int slot);
int  arrow_timer_elapsed_ms(arrow_ctx *ctx, int slot, float *ms);   /* synchronises on the stop event */
/* number of kernels this context has launched so far (bench.py's gpu_launches) */
int  arrow_launch_count(arrow_ctx *ctx, int64_t *count);

/* Run every kernel a step with `k` feature columns can launch once, on tiny operands.  CUDA loads a kernel lazily at
 * its first launch and loading synchronises the context: if that happens while arrow_peer_barrier spins on another lane
 * (or, with several rank threads in one process, in another rank) the step hangs until the barrier times out.  Call it
 * after arrow_ctx_create, before the first barrier -- or start the process with CUDA_MODULE_LOADING=EAGER. */
int  arrow_preload_kernels(arrow_ctx *ctx, int k);

/* measurement helpers used by bench.py: write `bytes` of scratch (L2 flush) */
int  arrow_l2_flush(arrow_ctx *ctx);

#ifdef __cplusplus
}
#endif
#endif /* ARROW_B200_H */
