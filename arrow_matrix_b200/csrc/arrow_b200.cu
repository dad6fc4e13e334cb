// libarrow_b200.so -- hand-written sm_90a kernels + C ABI for the arrow-decomposed SpMM hot path.
//
// What each piece replaces in the reference (spcl/arrow-matrix, paths relative to its repository root):
//   k_spmm_*            scipy `csr @ dense` / cupy->cuSPARSE SpMM at arrow_slim_mpi.py:109-111,125-127,
//                       142-144,190,211,231 and arrow_mpi.py:198-219,250-269,289-291,323
//   csr upload (once)   common/sp2cp.py:6-16 (_sp2cp, redone every iteration by the reference)
//   rowmap epilogue     arrow_dec_mpi.py:421,437  (pack + alltoallv + `C_i[perm] += recvbuf`)
//   remapped columns    arrow_dec_mpi.py:526,544  (`feature_tile()[perm]` + `C_i[perm] = recvbuf`)
//   k_gather_rows*      the same two exchanges as standalone (un-fused / cross-GPU) steps
//
// Layout: CSR = int32 indptr (rebased to 0) / int32 indices / fp32 values; dense tiles row-major fp32.
// All kernels are HBM/L2-bandwidth bound gathers (about 2 FLOP/B): no tensor cores on purpose.
#include "../../include/arrow_b200.h"

#include <cuda_runtime.h>
#include <ctype.h>
#include <dlfcn.h>
#include <sched.h>
#include <sys/mman.h>
#include <sys/syscall.h>
#include <unistd.h>
#include <stdint.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <cub/device/device_radix_sort.cuh>

#include <algorithm>
#include <cmath>
#include <map>
#include <mutex>
#include <type_traits>
#include <string>
#include <vector>

// ------------------------------------------------------------------------------------------------
// context + handle tables
// ------------------------------------------------------------------------------------------------
namespace {

struct DenseBuf {
    float *p = nullptr;               // element type per `dtype` (double * for ARROW_F64, int * for ARROW_I32)
    int64_t rows = 0;
    int k = 0;
    int dtype = ARROW_F32;
    bool owned = false;
    bool ipc = false;
    void *ipc_base = nullptr;
    bool live = false;
};

struct LongTask {      // one segment of a long row
    int row;
    int begin;         // nnz offsets (rebased)
    int end;
    int slot;          // partial-sum slot
};

struct Csr {
    int64_t n_rows = 0, n_cols = 0, nnz = 0;
    int *indptr = nullptr;
    int *indices = nullptr;
    float *vals = nullptr;            // element type per `dtype` (double * for ARROW_F64)
    int dtype = ARROW_F32;
    bool owns_indptr = false, owns_indices = false, owns_vals = false;
    bool may_skip = false;            // indices may contain -1 (remapped through a partial map)
    int64_t max_row_nnz = 0;
    // long rows (nnz > threshold) are processed by whole CTAs in segments, then reduced in order
    int n_long_rows = 0;
    int n_long_tasks = 0;
    LongTask *long_tasks = nullptr;   // device
    int *long_rows = nullptr;         // device: row ids
    int *long_first = nullptr;        // device: first slot of each long row (n_long_rows+1)
    bool owns_long = false;
    int long_threshold = 0;
    // row tiles for the CSR-streaming kernels: {row_begin, row_end, nnz_begin, nnz_end}, one list per TILE_LISTS entry
    // (every list is empty or none is: each covers every row that is not long)
    int4 *tiles[4] = {};
    int n_tiles[4] = {};
    int parent = -1;                  // handle of the block whose indptr / values / tiles this one shares (remapped copy)
    int children = 0;                 // live remapped copies that share this block's arrays
    bool live = false;
};

struct IdxMap {
    int *p = nullptr;
    int64_t n = 0;
    int64_t limit = 0;
    bool live = false;
};

struct Timer {
    cudaEvent_t a = nullptr, b = nullptr;
};

struct PtrTable {                     // one device pointer per row: where a SpMM / reduction writes that row
    float **p = nullptr;
    int64_t n = 0;
    int k = 0;
    bool live = false;
};

struct Adj {                          // push adjacency (arrow_adj_build / arrow_adj_build_weighted) and its frontier record
    int64_t n = 0, m = 0;             // vertices (level-0 rows), edges
    int *indptr = nullptr;            // device: n + 1 row pointers of the transposed matrix (row u: destinations v)
    int *indices = nullptr;           // device: m destinations
    float *values = nullptr;          // device: m fp32 weights, beside indices (weighted adjacency only)
    bool weighted = false;
    int *front_rows = nullptr;        // device, n: rows of the last arrow_bits_mark_frontier, in list order
    int *front_off = nullptr;         // device, n: first edge offset of each of them, increasing with the list position
    int64_t n_front = 0, front_edges = 0;
    int tag = -1;                     // dense handle whose fresh rows the record holds (-1: no record)
    const void *tag_p = nullptr;      // and its storage and width (a freed and re-used handle does not match)
    int tag_k = 0;
    bool incoming = false;            // in-adjacency (arrow_adj_build_in): row v lists its sources u; no frontier record
    int4 *segs = nullptr;             // device: {v, first, end, 0} per segment of the rows longer than PARENT_SEG entries,
    int n_segs = 0;                   //   which arrow_bits_parents and the betweenness passes split across warps
    bool has_segs = false;            // segs lists every list longer than PARENT_SEG (built for the in-adjacency, and on
                                      //   arrow_bits_dependencies' first call for the push adjacency)
    double *seg_part = nullptr;       // device: [n_segs x k] partial sums of the betweenness segment passes
    size_t seg_part_bytes = 0;
    int *hist = nullptr;              // device: the frontier records kept by arrow_adj_keep_record, level after level
    int64_t hist_cap = 0;             //   (its capacity in rows)
    std::vector<int64_t> hist_off;    // host: level h's rows are hist[hist_off[h], hist_off[h + 1])
    bool loopfree = false;            // weighted without the edges u == v (arrow_adj_build_loopfree)
    const void *wp_tag_p = nullptr;   // the state tile whose rounds the history holds (arrow_wpaths_counts), and its width
    int wp_tag_k = 0;
    bool live = false;
};

thread_local std::string g_create_error;
std::mutex g_numa_mu;                         // arrow_host_alloc_numa bookkeeping (pointer -> mapped length)
std::map<void *, size_t> g_numa_allocs;

}  // namespace

struct arrow_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    int sm_count = 132;
    long long l2_bytes = 50LL << 20;  // cudaDeviceProp::l2CacheSize
    std::string err;
    std::vector<DenseBuf> dense;
    std::vector<Csr> csrs;
    std::vector<IdxMap> maps;
    std::vector<Adj> adjs;
    Timer timers[ARROW_MAX_TIMERS];
    int64_t launches = 0;
    int long_threshold = 512;
    int long_segment = 2048;
    int l2_hints_plain = 3;           // arrow_set_option(ARROW_OPT_L2_HINTS_PLAIN)
    int l2_hints_fused = 0;           // arrow_set_option(ARROW_OPT_L2_HINTS_FUSED)
    int big_tiles = 1;                // arrow_set_option(ARROW_OPT_BIG_TILES): 128-row tiles when k <= 32
    int tile_rows = 0;                // arrow_set_option(ARROW_OPT_TILE_ROWS): 0 = the L2 budget picks the tile list, else its rows
    int spmm_ctas_per_sm = 0;         // arrow_set_option(ARROW_OPT_SPMM_CTAS_PER_SM): 0 = as many as fit
    int prefetch_plain = 0;           // arrow_set_option(ARROW_OPT_PREFETCH): low nibble = plain launches, high nibble = fused launches;
    int prefetch_fused = 0;           //   0 none, 1 bulk L2 prefetch of the current tile's X rows, 2 of the next tile's (look-ahead)
    int rows_per_group = 0;           // arrow_set_option(ARROW_OPT_ROWS_PER_GROUP): 0 = default (one row), 1 / 2 forced
    int spmm_sm_limit = 0;            // arrow_set_option(ARROW_OPT_SPMM_SM_LIMIT): cap on the SMs a SpMM grid covers (0 = all)
    int clock_khz = 2000000;          // SM clock (kHz) for the barrier time-out
    int tile_kernel = 1;              // arrow_set_option(ARROW_OPT_TILE_KERNEL): 1 = round-1 kernel for the launches it covers, 0 = generalised kernel everywhere
    int force_skip_path = 0;          // arrow_set_option(ARROW_OPT_FORCE_PREDICATED): measurement switch
    int smem_carveout = -1;           // arrow_set_option(ARROW_OPT_SMEM_CARVEOUT): preferred shared-memory carve-out (percent) of the tile kernel
    int push_interleave = 1;          // arrow_set_option(ARROW_OPT_PUSH_INTERLEAVE): 1 = the push grid serves all destinations at once
    int push_ctas = 0;                // arrow_set_option(ARROW_OPT_PUSH_CTAS): grid of the NVLink push kernel (0 = default)
    long long barrier_timeout_ms = 30000;   // arrow_set_option(ARROW_OPT_BARRIER_TIMEOUT_MS)
    bool poisoned = false;            // a peer barrier timed out: later launches are refused (results would be racy)
    float *long_scratch[ARROW_N_LANES] = {};    // [slots][k] partial sums of long-row segments, per lane
    size_t long_scratch_bytes[ARROW_N_LANES] = {};
    void *flush_buf = nullptr;
    size_t flush_bytes = 0;
    unsigned int *barrier_epoch = nullptr;        // device: one epoch counter per lane (each lane has its own flag set);
                                                  // device-resident so that a captured CUDA graph can be replayed
    int cur_lane = 0;                             // lane used by the launches that follow (arrow_set_lane)
    int *dev_status = nullptr;        // device-side status word (barrier timeout)
    int *tile_ticket = nullptr;       // device: per lane {next tile, finished CTAs} of the dynamic tile scheduler
    std::vector<PtrTable> ptrtabs;
    std::vector<cudaGraphExec_t> graphs;
    std::vector<int64_t> graph_kernels;           // kernels recorded in each graph (arrow_launch_count stays truthful under replay)
    int64_t capture_launches0 = 0;
    bool capturing = false;
    cudaStream_t lanes[ARROW_N_LANES] = {};   // lane 0 = main stream
    cudaEvent_t lane_events[ARROW_N_LANES] = {};
    cudaEvent_t user_events[ARROW_MAX_EVENTS] = {};
};

namespace {

int fail(arrow_ctx *ctx, int code, const char *fmt, ...) __attribute__((format(printf, 3, 4)));
int fail(arrow_ctx *ctx, int code, const char *fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    if (ctx) ctx->err = buf; else g_create_error = buf;
    return code;
}

cudaStream_t cur_stream(arrow_ctx *ctx) {
    return (ctx->cur_lane > 0 && ctx->lanes[ctx->cur_lane]) ? ctx->lanes[ctx->cur_lane] : ctx->stream;
}

#define CUDA_TRY(ctx, expr)                                                                   \
    do {                                                                                      \
        cudaError_t _e = (expr);                                                              \
        if (_e != cudaSuccess)                                                                \
            return fail((ctx), ARROW_ERR_CUDA, "%s failed: %s (%s:%d)", #expr,                \
                        cudaGetErrorString(_e), __FILE__, __LINE__);                          \
    } while (0)

#define CHECK_CTX(ctx)                                                                        \
    do {                                                                                      \
        if (!(ctx)) return fail(nullptr, ARROW_ERR_ARG, "null context");                      \
        cudaError_t _e = cudaSetDevice((ctx)->device);                                        \
        if (_e != cudaSuccess)                                                                \
            return fail((ctx), ARROW_ERR_CUDA, "cudaSetDevice(%d): %s", (ctx)->device,        \
                        cudaGetErrorString(_e));                                              \
    } while (0)

cudaStream_t cur_stream(arrow_ctx *ctx);

template <class T>
int new_slot(std::vector<T> &v) {
    for (size_t i = 0; i < v.size(); ++i)
        if (!v[i].live) return (int)i;
    v.emplace_back();
    return (int)v.size() - 1;
}

DenseBuf *get_dense(arrow_ctx *ctx, int h) {
    if (h < 0 || h >= (int)ctx->dense.size() || !ctx->dense[h].live) return nullptr;
    return &ctx->dense[h];
}
Csr *get_csr(arrow_ctx *ctx, int h) {
    if (h < 0 || h >= (int)ctx->csrs.size() || !ctx->csrs[h].live) return nullptr;
    return &ctx->csrs[h];
}
IdxMap *get_map(arrow_ctx *ctx, int h) {
    if (h < 0 || h >= (int)ctx->maps.size() || !ctx->maps[h].live) return nullptr;
    return &ctx->maps[h];
}
Adj *get_adj(arrow_ctx *ctx, int h) {
    if (h < 0 || h >= (int)ctx->adjs.size() || !ctx->adjs[h].live) return nullptr;
    return &ctx->adjs[h];
}

inline size_t dtype_size(int dtype) { return dtype == ARROW_F64 ? 8 : 4; }
inline const char *dtype_name(int dtype) {
    return dtype == ARROW_F64 ? "float64" : (dtype == ARROW_I32 ? "int32" : (dtype == ARROW_B1 ? "bits" : "float32"));
}
// int32 tiles hold labels (arrow_spmm_sr_witness): only the allocation, copies and that launch accept them
#define REFUSE_I32(ctx, d, what)                                                                                   \
    do {                                                                                                           \
        if ((d) != nullptr && (d)->dtype == ARROW_I32)                                                             \
            return fail((ctx), ARROW_ERR_ARG, "%s: int32 tiles hold labels, no arithmetic runs on them", (what));  \
    } while (0)
// bit tiles run the (or, and) launches of one GPU only
#define REFUSE_B1(ctx, d, what)                                                                                    \
    do {                                                                                                           \
        if ((d) != nullptr && (d)->dtype == ARROW_B1)                                                              \
            return fail((ctx), ARROW_ERR_ARG, "%s: bit tiles run the (or, and) launches of one GPU only", (what)); \
    } while (0)
// uint32 words per row of a bit tile: one bit per column; a row of k <= 32 columns is one word (its own kernel instances,
// 4-byte gathers: measured faster than a padded 16-byte row, DESIGN.md section 2), wider rows are padded to a multiple of
// 4 words so that they are whole 16-byte vectors (the uint4 gathers of the bit kernels)
inline int bit_row_words(int k) { return k <= 32 ? 1 : (((k + 31) / 32) + 3) & ~3; }
inline size_t row_bytes(int dtype, int k) { return dtype == ARROW_B1 ? (size_t)bit_row_words(k) * 4 : (size_t)k * dtype_size(dtype); }
// first byte of row `r` of a dense tile
inline char *dense_row(const DenseBuf *d, int64_t r) { return (char *)d->p + (size_t)r * row_bytes(d->dtype, d->k); }

// frees whatever device arrays the block owns (cudaFree waits for the device, so no launch can still read them)
void csr_release(Csr &c) {
    if (c.owns_indptr) cudaFree(c.indptr);
    if (c.owns_indices) cudaFree(c.indices);
    if (c.owns_vals) cudaFree(c.vals);
    if (c.owns_long) {
        cudaFree(c.long_tasks);
        cudaFree(c.long_rows);
        cudaFree(c.long_first);
        for (int4 *p : c.tiles) cudaFree(p);
    }
    c = Csr();
}

void adj_release(Adj &a) {
    cudaFree(a.indptr);
    cudaFree(a.indices);
    cudaFree(a.values);
    cudaFree(a.front_rows);
    cudaFree(a.front_off);
    cudaFree(a.segs);
    cudaFree(a.hist);
    cudaFree(a.seg_part);
    a = Adj();
}

struct DevTmp {                       // scratch allocation released on every exit path
    void *p = nullptr;
    ~DevTmp() { if (p) cudaFree(p); }
};

// ------------------------------------------------------------------------------------------------
// device helpers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float4 f4_zero() { return make_float4(0.f, 0.f, 0.f, 0.f); }
__device__ __forceinline__ void f4_fma(float4 &acc, float a, const float4 &x) {
    acc.x = fmaf(a, x.x, acc.x);
    acc.y = fmaf(a, x.y, acc.y);
    acc.z = fmaf(a, x.z, acc.z);
    acc.w = fmaf(a, x.w, acc.w);
}
__device__ __forceinline__ void f4_add(float4 &acc, const float4 &x) {
    acc.x += x.x; acc.y += x.y; acc.z += x.z; acc.w += x.w;
}
__device__ __forceinline__ double2 d2_zero() { return make_double2(0.0, 0.0); }
__device__ __forceinline__ void d2_fma(double2 &acc, double a, const double2 &x) {
    acc.x = fma(a, x.x, acc.x);
    acc.y = fma(a, x.y, acc.y);
}
__device__ __forceinline__ void d2_add(double2 &acc, const double2 &x) {
    acc.x += x.x; acc.y += x.y;
}

struct SpmmArgs {
    const int *__restrict__ indptr;
    const int *__restrict__ indices;
    const float *__restrict__ vals;
    const float *__restrict__ X;
    float *__restrict__ C;
    const int *__restrict__ rowmap;   // nullptr: identity
    long long n_rows;
    int k;                            // feature columns
    int k4;                           // k / 4 (vector kernels)
    int long_threshold;               // rows with more entries are left to the long-row kernels
    const float *__restrict__ add_src;   // optional addend: C[r] = sum + add_src[add_map[r]] (add_map[r] >= 0), else nullptr
    const int *__restrict__ add_map;
    const float *__restrict__ X2;        // optional second X base: columns >= x_split address X2[col - x_split] (else nullptr)
    int x_split;
    float *const *__restrict__ out_ptr;  // optional destination pointer per row (nullptr entry = row dropped); overrides C / rowmap
};

// row `c` of the X operand of SpmmArgs / LongArgs, whose X pointers carry elements of type T.  Only float operands come
// in two parts (the C ABI refuses X2 for float64); for the others the test is compiled out, which lets ptxas unroll the
// entry loops of the row-parallel kernels.
template <class T, class Args>
__device__ __forceinline__ const T *x_row_ptr(const Args &a, int c) {
    if (std::is_same<T, float>::value && a.X2 != nullptr && c >= a.x_split)
        return reinterpret_cast<const T *>(a.X2) + (long long)(c - a.x_split) * a.k;
    return reinterpret_cast<const T *>(a.X) + (long long)c * a.k;
}

// ------------------------------------------------------------------------------------------------
// variant 0: a group of G lanes owns one row; every lane of the group reads the same index/value
// (hardware broadcast) and its own float4 slice of the X row.  UNROLL independent X gathers in flight.
// ------------------------------------------------------------------------------------------------
// __launch_bounds__(256, 4): without the min-blocks bound ptxas aims at full occupancy (<= 40 registers)
// and serialises every gather behind the FFMAs of the previous one; with it all UNROLL gathers of a
// batch are issued back to back (checked in SASS), which is what hides the L2 / HBM latency.
template <int G, int VPL, bool ROWMAP, bool ACC>
__global__ void __launch_bounds__(256, 4) k_spmm_direct(SpmmArgs a) {
    constexpr int RPW = 32 / G;
    constexpr int UNROLL = (VPL == 1) ? 8 : 4;
    const int lane = threadIdx.x & 31;
    const int gl = lane % G;                      // lane inside the group
    const int gi = lane / G;                      // group inside the warp
    const long long warps_total = (long long)gridDim.x * (blockDim.x >> 5);
    const long long warp_id = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const float4 *__restrict__ X4 = reinterpret_cast<const float4 *>(a.X);
    float4 *__restrict__ C4 = reinterpret_cast<float4 *>(a.C);
    const int k4 = a.k4;

    for (long long row = warp_id * RPW + gi; row < a.n_rows; row += warps_total * RPW) {
        const int s = __ldg(a.indptr + row);
        const int e = __ldg(a.indptr + row + 1);
        if (e - s > a.long_threshold) continue;
        long long orow = row;
        if (ROWMAP) {
            orow = __ldg(a.rowmap + row);
            if (orow < 0) continue;
        }
        float4 acc[VPL];
#pragma unroll
        for (int i = 0; i < VPL; ++i) acc[i] = f4_zero();

        for (int p = s; p < e; p += UNROLL) {
            int c[UNROLL];
            float v[UNROLL];
#pragma unroll
            for (int u = 0; u < UNROLL; ++u) {
                const bool ok = p + u < e;
                c[u] = ok ? __ldcs(a.indices + p + u) : -1;
                v[u] = ok ? __ldcs(a.vals + p + u) : 0.f;
            }
            float4 x[UNROLL][VPL];
#pragma unroll
            for (int u = 0; u < UNROLL; ++u)
#pragma unroll
                for (int i = 0; i < VPL; ++i) {
                    const int vec = gl + i * G;
                    x[u][i] = (c[u] >= 0 && vec < k4) ? __ldg(X4 + (long long)c[u] * k4 + vec) : f4_zero();
                }
#pragma unroll
            for (int u = 0; u < UNROLL; ++u)
#pragma unroll
                for (int i = 0; i < VPL; ++i) f4_fma(acc[i], v[u], x[u][i]);
        }
#pragma unroll
        for (int i = 0; i < VPL; ++i) {
            const int vec = gl + i * G;
            if (vec < k4) {
                float4 *dst = C4 + orow * k4 + vec;
                if (ACC) {
                    float4 old = *dst;
                    f4_add(acc[i], old);
                    *dst = acc[i];
                } else {
                    __stcs(dst, acc[i]);
                }
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// variant 1: the group loads G consecutive (index, value) pairs of its row with ONE coalesced request
// each and broadcasts them with width-G shuffles; the X gathers are issued UNROLL at a time.
// ------------------------------------------------------------------------------------------------
template <int G, int VPL, bool ROWMAP, bool ACC>
__global__ void __launch_bounds__(256, 4) k_spmm_shfl(SpmmArgs a) {
    constexpr int RPW = 32 / G;
    constexpr int UWANT = (VPL == 1) ? 8 : 4;
    constexpr int UNROLL = (G >= UWANT) ? UWANT : G;
    const int lane = threadIdx.x & 31;
    const int gl = lane % G;
    const int gi = lane / G;
    const long long warps_total = (long long)gridDim.x * (blockDim.x >> 5);
    const long long warp_id = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const float4 *__restrict__ X4 = reinterpret_cast<const float4 *>(a.X);
    float4 *__restrict__ C4 = reinterpret_cast<float4 *>(a.C);
    const int k4 = a.k4;

    // warp-uniform trip count: every lane of the warp runs the same number of row iterations
    for (long long row0 = warp_id * RPW; row0 < a.n_rows; row0 += warps_total * RPW) {
        const long long row = row0 + gi;
        int s = 0, e = 0;
        long long orow = -1;
        if (row < a.n_rows) {
            s = __ldg(a.indptr + row);
            e = __ldg(a.indptr + row + 1);
            orow = row;
            if (ROWMAP) orow = __ldg(a.rowmap + row);
            if (e - s > a.long_threshold || orow < 0) { e = s; orow = -1; }
        }
        const int len = e - s;
        const int maxlen = __reduce_max_sync(0xffffffffu, len);
        float4 acc[VPL];
#pragma unroll
        for (int i = 0; i < VPL; ++i) acc[i] = f4_zero();

        for (int base = 0; base < maxlen; base += G) {
            int myc = -1;
            float myv = 0.f;
            if (base + gl < len) {
                myc = __ldcs(a.indices + s + base + gl);
                myv = __ldcs(a.vals + s + base + gl);
            }
            const int cnt = min(G, maxlen - base);               // warp-uniform
            for (int u0 = 0; u0 < cnt; u0 += UNROLL) {
                int c[UNROLL];
                float v[UNROLL];
#pragma unroll
                for (int u = 0; u < UNROLL; ++u) {
                    c[u] = __shfl_sync(0xffffffffu, myc, (u0 + u) % G, G);
                    v[u] = __shfl_sync(0xffffffffu, myv, (u0 + u) % G, G);
                    if (u0 + u >= G) c[u] = -1;
                }
                float4 x[UNROLL][VPL];
#pragma unroll
                for (int u = 0; u < UNROLL; ++u)
#pragma unroll
                    for (int i = 0; i < VPL; ++i) {
                        const int vec = gl + i * G;
                        x[u][i] = (c[u] >= 0 && vec < k4) ? __ldg(X4 + (long long)c[u] * k4 + vec) : f4_zero();
                    }
#pragma unroll
                for (int u = 0; u < UNROLL; ++u)
#pragma unroll
                    for (int i = 0; i < VPL; ++i) f4_fma(acc[i], v[u], x[u][i]);
            }
        }
        if (orow >= 0) {
#pragma unroll
            for (int i = 0; i < VPL; ++i) {
                const int vec = gl + i * G;
                if (vec < k4) {
                    float4 *dst = C4 + orow * k4 + vec;
                    if (ACC) {
                        float4 old = *dst;
                        f4_add(acc[i], old);
                        *dst = acc[i];
                    } else {
                        __stcs(dst, acc[i]);
                    }
                }
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// variant 2: TMA-style staging.  Each warp stages the X rows its rows reference into shared memory
// with one cp.async.bulk (UBLKCP) per non-zero, completion tracked by a per-warp mbarrier, two stages
// deep, and accumulates out of shared memory.  No registers are spent on in-flight gathers.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t *bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra WAIT_DONE;\n"
        "bra WAIT_LOOP;\n"
        "WAIT_DONE:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
            smem_u32(dst_smem)),
        "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}

// ---- L2 eviction policies (createpolicy + .L2::cache_hint) ---------------------------------------------
// The X rows are the only data with reuse (each row of a block's panel is hit ~nnz/row times from L2);
// CSR streams and the C tile are touched once.  Marking the gathers evict_last and everything else
// evict_first keeps the streams from pushing the panels out of L2 (fused level > 0: DRAM traffic was
// 13.9 GB vs 8.1 GB algorithmic before the hints).
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
    uint64_t p;
    asm("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
    uint64_t p;
    asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ uint64_t l2_policy_evict_normal() {
    uint64_t p;
    asm("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ float4 ldg_f4_hint(const float4 *ptr, uint64_t pol) {
    float4 r;
    asm("ld.global.nc.L2::cache_hint.v4.f32 {%0,%1,%2,%3}, [%4], %5;"
        : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
        : "l"(ptr), "l"(pol));
    return r;
}
__device__ __forceinline__ float4 ld_f4_hint(const float4 *ptr, uint64_t pol) {      // coherent load (C tile RMW)
    float4 r;
    asm("ld.global.L2::cache_hint.v4.f32 {%0,%1,%2,%3}, [%4], %5;"
        : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
        : "l"(ptr), "l"(pol));
    return r;
}
__device__ __forceinline__ void st_f4_hint(float4 *ptr, const float4 &v, uint64_t pol) {
    asm volatile("st.global.L2::cache_hint.v4.f32 [%0], {%1,%2,%3,%4}, %5;" ::"l"(ptr), "f"(v.x), "f"(v.y), "f"(v.z),
                 "f"(v.w), "l"(pol)
                 : "memory");
}
// the same three accesses on 16 bytes of bits (ARROW_B1 tiles), and on the 4 bytes of a one-word bit row further below
__device__ __forceinline__ uint4 ldg_u4_hint(const uint4 *ptr, uint64_t pol) {
    uint4 r;
    asm("ld.global.nc.L2::cache_hint.v4.b32 {%0,%1,%2,%3}, [%4], %5;"
        : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
        : "l"(ptr), "l"(pol));
    return r;
}
__device__ __forceinline__ uint4 ld_u4_hint(const uint4 *ptr, uint64_t pol) {
    uint4 r;
    asm("ld.global.L2::cache_hint.v4.b32 {%0,%1,%2,%3}, [%4], %5;"
        : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
        : "l"(ptr), "l"(pol));
    return r;
}
__device__ __forceinline__ void st_u4_hint(uint4 *ptr, const uint4 &v, uint64_t pol) {
    asm volatile("st.global.L2::cache_hint.v4.b32 [%0], {%1,%2,%3,%4}, %5;" ::"l"(ptr), "r"(v.x), "r"(v.y), "r"(v.z),
                 "r"(v.w), "l"(pol)
                 : "memory");
}
__device__ __forceinline__ void bulk_g2s_hint(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar,
                                              uint64_t pol) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(
            smem_u32(dst_smem)),
        "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)), "l"(pol)
        : "memory");
}

constexpr int TMA_WARPS = 8;      // warps per CTA
constexpr int TMA_SLOTS = 16;     // X rows staged per stage per warp
constexpr int TMA_STAGES = 2;

// One warp per row (VPL float4 per lane).  The warp walks a stream of work items -- (row, chunk of up
// to TMA_SLOTS non-zeros) -- and keeps the NEXT item's X rows in flight while it accumulates the
// current one out of shared memory, so the pipeline spans row boundaries.
struct TmaItem {
    long long row;     // -1: end of stream
    long long orow;
    int p0;            // first nnz of this chunk
    int cnt;           // nnz in this chunk
    int last;          // chunk closes its row
    int myc;           // this lane's column (lane < cnt), -1 otherwise
    float myv;
};

template <int VPL, bool ROWMAP, bool ACC>
__global__ void __launch_bounds__(TMA_WARPS * 32) k_spmm_tma(SpmmArgs a) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int k4 = a.k4;
    const uint32_t row_bytes = (uint32_t)a.k * 4u;
    float *wbase = reinterpret_cast<float *>(smem_raw) + (size_t)warp * TMA_STAGES * TMA_SLOTS * a.k;
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem_raw + (size_t)TMA_WARPS * TMA_STAGES * TMA_SLOTS * row_bytes) +
                     warp * TMA_STAGES;
    if (lane == 0) {
        for (int st = 0; st < TMA_STAGES; ++st) mbar_init(&bars[st], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncwarp();
    uint32_t parity0 = 0u, parity1 = 0u;

    const long long warps_total = (long long)gridDim.x * TMA_WARPS;
    const long long warp_id = (long long)blockIdx.x * TMA_WARPS + warp;
    float4 *__restrict__ C4 = reinterpret_cast<float4 *>(a.C);

    // work-item iterator (all lanes hold identical copies)
    long long it_row = warp_id - warps_total;
    int it_p = 0, it_e = 0;
    long long it_orow = -1;
    auto next_item = [&](TmaItem &t) {
        while (it_p >= it_e) {                       // advance to the next non-empty, non-long, routed row
            it_row += warps_total;
            if (it_row >= a.n_rows) { t.row = -1; t.cnt = 0; t.myc = -1; t.myv = 0.f; t.last = 0; return; }
            const int s = __ldg(a.indptr + it_row);
            const int e = __ldg(a.indptr + it_row + 1);
            long long orow = it_row;
            if (ROWMAP) orow = __ldg(a.rowmap + it_row);
            if (orow < 0 || e - s > a.long_threshold) continue;
            it_orow = orow;
            it_p = s;
            it_e = e;
            if (s == e) {                            // empty row still has to store zeros / keep C
                t.row = it_row; t.orow = orow; t.p0 = s; t.cnt = 0; t.last = 1; t.myc = -1; t.myv = 0.f;
                return;
            }
        }
        t.row = it_row;
        t.orow = it_orow;
        t.p0 = it_p;
        t.cnt = min(TMA_SLOTS, it_e - it_p);
        it_p += t.cnt;
        t.last = (it_p >= it_e);
        t.myc = -1;
        t.myv = 0.f;
        if (lane < t.cnt) {
            t.myc = __ldcs(a.indices + t.p0 + lane);
            t.myv = __ldcs(a.vals + t.p0 + lane);
        }
    };
    auto issue = [&](const TmaItem &t, int st) {
        const unsigned valid = __ballot_sync(0xffffffffu, t.myc >= 0);
        if (lane == 0) mbar_expect_tx(&bars[st], (uint32_t)__popc(valid) * row_bytes);
        __syncwarp();
        if (t.myc >= 0)
            bulk_g2s(wbase + ((size_t)st * TMA_SLOTS + lane) * a.k, a.X + (long long)t.myc * a.k, row_bytes, &bars[st]);
    };

    float4 acc[VPL];
#pragma unroll
    for (int i = 0; i < VPL; ++i) acc[i] = f4_zero();

    TmaItem cur, nxt;
    int stage = 0;
    next_item(cur);
    if (cur.row >= 0) issue(cur, stage);
    while (cur.row >= 0) {
        next_item(nxt);
        if (nxt.row >= 0) issue(nxt, stage ^ 1);
        if (stage == 0) { mbar_wait(&bars[0], parity0); parity0 ^= 1u; }
        else            { mbar_wait(&bars[1], parity1); parity1 ^= 1u; }
        const float4 *sm4 = reinterpret_cast<const float4 *>(wbase + (size_t)stage * TMA_SLOTS * a.k);
        for (int u = 0; u < cur.cnt; ++u) {
            const int c = __shfl_sync(0xffffffffu, cur.myc, u);
            const float v = __shfl_sync(0xffffffffu, cur.myv, u);
            if (c >= 0) {
#pragma unroll
                for (int i = 0; i < VPL; ++i) {
                    const int vec = lane + i * 32;
                    if (vec < k4) f4_fma(acc[i], v, sm4[(size_t)u * k4 + vec]);
                }
            }
        }
        if (cur.last) {
#pragma unroll
            for (int i = 0; i < VPL; ++i) {
                const int vec = lane + i * 32;
                if (vec < k4) {
                    float4 *dst = C4 + cur.orow * k4 + vec;
                    if (ACC) {
                        float4 old = *dst;
                        f4_add(acc[i], old);
                        *dst = acc[i];
                    } else {
                        __stcs(dst, acc[i]);
                    }
                }
                acc[i] = f4_zero();
            }
        }
        __syncwarp();           // every lane is done with this stage before it is refilled
        cur = nxt;
        stage ^= 1;
    }
}

// ------------------------------------------------------------------------------------------------
// variant 3 (default): CSR streamed by TMA.  A persistent CTA walks row tiles (<= TILE_ROWS rows,
// <= TILE_NNZ non-zeros, built at upload).  One elected thread brings the tile's slice of indptr /
// indices / values into shared memory with three cp.async.bulk copies (UBLKCP) that complete on an
// mbarrier, one tile ahead of the math (two stages).  Warps then only issue the X gathers: a group of
// G lanes owns a row, reads (col, val) from shared memory (broadcast) and VPL float4 of the X row.
// ------------------------------------------------------------------------------------------------
constexpr int TILE_ROWS = 64;       // bounds of the tiles the TR = 64 kernel instances take
constexpr int TILE_NNZ = 1024;
constexpr int TILE_ROWS_BIG = 128;  // k <= 32: the panels are small, bigger tiles amortise the per-tile fixed cost
constexpr int TILE_NNZ_BIG = 2048;
// The row-tile lists every CSR carries (Csr::tiles[i]: <= rows, <= nnz entries).  The lists below TILE_LIST_SMALL fit the
// TR = 64 instances' bounds, so they run on the same kernels; only the window of rows in flight changes (tile_list_for).
struct TileListCaps { int rows, nnz; };
constexpr TileListCaps TILE_LISTS[] = {{16, 256}, {32, 512}, {TILE_ROWS, TILE_NNZ}, {TILE_ROWS_BIG, TILE_NNZ_BIG}};
constexpr int N_TILE_LISTS = 4;
constexpr int TILE_LIST_SMALL = 2;  // the TILE_ROWS list
constexpr int TILE_LIST_BIG = 3;    // the TILE_ROWS_BIG list (TR = 128 instances, k <= 32)
constexpr int TILE_CTAS_PER_SM = 4; // __launch_bounds__(TILE_THREADS, 4) of every tile kernel: the resident CTAs per SM
constexpr int TILE_L2_WINDOW_DIV = 4;   // the X rows of the window in flight may take 1/4 of the L2 (DESIGN section 3, lesson 2)
static_assert(sizeof(Csr::tiles) / sizeof(Csr::tiles[0]) == N_TILE_LISTS, "one tile list per TILE_LISTS entry");
constexpr int TILE_THREADS = 256;
constexpr int TILE_STAGES = 2;      // CSR slices in shared memory: tile t (math), t+1 (in flight).  A third stage (tried in round 2 for a
                                    // look-ahead prefetch) cost more L1 than it bought: the L1 data array is the landing buffer of the gathers in flight
template <int TR, int TN>
struct TileCfg {
    static constexpr int PTR_WORDS = TR + 8;           // row pointer slice (+ alignment slack)
    static constexpr int NNZ_WORDS = TN + 8;
    static constexpr int STAGE_WORDS = PTR_WORDS + 2 * NNZ_WORDS;
    static constexpr size_t SMEM_BYTES = (size_t)TILE_STAGES * STAGE_WORDS * 4 + 64;
};

// where a result row goes
constexpr int OUT_IDENTITY = 0;     // C[r]
constexpr int OUT_ROWMAP = 1;       // C[rowmap[r]]           (rows with rowmap[r] < 0 are dropped)
constexpr int OUT_ROWPTR = 2;       // *(out_ptr[r])          (device pointer per row: a local tile or a peer GPU's staging slot)

struct TileArgs {
    SpmmArgs a;
    const int4 *__restrict__ tiles;
    int n_tiles;
    int skip;            // indices may hold -1
    int *ticket;         // dynamic tile scheduler: [0] next tile, [1] CTAs that finished (the last one re-arms both)
    int l2_hints;        // bit 0: X gathers evict_last, bit 1: CSR / C streams evict_first
    int prefetch;        // 1: bulk L2 prefetch of the tile's X rows before the math (A/B switch, off by default)
};

__device__ __forceinline__ void bulk_prefetch_l2(const void *gptr, uint32_t bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(gptr), "r"(bytes) : "memory");
}
// ------------------------------------------------------------------------------------------------
// The round-1 tile kernel, verbatim (one row per lane group, identity / row-map output, no dual operand): kept as the
// production path of those launches.  The generalised kernel below produces the same numbers but its fused level-1
// launch (scattered first-touch gathers, latency bound) was slower than this code; ARROW_OPT_TILE_KERNEL switches
// between the two.
// ------------------------------------------------------------------------------------------------
template <int G, int VPL, bool ROWMAP, bool ACC, int TR, int TN>
__global__ void __launch_bounds__(TILE_THREADS, 4) k_spmm_tiles_v1(TileArgs t) {
    constexpr int TILE_PTR_WORDS = TileCfg<TR, TN>::PTR_WORDS;
    constexpr int TILE_NNZ_WORDS = TileCfg<TR, TN>::NNZ_WORDS;
    constexpr int TILE_STAGE_WORDS = TileCfg<TR, TN>::STAGE_WORDS;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    int *stage_base = reinterpret_cast<int *>(smem_raw);
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem_raw + (size_t)2 * TILE_STAGE_WORDS * 4);
    const SpmmArgs &a = t.a;
    constexpr int RPW = 32 / G;
    constexpr int UNROLL = (VPL >= 4) ? 2 : (VPL == 2 ? 4 : 8);
    constexpr int TAIL = (UNROLL >= 4) ? UNROLL / 2 : UNROLL;     // predicated tail batches
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const bool EXACT = (t.a.k4 == G * VPL);                       // every lane owns valid columns
    const int gl = lane % G;
    const int gi = lane / G;
    const int k4 = a.k4;
    const float4 *__restrict__ Xl = reinterpret_cast<const float4 *>(a.X) + gl;
    float4 *__restrict__ Cl = reinterpret_cast<float4 *>(a.C) + gl;
    const uint64_t pol_keep = (t.l2_hints & 1) ? l2_policy_evict_last() : l2_policy_evict_normal();
    const uint64_t pol_stream = (t.l2_hints & 2) ? l2_policy_evict_first() : l2_policy_evict_normal();

    if (threadIdx.x == 0) {
        mbar_init(&bars[0], 1);
        mbar_init(&bars[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    auto prefetch = [&](int tile, int st) {
        const int4 d = __ldg(t.tiles + tile);
        const int rb4 = d.x & ~3;
        const int a0 = d.z & ~3;
        const uint32_t ptr_bytes = (uint32_t)(((d.y - rb4 + 1) + 3) & ~3) * 4u;
        const uint32_t nnz_bytes = (uint32_t)(((d.w - a0) + 3) & ~3) * 4u;
        int *sp = stage_base + (size_t)st * TILE_STAGE_WORDS;
        mbar_expect_tx(&bars[st], ptr_bytes + 2u * nnz_bytes);
        bulk_g2s_hint(sp, a.indptr + rb4, ptr_bytes, &bars[st], pol_stream);
        if (nnz_bytes) {
            bulk_g2s_hint(sp + TILE_PTR_WORDS, a.indices + a0, nnz_bytes, &bars[st], pol_stream);
            bulk_g2s_hint(sp + TILE_PTR_WORDS + TILE_NNZ_WORDS, a.vals + a0, nnz_bytes, &bars[st], pol_stream);
        }
    };

    // Dynamic scheduling: the first tile is blockIdx.x, every further tile comes from an atomic ticket.  All CTAs
    // therefore work on one compact, moving window of ~gridDim.x consecutive tiles; a static round-robin lets
    // CTAs drift apart over the ~260 tiles each one processes at 10M rows and the live X panels fall out of L2
    // (measured: 62 % L2 hit rate, DRAM traffic 1.30x algorithmic before this change).
    __shared__ int s_next[2];
    uint32_t parity0 = 0u, parity1 = 0u;
    int tile = blockIdx.x;
    int st = 0;
    if (tile < t.n_tiles && threadIdx.x == 0) prefetch(tile, 0);
    for (; tile < t.n_tiles; st ^= 1) {
        if (threadIdx.x == 0) {
            const int next = atomicAdd(t.ticket, 1) + (int)gridDim.x;
            s_next[st] = next;
            if (next < t.n_tiles) prefetch(next, st ^ 1);
        }
        const int4 d = __ldg(t.tiles + tile);
        if (st == 0) { mbar_wait(&bars[0], parity0); parity0 ^= 1u; }
        else         { mbar_wait(&bars[1], parity1); parity1 ^= 1u; }
        const int *sp = stage_base + (size_t)st * TILE_STAGE_WORDS;
        const int *s_ptr = sp + (d.x - (d.x & ~3));
        const int a0 = d.z & ~3;
        const int *s_idx = sp + TILE_PTR_WORDS - a0;                    // index with global nnz offsets
        const float *s_val = reinterpret_cast<const float *>(sp + TILE_PTR_WORDS + TILE_NNZ_WORDS) - a0;
        const int n_rows_tile = d.y - d.x;

        for (int lr = warp * RPW + gi; lr < n_rows_tile; lr += (TILE_THREADS / 32) * RPW) {
            const int s = s_ptr[lr];
            const int e = s_ptr[lr + 1];
            if (e - s > a.long_threshold) continue;
            const long long row = (long long)d.x + lr;
            long long orow = row;
            if (ROWMAP) {
                orow = __ldg(a.rowmap + row);
                if (orow < 0) continue;
            }
            if (false && t.prefetch) {
                // software prefetch into L2: the X rows the group's NEXT row of this tile will gather (their column
                // indices are already in shared memory); hides DRAM latency of first-touch / scattered rows
                const int nlr = lr + (TILE_THREADS / 32) * RPW;
                if (nlr < n_rows_tile) {
                    const int ns = s_ptr[nlr], ne = s_ptr[nlr + 1];
                    if (ne - ns <= a.long_threshold) {
                        const int lines = (a.k * 4 + 127) >> 7;
                        for (int q = ns + gl; q < ne; q += G) {
                            const int cq = s_idx[q];
                            if (cq >= 0) {
                                const char *xr = reinterpret_cast<const char *>(a.X) + (long long)cq * a.k * 4;
                                for (int l = 0; l < lines; ++l)
                                    asm volatile("prefetch.global.L2 [%0];" ::"l"(xr + l * 128));
                            }
                        }
                    }
                }
            }
            // accumulate mode: the old C row is read FIRST so that its latency hides behind the gathers (only this
            // group ever touches the row: the row maps are injective)
            float4 acc[VPL];
            float4 *cr = Cl + orow * k4;
#pragma unroll
            for (int i = 0; i < VPL; ++i)
                acc[i] = (ACC && gl + i * G < k4) ? ld_f4_hint(cr + i * G, pol_stream) : f4_zero();
            if (a.add_map != nullptr) {
                // epilogue gather-add, issued first so its latency hides behind the gathers: the backward exchange
                // C_{j-1}[to_prev[r]] += C_j[r] (arrow_dec_mpi.py:437) seen from the receiving row
                const int am = __ldg(a.add_map + row);
                if (am >= 0) {
                    const float4 *ar = reinterpret_cast<const float4 *>(a.add_src) + (long long)am * k4 + gl;
#pragma unroll
                    for (int i = 0; i < VPL; ++i)
                        if (gl + i * G < k4) f4_add(acc[i], ld_f4_hint(ar + i * G, pol_stream));
                }
            }
            int p = s;
            if (EXACT && !t.skip) {
                // unpredicated batches: full UNROLL batches, then the remainder as 4 / 2 / 1 (binary decomposition) --
                // a predicated tail batch costs as many instructions as a full one
                auto batch = [&](auto n_tag) {
                    constexpr int N = decltype(n_tag)::value;
                    int c[N];
                    float v[N];
#pragma unroll
                    for (int u = 0; u < N; ++u) {
                        c[u] = s_idx[p + u];
                        v[u] = s_val[p + u];
                    }
                    float4 x[N][VPL];
#pragma unroll
                    for (int u = 0; u < N; ++u) {
                        const float4 *xr = Xl + (long long)c[u] * k4;
#pragma unroll
                        for (int i = 0; i < VPL; ++i) x[u][i] = ldg_f4_hint(xr + i * G, pol_keep);
                    }
#pragma unroll
                    for (int u = 0; u < N; ++u)
#pragma unroll
                        for (int i = 0; i < VPL; ++i) f4_fma(acc[i], v[u], x[u][i]);
                    p += N;
                };
                while (p + UNROLL <= e) batch(std::integral_constant<int, UNROLL>{});
                if constexpr (UNROLL >= 8) { if (e - p >= 4) batch(std::integral_constant<int, 4>{}); }
                if constexpr (UNROLL >= 4) { if (e - p >= 2) batch(std::integral_constant<int, 2>{}); }
                if (e - p >= 1) batch(std::integral_constant<int, 1>{});
            }
            // tail (and the general case): predicated batches of TAIL
            for (; p < e; p += TAIL) {
                int c[TAIL];
                float v[TAIL];
#pragma unroll
                for (int u = 0; u < TAIL; ++u) {
                    const bool ok = p + u < e;
                    c[u] = ok ? s_idx[p + u] : -1;
                    v[u] = ok ? s_val[p + u] : 0.f;
                }
                float4 x[TAIL][VPL];
#pragma unroll
                for (int u = 0; u < TAIL; ++u) {
                    const float4 *xr = Xl + (long long)c[u] * k4;
#pragma unroll
                    for (int i = 0; i < VPL; ++i)
                        x[u][i] = (c[u] >= 0 && gl + i * G < k4) ? ldg_f4_hint(xr + i * G, pol_keep) : f4_zero();
                }
#pragma unroll
                for (int u = 0; u < TAIL; ++u)
#pragma unroll
                    for (int i = 0; i < VPL; ++i) f4_fma(acc[i], v[u], x[u][i]);
            }
#pragma unroll
            for (int i = 0; i < VPL; ++i)
                if (gl + i * G < k4) st_f4_hint(cr + i * G, acc[i], pol_stream);
        }
        __syncthreads();            // stage `st` may be refilled by the next iteration's prefetch
        tile = s_next[st];
    }
}

// G lanes own a row (VPL float4 each).  RPG = 2: a group works on two rows at once (rows lr and lr + rows-per-pass) with
// half the batch size per row: the gathers of both rows are issued before either row's FMAs.  Same registers, but the
// short tail batch of one row (a 10-entry row is 8 + 2 gathers: the second round trip keeps 2 of 8 slots busy) overlaps
// the other row's -- narrow feature tiles (k <= 32) are bound by gathers in flight, not by bandwidth.
template <int G, int VPL, int OUT, bool ACC, int TR, int TN, int RPG, int MINB, bool DUALX>
__global__ void __launch_bounds__(TILE_THREADS, 4) k_spmm_tiles(TileArgs t) {
    constexpr int TILE_PTR_WORDS = TileCfg<TR, TN>::PTR_WORDS;
    constexpr int TILE_NNZ_WORDS = TileCfg<TR, TN>::NNZ_WORDS;
    constexpr int TILE_STAGE_WORDS = TileCfg<TR, TN>::STAGE_WORDS;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    int *stage_base = reinterpret_cast<int *>(smem_raw);
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem_raw + (size_t)TILE_STAGES * TILE_STAGE_WORDS * 4);
    const SpmmArgs &a = t.a;
    constexpr int RPW = 32 / G;
    constexpr int ROWS_PER_PASS = (TILE_THREADS / 32) * RPW;
    // gathers a group keeps in flight: UNROLL per row x RPG rows = the same 32 registers of X data per lane in every shape
    constexpr int UNROLL = ((VPL >= 4) ? 2 : (VPL == 2 ? 4 : 8)) / RPG;
    constexpr int TAIL = (UNROLL >= 4) ? UNROLL / 2 : UNROLL;     // predicated tail batches
    static_assert(MINB == 4 && UNROLL >= 1, "tile kernel shape");
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const bool EXACT = (t.a.k4 == G * VPL);                       // every lane owns valid columns
    const int gl = lane % G;
    const int gi = lane / G;
    const int k4 = a.k4;
    const float4 *__restrict__ Xl = reinterpret_cast<const float4 *>(a.X) + gl;
    const float4 *__restrict__ X2l = reinterpret_cast<const float4 *>(a.X2) + gl;
    float4 *__restrict__ Cl = reinterpret_cast<float4 *>(a.C) + gl;
    const uint64_t pol_keep = (t.l2_hints & 1) ? l2_policy_evict_last() : l2_policy_evict_normal();
    const uint64_t pol_stream = (t.l2_hints & 2) ? l2_policy_evict_first() : l2_policy_evict_normal();

    auto xrow = [&](int c) -> const float4 * {
        if constexpr (DUALX) {
            return (c < a.x_split) ? Xl + (long long)c * k4 : X2l + (long long)(c - a.x_split) * k4;
        } else {
            return Xl + (long long)c * k4;
        }
    };

    __shared__ int s_tile[TILE_STAGES];
    auto issue_csr = [&](int tile, int st) {
        const int4 d = __ldg(t.tiles + tile);
        const int rb4 = d.x & ~3;
        const int a0 = d.z & ~3;
        const uint32_t ptr_bytes = (uint32_t)(((d.y - rb4 + 1) + 3) & ~3) * 4u;
        const uint32_t nnz_bytes = (uint32_t)(((d.w - a0) + 3) & ~3) * 4u;
        int *sp = stage_base + (size_t)st * TILE_STAGE_WORDS;
        mbar_expect_tx(&bars[st], ptr_bytes + 2u * nnz_bytes);
        bulk_g2s_hint(sp, a.indptr + rb4, ptr_bytes, &bars[st], pol_stream);
        if (nnz_bytes) {
            bulk_g2s_hint(sp + TILE_PTR_WORDS, a.indices + a0, nnz_bytes, &bars[st], pol_stream);
            bulk_g2s_hint(sp + TILE_PTR_WORDS + TILE_NNZ_WORDS, a.vals + a0, nnz_bytes, &bars[st], pol_stream);
        }
    };

    // Dynamic scheduling: the first tile is blockIdx.x, every further tile comes from an atomic ticket.  All CTAs
    // therefore work on one compact, moving window of ~gridDim.x consecutive tiles; a static round-robin lets
    // CTAs drift apart over the ~260 tiles each one processes at 10M rows and the live X panels fall out of L2
    // (measured: 62 % L2 hit rate, DRAM traffic 1.30x algorithmic before this change).
    if (threadIdx.x == 0) {
#pragma unroll
        for (int s = 0; s < TILE_STAGES; ++s) mbar_init(&bars[s], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        if ((int)blockIdx.x < t.n_tiles) issue_csr(blockIdx.x, 0);
    }
    __syncthreads();

    uint32_t phase = 0u;                  // bit s = parity the next wait on stage s expects
    int tile = blockIdx.x;
    for (int st = 0; tile < t.n_tiles; st ^= 1) {
        if (threadIdx.x == 0) {
            const int nn = atomicAdd(t.ticket, 1) + (int)gridDim.x;
            s_tile[st] = nn;
            if (nn < t.n_tiles) issue_csr(nn, st ^ 1);
        }
        const int4 d = __ldg(t.tiles + tile);
        mbar_wait(&bars[st], (phase >> st) & 1u);
        phase ^= (1u << st);
        const int *sp = stage_base + (size_t)st * TILE_STAGE_WORDS;
        const int *s_ptr = sp + (d.x - (d.x & ~3));
        const int a0 = d.z & ~3;
        const int *s_idx = sp + TILE_PTR_WORDS - a0;                    // index with global nnz offsets
        const float *s_val = reinterpret_cast<const float *>(sp + TILE_PTR_WORDS + TILE_NNZ_WORDS) - a0;
        const int n_rows_tile = d.y - d.x;

        if (t.prefetch) {
            // Bulk L2 prefetch of this tile's X rows (one cp.async.bulk.prefetch.L2 per row, issued by the TMA unit: no
            // registers, no LSU wavefronts).  Measured as a LOSS at every k -- the request rate of the unit, not DRAM
            // latency, becomes the bound.  Off by default; kept as the A/B switch.
            const uint32_t row_bytes = (uint32_t)a.k * 4u;
            for (int q = d.z + (int)threadIdx.x; q < d.w; q += TILE_THREADS) {
                const int cq = s_idx[q];
                if (cq >= 0) bulk_prefetch_l2(xrow(cq) - gl, row_bytes);
            }
        }

        // one or RPG rows of this lane group: setup, joint batches, store
        auto do_rows = [&](auto nr_tag, int lr0) {
            constexpr int NR = decltype(nr_tag)::value;
            int p[NR], e[NR];
            bool live[NR];
            float4 *cr[NR];
            float4 acc[NR][VPL];
#pragma unroll
            for (int r = 0; r < NR; ++r) {
                const int lr = lr0 + r * ROWS_PER_PASS;
                live[r] = lr < n_rows_tile;
                p[r] = e[r] = 0;
                cr[r] = nullptr;
                if (live[r]) {
                    p[r] = s_ptr[lr];
                    e[r] = s_ptr[lr + 1];
                    if (e[r] - p[r] > a.long_threshold) { live[r] = false; e[r] = p[r]; }
                }
                const long long row = (long long)d.x + lr;
                if (live[r]) {
                    if constexpr (OUT == OUT_ROWMAP) {
                        const long long orow = __ldg(a.rowmap + row);
                        if (orow < 0) { live[r] = false; e[r] = p[r]; } else cr[r] = Cl + orow * k4;
                    } else if constexpr (OUT == OUT_ROWPTR) {
                        float *dst = reinterpret_cast<float *>(__ldg(reinterpret_cast<const unsigned long long *>(a.out_ptr) + row));
                        if (dst == nullptr) { live[r] = false; e[r] = p[r]; } else cr[r] = reinterpret_cast<float4 *>(dst) + gl;
                    } else {
                        cr[r] = Cl + row * k4;
                    }
                }
                if constexpr (NR == 1) {
                    if (!live[0]) return;               // one row per group: nothing to keep predicated past this point
                    live[0] = true;
                }
                // accumulate mode: the old C row is read FIRST so that its latency hides behind the gathers (only this
                // group ever touches the row: the row maps are injective)
#pragma unroll
                for (int i = 0; i < VPL; ++i)
                    acc[r][i] = (ACC && live[r] && gl + i * G < k4) ? ld_f4_hint(cr[r] + i * G, pol_stream) : f4_zero();
                if (a.add_map != nullptr && live[r]) {
                    // epilogue gather-add, issued first so its latency hides behind the gathers: the backward exchange
                    // C_{j-1}[to_prev[r]] += C_j[r] (arrow_dec_mpi.py:437) seen from the receiving row
                    const int am = __ldg(a.add_map + row);
                    if (am >= 0) {
                        const float4 *ar = reinterpret_cast<const float4 *>(a.add_src) + (long long)am * k4 + gl;
#pragma unroll
                        for (int i = 0; i < VPL; ++i)
                            if (gl + i * G < k4) f4_add(acc[r][i], ld_f4_hint(ar + i * G, pol_stream));
                    }
                }
            }
            if (EXACT && !t.skip) {
                if constexpr (NR == 1) {
                    // unpredicated batches: full UNROLL batches, then the remainder as 4 / 2 / 1 (binary decomposition) --
                    // a predicated tail batch costs as many instructions as a full one
                    auto batch = [&](auto n_tag) {
                        constexpr int N = decltype(n_tag)::value;
                        float v[N];
                        float4 x[N][VPL];
#pragma unroll
                        for (int u = 0; u < N; ++u) {
                            const int c = s_idx[p[0] + u];
                            v[u] = s_val[p[0] + u];
                            const float4 *xr = xrow(c);
#pragma unroll
                            for (int i = 0; i < VPL; ++i) x[u][i] = ldg_f4_hint(xr + i * G, pol_keep);
                        }
#pragma unroll
                        for (int u = 0; u < N; ++u)
#pragma unroll
                            for (int i = 0; i < VPL; ++i) f4_fma(acc[0][i], v[u], x[u][i]);
                        p[0] += N;
                    };
                    while (p[0] + UNROLL <= e[0]) batch(std::integral_constant<int, UNROLL>{});
                    if constexpr (UNROLL >= 8) { if (e[0] - p[0] >= 4) batch(std::integral_constant<int, 4>{}); }
                    if constexpr (UNROLL >= 4) { if (e[0] - p[0] >= 2) batch(std::integral_constant<int, 2>{}); }
                    if (e[0] - p[0] >= 1) batch(std::integral_constant<int, 1>{});
                } else {
                    // paired rows: while both have a full batch left, 2 x UNROLL unpredicated gathers go out back to back;
                    // the values are read from shared memory when the gathers are back (registers)
                    while (e[0] - p[0] >= UNROLL && e[1] - p[1] >= UNROLL) {
                        float4 x[NR][UNROLL][VPL];
#pragma unroll
                        for (int r = 0; r < NR; ++r)
#pragma unroll
                            for (int u = 0; u < UNROLL; ++u) {
                                const float4 *xr = xrow(s_idx[p[r] + u]);
#pragma unroll
                                for (int i = 0; i < VPL; ++i) x[r][u][i] = __ldg(xr + i * G);
                            }
#pragma unroll
                        for (int r = 0; r < NR; ++r) {
#pragma unroll
                            for (int u = 0; u < UNROLL; ++u) {
                                const float v = s_val[p[r] + u];
#pragma unroll
                                for (int i = 0; i < VPL; ++i) f4_fma(acc[r][i], v, x[r][u][i]);
                            }
                            p[r] += UNROLL;
                        }
                    }
                    // remainders of both rows share predicated batches (one round trip for two short tails)
                    while (p[0] < e[0] || p[1] < e[1]) {
                        float4 x[NR][UNROLL][VPL];
#pragma unroll
                        for (int r = 0; r < NR; ++r)
#pragma unroll
                            for (int u = 0; u < UNROLL; ++u) {
                                const bool ok = p[r] + u < e[r];
                                const float4 *xr = xrow(ok ? s_idx[p[r] + u] : 0);
#pragma unroll
                                for (int i = 0; i < VPL; ++i) x[r][u][i] = ok ? __ldg(xr + i * G) : f4_zero();
                            }
#pragma unroll
                        for (int r = 0; r < NR; ++r) {
#pragma unroll
                            for (int u = 0; u < UNROLL; ++u) {
                                const float v = (p[r] + u < e[r]) ? s_val[p[r] + u] : 0.f;
#pragma unroll
                                for (int i = 0; i < VPL; ++i) f4_fma(acc[r][i], v, x[r][u][i]);
                            }
                            p[r] = min(p[r] + UNROLL, e[r]);
                        }
                    }
                }
            }
            // tail (and the general case): predicated batches of TAIL, one row at a time
#pragma unroll
            for (int r = 0; r < NR; ++r) {
                for (; p[r] < e[r]; p[r] += TAIL) {
                    int c[TAIL];
                    float v[TAIL];
#pragma unroll
                    for (int u = 0; u < TAIL; ++u) {
                        const bool ok = p[r] + u < e[r];
                        c[u] = ok ? s_idx[p[r] + u] : -1;
                        v[u] = ok ? s_val[p[r] + u] : 0.f;
                    }
                    float4 x[TAIL][VPL];
#pragma unroll
                    for (int u = 0; u < TAIL; ++u) {
                        const float4 *xr = xrow(c[u]);                    // c = -1: address arithmetic only, never dereferenced
#pragma unroll
                        for (int i = 0; i < VPL; ++i)
                            x[u][i] = (c[u] >= 0 && gl + i * G < k4) ? ldg_f4_hint(xr + i * G, pol_keep) : f4_zero();
                    }
#pragma unroll
                    for (int u = 0; u < TAIL; ++u)
#pragma unroll
                        for (int i = 0; i < VPL; ++i) f4_fma(acc[r][i], v[u], x[u][i]);
                }
                if (live[r]) {
#pragma unroll
                    for (int i = 0; i < VPL; ++i) {
                        if (gl + i * G < k4) {
                            if constexpr (OUT == OUT_ROWPTR) {
                                *(cr[r] + i * G) = acc[r][i];       // may be a peer GPU's memory (NVLink store): no L2 policy
                            } else {
                                st_f4_hint(cr[r] + i * G, acc[r][i], pol_stream);
                            }
                        }
                    }
                }
            }
        };

        if constexpr (RPG == 2) {
            for (int lr = warp * RPW + gi; lr < n_rows_tile; lr += 2 * ROWS_PER_PASS) do_rows(std::integral_constant<int, 2>{}, lr);
        } else {
            for (int lr = warp * RPW + gi; lr < n_rows_tile; lr += ROWS_PER_PASS) do_rows(std::integral_constant<int, 1>{}, lr);
        }
        __syncthreads();            // stage `st` may be refilled by the next iteration's CSR copy
        tile = s_tile[st];
    }
    // the last CTA to leave re-arms the scheduler for the next launch on this lane (no memset between launches)
    if (threadIdx.x == 0) {
        __threadfence();
        if (atomicAdd(t.ticket + 1, 1) == (int)gridDim.x - 1) {
            t.ticket[0] = 0;
            t.ticket[1] = 0;
            __threadfence();
        }
    }
}

// ------------------------------------------------------------------------------------------------
// Row-parallel kernels over a semiring: the generic kernel (k not a vector width; warp per row, lanes over columns,
// scalar accesses) and the long-row pair (hubs of the arrow head: one CTA per segment of `segment` non-zeros writes a
// partial to scratch, then one CTA per row reduces the partials in order -- deterministic, no atomics).  A semiring type
// gives the element T, zero() (the ⊕ identity), plus(a, b) = a ⊕ b, mac(acc, v, x) = acc ⊕ (v ⊗ x) and kValues (false:
// the CSR carries no values and `vals` is not read).  SpmmArgs / LongArgs carry T elements behind their float pointers.
// Per element every kernel keeps one order, so (+, x) results match the bounds in tests/spmm_bound*.py: generic, the
// ⊕-chain from zero() in entry order, then the old C row (accumulate), then the addend; long rows, each warp's chain
// over entries begin + w, begin + w + 8, ..., then warps 0..7, then the slots in order, the addend and the old C row.
// The partial kernel reduces each 128-column chunk through a fixed [8 warps][128] shared array before the next chunk,
// so its shared memory does not grow with k (a [warps][k] array passes the H100's 227 KB per block at k > 7264 in fp32).
// ------------------------------------------------------------------------------------------------
template <class V>
struct PlusTimes {
    using T = V;
    static constexpr bool kValues = true;
    __device__ __forceinline__ static V zero() { return V(0); }
    __device__ __forceinline__ static V plus(V a, V b) { return a + b; }
    __device__ __forceinline__ static V mac(V acc, V v, V x) { return fma(v, x, acc); }
};

template <class SR, bool ROWMAP, bool ACC>
__global__ void __launch_bounds__(256) k_spmm_generic(SpmmArgs a) {
    using T = typename SR::T;
    const T *vals = reinterpret_cast<const T *>(a.vals);
    const T *add_src = reinterpret_cast<const T *>(a.add_src);
    const int lane = threadIdx.x & 31;
    const long long warps_total = (long long)gridDim.x * (blockDim.x >> 5);
    const long long warp_id = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    for (long long row = warp_id; row < a.n_rows; row += warps_total) {
        const int s = __ldg(a.indptr + row);
        const int e = __ldg(a.indptr + row + 1);
        if (e - s > a.long_threshold) continue;
        long long orow = row;
        if (ROWMAP) {
            orow = __ldg(a.rowmap + row);
            if (orow < 0) continue;
        }
        T *crow = reinterpret_cast<T *>(a.C) + orow * a.k;
        if (a.out_ptr != nullptr) {
            crow = reinterpret_cast<T *>(a.out_ptr[row]);
            if (crow == nullptr) continue;
        }
        for (int c0 = 0; c0 < a.k; c0 += 128) {
            T acc[4] = {SR::zero(), SR::zero(), SR::zero(), SR::zero()};
            for (int p = s; p < e; ++p) {
                const int c = __ldg(a.indices + p);
                T v{};
                if constexpr (SR::kValues) v = __ldg(vals + p);
                if (c < 0) continue;
                const T *xr = x_row_ptr<T>(a, c);
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int col = c0 + lane + 32 * i;
                    if (col < a.k) acc[i] = SR::mac(acc[i], v, __ldg(xr + col));
                }
            }
            const int am = (a.add_map != nullptr) ? __ldg(a.add_map + row) : -1;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int col = c0 + lane + 32 * i;
                if (col < a.k) {
                    T *dst = crow + col;
                    T r = ACC ? SR::plus(*dst, acc[i]) : acc[i];
                    if (am >= 0) r = SR::plus(r, add_src[(long long)am * a.k + col]);
                    *dst = r;
                }
            }
        }
    }
}

constexpr int LONG_WARPS = 8;        // 256 threads per partial CTA
constexpr int LONG_CHUNK = 128;      // columns per chunk: 32 lanes x 4
struct LongArgs {
    const LongTask *__restrict__ tasks;
    const int *__restrict__ indices;
    const float *__restrict__ vals;
    const float *__restrict__ X;
    float *__restrict__ scratch;      // [slot][k]
    int k;
    const float *__restrict__ X2;     // second X base (see SpmmArgs)
    int x_split;
};

template <class SR>
__global__ void __launch_bounds__(256) k_spmm_long_partial(LongArgs a) {
    using T = typename SR::T;
    __shared__ T red[LONG_WARPS][LONG_CHUNK];
    const T *vals = reinterpret_cast<const T *>(a.vals);
    const LongTask t = a.tasks[blockIdx.x];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int c0 = 0; c0 < a.k; c0 += LONG_CHUNK) {
        T acc[4] = {SR::zero(), SR::zero(), SR::zero(), SR::zero()};
        for (int p = t.begin + warp; p < t.end; p += LONG_WARPS) {
            const int c = __ldg(a.indices + p);
            T v{};
            if constexpr (SR::kValues) v = __ldg(vals + p);
            if (c < 0) continue;
            const T *xr = x_row_ptr<T>(a, c);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int col = c0 + lane + 32 * i;
                if (col < a.k) acc[i] = SR::mac(acc[i], v, __ldg(xr + col));
            }
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) red[warp][lane + 32 * i] = acc[i];
        __syncthreads();
        const int col = c0 + threadIdx.x;
        if (threadIdx.x < LONG_CHUNK && col < a.k) {
            T sum = SR::zero();
            for (int w = 0; w < LONG_WARPS; ++w) sum = SR::plus(sum, red[w][threadIdx.x]);
            reinterpret_cast<T *>(a.scratch)[(long long)t.slot * a.k + col] = sum;
        }
        __syncthreads();
    }
}

template <class SR, bool ROWMAP, bool ACC>
__global__ void __launch_bounds__(128) k_spmm_long_reduce(SpmmArgs a, const int *__restrict__ long_rows,
                                                          const int *__restrict__ long_first,
                                                          const typename SR::T *__restrict__ scratch) {
    using T = typename SR::T;
    const T *add_src = reinterpret_cast<const T *>(a.add_src);
    const int k = a.k;
    const int r = long_rows[blockIdx.x];
    long long orow = r;
    if (ROWMAP) {
        orow = a.rowmap[r];
        if (orow < 0) return;
    }
    T *crow = reinterpret_cast<T *>(a.C) + orow * k;
    if (a.out_ptr != nullptr) {
        crow = reinterpret_cast<T *>(a.out_ptr[r]);
        if (crow == nullptr) return;
    }
    const int s0 = long_first[blockIdx.x], s1 = long_first[blockIdx.x + 1];
    for (int col = threadIdx.x; col < k; col += blockDim.x) {
        T sum = SR::zero();
        for (int s = s0; s < s1; ++s) sum = SR::plus(sum, scratch[(long long)s * k + col]);
        if (a.add_map != nullptr) {
            const int am = a.add_map[r];
            if (am >= 0) sum = SR::plus(sum, add_src[(long long)am * k + col]);
        }
        T *dst = crow + col;
        *dst = ACC ? SR::plus(*dst, sum) : sum;
    }
}

// ------------------------------------------------------------------------------------------------
// float64 (ARROW_F64 CSR values and tiles; one GPU).  The tile kernel keeps the pipeline of k_spmm_tiles_v1 -- the CSR
// slices streamed by cp.async.bulk on an mbarrier, two stages, persistent CTAs on the atomic ticket, a lane group per
// row -- with X and C moved as double2 (16 B: the vector path needs k % 2 == 0) and 8-byte values in shared memory.
// Every element is one fma chain in entry order (after the old C row or the addend), so a result does not depend on
// the grid.  The generic and long-row kernels are the row-parallel templates on PlusTimes<double>.
// ------------------------------------------------------------------------------------------------
struct SpmmArgsF64 {
    const int *__restrict__ indptr;
    const int *__restrict__ indices;
    const double *__restrict__ vals;
    const double *__restrict__ X;
    double *__restrict__ C;
    const int *__restrict__ rowmap;      // nullptr: identity
    long long n_rows;
    int k;
    int k2;                              // k / 2 (tile kernel)
    int long_threshold;
    const double *__restrict__ add_src;  // optional addend: C[r] = sum + add_src[add_map[r]] (add_map[r] >= 0)
    const int *__restrict__ add_map;
};

struct TileArgsF64 {
    SpmmArgsF64 a;
    const int4 *__restrict__ tiles;
    int n_tiles;
    int skip;            // indices may hold -1
    int *ticket;         // dynamic tile scheduler: [0] next tile
    int l2_hints;        // bit 0: X gathers evict_last, bit 1: CSR / C streams evict_first
};

// one stage: row pointers (int) | indices (int) | values (double), every part 16-byte aligned for cp.async.bulk
struct TileCfgF64 {
    static constexpr int PTR_WORDS = TILE_ROWS + 8;
    static constexpr int NNZ_WORDS = TILE_NNZ + 8;
    static constexpr int IDX_OFF = PTR_WORDS * 4;
    static constexpr int VAL_OFF = IDX_OFF + NNZ_WORDS * 4;
    static constexpr int STAGE_BYTES = VAL_OFF + NNZ_WORDS * 8;
    static constexpr size_t SMEM_BYTES = (size_t)TILE_STAGES * STAGE_BYTES + 64;
    static_assert(IDX_OFF % 16 == 0 && VAL_OFF % 16 == 0 && STAGE_BYTES % 16 == 0, "bulk copies need 16-byte alignment");
};

__device__ __forceinline__ double2 ldg_d2_hint(const double2 *ptr, uint64_t pol) {
    double2 r;
    asm("ld.global.nc.L2::cache_hint.v2.f64 {%0,%1}, [%2], %3;" : "=d"(r.x), "=d"(r.y) : "l"(ptr), "l"(pol));
    return r;
}
__device__ __forceinline__ double2 ld_d2_hint(const double2 *ptr, uint64_t pol) {      // coherent load (C tile RMW)
    double2 r;
    asm("ld.global.L2::cache_hint.v2.f64 {%0,%1}, [%2], %3;" : "=d"(r.x), "=d"(r.y) : "l"(ptr), "l"(pol));
    return r;
}
__device__ __forceinline__ void st_d2_hint(double2 *ptr, const double2 &v, uint64_t pol) {
    asm volatile("st.global.L2::cache_hint.v2.f64 [%0], {%1,%2}, %3;" ::"l"(ptr), "d"(v.x), "d"(v.y), "l"(pol) : "memory");
}

// G lanes own a row, VPL double2 each.  A value takes 2 registers here (1 in fp32): the values are read from shared memory
// only when the gathers of a batch are back, the UNROLL-8 batch of the narrow shapes shrinks to 4, and accumulate mode adds
// the old C row after the products instead of starting from it: every instance stays inside the 64 registers of
// __launch_bounds__(256, 4) without spills (-Xptxas -v).
template <int G, int VPL, bool ROWMAP, bool ACC>
__global__ void __launch_bounds__(TILE_THREADS, 4) k_spmm_tiles_f64(TileArgsF64 t) {
    using Cfg = TileCfgF64;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem_raw + (size_t)TILE_STAGES * Cfg::STAGE_BYTES);
    const SpmmArgsF64 &a = t.a;
    constexpr int RPW = 32 / G;
    constexpr int UNROLL = (VPL >= 4) ? 2 : 4;
    constexpr int TAIL = (UNROLL >= 4) ? UNROLL / 2 : UNROLL;     // predicated tail batches
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const bool EXACT = (a.k2 == G * VPL);                         // every lane owns valid columns
    const int gl = lane % G;
    const int gi = lane / G;
    const int k2 = a.k2;
    const double2 *__restrict__ Xl = reinterpret_cast<const double2 *>(a.X) + gl;
    double2 *__restrict__ Cl = reinterpret_cast<double2 *>(a.C) + gl;
    const uint64_t pol_keep = (t.l2_hints & 1) ? l2_policy_evict_last() : l2_policy_evict_normal();
    const uint64_t pol_stream = (t.l2_hints & 2) ? l2_policy_evict_first() : l2_policy_evict_normal();

    if (threadIdx.x == 0) {
        mbar_init(&bars[0], 1);
        mbar_init(&bars[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    // the slices start at the 4-entry boundary below the tile and round up to 4 entries: 16-byte copies of the 4-byte
    // arrays, 32-byte copies of the values (the upload leaves 8 entries of slack behind every array)
    auto issue_csr = [&](int tile, int st) {
        const int4 d = __ldg(t.tiles + tile);
        const int rb4 = d.x & ~3;
        const int a0 = d.z & ~3;
        const uint32_t ptr_bytes = (uint32_t)(((d.y - rb4 + 1) + 3) & ~3) * 4u;
        const uint32_t n_nnz = (uint32_t)(((d.w - a0) + 3) & ~3);
        unsigned char *sp = smem_raw + (size_t)st * Cfg::STAGE_BYTES;
        mbar_expect_tx(&bars[st], ptr_bytes + n_nnz * 12u);
        bulk_g2s_hint(sp, a.indptr + rb4, ptr_bytes, &bars[st], pol_stream);
        if (n_nnz) {
            bulk_g2s_hint(sp + Cfg::IDX_OFF, a.indices + a0, n_nnz * 4u, &bars[st], pol_stream);
            bulk_g2s_hint(sp + Cfg::VAL_OFF, a.vals + a0, n_nnz * 8u, &bars[st], pol_stream);
        }
    };

    __shared__ int s_next[TILE_STAGES];
    uint32_t phase = 0u;                  // bit s = parity the next wait on stage s expects
    int tile = blockIdx.x;
    if (tile < t.n_tiles && threadIdx.x == 0) issue_csr(tile, 0);
    for (int st = 0; tile < t.n_tiles; st ^= 1) {
        if (threadIdx.x == 0) {
            const int next = atomicAdd(t.ticket, 1) + (int)gridDim.x;
            s_next[st] = next;
            if (next < t.n_tiles) issue_csr(next, st ^ 1);
        }
        const int4 d = __ldg(t.tiles + tile);
        mbar_wait(&bars[st], (phase >> st) & 1u);
        phase ^= (1u << st);
        const unsigned char *sp = smem_raw + (size_t)st * Cfg::STAGE_BYTES;
        const int *s_ptr = reinterpret_cast<const int *>(sp) + (d.x - (d.x & ~3));
        const int a0 = d.z & ~3;
        const int *s_idx = reinterpret_cast<const int *>(sp + Cfg::IDX_OFF) - a0;        // index with global nnz offsets
        const double *s_val = reinterpret_cast<const double *>(sp + Cfg::VAL_OFF) - a0;
        const int n_rows_tile = d.y - d.x;

        for (int lr = warp * RPW + gi; lr < n_rows_tile; lr += (TILE_THREADS / 32) * RPW) {
            const int s = s_ptr[lr];
            const int e = s_ptr[lr + 1];
            if (e - s > a.long_threshold) continue;
            const long long row = (long long)d.x + lr;
            long long orow = row;
            if (ROWMAP) {
                orow = __ldg(a.rowmap + row);
                if (orow < 0) continue;
            }
            // the addend is read first so that its latency hides behind the gathers
            double2 acc[VPL];
            double2 *cr = Cl + orow * k2;
#pragma unroll
            for (int i = 0; i < VPL; ++i) acc[i] = d2_zero();
            if (a.add_map != nullptr) {
                const int am = __ldg(a.add_map + row);
                if (am >= 0) {
                    const double2 *ar = reinterpret_cast<const double2 *>(a.add_src) + (long long)am * k2 + gl;
#pragma unroll
                    for (int i = 0; i < VPL; ++i)
                        if (gl + i * G < k2) d2_add(acc[i], ld_d2_hint(ar + i * G, pol_stream));
                }
            }
            int p = s;
            if (EXACT && !t.skip) {
                // unpredicated batches: full UNROLL batches, then the remainder as 2 / 1
                auto batch = [&](auto n_tag) {
                    constexpr int N = decltype(n_tag)::value;
                    double2 x[N][VPL];
#pragma unroll
                    for (int u = 0; u < N; ++u) {
                        const double2 *xr = Xl + (long long)s_idx[p + u] * k2;
#pragma unroll
                        for (int i = 0; i < VPL; ++i) x[u][i] = ldg_d2_hint(xr + i * G, pol_keep);
                    }
#pragma unroll
                    for (int u = 0; u < N; ++u) {
                        const double v = s_val[p + u];
#pragma unroll
                        for (int i = 0; i < VPL; ++i) d2_fma(acc[i], v, x[u][i]);
                    }
                    p += N;
                };
                while (p + UNROLL <= e) batch(std::integral_constant<int, UNROLL>{});
                if constexpr (UNROLL >= 4) { if (e - p >= 2) batch(std::integral_constant<int, 2>{}); }
                if (e - p >= 1) batch(std::integral_constant<int, 1>{});
            }
            // tail (and the general case): predicated batches of TAIL; a skipped entry (column -1) adds nothing
            for (; p < e; p += TAIL) {
                double2 x[TAIL][VPL];
#pragma unroll
                for (int u = 0; u < TAIL; ++u) {
                    const int c = (p + u < e) ? s_idx[p + u] : -1;
                    const double2 *xr = Xl + (long long)c * k2;             // c = -1: address arithmetic only
#pragma unroll
                    for (int i = 0; i < VPL; ++i)
                        x[u][i] = (c >= 0 && gl + i * G < k2) ? ldg_d2_hint(xr + i * G, pol_keep) : d2_zero();
                }
#pragma unroll
                for (int u = 0; u < TAIL; ++u) {
                    const double v = (p + u < e) ? s_val[p + u] : 0.0;     // 0 * 0 added: no rounding
#pragma unroll
                    for (int i = 0; i < VPL; ++i) d2_fma(acc[i], v, x[u][i]);
                }
            }
            // accumulate mode: C += the products (only this group ever touches the row: the row maps are injective)
#pragma unroll
            for (int i = 0; i < VPL; ++i) {
                if (gl + i * G < k2) {
                    if (ACC) d2_add(acc[i], ld_d2_hint(cr + i * G, pol_stream));
                    st_d2_hint(cr + i * G, acc[i], pol_stream);
                }
            }
        }
        __syncthreads();            // stage `st` may be refilled by the next iteration's copy
        tile = s_next[st];
    }
}

// ------------------------------------------------------------------------------------------------
// exchange kernels: dst[r] (+)= src[map[r]]
// ------------------------------------------------------------------------------------------------
constexpr int MAX_SRC = 16;
struct MultiSrc {
    const float *p[MAX_SRC];
    long long bound[MAX_SRC + 1];
    int n;
};

// A group of G lanes moves one row (VPR vectors of VT); rows are taken warp-strided so that a warp's
// destination rows are consecutive (coalesced stores) while the sources are wherever the map points --
// local HBM, or a peer GPU's memory over NVLink when MULTI.
template <typename VT, int G, bool ACC, bool MULTI>
__global__ void __launch_bounds__(256) k_gather_rows(VT *__restrict__ dst, const VT *__restrict__ src, MultiSrc ms,
                                                     const int *__restrict__ map, long long n_rows, int vec_per_row) {
    constexpr int RPW = 32 / G;
    const int lane = threadIdx.x & 31;
    const int gl = lane % G, gi = lane / G;
    const long long warps_total = (long long)gridDim.x * (blockDim.x >> 5);
    const long long warp_id = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    for (long long r = warp_id * RPW + gi; r < n_rows; r += warps_total * RPW) {
        const int m = __ldg(map + r);
        if (m < 0) continue;
        const VT *sp;
        if (MULTI) {
            int s = 0;
#pragma unroll 1
            while (s + 1 < ms.n && (long long)m >= ms.bound[s + 1]) ++s;
            sp = reinterpret_cast<const VT *>(ms.p[s]) + ((long long)m - ms.bound[s]) * vec_per_row;
        } else {
            sp = src + (long long)m * vec_per_row;
        }
        VT *dp = dst + r * vec_per_row;
        for (int v0 = gl; v0 < vec_per_row; v0 += 4 * G) {
            VT val[4];
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (v0 + j * G < vec_per_row) val[j] = sp[v0 + j * G];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (v0 + j * G < vec_per_row) {
                    if (ACC) {
                        VT old = dp[v0 + j * G];
                        if constexpr (std::is_same<VT, float4>::value) {
                            f4_add(val[j], old);
                        } else if constexpr (std::is_same<VT, double2>::value) {
                            d2_add(val[j], old);
                        } else {
                            val[j] += old;
                        }
                    }
                    dp[v0 + j * G] = val[j];
                }
            }
        }
    }
}

// Push: dst_d[i - bound[d]] = src[map[i]] for item i in [bound[d], bound[d+1]) -- the forward exchange of the fused
// multi-GPU step.  The items are sorted by destination GPU and, inside one destination, by the slot of its receive
// region, so every destination sees ONE sequential stream of 512-byte rows arriving over NVLink (posted stores: the
// sender never waits for the link) while the reads are local HBM gathers.  Replaces pack kernel + all-to-all + unpack
// kernel (arrow_dec_mpi.py:526, 584-610, 544) by a single pass.
struct MultiDst {
    float *p[MAX_SRC];
    long long bound[MAX_SRC + 1];
    int n;
    long long max_len;        // longest block; > 0: the grid walks the blocks interleaved (item q -> block q % n, position q / n)
};

// `md.max_len > 0`: consecutive lane groups serve DIFFERENT destinations, so at every instant a GPU sends to all its peers
// at once and every receiver hears from all senders at once -- the uniform all-to-all an NVSwitch serves at full rate
// whatever the relative timing of the GPUs.  Block after block (max_len == 0) depends on the GPUs staying in lockstep.
template <typename VT, int G>
__global__ void __launch_bounds__(256) k_push_rows(MultiDst md, const VT *__restrict__ src, const int *__restrict__ map,
                                                   long long n_items, int vec_per_row) {
    constexpr int RPW = 32 / G;
    const int lane = threadIdx.x & 31;
    const int gl = lane % G, gi = lane / G;
    const long long warps_total = (long long)gridDim.x * (blockDim.x >> 5);
    const long long warp_id = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const long long n_walk = md.max_len > 0 ? md.max_len * md.n : n_items;
    for (long long q = warp_id * RPW + gi; q < n_walk; q += warps_total * RPW) {
        long long i = q;
        int d = 0;
        if (md.max_len > 0) {
            d = (int)(q % md.n);
            const long long pos = q / md.n;
            if (pos >= md.bound[d + 1] - md.bound[d]) continue;
            i = md.bound[d] + pos;
        }
        const int m = __ldg(map + i);
        if (m < 0) continue;
        if (md.max_len == 0) {
#pragma unroll 1
            while (d + 1 < md.n && i >= md.bound[d + 1]) ++d;
        }
        const VT *sp = src + (long long)m * vec_per_row;
        VT *dp = reinterpret_cast<VT *>(md.p[d]) + (i - md.bound[d]) * vec_per_row;
        for (int v0 = gl; v0 < vec_per_row; v0 += 4 * G) {
            VT val[4];
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (v0 + j * G < vec_per_row) val[j] = sp[v0 + j * G];
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (v0 + j * G < vec_per_row) dp[v0 + j * G] = val[j];
        }
    }
}

// out(r) = sum_s src_s[r] in source order (deterministic): the reduction of the partial head tiles
// (C_0 = sum_i A_0i X_i, arrow_slim_mpi.py:116) in one launch; the sources are peer tiles read over NVLink.  With a
// pointer table the sum goes wherever the row is routed (a peer's staging slot: head rows of a level > 0 on their way
// to the level below), else into dst.
template <typename VT>
__global__ void __launch_bounds__(256) k_reduce_rows(VT *__restrict__ dst, float *const *__restrict__ out_ptr, MultiSrc ms,
                                                     long long n_rows, int vec_per_row) {
    const long long total = n_rows * vec_per_row;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
        const long long r = i / vec_per_row;
        const int v = (int)(i - r * vec_per_row);
        VT *o = dst ? dst + i : nullptr;
        if (out_ptr != nullptr) {
            float *q = out_ptr[r];
            if (q != nullptr) o = reinterpret_cast<VT *>(q) + v;
        }
        if (o == nullptr) continue;
        VT sum = reinterpret_cast<const VT *>(ms.p[0])[i];
        for (int s = 1; s < ms.n; ++s) {
            const VT x = reinterpret_cast<const VT *>(ms.p[s])[i];
            if constexpr (sizeof(VT) == 16) {
                f4_add(sum, x);
            } else {
                sum += x;
            }
        }
        *o = sum;
    }
}

__global__ void k_fill_ptr_table(float **table, const int *__restrict__ which, const long long *__restrict__ row,
                                 const unsigned long long *__restrict__ bases, long long n, int k) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const int w = which[i];
        table[i] = (w < 0) ? nullptr : reinterpret_cast<float *>(bases[w]) + row[i] * k;
    }
}

// ------------------------------------------------------------------------------------------------
// small utility kernels
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void k_fill(T *p, T v, long long n) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) p[i] = v;
}

template <typename SrcT>
__global__ void k_to_i32(const SrcT *__restrict__ in, int *__restrict__ out, long long n, long long base, int *bad) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const long long v = (long long)in[i] - base;
        if (v < 0 || v > 2147483647LL) atomicExch(bad, 1);
        out[i] = (int)v;
    }
}

__global__ void k_check_cols(const int *__restrict__ idx, long long n, long long n_cols, int *bad) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const int c = idx[i];
        if (c < 0 || c >= n_cols) atomicExch(bad, 1);
    }
}

__global__ void k_map_from_i64(const long long *__restrict__ in, int *__restrict__ out, long long n, long long limit) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const long long v = in[i];
        out[i] = (v < 0 || v >= limit) ? -1 : (int)v;
    }
}

__global__ void k_remap(const int *__restrict__ idx, const int *__restrict__ map, long long map_n, int *__restrict__ out,
                        long long n, int *any_invalid) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    bool bad = false;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const int c = idx[i];
        const int m = (c < 0 || c >= map_n) ? -1 : map[c];
        out[i] = m;
        bad = bad || m < 0;
    }
    if (bad && any_invalid != nullptr) atomicExch(any_invalid, 1);
}

__global__ void k_map_invert(const int *__restrict__ map, long long n, int *__restrict__ out, long long n_out) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const int q = map[i];
        if (q >= 0 && q < n_out) out[q] = (int)i;
    }
}

// Cross-GPU barrier over peer-mapped flag words: rank r writes the lane's next epoch into slot r of every peer's
// flag array, then waits until every slot of its own array reached that epoch.  The epoch counter lives in device
// memory (one per lane) so the launch carries no per-call state: a captured CUDA graph replays it unchanged.
struct PeerFlags {
    unsigned int *p[MAX_SRC];
};
__global__ void k_peer_barrier(PeerFlags flags, int rank, int world, unsigned int *epoch_ctr, int *status, long long timeout_clocks) {
    __shared__ unsigned int s_epoch;
    __threadfence_system();
    if (threadIdx.x == 0) {
        s_epoch = *epoch_ctr + 1u;
        *epoch_ctr = s_epoch;
    }
    __syncthreads();
    const unsigned int epoch = s_epoch;
    const int s = threadIdx.x;
    if (s < world) {
        volatile unsigned int *remote = flags.p[s] + rank;
        *remote = epoch;
        __threadfence_system();
        volatile unsigned int *mine = flags.p[rank] + s;
        const long long t0 = clock64();
        while ((int)(*mine - epoch) < 0) {
            if (clock64() - t0 > timeout_clocks) {    // give up instead of hanging the box; the context is poisoned
                atomicExch(status, 1);
                break;
            }
        }
    }
    __syncthreads();
    __threadfence_system();
}

// ------------------------------------------------------------------------------------------------
// launch helpers
// ------------------------------------------------------------------------------------------------
int grid_for(arrow_ctx *ctx, const void *fn, int threads, size_t smem, long long work_ctas) {
    int occ = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fn, threads, smem) != cudaSuccess || occ < 1) occ = 1;
    long long resident = (long long)occ * ctx->sm_count;
    long long g = std::min<long long>(std::max<long long>(work_ctas, 1), resident);
    return (int)g;
}

// f(ROWMAP, ACC) with both as std::bool_constant; only (+, x) has the row-map and accumulate epilogues
template <class SR, class F>
void with_epilogue(bool rowmap, bool acc, F &&f) {
    if constexpr (std::is_same<SR, PlusTimes<typename SR::T>>::value) {
        if (rowmap && acc) f(std::true_type{}, std::true_type{});
        else if (rowmap) f(std::true_type{}, std::false_type{});
        else if (acc) f(std::false_type{}, std::true_type{});
        else f(std::false_type{}, std::false_type{});
    } else {
        f(std::false_type{}, std::false_type{});
    }
}

// the generic kernel over every row of `a` (rows past the long-row threshold are left to launch_long_rows)
template <class SR>
void launch_generic(arrow_ctx *ctx, const SpmmArgs &a, bool rowmap, bool acc) {
    with_epilogue<SR>(rowmap, acc, [&](auto rm, auto ac) {
        auto fn = k_spmm_generic<SR, decltype(rm)::value, decltype(ac)::value>;
        const int grid = grid_for(ctx, (const void *)fn, 256, 0, (a.n_rows + 7) / 8);
        fn<<<grid, 256, 0, cur_stream(ctx)>>>(a);
    });
    ctx->launches++;
}

// Grows the current lane's long-row scratch to at least `need` bytes.  Growing frees and allocates, which a graph
// capture cannot record: the step has to run once outside the capture first.
int grow_long_scratch(arrow_ctx *ctx, size_t need) {
    const int lane = ctx->cur_lane;
    if (need <= ctx->long_scratch_bytes[lane]) return ARROW_OK;
    if (ctx->capturing) return fail(ctx, ARROW_ERR_UNSUPPORTED, "long-row scratch would grow during graph capture: run the step once first");
    CUDA_TRY(ctx, cudaStreamSynchronize(cur_stream(ctx)));
    if (ctx->long_scratch[lane]) cudaFree(ctx->long_scratch[lane]);
    ctx->long_scratch[lane] = nullptr;
    ctx->long_scratch_bytes[lane] = 0;
    CUDA_TRY(ctx, cudaMalloc(&ctx->long_scratch[lane], need));
    ctx->long_scratch_bytes[lane] = need;
    return ARROW_OK;
}

// the long rows of A: segment partials into the lane's scratch, then the in-order reduction with a's epilogue
template <class SR>
int launch_long_rows(arrow_ctx *ctx, const Csr *A, const SpmmArgs &a, bool rowmap, bool acc) {
    using T = typename SR::T;
    if (A->n_long_tasks == 0) return ARROW_OK;
    const int rc = grow_long_scratch(ctx, (size_t)A->n_long_tasks * a.k * sizeof(T));
    if (rc != ARROW_OK) return rc;
    cudaStream_t stream = cur_stream(ctx);
    LongArgs la;
    la.tasks = A->long_tasks;
    la.indices = a.indices;
    la.vals = a.vals;
    la.X = a.X;
    la.scratch = ctx->long_scratch[ctx->cur_lane];
    la.k = a.k;
    la.X2 = a.X2;
    la.x_split = a.x_split;
    k_spmm_long_partial<SR><<<A->n_long_tasks, 256, 0, stream>>>(la);
    ctx->launches++;
    with_epilogue<SR>(rowmap, acc, [&](auto rm, auto ac) {
        k_spmm_long_reduce<SR, decltype(rm)::value, decltype(ac)::value><<<A->n_long_rows, 128, 0, stream>>>(
            a, A->long_rows, A->long_first, reinterpret_cast<const T *>(la.scratch));
    });
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
    return ARROW_OK;
}

// A persistent tile kernel: as many CTAs as are resident (capped by ARROW_OPT_SPMM_CTAS_PER_SM / _SPMM_SM_LIMIT), at
// most one per tile, taking tiles from the atomic ticket.  KERNEL is a template argument so that each kernel keeps its
// own per-device attribute and occupancy cache.
template <auto KERNEL, size_t SMEM, class Args>
int launch_persistent(arrow_ctx *ctx, const Args &args, int n_tiles, int *ticket) {
    static bool attr_set[64] = {};            /* function attributes are per device */
    static int occ_dev[64] = {};
    const int dv = ctx->device & 63;
    if (!attr_set[dv]) {
        cudaFuncSetAttribute(KERNEL, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM);
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_dev[dv], KERNEL, TILE_THREADS, SMEM) != cudaSuccess || occ_dev[dv] < 1) occ_dev[dv] = 1;
        attr_set[dv] = true;
    }
    const int occ = occ_dev[dv];
    const int per_sm = (ctx->spmm_ctas_per_sm > 0) ? std::min(occ, ctx->spmm_ctas_per_sm) : occ;
    int sms = ctx->sm_count;
    if (ctx->spmm_sm_limit > 0) sms = std::min(sms, ctx->spmm_sm_limit);
    int grid = (int)std::min<long long>((long long)per_sm * sms, n_tiles);
    // the scheduler words are zeroed before every launch: the round-1 kernel (which shares them) leaves its ticket behind,
    // and a launch must never depend on how the previous one on this lane ended
    cudaMemsetAsync(ticket, 0, 2 * sizeof(int), cur_stream(ctx));
    KERNEL<<<grid, TILE_THREADS, SMEM, cur_stream(ctx)>>>(args);
    ctx->launches++;
    return ARROW_OK;
}

template <int G, int VPL>
int launch_vec(arrow_ctx *ctx, const SpmmArgs &a, bool rowmap, bool acc, int variant) {
    constexpr int RPW = 32 / G;
    const int threads = 256;
    const long long rows_per_cta = (long long)(threads / 32) * RPW;
    const long long ctas = (a.n_rows + rows_per_cta - 1) / rows_per_cta;
#define LAUNCH_K(KERNEL)                                                                              \
    do {                                                                                              \
        auto fn = KERNEL;                                                                             \
        int grid = grid_for(ctx, (const void *)fn, threads, 0, ctas);                                 \
        fn<<<grid, threads, 0, cur_stream(ctx)>>>(a);                                                     \
    } while (0)
    if (variant == ARROW_VARIANT_SHFL) {
        if (rowmap && acc) LAUNCH_K((k_spmm_shfl<G, VPL, true, true>));
        else if (rowmap) LAUNCH_K((k_spmm_shfl<G, VPL, true, false>));
        else if (acc) LAUNCH_K((k_spmm_shfl<G, VPL, false, true>));
        else LAUNCH_K((k_spmm_shfl<G, VPL, false, false>));
    } else {
        if (rowmap && acc) LAUNCH_K((k_spmm_direct<G, VPL, true, true>));
        else if (rowmap) LAUNCH_K((k_spmm_direct<G, VPL, true, false>));
        else if (acc) LAUNCH_K((k_spmm_direct<G, VPL, false, true>));
        else LAUNCH_K((k_spmm_direct<G, VPL, false, false>));
    }
#undef LAUNCH_K
    ctx->launches++;
    return ARROW_OK;
}

template <int VPL>
int launch_tma(arrow_ctx *ctx, const SpmmArgs &a, bool rowmap, bool acc) {
    const int threads = TMA_WARPS * 32;
    const size_t smem = (size_t)TMA_WARPS * TMA_STAGES * TMA_SLOTS * a.k * 4 + TMA_WARPS * TMA_STAGES * 8;
    const long long ctas = (a.n_rows + TMA_WARPS - 1) / TMA_WARPS;
#define LAUNCH_T(KERNEL)                                                                              \
    do {                                                                                              \
        auto fn = KERNEL;                                                                             \
        cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);             \
        int grid = grid_for(ctx, (const void *)fn, threads, smem, ctas);                              \
        fn<<<grid, threads, smem, cur_stream(ctx)>>>(a);                                                  \
    } while (0)
    if (rowmap && acc) LAUNCH_T((k_spmm_tma<VPL, true, true>));
    else if (rowmap) LAUNCH_T((k_spmm_tma<VPL, true, false>));
    else if (acc) LAUNCH_T((k_spmm_tma<VPL, false, true>));
    else LAUNCH_T((k_spmm_tma<VPL, false, false>));
#undef LAUNCH_T
    ctx->launches++;
    return ARROW_OK;
}

// what a tile launch needs beyond the template parameters
struct TileLaunch {
    int out_mode = OUT_IDENTITY;     // OUT_*
    bool acc = false;
    bool dualx = false;
    int vpl_req = 0;                 // 0 = default float4-per-lane count
    int rpg_req = 0;                 // 0 = default rows per lane group, 1 / 2 forced
};

template <int G, int VPL, int OUT, bool ACC, int TR, int TN, int RPG, int MINB, bool DUALX>
int launch_tiles_one(arrow_ctx *ctx, const TileArgs &t) {
    constexpr auto fn = k_spmm_tiles<G, VPL, OUT, ACC, TR, TN, RPG, MINB, DUALX>;
    static int carve_dev[64];
    const int dv = ctx->device & 63;
    if (ctx->smem_carveout != carve_dev[dv] - 1000) {       // measurement switch: how much of the 256 KB is L1
        cudaFuncSetAttribute(fn, cudaFuncAttributePreferredSharedMemoryCarveout, ctx->smem_carveout);
        carve_dev[dv] = ctx->smem_carveout + 1000;
    }
    return launch_persistent<fn, TileCfg<TR, TN>::SMEM_BYTES>(ctx, t, t.n_tiles, t.ticket);
}

template <int G, int VPL, bool ROWMAP, bool ACC, int TR, int TN>
int launch_tiles_v1(arrow_ctx *ctx, const TileArgs &t) {
    return launch_persistent<k_spmm_tiles_v1<G, VPL, ROWMAP, ACC, TR, TN>, TileCfg<TR, TN>::SMEM_BYTES>(ctx, t, t.n_tiles, t.ticket);
}

template <int G, int VPL, int TR, int TN, int RPG, int MINB>
int launch_tiles_gv(arrow_ctx *ctx, const TileArgs &t, const TileLaunch &L) {
    if (L.out_mode == OUT_ROWPTR) {
        // the multi-GPU fused path: row-pointer epilogue, optionally the [recv region | local tile] dual X base
        if (L.acc) return fail(ctx, ARROW_ERR_UNSUPPORTED, "row-pointer epilogue does not accumulate");
        if (L.dualx) return launch_tiles_one<G, VPL, OUT_ROWPTR, false, TR, TN, RPG, MINB, true>(ctx, t);
        return launch_tiles_one<G, VPL, OUT_ROWPTR, false, TR, TN, RPG, MINB, false>(ctx, t);
    }
    if (L.dualx) {
        if (L.out_mode != OUT_IDENTITY || L.acc) return fail(ctx, ARROW_ERR_UNSUPPORTED, "dual X base needs a plain or row-pointer epilogue");
        return launch_tiles_one<G, VPL, OUT_IDENTITY, false, TR, TN, RPG, MINB, true>(ctx, t);
    }
    if constexpr (RPG == 2) {
        // the two-rows-per-group family exists for plain and row-pointer launches (the narrow-k fast path)
        if (L.out_mode == OUT_IDENTITY && !L.acc) return launch_tiles_one<G, VPL, OUT_IDENTITY, false, TR, TN, 2, MINB, false>(ctx, t);
        return launch_tiles_gv<G, VPL, TR, TN, 1, 4>(ctx, t, L);
    } else {
        const bool rowmap = L.out_mode == OUT_ROWMAP;
        if (ctx->tile_kernel == 1) {
            if (rowmap && L.acc) return launch_tiles_v1<G, VPL, true, true, TR, TN>(ctx, t);
            if (rowmap) return launch_tiles_v1<G, VPL, true, false, TR, TN>(ctx, t);
            if (L.acc) return launch_tiles_v1<G, VPL, false, true, TR, TN>(ctx, t);
            return launch_tiles_v1<G, VPL, false, false, TR, TN>(ctx, t);
        }
        if (rowmap && L.acc) return launch_tiles_one<G, VPL, OUT_ROWMAP, true, TR, TN, 1, MINB, false>(ctx, t);
        if (rowmap) return launch_tiles_one<G, VPL, OUT_ROWMAP, false, TR, TN, 1, MINB, false>(ctx, t);
        if (L.acc) return launch_tiles_one<G, VPL, OUT_IDENTITY, true, TR, TN, 1, MINB, false>(ctx, t);
        return launch_tiles_one<G, VPL, OUT_IDENTITY, false, TR, TN, 1, MINB, false>(ctx, t);
    }
}

// Which row-tile list a launch walks (an index into TILE_LISTS).  The CTAs share one atomic ticket, so the rows in flight
// are about resident CTAs x rows per tile, and the X rows those rows gather from must stay in L2 until the last of their
// ~10 gathers: at k = 128 fp32 on H100, 528 CTAs x 64 rows span 3-4 block-rows whose panels and the head panel take
// about half of the 50 MB L2.  The rule counts the window's own X rows only (resident CTAs x rows x k x element size)
// and lets them take 1 / TILE_L2_WINDOW_DIV of the L2, leaving the rest to the block overlap, the head panel and the CSR
// and C streams; it picks the largest list that fits, never fewer than 16 rows.  The 128-row list needs a TR = 128
// instance (big_ok: k <= 32 on the fp32 paths).
int tile_list_rule(int k, int elem_bytes, long long l2_bytes, long long resident_ctas, bool big_ok) {
    int i = big_ok ? TILE_LIST_BIG : TILE_LIST_SMALL;
    while (i > 0 && resident_ctas * TILE_LISTS[i].rows * k * elem_bytes > l2_bytes / TILE_L2_WINDOW_DIV) --i;
    return i;
}

int tile_list_for(const arrow_ctx *ctx, int k, int elem_bytes, bool big_ok) {
    for (int i = 0; i < N_TILE_LISTS; ++i)                     // forced by ARROW_OPT_TILE_ROWS
        if (TILE_LISTS[i].rows == ctx->tile_rows) return (i == TILE_LIST_BIG && !big_ok) ? TILE_LIST_SMALL : i;
    const int per_sm = ctx->spmm_ctas_per_sm > 0 ? std::min(TILE_CTAS_PER_SM, ctx->spmm_ctas_per_sm) : TILE_CTAS_PER_SM;
    const int sms = ctx->spmm_sm_limit > 0 ? std::min(ctx->sm_count, ctx->spmm_sm_limit) : ctx->sm_count;
    return tile_list_rule(k, elem_bytes, ctx->l2_bytes, (long long)per_sm * sms, big_ok && ctx->big_tiles);
}

// (lanes per row, float4 per lane) for a k4 = k/4; vpl_req = 0 picks the default
int launch_tiles(arrow_ctx *ctx, TileArgs &t, const Csr *A, const TileLaunch &L) {
    const int k4 = t.a.k4;
    int vpl = L.vpl_req;
    // ~8 lanes per row (scripts/kbench.py sweeps the alternatives)
    if (vpl != 1 && vpl != 2 && vpl != 4) vpl = (k4 >= 32) ? 4 : (k4 >= 8 ? 2 : 1);
    while (vpl > 1 && k4 < vpl) vpl >>= 1;
    int lanes = (k4 + vpl - 1) / vpl;                 // lanes needed per row
    if (lanes > 32) { vpl = (k4 + 31) / 32 <= 2 ? 2 : 4; lanes = (k4 + vpl - 1) / vpl; }
    int g = 1;
    while (g < lanes) g <<= 1;
    const int list = tile_list_for(ctx, t.a.k, 4, k4 <= 8);                  // k <= 32: TLB / TLP shapes exist
    const bool big = list == TILE_LIST_BIG;
    t.tiles = A->tiles[list];
    t.n_tiles = A->n_tiles[list];
    // one row per lane group unless asked: on H100 at 10M rows pairs lose at k = 32 (1.75 vs 1.67 ms, scripts/kbench.py
    // variants 3 and 259)
    int rpg = L.rpg_req ? L.rpg_req : (ctx->rows_per_group ? ctx->rows_per_group : 1);
    if (!big || rpg != 2) rpg = 1;                                           // pairs need >= 2 passes per tile
#define TL(GG, VV)                                                                                       \
    if (g == GG && vpl == VV) return launch_tiles_gv<GG, VV, TILE_ROWS, TILE_NNZ, 1, 4>(ctx, t, L)
#define TLB(GG, VV)                                                                                      \
    if (big && rpg == 1 && g == GG && vpl == VV) return launch_tiles_gv<GG, VV, TILE_ROWS_BIG, TILE_NNZ_BIG, 1, 4>(ctx, t, L)
#define TLP(GG, VV)                                                                                      \
    if (big && rpg == 2 && g == GG && vpl == VV) return launch_tiles_gv<GG, VV, TILE_ROWS_BIG, TILE_NNZ_BIG, 2, 4>(ctx, t, L)
    TLP(4, 1); TLP(8, 1); TLP(2, 2); TLP(4, 2);
    if (rpg == 2) rpg = 1;                                                   // no paired kernel for this shape
    TLB(1, 1); TLB(2, 1); TLB(4, 1); TLB(8, 1); TLB(1, 2); TLB(2, 2); TLB(4, 2); TLB(1, 4); TLB(2, 4);
    TL(1, 1); TL(2, 1); TL(4, 1); TL(8, 1); TL(16, 1); TL(32, 1);
    TL(1, 2); TL(2, 2); TL(4, 2); TL(8, 2); TL(16, 2); TL(32, 2);
    TL(1, 4); TL(2, 4); TL(4, 4); TL(8, 4); TL(16, 4);
#undef TL
#undef TLB
#undef TLP
    return fail(ctx, ARROW_ERR_UNSUPPORTED, "no tile kernel for k4=%d vpl=%d", k4, vpl);
}

int pick_variant(int k) {
    (void)k;
    return 3;
}

// ---- float64 dispatch (one GPU): the tile kernel for even k <= 256, the generic kernel otherwise, long rows as fp32 ----
template <int G, int VPL, bool ROWMAP, bool ACC>
int launch_tiles_f64_one(arrow_ctx *ctx, const TileArgsF64 &t) {
    return launch_persistent<k_spmm_tiles_f64<G, VPL, ROWMAP, ACC>, TileCfgF64::SMEM_BYTES>(ctx, t, t.n_tiles, t.ticket);
}

template <int G, int VPL>
int launch_tiles_f64_epi(arrow_ctx *ctx, const TileArgsF64 &t, bool rowmap, bool acc) {
    if (rowmap && acc) return launch_tiles_f64_one<G, VPL, true, true>(ctx, t);
    if (rowmap) return launch_tiles_f64_one<G, VPL, true, false>(ctx, t);
    if (acc) return launch_tiles_f64_one<G, VPL, false, true>(ctx, t);
    return launch_tiles_f64_one<G, VPL, false, false>(ctx, t);
}

// (lanes per row, double2 per lane) from k2 = k/2 the way launch_tiles picks them from k/4: ~8 lanes per row
int launch_tiles_f64(arrow_ctx *ctx, const TileArgsF64 &t, bool rowmap, bool acc) {
    const int k2 = t.a.k2;
    const int vpl = (k2 >= 32) ? 4 : (k2 >= 8 ? 2 : 1);
    const int lanes = (k2 + vpl - 1) / vpl;           // <= 32: k2 <= 128
    int g = 1;
    while (g < lanes) g <<= 1;
#define TF(GG, VV) \
    if (g == GG && vpl == VV) return launch_tiles_f64_epi<GG, VV>(ctx, t, rowmap, acc)
    TF(1, 1); TF(2, 1); TF(4, 1); TF(8, 1);
    TF(4, 2); TF(8, 2); TF(16, 2);
    TF(8, 4); TF(16, 4); TF(32, 4);
#undef TF
    return fail(ctx, ARROW_ERR_UNSUPPORTED, "no float64 tile kernel for k2=%d vpl=%d", k2, vpl);
}

// the product of spmm_impl for float64 operands; `a` carries the validated operands (value / tile pointers are double)
int spmm_f64(arrow_ctx *ctx, const Csr *A, const SpmmArgs &a, bool rowmap, bool acc) {
    const int k = a.k;
    if (k % 2 != 0 || k > 256) {
        launch_generic<PlusTimes<double>>(ctx, a, rowmap, acc);
    } else if (A->n_tiles[TILE_LIST_SMALL] > 0) {
        TileArgsF64 t;
        t.a.indptr = a.indptr;
        t.a.indices = a.indices;
        t.a.vals = reinterpret_cast<const double *>(a.vals);
        t.a.X = reinterpret_cast<const double *>(a.X);
        t.a.C = reinterpret_cast<double *>(a.C);
        t.a.rowmap = a.rowmap;
        t.a.n_rows = a.n_rows;
        t.a.k = k;
        t.a.k2 = k / 2;
        t.a.long_threshold = a.long_threshold;
        t.a.add_src = reinterpret_cast<const double *>(a.add_src);
        t.a.add_map = a.add_map;
        const int list = tile_list_for(ctx, k, 8, false);              // one tile kernel size: TR = 64
        t.tiles = A->tiles[list];
        t.n_tiles = A->n_tiles[list];
        t.skip = (A->may_skip || ctx->force_skip_path) ? 1 : 0;
        t.ticket = ctx->tile_ticket + 2 * ctx->cur_lane;
        t.l2_hints = (rowmap || acc) ? ctx->l2_hints_fused : ctx->l2_hints_plain;
        const int rc = launch_tiles_f64(ctx, t, rowmap, acc);
        if (rc != ARROW_OK) return rc;
    }
    CUDA_TRY(ctx, cudaGetLastError());
    return launch_long_rows<PlusTimes<double>>(ctx, A, a, rowmap, acc);
}

// ------------------------------------------------------------------------------------------------
// tropical semirings (one GPU, fp32): C[r] = (⊕_p A[r,p] ⊗ X[col_p]) ⊕ add[add_map[r]] with ⊗ = the fp32 add (one
// rounding per term) and ⊕ = min / max.  ⊕ is exact and does not depend on the order of the terms, so every kernel below
// gives the same bits on every grid, tile size and lane split.  A semiring is a type with zero() (the ⊕ identity), plus()
// and times(); (+, x) keeps the kernels above.
// ------------------------------------------------------------------------------------------------
struct SrMinPlus {
    using T = float;
    static constexpr bool kValues = true;
    __device__ __forceinline__ static float zero() { return __int_as_float(0x7f800000); }       // +inf
    __device__ __forceinline__ static float one() { return 0.0f; }                               // the ⊗ identity
    __device__ __forceinline__ static float plus(float a, float b) { return fminf(a, b); }
    __device__ __forceinline__ static float times(float a, float x) { return __fadd_rn(a, x); }
    __device__ __forceinline__ static float mac(float acc, float v, float x) { return plus(acc, times(v, x)); }
};
struct SrMaxPlus {
    using T = float;
    static constexpr bool kValues = true;
    __device__ __forceinline__ static float zero() { return __int_as_float(0xff800000); }       // -inf
    __device__ __forceinline__ static float one() { return 0.0f; }
    __device__ __forceinline__ static float plus(float a, float b) { return fmaxf(a, b); }
    __device__ __forceinline__ static float times(float a, float x) { return __fadd_rn(a, x); }
    __device__ __forceinline__ static float mac(float acc, float v, float x) { return plus(acc, times(v, x)); }
};
// The bottleneck semirings: ⊕ and ⊗ are both min or max, so every result is one of the operands (no rounding).  FMNMX
// drops a NaN operand (a NaN weight passes the feature through, a NaN feature becomes the ⊗ identity at the first level
// with the identity) and orders -0 below +0 (DESIGN.md §4).  (max, min): widest paths; (min, max): minimax paths.
struct SrMaxMin {
    using T = float;
    static constexpr bool kValues = true;
    __device__ __forceinline__ static float zero() { return __int_as_float(0xff800000); }       // -inf
    __device__ __forceinline__ static float one() { return __int_as_float(0x7f800000); }        // +inf
    __device__ __forceinline__ static float plus(float a, float b) { return fmaxf(a, b); }
    __device__ __forceinline__ static float times(float a, float x) { return fminf(a, x); }
    __device__ __forceinline__ static float mac(float acc, float v, float x) { return plus(acc, times(v, x)); }
};
struct SrMinMax {
    using T = float;
    static constexpr bool kValues = true;
    __device__ __forceinline__ static float zero() { return __int_as_float(0x7f800000); }       // +inf
    __device__ __forceinline__ static float one() { return __int_as_float(0xff800000); }        // -inf
    __device__ __forceinline__ static float plus(float a, float b) { return fminf(a, b); }
    __device__ __forceinline__ static float times(float a, float x) { return fmaxf(a, x); }
    __device__ __forceinline__ static float mac(float acc, float v, float x) { return plus(acc, times(v, x)); }
};
// the semirings of arrow_spmm_sr / arrow_gather_rows_sr on fp32 tiles
bool fp32_semiring(int semiring) {
    return semiring == ARROW_SR_MIN_PLUS || semiring == ARROW_SR_MAX_PLUS || semiring == ARROW_SR_MAX_MIN ||
           semiring == ARROW_SR_MIN_MAX;
}

template <class SR>
__device__ __forceinline__ float4 sr4_zero() {
    const float z = SR::zero();
    return make_float4(z, z, z, z);
}
template <class SR>
__device__ __forceinline__ void sr_plus(float4 &acc, const float4 &x) {
    acc.x = SR::plus(acc.x, x.x);
    acc.y = SR::plus(acc.y, x.y);
    acc.z = SR::plus(acc.z, x.z);
    acc.w = SR::plus(acc.w, x.w);
}
template <class SR>
__device__ __forceinline__ void sr_plus(float &acc, const float &x) {
    acc = SR::plus(acc, x);
}
// acc = acc ⊕ (a ⊗ x): FADD + FMNMX per element
template <class SR>
__device__ __forceinline__ void sr4_mac(float4 &acc, float a, const float4 &x) {
    acc.x = SR::plus(acc.x, SR::times(a, x.x));
    acc.y = SR::plus(acc.y, SR::times(a, x.y));
    acc.z = SR::plus(acc.z, SR::times(a, x.z));
    acc.w = SR::plus(acc.w, SR::times(a, x.w));
}

// The k_spmm_tiles_v1 pipeline (CSR slices by cp.async.bulk on an mbarrier, two stages, persistent CTAs on the atomic
// ticket, a lane group per row, float4 gathers under the L2 policies) with the semiring's inner step and one epilogue:
// C[r] = the product, ⊕ the addend row when add_map[r] >= 0.
template <int G, int VPL, class SR, int TR, int TN>
__global__ void __launch_bounds__(TILE_THREADS, 4) k_spmm_tiles_sr(TileArgs t) {
    constexpr int TILE_PTR_WORDS = TileCfg<TR, TN>::PTR_WORDS;
    constexpr int TILE_NNZ_WORDS = TileCfg<TR, TN>::NNZ_WORDS;
    constexpr int TILE_STAGE_WORDS = TileCfg<TR, TN>::STAGE_WORDS;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    int *stage_base = reinterpret_cast<int *>(smem_raw);
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem_raw + (size_t)2 * TILE_STAGE_WORDS * 4);
    const SpmmArgs &a = t.a;
    constexpr int RPW = 32 / G;
    constexpr int UNROLL = (VPL >= 4) ? 2 : (VPL == 2 ? 4 : 8);
    constexpr int TAIL = (UNROLL >= 4) ? UNROLL / 2 : UNROLL;     // predicated tail batches
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const bool EXACT = (t.a.k4 == G * VPL);                       // every lane owns valid columns
    const int gl = lane % G;
    const int gi = lane / G;
    const int k4 = a.k4;
    const float4 *__restrict__ Xl = reinterpret_cast<const float4 *>(a.X) + gl;
    float4 *__restrict__ Cl = reinterpret_cast<float4 *>(a.C) + gl;
    const uint64_t pol_keep = (t.l2_hints & 1) ? l2_policy_evict_last() : l2_policy_evict_normal();
    const uint64_t pol_stream = (t.l2_hints & 2) ? l2_policy_evict_first() : l2_policy_evict_normal();

    if (threadIdx.x == 0) {
        mbar_init(&bars[0], 1);
        mbar_init(&bars[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    auto issue_csr = [&](int tile, int st) {
        const int4 d = __ldg(t.tiles + tile);
        const int rb4 = d.x & ~3;
        const int a0 = d.z & ~3;
        const uint32_t ptr_bytes = (uint32_t)(((d.y - rb4 + 1) + 3) & ~3) * 4u;
        const uint32_t nnz_bytes = (uint32_t)(((d.w - a0) + 3) & ~3) * 4u;
        int *sp = stage_base + (size_t)st * TILE_STAGE_WORDS;
        mbar_expect_tx(&bars[st], ptr_bytes + 2u * nnz_bytes);
        bulk_g2s_hint(sp, a.indptr + rb4, ptr_bytes, &bars[st], pol_stream);
        if (nnz_bytes) {
            bulk_g2s_hint(sp + TILE_PTR_WORDS, a.indices + a0, nnz_bytes, &bars[st], pol_stream);
            bulk_g2s_hint(sp + TILE_PTR_WORDS + TILE_NNZ_WORDS, a.vals + a0, nnz_bytes, &bars[st], pol_stream);
        }
    };

    // the n-th tile of a CTA uses stage n & 1 and waits for completion (n >> 1) & 1 of that stage's barrier: one counter
    // instead of a stage index and a parity word keeps the VPL = 4 instances free of spills
    __shared__ int s_next[TILE_STAGES];
    int tile = blockIdx.x;
    if (tile < t.n_tiles && threadIdx.x == 0) issue_csr(tile, 0);
    for (unsigned int n = 0; tile < t.n_tiles; ++n) {
        const int st = (int)(n & 1u);
        if (threadIdx.x == 0) {
            const int next = atomicAdd(t.ticket, 1) + (int)gridDim.x;
            s_next[st] = next;
            if (next < t.n_tiles) issue_csr(next, st ^ 1);
        }
        const int4 d = __ldg(t.tiles + tile);
        mbar_wait(&bars[st], (n >> 1) & 1u);
        const int *sp = stage_base + (size_t)st * TILE_STAGE_WORDS;
        const int *s_ptr = sp + (d.x - (d.x & ~3));
        const int a0 = d.z & ~3;
        const int *s_idx = sp + TILE_PTR_WORDS - a0;                    // index with global nnz offsets
        const float *s_val = reinterpret_cast<const float *>(sp + TILE_PTR_WORDS + TILE_NNZ_WORDS) - a0;
        const int n_rows_tile = d.y - d.x;

        for (int lr = warp * RPW + gi; lr < n_rows_tile; lr += (TILE_THREADS / 32) * RPW) {
            const int s = s_ptr[lr];
            const int e = s_ptr[lr + 1];
            if (e - s > a.long_threshold) continue;
            const long long row = (long long)d.x + lr;
            float4 acc[VPL];
#pragma unroll
            for (int i = 0; i < VPL; ++i) acc[i] = sr4_zero<SR>();
            if (a.add_map != nullptr) {
                // the addend is requested first so that its latency hides behind the gathers
                const int am = __ldg(a.add_map + row);
                if (am >= 0) {
                    const float4 *ar = reinterpret_cast<const float4 *>(a.add_src) + (long long)am * k4 + gl;
#pragma unroll
                    for (int i = 0; i < VPL; ++i)
                        if (gl + i * G < k4) acc[i] = ld_f4_hint(ar + i * G, pol_stream);
                }
            }
            int p = s;
            if (EXACT && !t.skip) {
                // unpredicated batches: full UNROLL batches, then the remainder as 4 / 2 / 1
                auto batch = [&](auto n_tag) {
                    constexpr int N = decltype(n_tag)::value;
                    float4 x[N][VPL];
#pragma unroll
                    for (int u = 0; u < N; ++u) {
                        const float4 *xr = Xl + (long long)s_idx[p + u] * k4;
#pragma unroll
                        for (int i = 0; i < VPL; ++i) x[u][i] = ldg_f4_hint(xr + i * G, pol_keep);
                    }
#pragma unroll
                    for (int u = 0; u < N; ++u) {
                        const float v = s_val[p + u];
#pragma unroll
                        for (int i = 0; i < VPL; ++i) sr4_mac<SR>(acc[i], v, x[u][i]);
                    }
                    p += N;
                };
                while (p + UNROLL <= e) batch(std::integral_constant<int, UNROLL>{});
                if constexpr (UNROLL >= 8) { if (e - p >= 4) batch(std::integral_constant<int, 4>{}); }
                if constexpr (UNROLL >= 4) { if (e - p >= 2) batch(std::integral_constant<int, 2>{}); }
                if (e - p >= 1) batch(std::integral_constant<int, 1>{});
            }
            // tail (and the general case): predicated batches of TAIL.  A skipped entry (column -1) or a slot past the
            // row's end gets the ⊕ identity as its weight and zeros as its X row, whose term is the ⊕ identity again and
            // leaves acc unchanged: ∓inf + 0 = ∓inf in (min, +) / (max, +), min(-inf, 0) = -inf in (max, min) and
            // max(+inf, 0) = +inf in (min, max) (one select per slot instead of one per element).  Columns past k4 are computed on zeros and never stored.
            // Here and in the batches the weights are read from shared memory once the gathers are back (fewer live
            // registers across the gathers).
            for (; p < e; p += TAIL) {
                float4 x[TAIL][VPL];
#pragma unroll
                for (int u = 0; u < TAIL; ++u) {
                    const int c = (p + u < e) ? s_idx[p + u] : -1;
                    const float4 *xr = Xl + (long long)c * k4;              // c = -1: address arithmetic only
#pragma unroll
                    for (int i = 0; i < VPL; ++i)
                        x[u][i] = (c >= 0 && gl + i * G < k4) ? ldg_f4_hint(xr + i * G, pol_keep) : f4_zero();
                }
#pragma unroll
                for (int u = 0; u < TAIL; ++u) {
                    const int c = (p + u < e) ? s_idx[p + u] : -1;
                    const float v = (c >= 0) ? s_val[p + u] : SR::zero();
#pragma unroll
                    for (int i = 0; i < VPL; ++i) sr4_mac<SR>(acc[i], v, x[u][i]);
                }
            }
            float4 *cr = Cl + row * k4;
#pragma unroll
            for (int i = 0; i < VPL; ++i)
                if (gl + i * G < k4) st_f4_hint(cr + i * G, acc[i], pol_stream);
        }
        __syncthreads();            // stage `st` may be refilled by the next iteration's copy
        tile = s_next[st];
    }
}

// dst[r] = dst[r] ⊕ src[map[r]] (map[r] >= 0): the backward exchange of a semiring step (k_gather_rows without peers)
template <typename VT, int G, class SR>
__global__ void __launch_bounds__(256) k_gather_rows_sr(VT *__restrict__ dst, const VT *__restrict__ src,
                                                        const int *__restrict__ map, long long n_rows, int vec_per_row) {
    constexpr int RPW = 32 / G;
    const int lane = threadIdx.x & 31;
    const int gl = lane % G, gi = lane / G;
    const long long warps_total = (long long)gridDim.x * (blockDim.x >> 5);
    const long long warp_id = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    for (long long r = warp_id * RPW + gi; r < n_rows; r += warps_total * RPW) {
        const int m = __ldg(map + r);
        if (m < 0) continue;
        const VT *sp = src + (long long)m * vec_per_row;
        VT *dp = dst + r * vec_per_row;
        for (int v0 = gl; v0 < vec_per_row; v0 += 4 * G) {
            VT val[4];
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (v0 + j * G < vec_per_row) val[j] = sp[v0 + j * G];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (v0 + j * G < vec_per_row) {
                    VT old = dp[v0 + j * G];
                    sr_plus<SR>(old, val[j]);
                    dp[v0 + j * G] = old;
                }
            }
        }
    }
}

// rows (warp per row) in which two equally shaped tiles differ in some element, compared by value (-0 == +0, NaN != NaN)
template <typename T>
__global__ void __launch_bounds__(256) k_count_diff(const T *__restrict__ a, const T *__restrict__ b, long long rows,
                                                    int k, unsigned long long *__restrict__ count) {
    __shared__ unsigned int s_count;
    if (threadIdx.x == 0) s_count = 0u;
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const long long warps_total = (long long)gridDim.x * (blockDim.x >> 5);
    const long long warp_id = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    for (long long r = warp_id; r < rows; r += warps_total) {
        bool diff = false;
        for (int c = lane; c < k; c += 32) diff |= (a[r * k + c] != b[r * k + c]);
        if (__any_sync(0xffffffffu, diff) && lane == 0) atomicAdd(&s_count, 1u);
    }
    __syncthreads();
    if (threadIdx.x == 0 && s_count) atomicAdd(count, (unsigned long long)s_count);
}

template <int G, int VPL, class SR, int TR, int TN>
int launch_tiles_sr_one(arrow_ctx *ctx, const TileArgs &t) {
    return launch_persistent<k_spmm_tiles_sr<G, VPL, SR, TR, TN>, TileCfg<TR, TN>::SMEM_BYTES>(ctx, t, t.n_tiles, t.ticket);
}

// (lanes per row, float4 per lane) and tile size as launch_tiles picks them for a plain launch with the default options
template <class SR>
int launch_tiles_sr_shape(arrow_ctx *ctx, TileArgs &t, const Csr *A) {
    const int k4 = t.a.k4;
    const int vpl = (k4 >= 32) ? 4 : (k4 >= 8 ? 2 : 1);
    const int lanes = (k4 + vpl - 1) / vpl;           // <= 16: k4 <= 64
    int g = 1;
    while (g < lanes) g <<= 1;
    const int list = tile_list_for(ctx, t.a.k, 4, k4 <= 8);                  // k <= 32: SRB shapes exist
    const bool big = list == TILE_LIST_BIG;
    t.tiles = A->tiles[list];
    t.n_tiles = A->n_tiles[list];
#define TSR(GG, VV, TR, TN) return launch_tiles_sr_one<GG, VV, SR, TR, TN>(ctx, t)
#define SRB(GG, VV) if (big && g == GG && vpl == VV) TSR(GG, VV, TILE_ROWS_BIG, TILE_NNZ_BIG)
#define SRS(GG, VV) if (g == GG && vpl == VV) TSR(GG, VV, TILE_ROWS, TILE_NNZ)
    SRB(1, 1); SRB(2, 1); SRB(4, 1); SRB(8, 1); SRB(4, 2);
    SRS(1, 1); SRS(2, 1); SRS(4, 1); SRS(8, 1); SRS(4, 2); SRS(8, 2); SRS(16, 2); SRS(8, 4); SRS(16, 4);
#undef SRS
#undef SRB
#undef TSR
    return fail(ctx, ARROW_ERR_UNSUPPORTED, "no semiring tile kernel for k4=%d vpl=%d", k4, vpl);
}

// the product of arrow_spmm_sr for the fp32 semirings; `a` carries the validated fp32 operands (identity output rows)
template <class SR>
int spmm_sr(arrow_ctx *ctx, const Csr *A, const SpmmArgs &a) {
    const int k = a.k;
    if (k % 4 != 0 || k > 256) {
        launch_generic<SR>(ctx, a, false, false);
    } else if (A->n_tiles[TILE_LIST_SMALL] > 0) {
        TileArgs t;
        t.a = a;
        t.skip = (A->may_skip || ctx->force_skip_path) ? 1 : 0;
        t.ticket = ctx->tile_ticket + 2 * ctx->cur_lane;
        t.l2_hints = ctx->l2_hints_plain;
        t.prefetch = 0;
        const int rc = launch_tiles_sr_shape<SR>(ctx, t, A);
        if (rc != ARROW_OK) return rc;
    }
    CUDA_TRY(ctx, cudaGetLastError());
    return launch_long_rows<SR>(ctx, A, a, false, false);
}

template <class SR>
int gather_rows_sr(arrow_ctx *ctx, DenseBuf *D, const DenseBuf *S, const IdxMap *m) {
    const long long n_rows = m->n;
    if (n_rows == 0) return ARROW_OK;
    const int k = D->k;
    const bool vec = (k % 4 == 0);
    const int vpr = vec ? k / 4 : k;
    int g = 1;
    while (g < vpr && g < 32) g <<= 1;                       // lanes per row
    if (g > 8 && vpr <= 32) g = 8;                           // 8 lanes x 4 vectors cover k <= 128 in one pass
    const int threads = 256;
    const long long rows_per_cta = (threads / 32) * (32 / g);
    int grid = (int)std::min<long long>((n_rows + rows_per_cta - 1) / rows_per_cta, (long long)ctx->sm_count * 8);
    grid = std::max(grid, 1);
#define LAUNCH_GS(VT, GG)                                                                                        \
    k_gather_rows_sr<VT, GG, SR><<<grid, threads, 0, cur_stream(ctx)>>>(reinterpret_cast<VT *>(D->p),            \
                                                                        reinterpret_cast<const VT *>(S->p), m->p, n_rows, vpr)
#define DISPATCH_GS(VT)                                                                                          \
    do {                                                                                                         \
        switch (g) {                                                                                             \
            case 1: LAUNCH_GS(VT, 1); break;                                                                     \
            case 2: LAUNCH_GS(VT, 2); break;                                                                     \
            case 4: LAUNCH_GS(VT, 4); break;                                                                     \
            case 8: LAUNCH_GS(VT, 8); break;                                                                     \
            case 16: LAUNCH_GS(VT, 16); break;                                                                   \
            default: LAUNCH_GS(VT, 32); break;                                                                   \
        }                                                                                                        \
    } while (0)
    if (vec) DISPATCH_GS(float4);
    else DISPATCH_GS(float);
#undef DISPATCH_GS
#undef LAUNCH_GS
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
    return ARROW_OK;
}

// ------------------------------------------------------------------------------------------------
// the boolean semiring (or, and) on bit tiles (ARROW_B1, one GPU): C[r] = (OR_p X[col_p]) | add[add_map[r]].  ⊗ is "the
// entry exists", so the CSR values are never read (the CSR stage copy carries row pointers and column indices only); ⊕ is
// OR.  A row of k columns is bit_row_words(k) uint32 words, a multiple of 4: the fp32 tile pipeline with k4 = words / 4
// uint4 per row.  OR is exact, associative, commutative and idempotent: every kernel, grid and tile list gives the same bits.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void u4_or(uint4 &acc, const uint4 &x) {
    acc.x |= x.x; acc.y |= x.y; acc.z |= x.z; acc.w |= x.w;
}
__device__ __forceinline__ void u4_or(unsigned &acc, const unsigned &x) { acc |= x; }        // one-word rows
template <class V> __device__ __forceinline__ V v_zero();
template <> __device__ __forceinline__ uint4 v_zero<uint4>() { return make_uint4(0u, 0u, 0u, 0u); }
template <> __device__ __forceinline__ unsigned v_zero<unsigned>() { return 0u; }
__device__ __forceinline__ unsigned ldg_u4_hint(const unsigned *ptr, uint64_t pol) {
    unsigned r;
    asm("ld.global.nc.L2::cache_hint.b32 %0, [%1], %2;" : "=r"(r) : "l"(ptr), "l"(pol));
    return r;
}
__device__ __forceinline__ unsigned ld_u4_hint(const unsigned *ptr, uint64_t pol) {
    unsigned r;
    asm("ld.global.L2::cache_hint.b32 %0, [%1], %2;" : "=r"(r) : "l"(ptr), "l"(pol));
    return r;
}
__device__ __forceinline__ void st_u4_hint(unsigned *ptr, const unsigned &v, uint64_t pol) {
    asm volatile("st.global.L2::cache_hint.b32 [%0], %1, %2;" ::"l"(ptr), "r"(v), "l"(pol) : "memory");
}

template <int TR, int TN>
struct TileCfgBits {                                   // TileCfg without the values stream
    static constexpr int PTR_WORDS = TileCfg<TR, TN>::PTR_WORDS;
    static constexpr int NNZ_WORDS = TileCfg<TR, TN>::NNZ_WORDS;
    static constexpr int STAGE_WORDS = PTR_WORDS + NNZ_WORDS;
    static constexpr size_t SMEM_BYTES = (size_t)TILE_STAGES * STAGE_WORDS * 4 + 64;
};

// G lanes own a row, VPL vectors V each (uint4; one uint32 for the one-word rows of k <= 32).  Splitting a row's entries over S groups of G lanes (OR-reduced with shuffles) was
// measured slower for every S > 1 (DESIGN.md section 3), so one lane group walks all of a row's entries.
template <int G, int VPL, int TR, int TN, class V = uint4>
__global__ void __launch_bounds__(TILE_THREADS, 4) k_spmm_tiles_bits(TileArgs t) {
    constexpr int TILE_PTR_WORDS = TileCfgBits<TR, TN>::PTR_WORDS;
    constexpr int TILE_STAGE_WORDS = TileCfgBits<TR, TN>::STAGE_WORDS;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    int *stage_base = reinterpret_cast<int *>(smem_raw);
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem_raw + (size_t)TILE_STAGES * TILE_STAGE_WORDS * 4);
    const SpmmArgs &a = t.a;
    constexpr int RPW = 32 / G;
    constexpr int UNROLL = (VPL == 2) ? 4 : 8;
    constexpr int TAIL = UNROLL / 2;                              // predicated tail batches
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const bool EXACT = (t.a.k4 == G * VPL);                       // every lane owns valid columns
    const int gc = lane % G;                                      // the lane's first V of the row
    const int gi = lane / G;
    const int k4 = a.k4;
    const uint64_t pol_keep = (t.l2_hints & 1) ? l2_policy_evict_last() : l2_policy_evict_normal();
    const uint64_t pol_stream = (t.l2_hints & 2) ? l2_policy_evict_first() : l2_policy_evict_normal();

    if (threadIdx.x == 0) {
        mbar_init(&bars[0], 1);
        mbar_init(&bars[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    auto issue_csr = [&](int tile, int st) {
        const int4 d = __ldg(t.tiles + tile);
        const int rb4 = d.x & ~3;
        const int a0 = d.z & ~3;
        const uint32_t ptr_bytes = (uint32_t)(((d.y - rb4 + 1) + 3) & ~3) * 4u;
        const uint32_t nnz_bytes = (uint32_t)(((d.w - a0) + 3) & ~3) * 4u;
        int *sp = stage_base + (size_t)st * TILE_STAGE_WORDS;
        mbar_expect_tx(&bars[st], ptr_bytes + nnz_bytes);     // no values stream
        bulk_g2s_hint(sp, a.indptr + rb4, ptr_bytes, &bars[st], pol_stream);
        if (nnz_bytes) bulk_g2s_hint(sp + TILE_PTR_WORDS, a.indices + a0, nnz_bytes, &bars[st], pol_stream);
    };

    __shared__ int s_next[TILE_STAGES];
    int tile = blockIdx.x;
    if (tile < t.n_tiles && threadIdx.x == 0) issue_csr(tile, 0);
    for (unsigned int n = 0; tile < t.n_tiles; ++n) {
        const int st = (int)(n & 1u);
        if (threadIdx.x == 0) {
            const int next = atomicAdd(t.ticket, 1) + (int)gridDim.x;
            s_next[st] = next;
            if (next < t.n_tiles) issue_csr(next, st ^ 1);
        }
        const int4 d = __ldg(t.tiles + tile);
        mbar_wait(&bars[st], (n >> 1) & 1u);
        const int *sp = stage_base + (size_t)st * TILE_STAGE_WORDS;
        const int *s_ptr = sp + (d.x - (d.x & ~3));
        const int a0 = d.z & ~3;
        const int *s_idx = sp + TILE_PTR_WORDS - a0;                    // index with global nnz offsets
        const int n_rows_tile = d.y - d.x;

        for (int lr = warp * RPW + gi; lr < n_rows_tile; lr += (TILE_THREADS / 32) * RPW) {
            const int s = s_ptr[lr];
            const int e = s_ptr[lr + 1];
            if (e - s > a.long_threshold) continue;
            const long long row = (long long)d.x + lr;
            V acc[VPL];
#pragma unroll
            for (int i = 0; i < VPL; ++i) acc[i] = v_zero<V>();
            if (a.add_map != nullptr) {
                const int am = __ldg(a.add_map + row);
                if (am >= 0) {
                    const V *ar = reinterpret_cast<const V *>(a.add_src) + (long long)am * k4 + gc;
#pragma unroll
                    for (int i = 0; i < VPL; ++i)
                        if (gc + i * G < k4) acc[i] = ld_u4_hint(ar + i * G, pol_stream);
                }
            }
            int p = s;
            if (EXACT && !t.skip) {
                // unpredicated batches: full UNROLL batches, then the remainder as 4 / 2 / 1
                auto batch = [&](auto n_tag) {
                    constexpr int N = decltype(n_tag)::value;
                    V x[N][VPL];
#pragma unroll
                    for (int u = 0; u < N; ++u) {
                        const V *xr = reinterpret_cast<const V *>(a.X) + (long long)s_idx[p + u] * k4 + gc;
#pragma unroll
                        for (int i = 0; i < VPL; ++i) x[u][i] = ldg_u4_hint(xr + i * G, pol_keep);
                    }
#pragma unroll
                    for (int u = 0; u < N; ++u)
#pragma unroll
                        for (int i = 0; i < VPL; ++i) u4_or(acc[i], x[u][i]);
                    p += N;
                };
                while (p + UNROLL <= e) batch(std::integral_constant<int, UNROLL>{});
                if constexpr (UNROLL >= 8) { if (e - p >= 4) batch(std::integral_constant<int, 4>{}); }
                if (e - p >= 2) batch(std::integral_constant<int, 2>{});
                if (e - p >= 1) batch(std::integral_constant<int, 1>{});
            }
            // tail (and the general case): predicated batches; a skipped entry (column -1) or a slot past the row's end
            // ORs zeros
            for (; p < e; p += TAIL) {
                V x[TAIL][VPL];
#pragma unroll
                for (int u = 0; u < TAIL; ++u) {
                    const int c = (p + u < e) ? s_idx[p + u] : -1;
                    const V *xr = reinterpret_cast<const V *>(a.X) + (long long)c * k4 + gc;   // c = -1: address arithmetic only
#pragma unroll
                    for (int i = 0; i < VPL; ++i)
                        x[u][i] = (c >= 0 && gc + i * G < k4) ? ldg_u4_hint(xr + i * G, pol_keep) : v_zero<V>();
                }
#pragma unroll
                for (int u = 0; u < TAIL; ++u)
#pragma unroll
                    for (int i = 0; i < VPL; ++i) u4_or(acc[i], x[u][i]);
            }
            V *cr = reinterpret_cast<V *>(a.C) + row * k4 + gc;
#pragma unroll
            for (int i = 0; i < VPL; ++i)
                if (gc + i * G < k4) st_u4_hint(cr + i * G, acc[i], pol_stream);
        }
        __syncthreads();            // stage `st` may be refilled by the next iteration's copy
        tile = s_next[st];
    }
}

// (or, and) for the row-parallel long-row kernels, on uint32 words (a.k carries the row's words)
struct OrAnd {
    using T = unsigned;
    static constexpr bool kValues = false;
    __device__ __forceinline__ static unsigned zero() { return 0u; }
    __device__ __forceinline__ static unsigned plus(unsigned a, unsigned b) { return a | b; }
    __device__ __forceinline__ static unsigned mac(unsigned acc, unsigned, unsigned x) { return acc | x; }
};

// dst[r] |= src[map[r]] (map[r] >= 0): the backward exchange of an (or, and) step; a lane group of G lanes per row,
// whole uint4 of the padded rows
template <int G>
__global__ void __launch_bounds__(256) k_gather_rows_or(uint4 *__restrict__ dst, const uint4 *__restrict__ src,
                                                        const int *__restrict__ map, long long n_rows, int vec_per_row) {
    constexpr int RPW = 32 / G;
    const int lane = threadIdx.x & 31;
    const int gl = lane % G, gi = lane / G;
    const long long warps_total = (long long)gridDim.x * (blockDim.x >> 5);
    const long long warp_id = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    for (long long r = warp_id * RPW + gi; r < n_rows; r += warps_total * RPW) {
        const int m = __ldg(map + r);
        if (m < 0) continue;
        const uint4 *sp = src + (long long)m * vec_per_row;
        uint4 *dp = dst + r * vec_per_row;
        for (int v = gl; v < vec_per_row; v += G) {
            uint4 x = sp[v];
            u4_or(x, dp[v]);
            dp[v] = x;
        }
    }
}

// dst[r] |= src[map[r]] on one-word rows
__global__ void __launch_bounds__(256) k_gather_rows_or_word(unsigned *__restrict__ dst, const unsigned *__restrict__ src,
                                                             const int *__restrict__ map, long long n) {
    for (long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (long long)gridDim.x * blockDim.x) {
        const int m = __ldg(map + r);
        if (m >= 0) dst[r] |= src[m];
    }
}

// bits of the k columns of word w of a row (the padding bits of the last word and of the padding words are outside)
__device__ __forceinline__ unsigned int bit_col_mask(int w, int k) {
    const int lo = w * 32;
    if (lo >= k) return 0u;
    return (k - lo >= 32) ? 0xffffffffu : ((1u << (k - lo)) - 1u);
}

// rows (warp per row) of two bit tiles that differ in one of the k columns
__global__ void __launch_bounds__(256) k_count_diff_bits(const unsigned int *__restrict__ a, const unsigned int *__restrict__ b,
                                                         long long rows, int k, int words, unsigned long long *__restrict__ count) {
    __shared__ unsigned int s_count;
    if (threadIdx.x == 0) s_count = 0u;
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const long long warps_total = (long long)gridDim.x * (blockDim.x >> 5);
    const long long warp_id = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    for (long long r = warp_id; r < rows; r += warps_total) {
        bool diff = false;
        for (int w = lane; w * 32 < k; w += 32) diff |= ((a[r * words + w] ^ b[r * words + w]) & bit_col_mask(w, k)) != 0u;
        if (__any_sync(0xffffffffu, diff) && lane == 0) atomicAdd(&s_count, 1u);
    }
    __syncthreads();
    if (threadIdx.x == 0 && s_count) atomicAdd(count, (unsigned long long)s_count);
}

// dist[r, c] = level for every column c < k whose bit is set in `nw` and clear in `old`; counts those bits.  One thread
// per (row, word).
__global__ void __launch_bounds__(256) k_bits_mark_new(const unsigned int *__restrict__ nw, const unsigned int *__restrict__ old,
                                                       int *__restrict__ dist, long long rows, int k, int words, int level,
                                                       unsigned long long *__restrict__ count) {
    const int used = (k + 31) / 32;
    const long long total = rows * used;
    const long long stride = (long long)gridDim.x * blockDim.x;
    unsigned long long mine = 0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
        const long long r = i / used;
        const int w = (int)(i - r * used);
        unsigned int fresh = nw[r * words + w] & ~old[r * words + w] & bit_col_mask(w, k);
        mine += (unsigned long long)__popc(fresh);
        int *drow = dist + r * k + w * 32;
        while (fresh) {
            const int c = __ffs(fresh) - 1;
            drow[c] = level;
            fresh &= fresh - 1u;
        }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, off);
    if ((threadIdx.x & 31) == 0 && mine) atomicAdd(count, mine);
}

template <int G, int VPL, int TR, int TN, class V = uint4>
int launch_tiles_bits_one(arrow_ctx *ctx, const TileArgs &t) {
    return launch_persistent<k_spmm_tiles_bits<G, VPL, TR, TN, V>, TileCfgBits<TR, TN>::SMEM_BYTES>(ctx, t, t.n_tiles, t.ticket);
}

// (lanes per row, uint4 per lane) from k4 = words / 4 as launch_tiles_sr_shape picks them from an fp32 row of `words`
// columns, except that rows of more than 32 uint4 take 32 lanes of 2 (the VPL = 4 instances spill)
int launch_tiles_bits_shape(arrow_ctx *ctx, TileArgs &t, const Csr *A) {
    if (t.a.k == 1) {                  // one-word rows (k <= 32): a lane per row, one uint32 gather per entry
        t.a.k4 = 1;
        const int list = tile_list_for(ctx, 1, 4, true);
        t.tiles = A->tiles[list];
        t.n_tiles = A->n_tiles[list];
#define BIW(TR, TN) return launch_tiles_bits_one<1, 1, TR, TN, unsigned>(ctx, t)
        if (list == TILE_LIST_BIG) BIW(TILE_ROWS_BIG, TILE_NNZ_BIG);
        BIW(TILE_ROWS, TILE_NNZ);
#undef BIW
    }
    const int k4 = t.a.k4;
    const int vpl = k4 >= 8 ? 2 : 1;
    const int lanes = (k4 + vpl - 1) / vpl;           // <= 32: k4 <= 64
    int g = 1;
    while (g < lanes) g <<= 1;
    const int list = tile_list_for(ctx, 4 * k4, 4, k4 <= 8);                 // the row's bytes as an fp32 row
    const bool big = list == TILE_LIST_BIG;
    t.tiles = A->tiles[list];
    t.n_tiles = A->n_tiles[list];
#define TBI(GG, VV, TR, TN) return launch_tiles_bits_one<GG, VV, TR, TN>(ctx, t)
#define BIB(GG, VV) if (big && g == GG && vpl == VV) TBI(GG, VV, TILE_ROWS_BIG, TILE_NNZ_BIG)
#define BIS(GG, VV) if (g == GG && vpl == VV) TBI(GG, VV, TILE_ROWS, TILE_NNZ)
    BIB(1, 1); BIB(2, 1); BIB(4, 1); BIB(8, 1); BIB(4, 2);
    BIS(1, 1); BIS(2, 1); BIS(4, 1); BIS(8, 1); BIS(4, 2); BIS(8, 2); BIS(16, 2); BIS(32, 2);
#undef BIS
#undef BIB
#undef TBI
    return fail(ctx, ARROW_ERR_UNSUPPORTED, "no bit tile kernel for k4=%d vpl=%d", k4, vpl);
}

// the product of arrow_spmm_sr in (or, and); `a` carries the validated bit operands, a.k = the row's words
int spmm_bits(arrow_ctx *ctx, const Csr *A, const SpmmArgs &a) {
    if (A->n_tiles[TILE_LIST_SMALL] > 0) {
        TileArgs t;
        t.a = a;
        t.skip = (A->may_skip || ctx->force_skip_path) ? 1 : 0;
        t.ticket = ctx->tile_ticket + 2 * ctx->cur_lane;
        t.l2_hints = ctx->l2_hints_plain;
        t.prefetch = 0;
        const int rc = launch_tiles_bits_shape(ctx, t, A);
        if (rc != ARROW_OK) return rc;
    }
    CUDA_TRY(ctx, cudaGetLastError());
    return launch_long_rows<OrAnd>(ctx, A, a, false, false);
}

constexpr int BITS_MAX_K = 8192;    // 256 words = 64 uint4 per row: the widest (G, VPL) = (32, 2) tile shape

int gather_rows_or(arrow_ctx *ctx, DenseBuf *D, const DenseBuf *S, const IdxMap *m) {
    const long long n_rows = m->n;
    if (n_rows == 0) return ARROW_OK;
    if (bit_row_words(D->k) == 1) {    // one-word rows: a thread per row
        int grid = (int)std::max<long long>(1, std::min<long long>((n_rows + 255) / 256, (long long)ctx->sm_count * 8));
        k_gather_rows_or_word<<<grid, 256, 0, cur_stream(ctx)>>>(reinterpret_cast<unsigned *>(D->p), reinterpret_cast<const unsigned *>(S->p), m->p, n_rows);
        ctx->launches++;
        CUDA_TRY(ctx, cudaGetLastError());
        return ARROW_OK;
    }
    const int vpr = bit_row_words(D->k) / 4;
    int g = 1;
    while (g < vpr && g < 8) g <<= 1;                        // lanes per row
    const int threads = 256;
    const long long rows_per_cta = (threads / 32) * (32 / g);
    int grid = (int)std::min<long long>((n_rows + rows_per_cta - 1) / rows_per_cta, (long long)ctx->sm_count * 8);
    grid = std::max(grid, 1);
    uint4 *dp = reinterpret_cast<uint4 *>(D->p);
    const uint4 *sp = reinterpret_cast<const uint4 *>(S->p);
    switch (g) {
        case 1: k_gather_rows_or<1><<<grid, threads, 0, cur_stream(ctx)>>>(dp, sp, m->p, n_rows, vpr); break;
        case 2: k_gather_rows_or<2><<<grid, threads, 0, cur_stream(ctx)>>>(dp, sp, m->p, n_rows, vpr); break;
        case 4: k_gather_rows_or<4><<<grid, threads, 0, cur_stream(ctx)>>>(dp, sp, m->p, n_rows, vpr); break;
        default: k_gather_rows_or<8><<<grid, threads, 0, cur_stream(ctx)>>>(dp, sp, m->p, n_rows, vpr); break;
    }
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
    return ARROW_OK;
}

// ------------------------------------------------------------------------------------------------
// direction-optimising BFS on bit tiles.  With add_identity a fused (or, and) step is X' = X | M X, M the level-0 x level-0
// union of every level's entries (r, c) as edges cmap_j(c) -> cmap_j(r).  Inside a BFS, where X_h = X_{h-1} | M X_{h-1},
// the next level is X_h | M F_h with F_h the rows holding a bit of X_h & ~X_{h-1}: a push of the frontier rows along the
// transposed matrix (arrow_adj_build) gives the pull step's bits exactly, for the cost of the frontier's edges.
// ------------------------------------------------------------------------------------------------
struct AdjPart {
    const int *__restrict__ indptr;
    const int *__restrict__ indices;
    const int *__restrict__ map;      // nullptr: the identity
    long long nnz;
    int n_rows;
};

// the largest i in [lo, hi] with a[i] <= e (a non-decreasing, a[lo] <= e): the row of entry e given row pointers, the
// frontier row of edge slot e given first edge offsets (rows without entries share their offset with the next row)
__device__ __forceinline__ int last_le(const int *__restrict__ a, int lo, int hi, long long e) {
    while (lo < hi) {
        const int mid = (int)(((long long)lo + hi + 1) >> 1);
        if ((long long)__ldg(a + mid) <= e) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// edges of one block: entry (r, c) with c >= 0 gives u -> v = map(c) -> map(r); an end at -1 drops it, and so does u == v
// unless LOOPS (the weighted push adjacency keeps self-loops: a negative one changes a min-plus step).  Counts them into
// *count; with `keys` also appends (u << 32) | v at a warp-aggregated cursor (the order is fixed by the sort), and with W
// the entry's value w_in[e] at the same slot of w_out.  IN appends (v << 32) | u instead: the in-adjacency, row v by source.
template <bool W, bool IN = false, bool LOOPS = W>
__global__ void __launch_bounds__(256) k_adj_edges(AdjPart p, unsigned long long *__restrict__ count,
                                                   unsigned long long *__restrict__ keys,
                                                   const float *__restrict__ w_in = nullptr, float *__restrict__ w_out = nullptr) {
    const int lane = threadIdx.x & 31;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long e0 = (long long)blockIdx.x * blockDim.x + (threadIdx.x & ~31); e0 < p.nnz; e0 += stride) {
        const long long e = e0 + lane;
        bool ok = false;
        unsigned long long key = 0;
        if (e < p.nnz) {
            const int c = __ldg(p.indices + e);
            if (c >= 0) {
                const int r = last_le(p.indptr, 0, p.n_rows - 1, e);
                const int u = p.map ? __ldg(p.map + c) : c;
                const int v = p.map ? __ldg(p.map + r) : r;
                ok = u >= 0 && v >= 0 && (LOOPS || u != v);
                key = IN ? ((unsigned long long)(unsigned)v << 32) | (unsigned)u
                         : ((unsigned long long)(unsigned)u << 32) | (unsigned)v;
            }
        }
        const unsigned ball = __ballot_sync(0xffffffffu, ok);
        if (ball == 0u) continue;
        unsigned long long base = 0;
        if (lane == 0) base = atomicAdd(count, (unsigned long long)__popc(ball));
        if (keys != nullptr) {
            base = __shfl_sync(0xffffffffu, base, 0);
            if (ok) {
                const unsigned long long at = base + __popc(ball & ((1u << lane) - 1u));
                keys[at] = key;
                if (W) w_out[at] = __ldg(w_in + e);
            }
        }
    }
}

// the CSR of the sorted keys: indices[e] = v of key e, indptr[u] = the first key of row u (lower bound of u << 32)
__global__ void __launch_bounds__(256) k_adj_csr(const unsigned long long *__restrict__ keys, long long m, long long n,
                                                 int *__restrict__ indptr, int *__restrict__ indices) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    for (long long e = t; e < m; e += stride) indices[e] = (int)(unsigned)keys[e];
    for (long long u = t; u <= n; u += stride) {
        const unsigned long long want = (unsigned long long)u << 32;
        long long lo = 0, hi = m;
        while (lo < hi) {
            const long long mid = (lo + hi) >> 1;
            if (keys[mid] < want) lo = mid + 1;
            else hi = mid;
        }
        indptr[u] = (int)lo;
    }
}

constexpr int MARK_THREADS = 256;

// k_bits_mark_new's level record and bit count, a thread per row, plus the frontier record: the rows with a fresh bit in a
// column < k, listed with their first edge offset in the push adjacency.  A CTA scans (1 << 32) + degree over its rows and
// claims its slice of the list with one 64-bit atomicAdd on counts[1], so list positions (high half) and edge offsets (low
// half) come from the same add and increase together; the edge sum stays below 2^31 and never carries into the rows.
__global__ void __launch_bounds__(MARK_THREADS) k_bits_mark_frontier(const unsigned int *__restrict__ nw,
                                                                     const unsigned int *__restrict__ old,
                                                                     int *__restrict__ dist, long long rows, int k, int words,
                                                                     int level, const int *__restrict__ adj_ptr,
                                                                     int *__restrict__ front_rows, int *__restrict__ front_off,
                                                                     unsigned long long *__restrict__ counts) {
    constexpr int WARPS = MARK_THREADS / 32;
    __shared__ unsigned long long s_warp[WARPS];
    __shared__ unsigned long long s_base;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int used = (k + 31) / 32;
    unsigned long long mine = 0;
    for (long long r0 = (long long)blockIdx.x * MARK_THREADS; r0 < rows; r0 += (long long)gridDim.x * MARK_THREADS) {
        const long long r = r0 + threadIdx.x;
        unsigned long long claim = 0;
        if (r < rows) {
            bool any = false;
            for (int w = 0; w < used; ++w) {
                unsigned int fresh = nw[r * words + w] & ~old[r * words + w] & bit_col_mask(w, k);
                any |= fresh != 0u;
                mine += (unsigned long long)__popc(fresh);
                int *drow = dist + r * k + w * 32;
                while (fresh) {
                    const int c = __ffs(fresh) - 1;
                    drow[c] = level;
                    fresh &= fresh - 1u;
                }
            }
            if (any) claim = (1ull << 32) | (unsigned)(__ldg(adj_ptr + r + 1) - __ldg(adj_ptr + r));
        }
        unsigned long long incl = claim;                      // inclusive scan over the warp
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            const unsigned long long y = __shfl_up_sync(0xffffffffu, incl, off);
            if (lane >= off) incl += y;
        }
        if (lane == 31) s_warp[warp] = incl;
        __syncthreads();
        if (threadIdx.x == 0) {
            unsigned long long total = 0;
            for (int i = 0; i < WARPS; ++i) {
                const unsigned long long t = s_warp[i];
                s_warp[i] = total;
                total += t;
            }
            s_base = total ? atomicAdd(counts + 1, total) : 0ull;
        }
        __syncthreads();
        if (claim) {
            const unsigned long long at = s_base + s_warp[warp] + incl - claim;
            front_rows[at >> 32] = (int)r;
            front_off[at >> 32] = (int)(unsigned)at;
        }
        __syncthreads();                                      // s_warp / s_base are rewritten by the next pass
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, off);
    if (lane == 0 && mine) atomicAdd(counts, mine);
}

__device__ __forceinline__ void red_or_b32(unsigned *p, unsigned v) {
    asm volatile("red.global.or.b32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void red_or_b64(unsigned long long *p, unsigned long long v) {
    asm volatile("red.global.or.b64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
// out[vec] |= x, skipping zero words: one 32-bit OR for a one-word row, two 64-bit ORs for a 16-byte vector of a padded row
__device__ __forceinline__ void push_or(unsigned *out, long long vec, unsigned x) {
    if (x) red_or_b32(out + vec, x);
}
__device__ __forceinline__ void push_or(unsigned *out, long long vec, const uint4 &x) {
    unsigned long long *p = reinterpret_cast<unsigned long long *>(out + 4 * vec);
    if (x.x | x.y) red_or_b64(p, ((unsigned long long)x.y << 32) | x.x);
    if (x.z | x.w) red_or_b64(p + 1, ((unsigned long long)x.w << 32) | x.z);
}

constexpr int PUSH_THREADS = 256, PUSH_ITEMS = 4;

// out[v] |= x[u] along every edge u -> v of the recorded frontier rows.  An item is (edge slot e, vector q of the row's
// first `vecs` vectors, those that hold columns < k); a CTA walks chunks of PUSH_THREADS * PUSH_ITEMS consecutive items, so
// a hub row's edges spread over many CTAs.  The frontier rows of a chunk come from one binary search over the record's
// edge offsets, each item's row from a search between them.
template <class V>
__global__ void __launch_bounds__(PUSH_THREADS) k_bits_push(const V *__restrict__ x, unsigned *__restrict__ out,
                                                            const int *__restrict__ adj_ptr, const int *__restrict__ adj_idx,
                                                            const int *__restrict__ front_rows,
                                                            const int *__restrict__ front_off, int n_front, long long n_items,
                                                            int vecs, int row_vecs) {
    constexpr long long CHUNK = (long long)PUSH_THREADS * PUSH_ITEMS;
    __shared__ int s_lo, s_hi;
    for (long long c0 = (long long)blockIdx.x * CHUNK; c0 < n_items; c0 += (long long)gridDim.x * CHUNK) {
        if (threadIdx.x == 0) {
            const long long c1 = (c0 + CHUNK < n_items ? c0 + CHUNK : n_items) - 1;
            s_lo = last_le(front_off, 0, n_front - 1, c0 / vecs);
            s_hi = last_le(front_off, s_lo, n_front - 1, c1 / vecs);
        }
        __syncthreads();
        const int lo = s_lo, hi = s_hi;
#pragma unroll
        for (int j = 0; j < PUSH_ITEMS; ++j) {
            const long long i = c0 + j * PUSH_THREADS + threadIdx.x;
            if (i < n_items) {
                const long long e = i / vecs;
                const int q = (int)(i - e * vecs);
                const int p = last_le(front_off, lo, hi, e);
                const int u = __ldg(front_rows + p);
                const int v = __ldg(adj_idx + __ldg(adj_ptr + u) + (int)(e - __ldg(front_off + p)));
                push_or(out, (long long)v * row_vecs + q, x[(long long)u * row_vecs + q]);
            }
        }
        __syncthreads();                                      // s_lo / s_hi are rewritten by the next chunk
    }
}

// ------------------------------------------------------------------------------------------------
// BFS parents on bit tiles.  Inside a BFS, X_h = X_{h-1} | M X_{h-1}.  A bit (v, s) fresh at level h (set in X_h, clear in
// X_{h-1}) has an in-neighbour u of v in M holding bit s in X_{h-1}, and every such u has hop level exactly h - 1 (had u
// reached s by level h - 2, v would hold s in X_{h-1}).  So the parent of (v, s), the smallest in-neighbour one hop
// closer, is the first u of v's ascending in-list (arrow_adj_build_in) whose bit s is set in X_{h-1}: a bottom-up search
// over the frontier rows that stops once every fresh bit of the row has its first hit.
// ------------------------------------------------------------------------------------------------
constexpr int PARENT_SEG = 512;     // in-edges per segment: longer rows are split into segments across warps

__device__ __forceinline__ unsigned bv_and(unsigned a, unsigned b) { return a & b; }
__device__ __forceinline__ unsigned bv_andn(unsigned a, unsigned b) { return a & ~b; }
__device__ __forceinline__ unsigned bv_or(unsigned a, unsigned b) { return a | b; }
__device__ __forceinline__ bool bv_any(unsigned a) { return a != 0u; }
__device__ __forceinline__ unsigned bv_zero(unsigned) { return 0u; }
__device__ __forceinline__ unsigned bv_shfl_up(unsigned a, int d) { return __shfl_up_sync(0xffffffffu, a, d); }
__device__ __forceinline__ unsigned bv_shfl(unsigned a, int l) { return __shfl_sync(0xffffffffu, a, l); }
__device__ __forceinline__ unsigned bv_word(unsigned a, int) { return a; }
__device__ __forceinline__ unsigned bv_cols(unsigned, int q, int k) { return bit_col_mask(q, k); }
__device__ __forceinline__ uint4 bv_and(uint4 a, uint4 b) { return make_uint4(a.x & b.x, a.y & b.y, a.z & b.z, a.w & b.w); }
__device__ __forceinline__ uint4 bv_andn(uint4 a, uint4 b) { return make_uint4(a.x & ~b.x, a.y & ~b.y, a.z & ~b.z, a.w & ~b.w); }
__device__ __forceinline__ uint4 bv_or(uint4 a, uint4 b) { return make_uint4(a.x | b.x, a.y | b.y, a.z | b.z, a.w | b.w); }
__device__ __forceinline__ bool bv_any(uint4 a) { return (a.x | a.y | a.z | a.w) != 0u; }
__device__ __forceinline__ uint4 bv_zero(uint4) { return make_uint4(0u, 0u, 0u, 0u); }
__device__ __forceinline__ uint4 bv_shfl_up(uint4 a, int d) {
    return make_uint4(__shfl_up_sync(0xffffffffu, a.x, d), __shfl_up_sync(0xffffffffu, a.y, d),
                      __shfl_up_sync(0xffffffffu, a.z, d), __shfl_up_sync(0xffffffffu, a.w, d));
}
__device__ __forceinline__ uint4 bv_shfl(uint4 a, int l) {
    return make_uint4(__shfl_sync(0xffffffffu, a.x, l), __shfl_sync(0xffffffffu, a.y, l), __shfl_sync(0xffffffffu, a.z, l),
                      __shfl_sync(0xffffffffu, a.w, l));
}
__device__ __forceinline__ unsigned bv_word(const uint4 &a, int i) { return i == 0 ? a.x : i == 1 ? a.y : i == 2 ? a.z : a.w; }
__device__ __forceinline__ uint4 bv_cols(uint4, int q, int k) {
    return make_uint4(bit_col_mask(4 * q, k), bit_col_mask(4 * q + 1, k), bit_col_mask(4 * q + 2, k), bit_col_mask(4 * q + 3, k));
}

struct ParentArgs {
    const void *__restrict__ nw;        // X_h (bit tile, row_vecs V per row)
    const void *__restrict__ old;       // X_{h-1}
    int *__restrict__ parent;           // int32 [rows x k]
    const int *__restrict__ in_ptr;     // in-adjacency
    const int *__restrict__ in_idx;
    const int *__restrict__ rows;       // frontier rows (row pass), or nullptr: the segment pass over segs
    const int4 *__restrict__ segs;
    int n_items;                        // frontier rows, or segments
    int k, row_vecs, vecs;              // columns, V per row, V that hold columns < k
    unsigned long long *__restrict__ scanned;   // optional: in-edges gathered
};

// A warp per item: a frontier row (row pass; a row of more than PARENT_SEG in-edges only has its fresh elements set to
// -1, its segments follow in the segment pass) or a segment {v, first, end} of a long row (segment pass: skipped unless v
// has a fresh bit).  Lane = (edge slot g, vector q): G lanes share an edge, 32 / G edges go at once, lane q holds vectors
// q, q + G, ... of the row's fresh bits.  For a batch of edges (ascending u) an exclusive OR-scan over the edge slots of
// X_{h-1}[u] & fresh gives each fresh bit's first hit, which is its parent within the batch; the row pass stores it, the
// segment pass folds it with a non-returning unsigned min (-1 is above every label, so the result is exact whatever the
// order of the segments).  A row or segment stops once no fresh bit is left.
// parent = -1 for the bits of f (every edge slot holds the same f: slot 0 writes)
template <class V, int G, int VPL>
__device__ __forceinline__ void set_no_parent(int *prow, const V (&f)[VPL], int g, int q) {
    constexpr int WORDS = (int)(sizeof(V) / 4);
    if (g != 0) return;
#pragma unroll
    for (int j = 0; j < VPL; ++j)
        for (int w = 0; w < WORDS; ++w)
            for (unsigned m = bv_word(f[j], w); m; m &= m - 1u) prow[((q + j * G) * WORDS + w) * 32 + __ffs(m) - 1] = -1;
}

template <class V, int G, int VPL>
__global__ void __launch_bounds__(256) k_bits_parents(ParentArgs a) {
    constexpr int E = 32 / G;                                 // edges per batch
    constexpr int WORDS = (int)(sizeof(V) / 4);
    const V *__restrict__ nw = reinterpret_cast<const V *>(a.nw);
    const V *__restrict__ old = reinterpret_cast<const V *>(a.old);
    const int lane = threadIdx.x & 31, g = lane / G, q = lane % G;
    const long long warps_total = (long long)gridDim.x * (blockDim.x >> 5);
    unsigned long long scanned = 0;
    for (long long it = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); it < a.n_items; it += warps_total) {
        int v, b, e;
        if (a.rows) {
            v = __ldg(a.rows + it);
            b = __ldg(a.in_ptr + v);
            e = __ldg(a.in_ptr + v + 1);
        } else {
            const int4 s = __ldg(a.segs + it);
            v = s.x, b = s.y, e = s.z;
        }
        const bool seg = a.rows == nullptr;
        const bool long_row = !seg && e - b > PARENT_SEG;
        V f[VPL];
        bool any = false;
#pragma unroll
        for (int j = 0; j < VPL; ++j) {
            const int qq = q + j * G;
            f[j] = bv_zero(V());
            if (qq < a.vecs) {
                const long long at = (long long)v * a.row_vecs + qq;
                f[j] = bv_and(bv_andn(nw[at], old[at]), bv_cols(V(), qq, a.k));
            }
            any |= bv_any(f[j]);
        }
        if (!__any_sync(0xffffffffu, any)) continue;
        int *prow = a.parent + (long long)v * a.k;
        if (long_row) {                                       // the segment pass folds into -1
            set_no_parent<V, G, VPL>(prow, f, g, q);
            continue;
        }
        for (int base = b; base < e; base += E) {
            const int edge = base + g;
            const int u = edge < e ? __ldg(a.in_idx + edge) : -1;
            bool left = false;
#pragma unroll
            for (int j = 0; j < VPL; ++j) {
                const int qq = q + j * G;
                V x = bv_zero(V());
                if (u >= 0 && qq < a.vecs) x = bv_and(old[(long long)u * a.row_vecs + qq], f[j]);
                V incl = x;                                   // inclusive OR-scan over the edge slots
#pragma unroll
                for (int d = G; d < 32; d <<= 1) {
                    const V y = bv_shfl_up(incl, d);
                    if (lane >= d) incl = bv_or(incl, y);
                }
                V first = x;                                  // bits whose first hit in the batch is this edge
                if (E > 1) {
                    const V before = bv_shfl_up(incl, G);
                    if (g > 0) first = bv_andn(x, before);
                }
                for (int w = 0; w < WORDS; ++w)
                    for (unsigned m = bv_word(first, w); m; m &= m - 1u) {
                        int *p = prow + (qq * WORDS + w) * 32 + __ffs(m) - 1;
                        if (seg) asm volatile("red.global.min.u32 [%0], %1;" ::"l"(p), "r"(u) : "memory");
                        else *p = u;
                    }
                f[j] = bv_andn(f[j], E > 1 ? bv_shfl(incl, 32 - G + q) : incl);
                left |= bv_any(f[j]);
            }
            scanned += (unsigned long long)min(E, e - base);
            if (!__any_sync(0xffffffffu, left)) break;
        }
        if (!seg) set_no_parent<V, G, VPL>(prow, f, g, q);      // fresh bits without a hit (none inside a BFS)
    }
    if (a.scanned && lane == 0 && scanned) atomicAdd(a.scanned, scanned);
}

template <class V, int G, int VPL>
void launch_parents(arrow_ctx *ctx, const ParentArgs &p, int grid) {
    k_bits_parents<V, G, VPL><<<grid, 256, 0, cur_stream(ctx)>>>(p);
    ctx->launches++;
}
// the row pass over the recorded frontier rows, then the segment pass over the long rows' segments
int bits_parents(arrow_ctx *ctx, ParentArgs p, const Adj *in, const Adj *a) {
    const int per_sm = ctx->spmm_ctas_per_sm > 0 ? std::min(ctx->spmm_ctas_per_sm, 8) : 8;
    const int sms = ctx->spmm_sm_limit > 0 ? std::min(ctx->sm_count, ctx->spmm_sm_limit) : ctx->sm_count;
    const bool word = p.row_vecs == 1 && p.k <= 32;
    int g = 1;
    while (g < 32 && g * (p.vecs > 32 ? 2 : 1) < p.vecs) g <<= 1;     // lanes per edge
    for (int pass = 0; pass < 2; ++pass) {
        p.rows = pass == 0 ? a->front_rows : nullptr;
        p.segs = pass == 0 ? nullptr : in->segs;
        p.n_items = pass == 0 ? (int)a->n_front : in->n_segs;
        if (p.n_items == 0) continue;
        const int grid = (int)std::min<long long>((p.n_items + 7) / 8, (long long)per_sm * sms);
        if (word) launch_parents<unsigned, 1, 1>(ctx, p, grid);
        else if (p.vecs > 32) launch_parents<uint4, 32, 2>(ctx, p, grid);
        else if (g == 1) launch_parents<uint4, 1, 1>(ctx, p, grid);
        else if (g == 2) launch_parents<uint4, 2, 1>(ctx, p, grid);
        else if (g == 4) launch_parents<uint4, 4, 1>(ctx, p, grid);
        else if (g == 8) launch_parents<uint4, 8, 1>(ctx, p, grid);
        else if (g == 16) launch_parents<uint4, 16, 1>(ctx, p, grid);
        else launch_parents<uint4, 32, 1>(ctx, p, grid);
        CUDA_TRY(ctx, cudaGetLastError());
    }
    return ARROW_OK;
}

// ------------------------------------------------------------------------------------------------
// Betweenness on bit tiles (Brandes over k source columns).  M is taken as a set: a list entry equal to its predecessor in
// the (sorted) list is skipped.  Path counts: a bit (v, s) fresh at level h has sigma[v, s] = the sum of sigma[u, s] over
// the in-neighbours u holding s in X_{h-1} (exactly those at level h - 1, see the parents pass).  Dependencies: for
// L[u, s] = h, delta[u, s] = sigma[u, s] * sum of fl((1 + delta[w, s]) / sigma[w, s]) over the out-neighbours w with
// L[w, s] = h + 1.  Both sums run over the list in ascending order, PATH_SEG entries at a time from the row's start: each
// segment's terms are summed left to right into a partial that starts at 0, and the partials are added in segment order.
// A warp takes one (row, 32-column word), a lane per column.  A list of at most PATH_SEG entries is summed by that warp;
// a longer one is split at the adjacency's segments (Adj::segs): a segment pass gives each (segment, word) its own warp,
// which stores its partial in Adj::seg_part, and the row pass adds the row's partials in segment order.  The order depends
// on the adjacency alone and no floating-point atomics are needed: the results are exact functions of the inputs.
// ------------------------------------------------------------------------------------------------
constexpr int PATH_SEG = PARENT_SEG;    // list entries per partial sum: the adjacencies' segment length

struct PathArgs {
    const unsigned *__restrict__ nw;    // X_h (path counts) -- bit tiles of `words` words per row
    const unsigned *__restrict__ old;   // X_{h-1}
    const int *__restrict__ dist;       // level tile (dependencies)
    double *sigma;                      // path counts: read at level h - 1, written at the fresh bits of level h
    double *delta;                      // dependencies: read at level h + 1, written at level h
    const int *__restrict__ ptr;        // in-adjacency (path counts) or push adjacency (dependencies)
    const int *__restrict__ idx;
    const int *__restrict__ rows;       // frontier rows of level h (row pass), or nullptr: the segment pass over segs
    const int4 *__restrict__ segs;      // {row, first, end, 0} per segment of the lists longer than PATH_SEG, by row
    int n_segs;
    double *seg_part;                   // [n_segs x k] partial sums of the segment pass
    int n_items;                        // (rows or segments) x used words (below 2^31 whenever the fp64 tiles fit)
    int k, words, used, level;
    unsigned long long *__restrict__ scanned;   // optional: list entries read, once per (row or segment, word) (a 64-bit
                                                //   sum kept in registers across the division's slow-path call would spill)
};

// the first segment of row v in segs (sorted by row; v has at least one)
__device__ __forceinline__ int first_seg(const int4 *__restrict__ segs, int n, int v) {
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (__ldg(&segs[mid].x) < v) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

// item `it` of a pass: (row, list [b, e) of the row, range [sb, se) summed here, word w, segment index or -1)
struct PathItem {
    int v, b, e, sb, se, w, seg;
};
__device__ __forceinline__ PathItem path_item(const PathArgs &a, int it) {
    PathItem t;
    const int i = it / a.used;
    t.w = it - i * a.used;
    if (a.rows) {
        t.v = __ldg(a.rows + i);
        t.b = __ldg(a.ptr + t.v);
        t.e = __ldg(a.ptr + t.v + 1);
        t.sb = t.b;
        t.se = t.e;
        t.seg = -1;
    } else {
        const int4 g = __ldg(a.segs + i);
        t.v = g.x;
        t.b = __ldg(a.ptr + t.v);
        t.e = __ldg(a.ptr + t.v + 1);
        t.sb = g.y;
        t.se = g.z;
        t.seg = i;
    }
    return t;
}

// the row pass's total for lane column c of a long row: its segment partials added in order (active lanes only)
__device__ __forceinline__ double seg_total(const PathArgs &a, int v, int c) {
    double total = 0.0;
    for (int j = first_seg(a.segs, a.n_segs, v); j < a.n_segs && __ldg(&a.segs[j].x) == v; ++j)
        total += a.seg_part[(long long)j * a.k + c];
    return total;
}

// sigma[v, c] for the fresh bits c of word w of every frontier row v.  Per batch of 32 list entries lane j loads entry j
// and the hit mask X_{h-1}[u] & fresh; then the entries with a hit are taken in order, each lane adding sigma[u, c] for its
// own column c when hit.  Only the sigma words of hit columns are read.
__global__ void __launch_bounds__(256) k_bits_path_counts(PathArgs a) {
    const int lane = threadIdx.x & 31;
    const int warps_total = gridDim.x * (blockDim.x >> 5);
    for (int it = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); it < a.n_items; it += warps_total) {
        const PathItem t = path_item(a, it);
        const long long vw = (long long)t.v * a.words + t.w;
        const unsigned fresh = __ldg(a.nw + vw) & ~__ldg(a.old + vw) & bit_col_mask(t.w, a.k);
        if (fresh == 0u) continue;
        const int c = t.w * 32 + lane;
        const bool on = (fresh >> lane) & 1u;
        const bool split = t.seg < 0 && t.e - t.b > PATH_SEG;     // a long row: its segments were summed by the segment pass
        double total = 0.0;
        if (split) {
            if (on) total = seg_total(a, t.v, c);
        } else {
            double part = 0.0;
            for (int base = t.sb; base < t.se; base += 32) {
                const int edge = base + lane;
                int u = 0;
                unsigned hit = 0u;
                if (edge < t.se) {
                    u = __ldg(a.idx + edge);
                    if (edge == t.b || __ldg(a.idx + edge - 1) != u) hit = __ldg(a.old + (long long)u * a.words + t.w) & fresh;
                }
                for (unsigned bal = __ballot_sync(0xffffffffu, hit != 0u); bal; bal &= bal - 1u) {
                    const int j = __ffs(bal) - 1;
                    const int uj = __shfl_sync(0xffffffffu, u, j);
                    const unsigned hj = __shfl_sync(0xffffffffu, hit, j);
                    if ((hj >> lane) & 1u) part += a.sigma[(long long)uj * a.k + c];
                }
            }
            total += part;
            if (a.scanned && lane == 0) atomicAdd(a.scanned, (unsigned long long)(t.se - t.sb));
        }
        if (!on) continue;
        if (t.seg >= 0) a.seg_part[(long long)t.seg * a.k + c] = total;
        else a.sigma[(long long)t.v * a.k + c] = total;
    }
}

// delta[u, c] for the columns c of word w of every recorded row u of level h with L[u, c] = h.  Per batch of 32 list
// entries the warp takes each distinct w in order and reads its level row (one 128-byte line per word); the lanes whose
// column is at level h + 1 there add (1 + delta[w, c]) / sigma[w, c].
__global__ void __launch_bounds__(256) k_bits_dependencies(PathArgs a) {
    const int lane = threadIdx.x & 31;
    const int warps_total = gridDim.x * (blockDim.x >> 5);
    for (int it = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); it < a.n_items; it += warps_total) {
        const PathItem t = path_item(a, it);
        const int c = t.w * 32 + lane;
        const bool mine = c < a.k && __ldg(a.dist + (long long)t.v * a.k + c) == a.level;
        if (!__any_sync(0xffffffffu, mine)) continue;
        const bool split = t.seg < 0 && t.e - t.b > PATH_SEG;
        double total = 0.0;
        if (split) {
            if (mine) total = seg_total(a, t.v, c);
        } else {
            double part = 0.0;
            for (int base = t.sb; base < t.se; base += 32) {
                const int edge = base + lane;
                int x = 0;
                bool ok = false;
                if (edge < t.se) {
                    x = __ldg(a.idx + edge);
                    ok = edge == t.b || __ldg(a.idx + edge - 1) != x;
                }
                for (unsigned bal = __ballot_sync(0xffffffffu, ok); bal; bal &= bal - 1u) {
                    const long long at = (long long)__shfl_sync(0xffffffffu, x, __ffs(bal) - 1) * a.k + c;
                    if (mine && __ldg(a.dist + at) == a.level + 1) part += (1.0 + a.delta[at]) / a.sigma[at];
                }
            }
            total += part;
            if (a.scanned && lane == 0) atomicAdd(a.scanned, (unsigned long long)(t.se - t.sb));
        }
        if (!mine) continue;
        if (t.seg >= 0) a.seg_part[(long long)t.seg * a.k + c] = total;
        else a.delta[(long long)t.v * a.k + c] = a.sigma[(long long)t.v * a.k + c] * total;
    }
}

// out[r, c] = value for every column c < k whose bit is set in `nw` and clear in `old` (fp64 tile); one thread per
// (row, word)
__global__ void __launch_bounds__(256) k_bits_fill_f64(const unsigned *__restrict__ nw, const unsigned *__restrict__ old,
                                                       double *__restrict__ out, long long rows, int k, int words, double value) {
    const int used = (k + 31) / 32;
    const long long total = rows * used;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long r = i / used;
        const int w = (int)(i - r * used);
        double *orow = out + r * k + w * 32;
        for (unsigned m = nw[r * words + w] & ~old[r * words + w] & bit_col_mask(w, k); m; m &= m - 1u) orow[__ffs(m) - 1] = value;
    }
}

// out[r] = x[r, 0] + x[r, 1] + ... + x[r, k - 1], left to right from 0 (fp64); a thread per row
__global__ void __launch_bounds__(256) k_row_sum_f64(const double *__restrict__ x, double *__restrict__ out, long long rows, int k) {
    for (long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += (long long)gridDim.x * blockDim.x) {
        const double *xr = x + r * k;
        double s = 0.0;
        for (int c = 0; c < k; ++c) s += xr[c];
        out[r] = s;
    }
}

// the segments of the lists longer than PATH_SEG entries, {row, first, end, 0} sorted by row and first (synchronises)
cudaError_t build_segs(Adj &a) {
    a.has_segs = true;
    if (a.m <= (int64_t)PATH_SEG) return cudaSuccess;
    std::vector<int> ptr((size_t)a.n + 1);
    cudaError_t e = cudaMemcpy(ptr.data(), a.indptr, ptr.size() * 4, cudaMemcpyDeviceToHost);
    std::vector<int4> segs;
    for (int64_t v = 0; e == cudaSuccess && v < a.n; ++v)
        if (ptr[v + 1] - ptr[v] > PATH_SEG)
            for (int b = ptr[v]; b < ptr[v + 1]; b += PATH_SEG)
                segs.push_back(make_int4((int)v, b, std::min(b + PATH_SEG, ptr[v + 1]), 0));
    if (e == cudaSuccess && !segs.empty()) e = cudaMalloc(&a.segs, segs.size() * sizeof(int4));
    if (e == cudaSuccess && !segs.empty()) e = cudaMemcpy(a.segs, segs.data(), segs.size() * sizeof(int4), cudaMemcpyHostToDevice);
    a.n_segs = e == cudaSuccess ? (int)segs.size() : 0;
    return e;
}

// the grid of a path pass over `items` warp items: the parents pass's CTAs per SM and SM cap
int path_grid(const arrow_ctx *ctx, long long items) {
    const int per_sm = ctx->spmm_ctas_per_sm > 0 ? std::min(ctx->spmm_ctas_per_sm, 8) : 8;
    const int sms = ctx->spmm_sm_limit > 0 ? std::min(ctx->sm_count, ctx->spmm_sm_limit) : ctx->sm_count;
    return (int)std::min<long long>((items + 7) / 8, (long long)per_sm * sms);
}

// the segment pass over the adjacency's segments (their partials into a.seg_part, grown to n_segs x k, unless the passes
// keep no partials), then the row pass over `n_rows` rows, each as launch(grid, args)
template <class Launch>
int launch_seg_passes(arrow_ctx *ctx, PathArgs p, Adj *adj, long long n_rows, Launch &&launch, bool partials = true) {
    if (n_rows == 0) return ARROW_OK;
    if (std::max<long long>(n_rows, adj->n_segs) * p.used > INT_MAX)
        return fail(ctx, ARROW_ERR_RANGE, "%lld rows x %d words exceed the int32 item count", std::max<long long>(n_rows, adj->n_segs), p.used);
    const size_t part_bytes = partials ? (size_t)adj->n_segs * p.k * sizeof(double) : 0;
    if (part_bytes > adj->seg_part_bytes) {
        cudaFree(adj->seg_part);                              // waits for the launches that read it
        adj->seg_part = nullptr;
        adj->seg_part_bytes = 0;
        CUDA_TRY(ctx, cudaMalloc(&adj->seg_part, part_bytes));
        adj->seg_part_bytes = part_bytes;
    }
    p.segs = adj->segs;
    p.n_segs = adj->n_segs;
    p.seg_part = partials ? adj->seg_part : nullptr;
    const int *rows = p.rows;
    for (int pass = 0; pass < 2; ++pass) {
        p.rows = pass == 0 ? nullptr : rows;
        p.n_items = (int)((pass == 0 ? adj->n_segs : n_rows) * p.used);
        if (p.n_items == 0) continue;
        launch(path_grid(ctx, p.n_items), p);
        ctx->launches++;
        CUDA_TRY(ctx, cudaGetLastError());
    }
    return ARROW_OK;
}

int launch_paths(arrow_ctx *ctx, PathArgs p, Adj *adj, long long n_rows, bool dependencies) {
    return launch_seg_passes(ctx, p, adj, n_rows, [&](int grid, const PathArgs &q) {
        if (dependencies) k_bits_dependencies<<<grid, 256, 0, cur_stream(ctx)>>>(q);
        else k_bits_path_counts<<<grid, 256, 0, cur_stream(ctx)>>>(q);
    });
}

// ------------------------------------------------------------------------------------------------
// Weighted betweenness on min-plus fp32 tiles.  D is the fixed point reached, X0 the features the loop started from, and
// the lists are the weighted loop-free adjacencies (arrow_adj_build_loopfree): the entries u -> v of M with u != v, each
// with its weight a.  An entry is tight in column s when D[u, s] < D[v, s] < +inf and fl(a + D[u, s]) == D[v, s]; a pair (u, v)
// is tight when one of its entries is, and counts once, at its first entry.  A tight pair strictly increases D, so the
// tight pairs of a column form a DAG, and Kahn rounds over it order every element after its tight predecessors:
// - the pending pass stores in `state` the number of tight pairs into every finite element (-1 elsewhere), and -2 (depth
//   0) where there is none; those elements' counts are [v in S] (S: D == X0, finite) and their rows round 0's;
// - round r sums sigma over the in-lists of its elements (state -(r + 2)), then releases their tight pairs out with an
//   integer atomic per pair: an element whose counter reaches 0 is at depth r + 1 and its row is listed for round r + 1;
// - the backward sweep visits the rounds from the deepest to 0 and sums the dependencies along the out-lists.
// Each element is written by one lane, after every value it reads is final, and the sums run in the bit passes' order
// (PATH_SEG segments, partials in order): every result depends on D, X0 and the lists alone, never on the schedule.
// ------------------------------------------------------------------------------------------------
enum { WP_PENDING, WP_COUNTS, WP_RELEASE, WP_DEPENDENCIES };

struct WPathArgs {
    PathArgs p;                         // lists, rows, segments, sigma, delta, k, used; p.level is the round
    const float *__restrict__ wt;       // the lists' weights
    const float *__restrict__ D;        // the fixed point reached [n x k]
    const float *__restrict__ x0;       // the features the loop started from [n x k]
    int *state;                         // [n x k]: -1 not finite, > 0 tight pairs still to release, -(depth + 2)
    int *mark;                          // [n]: the last round a row was listed for
    int *next;                          // the rows listed (pending pass: round 0, release pass: round + 1), at *cursor
    unsigned long long *cursor;
};

// u -> v (weight a) is tight: D[u] < D[v] < +inf and fl(a + D[u]) == D[v] (no FMA); the finite target keeps a +inf weight
// or an overflowing sum out of the pairs into an element that is not reached
__device__ __forceinline__ bool wp_tight(float a, float du, float dv) {
    return du < dv && dv < __int_as_float(0x7f800000) && __fadd_rn(a, du) == dv;
}

// lists row v for `round` unless it is already (one lane of the warp)
__device__ __forceinline__ void wp_list(const WPathArgs &a, int v, int round) {
    if (atomicExch(a.mark + v, round) != round) a.next[atomicAdd(a.cursor, 1ull)] = v;
}

// A warp takes one (row, 32-column word), a lane per column, as in the bit passes.  Per batch of 32 list entries lane j
// loads entry j; the first entries of their pairs are then taken in order, each lane testing its own column (a pair with
// duplicates is tight when one of them is: its later entries are read then, past the segment's end if need be).
// PENDING counts the tight pairs in over every row's whole in-list; COUNTS sums sigma over the in-lists of the round's
// elements and RELEASE decrements the counters along their out-lists; DEPENDENCIES sums fl((1 + delta) / sigma) along the
// out-lists.  The two sums split lists longer than PATH_SEG at the adjacency's segments, like the bit passes.
template <int PASS>
__global__ void __launch_bounds__(256) k_wpaths(WPathArgs a) {
    constexpr bool IN = PASS == WP_PENDING || PASS == WP_COUNTS;
    constexpr bool SUM = PASS == WP_COUNTS || PASS == WP_DEPENDENCIES;
    const int lane = threadIdx.x & 31;
    const int warps_total = gridDim.x * (blockDim.x >> 5);
    const int here = -(a.p.level + 2);                        // the state of the round's elements
    for (int it = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); it < a.p.n_items; it += warps_total) {
        PathItem t;
        if (PASS == WP_PENDING) {                             // every row
            t.v = it / a.p.used;
            t.w = it - t.v * a.p.used;
            t.b = t.sb = __ldg(a.p.ptr + t.v);
            t.e = t.se = __ldg(a.p.ptr + t.v + 1);
            t.seg = -1;
        } else {
            t = path_item(a.p, it);
        }
        const int c = t.w * 32 + lane;
        const long long vc = (long long)t.v * a.p.k + c;
        const float dv = c < a.p.k ? __ldg(a.D + vc) : 0.0f;
        const bool mine = c < a.p.k && (PASS == WP_PENDING ? isfinite(dv) : a.state[vc] == here);
        const bool any = __any_sync(0xffffffffu, mine);
        if (PASS != WP_PENDING && !any) continue;
        const bool split = SUM && t.seg < 0 && t.e - t.b > PATH_SEG;
        double part = 0.0;
        int pending = 0;
        if (any && !split) {
            for (int base = t.sb; base < t.se; base += 32) {
                const int e = base + lane;
                int x = 0;
                float w = 0.0f;
                bool first = false, dup = false;
                if (e < t.se) {
                    x = __ldg(a.p.idx + e);
                    w = __ldg(a.wt + e);
                    first = e == t.b || __ldg(a.p.idx + e - 1) != x;
                    dup = e + 1 < t.e && __ldg(a.p.idx + e + 1) == x;
                }
                for (unsigned bal = __ballot_sync(0xffffffffu, first); bal; bal &= bal - 1u) {
                    const int j = __ffs(bal) - 1;
                    const int xj = __shfl_sync(0xffffffffu, x, j);
                    const float wj = __shfl_sync(0xffffffffu, w, j);
                    const bool dj = __shfl_sync(0xffffffffu, dup, j);
                    const long long at = (long long)xj * a.p.k + c;
                    bool tight = false;
                    if (mine) {
                        const float dx = __ldg(a.D + at);
                        const float from = IN ? dx : dv, to = IN ? dv : dx;
                        tight = wp_tight(wj, from, to);
                        for (int d = base + j + 1; dj && !tight && d < t.e && __ldg(a.p.idx + d) == xj; ++d)
                            tight = wp_tight(__ldg(a.wt + d), from, to);
                    }
                    if (PASS == WP_PENDING) {
                        pending += tight;
                    } else if (PASS == WP_COUNTS) {
                        if (tight) part += a.p.sigma[at];
                    } else if (PASS == WP_DEPENDENCIES) {
                        if (tight) {                                  // a successor without paths adds nothing
                            const double sw = a.p.sigma[at];
                            if (sw != 0.0) part += (1.0 + a.p.delta[at]) / sw;
                        }
                    } else {
                        bool ready = false;
                        if (tight && atomicSub(a.state + at, 1) == 1) {
                            a.state[at] = here - 1;
                            ready = true;
                        }
                        if (__any_sync(0xffffffffu, ready) && lane == 0) wp_list(a, xj, a.p.level + 1);
                    }
                }
            }
            if (a.p.scanned && lane == 0) atomicAdd(a.p.scanned, (unsigned long long)(t.se - t.sb));
        }
        if (PASS == WP_PENDING) {
            if (c < a.p.k) {
                const int s = !mine ? -1 : pending > 0 ? pending : -2;
                a.state[vc] = s;
                if (s < 0) a.p.sigma[vc] = s == -2 && dv == __ldg(a.x0 + vc) ? 1.0 : 0.0;
            }
            if (__any_sync(0xffffffffu, mine && pending == 0) && lane == 0) wp_list(a, t.v, 0);
        }
        if (!SUM || !mine) continue;
        const double total = split ? seg_total(a.p, t.v, c) : part;
        if (t.seg >= 0) a.p.seg_part[(long long)t.seg * a.p.k + c] = total;
        else if (PASS == WP_COUNTS) a.p.sigma[vc] = (dv == __ldg(a.x0 + vc) ? 1.0 : 0.0) + total;
        else a.p.delta[vc] = dv == __ldg(a.x0 + vc) ? 0.0 : a.p.sigma[vc] * total;
    }
}

// ------------------------------------------------------------------------------------------------
// direction-optimising shortest and critical paths on fp32 tiles (min-plus, max-plus).  With add_identity a fused step is
// F(X)[v] = ⊕ over in-edges (u, a) of v of fl(a + X[u]), NaN terms dropped, the in-edges being the identity diagonal and
// every level's entries through its row map.  Inside a fixed-point loop, X_h = F(X_{h-1}) <= X_{h-1}; a row whose bits did
// not change contributes terms X_h already holds, so F(X_h)[v] = canon(X_h[v]) ⊕ (⊕ over the frontier rows u -> v of
// fl(a + X_h[u])), canon(x) = fl(0 + x) with NaN as the ⊕ identity: the push of the frontier along the weighted transposed
// operator (arrow_adj_build_weighted) gives the pull step's bits, provided no weight is -0 (fl(-0 + -0) = -0 breaks the
// bit order of the argument).
// ------------------------------------------------------------------------------------------------

// k_count_diff's figure (rows that differ by value: -0 == +0, NaN != NaN) and the frontier record of the rows that differ
// in bits, each with its first edge offset in the push adjacency.  A warp takes its 32 rows of a pass one at a time (lanes
// over the columns) and lane i keeps the claim of the i-th; a CTA claims its slice of the list with one 64-bit atomicAdd
// on counts[1], packed like k_bits_mark_frontier's.  STEPS (arrow_sr_mark_frontier_steps) also writes steps[r, c] = level
// where the two differ in bits, and 0 to every element at level 0.
template <bool STEPS>
__global__ void __launch_bounds__(MARK_THREADS) k_sr_mark_frontier(const float *__restrict__ nw, const float *__restrict__ old,
                                                                   long long rows, int k, const int *__restrict__ adj_ptr,
                                                                   int *__restrict__ front_rows, int *__restrict__ front_off,
                                                                   unsigned long long *__restrict__ counts,
                                                                   int *__restrict__ steps, int level) {
    constexpr int WARPS = MARK_THREADS / 32;
    __shared__ unsigned long long s_warp[WARPS];
    __shared__ unsigned long long s_base;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned long long changed = 0;                           // rows that differ by value (lane 0 counts them)
    for (long long r0 = (long long)blockIdx.x * MARK_THREADS; r0 < rows; r0 += (long long)gridDim.x * MARK_THREADS) {
        const long long w0 = r0 + (long long)warp * 32;
        unsigned long long claim = 0;
        for (int i = 0; i < 32 && w0 + i < rows; ++i) {
            const float *a = nw + (w0 + i) * k, *b = old + (w0 + i) * k;
            bool by_value = false, by_bits = false;
            for (int c = lane; c < k; c += 32) {
                const float x = a[c], y = b[c];
                by_value |= x != y;
                by_bits |= __float_as_uint(x) != __float_as_uint(y);
                if constexpr (STEPS) {
                    const bool differ = __float_as_uint(x) != __float_as_uint(y);
                    if (differ || level == 0) steps[(w0 + i) * k + c] = differ ? level : 0;
                }
            }
            by_value = __any_sync(0xffffffffu, by_value);
            by_bits = __any_sync(0xffffffffu, by_bits);
            changed += (lane == 0 && by_value);
            if (lane == i && by_bits)
                claim = (1ull << 32) | (unsigned)(__ldg(adj_ptr + w0 + i + 1) - __ldg(adj_ptr + w0 + i));
        }
        unsigned long long incl = claim;                      // inclusive scan over the warp
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            const unsigned long long y = __shfl_up_sync(0xffffffffu, incl, off);
            if (lane >= off) incl += y;
        }
        if (lane == 31) s_warp[warp] = incl;
        __syncthreads();
        if (threadIdx.x == 0) {
            unsigned long long total = 0;
            for (int i = 0; i < WARPS; ++i) {
                const unsigned long long t = s_warp[i];
                s_warp[i] = total;
                total += t;
            }
            s_base = total ? atomicAdd(counts + 1, total) : 0ull;
        }
        __syncthreads();
        if (claim) {
            const unsigned long long at = s_base + s_warp[warp] + incl - claim;
            front_rows[at >> 32] = (int)(w0 + lane);
            front_off[at >> 32] = (int)(unsigned)at;
        }
        __syncthreads();                                      // s_warp / s_base are rewritten by the next pass
    }
    if (changed) atomicAdd(counts, changed);
}

// canon(x) = (the ⊗ identity ⊗ x) ⊕ the ⊕ identity: what the identity diagonal contributes to a pull step.  Tropical:
// fl(0 + x), NaN -> the ⊕ identity, -0 -> +0.  Bottleneck: x, NaN -> the ⊗ identity (FMNMX drops it), -0 kept.
template <class SR>
__device__ __forceinline__ float sr_canon(float x) {
    return SR::plus(SR::zero(), SR::times(SR::one(), x));
}
template <class SR>
__global__ void __launch_bounds__(256) k_sr_canon(const float4 *__restrict__ x, float4 *__restrict__ out, long long n4,
                                                  const float *__restrict__ xs, float *__restrict__ outs, long long n) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    for (long long i = t; i < n4; i += stride) {
        const float4 v = x[i];
        out[i] = make_float4(sr_canon<SR>(v.x), sr_canon<SR>(v.y), sr_canon<SR>(v.z), sr_canon<SR>(v.w));
    }
    for (long long i = 4 * n4 + t; i < n; i += stride) outs[i] = sr_canon<SR>(xs[i]);
}

// a non-returning float min / max from integer reductions: a float with the sign bit clear orders like its bits as s32, one
// with the sign bit set in reverse of its bits as u32, and every sign-set bit pattern is above every sign-clear one as
// u32 and below it as s32.  t is never NaN, and the target never holds NaN or -0 (canon).
__device__ __forceinline__ void red_fold(SrMinPlus, float *p, float t) {
    if (__float_as_int(t) >= 0) asm volatile("red.global.min.s32 [%0], %1;" ::"l"(p), "r"(__float_as_int(t)) : "memory");
    else asm volatile("red.global.max.u32 [%0], %1;" ::"l"(p), "r"(__float_as_uint(t)) : "memory");
}
__device__ __forceinline__ void red_fold(SrMaxPlus, float *p, float t) {
    if (__float_as_int(t) >= 0) asm volatile("red.global.max.s32 [%0], %1;" ::"l"(p), "r"(__float_as_int(t)) : "memory");
    else asm volatile("red.global.min.u32 [%0], %1;" ::"l"(p), "r"(__float_as_uint(t)) : "memory");
}
__device__ __forceinline__ bool improves(SrMinPlus, float t, float c) { return t < c; }   // false for a NaN t
__device__ __forceinline__ bool improves(SrMaxPlus, float t, float c) { return t > c; }
// The bottleneck targets may hold -0 and t may be -0: the integer folds above already order -0 below +0 (sign set: below
// every sign-clear pattern), and so must the test, or a +0 term would be dropped against a -0 target.  Among equal
// values only the two zeros differ in bits, and there the signed integers order them the same way.
__device__ __forceinline__ void red_fold(SrMaxMin, float *p, float t) { red_fold(SrMaxPlus(), p, t); }
__device__ __forceinline__ void red_fold(SrMinMax, float *p, float t) { red_fold(SrMinPlus(), p, t); }
__device__ __forceinline__ bool improves(SrMaxMin, float t, float c) {
    return t > c || (t == c && __float_as_int(t) > __float_as_int(c));                   // false for a NaN t
}
__device__ __forceinline__ bool improves(SrMinMax, float t, float c) {
    return t < c || (t == c && __float_as_int(t) < __float_as_int(c));
}

// fold t = fl(a + xu) into *o when it improves on canon(xv), xv the read-only x[v] (failed relaxations cost no atomic)
template <class SR>
__device__ __forceinline__ void sr_relax(float *o, float a, float xu, float xv) {
    const float t = SR::times(a, xu);
    if (improves(SR(), t, sr_canon<SR>(xv))) red_fold(SR(), o, t);
}
template <class SR>
__device__ __forceinline__ void sr_relax(float *o, float a, const float4 &xu, const float4 &xv) {
    sr_relax<SR>(o, a, xu.x, xv.x);
    sr_relax<SR>(o + 1, a, xu.y, xv.y);
    sr_relax<SR>(o + 2, a, xu.z, xv.z);
    sr_relax<SR>(o + 3, a, xu.w, xv.w);
}

// out[v] ⊕= fl(a + x[u]) along every edge (u -> v, a) of the recorded frontier rows.  An item is (edge slot e, vector q of
// the row's `vecs` float4 groups, or columns when k % 4 != 0); CTAs walk chunks like k_bits_push, so a hub row's edges
// spread over many CTAs.
template <class SR, class V>
__global__ void __launch_bounds__(PUSH_THREADS) k_sr_push(const V *__restrict__ x, float *__restrict__ out,
                                                          const int *__restrict__ adj_ptr, const int *__restrict__ adj_idx,
                                                          const float *__restrict__ adj_val,
                                                          const int *__restrict__ front_rows,
                                                          const int *__restrict__ front_off, int n_front, long long n_items,
                                                          int vecs) {
    constexpr long long CHUNK = (long long)PUSH_THREADS * PUSH_ITEMS;
    constexpr int PER = (int)(sizeof(V) / sizeof(float));
    __shared__ int s_lo, s_hi;
    for (long long c0 = (long long)blockIdx.x * CHUNK; c0 < n_items; c0 += (long long)gridDim.x * CHUNK) {
        if (threadIdx.x == 0) {
            const long long c1 = (c0 + CHUNK < n_items ? c0 + CHUNK : n_items) - 1;
            s_lo = last_le(front_off, 0, n_front - 1, c0 / vecs);
            s_hi = last_le(front_off, s_lo, n_front - 1, c1 / vecs);
        }
        __syncthreads();
        const int lo = s_lo, hi = s_hi;
#pragma unroll
        for (int j = 0; j < PUSH_ITEMS; ++j) {
            const long long i = c0 + j * PUSH_THREADS + threadIdx.x;
            if (i < n_items) {
                const long long e = i / vecs;
                const int q = (int)(i - e * vecs);
                const int p = last_le(front_off, lo, hi, e);
                const int u = __ldg(front_rows + p);
                const int slot = __ldg(adj_ptr + u) + (int)(e - __ldg(front_off + p));
                const int v = __ldg(adj_idx + slot);
                const float a = __ldg(adj_val + slot);
                const long long vq = (long long)v * vecs + q;
                sr_relax<SR>(out + vq * PER, a, x[(long long)u * vecs + q], x[vq]);
            }
        }
        __syncthreads();                                      // s_lo / s_hi are rewritten by the next chunk
    }
}

// the push launch of the bottleneck semirings (arrow_sr_push_frontier): k_sr_push on float4 groups or floats
template <class SR>
void launch_bottleneck_push(cudaStream_t stream, int grid, const Adj *a, const DenseBuf *X, DenseBuf *O, long long items, int vecs) {
    if (X->k % 4 == 0)
        k_sr_push<SR, float4><<<grid, PUSH_THREADS, 0, stream>>>(reinterpret_cast<const float4 *>(X->p), O->p, a->indptr,
                                                                 a->indices, a->values, a->front_rows, a->front_off,
                                                                 (int)a->n_front, items, vecs);
    else
        k_sr_push<SR, float><<<grid, PUSH_THREADS, 0, stream>>>(X->p, O->p, a->indptr, a->indices, a->values, a->front_rows,
                                                                a->front_off, (int)a->n_front, items, vecs);
}

// ------------------------------------------------------------------------------------------------
// bottleneck path trees (max-min, min-max).  D is a fixed point of the step with the identity and T the level at which each
// element last changed (k_sr_mark_frontier<true>).  The parent of (v, s) is the smallest in-neighbour u != v with an entry
// of weight a such that a ⊗ D[u] == D[v] in bits and D[u] is strictly better than D[v] in the ⊕ order, or equal to it
// with T[u] < T[v]; -1 for T[v] == 0, for D[v] the ⊕ identity and where there is none.  The parent edges strictly improve D
// or strictly lower T, so they form a forest (DESIGN.md §4).
// ------------------------------------------------------------------------------------------------
struct TreeArgs {
    PathArgs p;                         // the loop-free in-lists, segments, k, used; p.rows: the row pass (every row)
    const float *__restrict__ wt;       // the lists' weights
    const float *__restrict__ D;        // the fixed point [n x k]
    const int *__restrict__ T;          // the step record [n x k]
    int *__restrict__ parent;           // [n x k], -1 everywhere before the passes
    bool seg_pass;                      // the segment pass (items: segments x used words), else rows x used words
};

// the ⊕ order as unsigned integers, -0 below +0 (D never holds NaN where T > 0)
__device__ __forceinline__ unsigned sr_order_key(float x) {
    const unsigned u = __float_as_uint(x);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
template <class SR>
__device__ __forceinline__ bool tree_better(float du, float dv) {
    if constexpr (std::is_same<SR, SrMaxMin>::value) return sr_order_key(du) > sr_order_key(dv);
    else return sr_order_key(du) < sr_order_key(dv);
}

// A warp takes one (row, 32-column word) -- a row's whole list (row pass; lists longer than PATH_SEG are left to the
// segment pass) or one segment of it (segment pass) -- with a lane per column.  Per batch of 32 list entries lane j loads
// entry j; the entries are then taken in order, each pending lane testing its own column, until no lane is pending.  The
// row pass stores a hit, the segment pass folds it with a non-returning unsigned min into the -1 already there.
template <class SR>
__global__ void __launch_bounds__(256) k_sr_tree(TreeArgs a) {
    const int lane = threadIdx.x & 31;
    const int warps_total = gridDim.x * (blockDim.x >> 5);
    unsigned long long scanned = 0;
    for (int it = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); it < a.p.n_items; it += warps_total) {
        PathItem t;
        if (a.seg_pass) {
            t = path_item(a.p, it);
        } else {
            t.v = it / a.p.used;
            t.w = it - t.v * a.p.used;
            t.b = t.sb = __ldg(a.p.ptr + t.v);
            t.e = t.se = __ldg(a.p.ptr + t.v + 1);
            if (t.e - t.b > PATH_SEG) continue;
        }
        const int c = t.w * 32 + lane;
        const long long vc = (long long)t.v * a.p.k + c;
        float dv = 0.0f;
        int tv = 0;
        if (c < a.p.k) {
            dv = __ldg(a.D + vc);
            tv = __ldg(a.T + vc);
        }
        bool pending = c < a.p.k && tv > 0 && dv != SR::zero();
        if (!__any_sync(0xffffffffu, pending)) continue;
        for (int base = t.sb; base < t.se; base += 32) {
            const int e = base + lane;
            int x = 0;
            float w = 0.0f;
            if (e < t.se) {
                x = __ldg(a.p.idx + e);
                w = __ldg(a.wt + e);
            }
            const int n = min(32, t.se - base);
            scanned += (unsigned long long)n;
            for (int j = 0; j < n; ++j) {
                const int u = __shfl_sync(0xffffffffu, x, j);
                const float wj = __shfl_sync(0xffffffffu, w, j);
                if (pending) {
                    const long long at = (long long)u * a.p.k + c;
                    const float du = __ldg(a.D + at);
                    if (__float_as_uint(SR::times(wj, du)) == __float_as_uint(dv) &&
                        (tree_better<SR>(du, dv) || (__float_as_uint(du) == __float_as_uint(dv) && __ldg(a.T + at) < tv))) {
                        if (a.seg_pass) asm volatile("red.global.min.u32 [%0], %1;" ::"l"(a.parent + vc), "r"(u) : "memory");
                        else a.parent[vc] = u;
                        pending = false;
                    }
                }
                if (!__any_sync(0xffffffffu, pending)) break;
            }
            if (!__any_sync(0xffffffffu, pending)) break;
        }
    }
    if (a.p.scanned && lane == 0 && scanned) atomicAdd(a.p.scanned, scanned);
}

// ------------------------------------------------------------------------------------------------
// predecessors of the tropical semirings: the product of arrow_spmm_sr carried over (value, label) pairs.  A candidate
// of row r is an entry p with a valid column c != self(r); its value is fl(A[r,p] + X[c]) and its label is c.  Pairs are
// ⊕-reduced lexicographically: the better value wins (smaller for (min, +), larger for (max, +)), equal values (by value,
// -0 == +0) go to the smaller label.  Labels compare as unsigned, so (⊕ identity, -1) is the identity of this ⊕ and a
// skipped slot is a no-op; a NaN term never wins.  The reduction is therefore exact, associative and commutative: the
// result does not depend on the kernel, the grid or the order of the terms.
// ------------------------------------------------------------------------------------------------
struct WitArgs {
    TileArgs t;                          // t.a: the product's operands; a.C = the value tile (nullptr: none), a.add_src =
                                         // the addend's values
    const int *__restrict__ self;        // row -> the label its own entries carry (-1: none); nullptr: the row index
    int *__restrict__ lab_out;           // labels (pair out) or parents (dist != nullptr)
    const int *__restrict__ add_lab;     // the addend's labels (same rows as a.add_src)
    const float *__restrict__ dist;      // parent epilogue: row r of dist is D[r]; nullptr: pair out
};

template <class SR>
__device__ __forceinline__ bool wit_better(float t, float acc) {
    if constexpr (std::is_same<SR, SrMinPlus>::value) return t < acc;
    else return t > acc;
}
// (av, al) = (av, al) ⊕ (t, l)
template <class SR>
__device__ __forceinline__ void wit_plus(float &av, int &al, float t, int l) {
    const bool take = wit_better<SR>(t, av) || (t == av && (unsigned)l < (unsigned)al);
    av = take ? t : av;
    al = take ? l : al;
}
template <class SR>
__device__ __forceinline__ void wit4_mac(float4 &av, int4 &al, float a, const float4 &x, int l) {
    wit_plus<SR>(av.x, al.x, SR::times(a, x.x), l);
    wit_plus<SR>(av.y, al.y, SR::times(a, x.y), l);
    wit_plus<SR>(av.z, al.z, SR::times(a, x.z), l);
    wit_plus<SR>(av.w, al.w, SR::times(a, x.w), l);
}
// the parent of one element: the witness label where D is not the ⊕ identity and the witness value equals it
template <class SR>
__device__ __forceinline__ int wit_parent(float d, float v, int l) {
    return (d != SR::zero() && v == d) ? l : -1;
}
__device__ __forceinline__ int4 i4_none() { return make_int4(-1, -1, -1, -1); }

// The k_spmm_tiles_sr pipeline with a label per element.  Epilogues (runtime): the addend pair ⊕-ed in where
// add_map[r] >= 0; out: the pair (values to a.C when given, labels to lab_out) or, with dist, the parents.
template <int G, int VPL, class SR, int TR, int TN>
__global__ void __launch_bounds__(TILE_THREADS, 4) k_spmm_tiles_wit(WitArgs w) {
    constexpr int TILE_PTR_WORDS = TileCfg<TR, TN>::PTR_WORDS;
    constexpr int TILE_NNZ_WORDS = TileCfg<TR, TN>::NNZ_WORDS;
    constexpr int TILE_STAGE_WORDS = TileCfg<TR, TN>::STAGE_WORDS;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    int *stage_base = reinterpret_cast<int *>(smem_raw);
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem_raw + (size_t)2 * TILE_STAGE_WORDS * 4);
    const TileArgs &t = w.t;
    const SpmmArgs &a = t.a;
    constexpr int RPW = 32 / G;
    constexpr int UNROLL = (VPL >= 2) ? 2 : 4;                    // a label per element doubles the accumulator
    constexpr int TAIL = 2;                                       // predicated tail batches
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const bool EXACT = (t.a.k4 == G * VPL);                       // every lane owns valid columns
    const int gl = lane % G;
    const int gi = lane / G;
    const int k4 = a.k4;
    const float4 *__restrict__ Xl = reinterpret_cast<const float4 *>(a.X) + gl;
    const uint64_t pol_keep = (t.l2_hints & 1) ? l2_policy_evict_last() : l2_policy_evict_normal();
    const uint64_t pol_stream = (t.l2_hints & 2) ? l2_policy_evict_first() : l2_policy_evict_normal();

    if (threadIdx.x == 0) {
        mbar_init(&bars[0], 1);
        mbar_init(&bars[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    auto issue_csr = [&](int tile, int st) {
        const int4 d = __ldg(t.tiles + tile);
        const int rb4 = d.x & ~3;
        const int a0 = d.z & ~3;
        const uint32_t ptr_bytes = (uint32_t)(((d.y - rb4 + 1) + 3) & ~3) * 4u;
        const uint32_t nnz_bytes = (uint32_t)(((d.w - a0) + 3) & ~3) * 4u;
        int *sp = stage_base + (size_t)st * TILE_STAGE_WORDS;
        mbar_expect_tx(&bars[st], ptr_bytes + 2u * nnz_bytes);
        bulk_g2s_hint(sp, a.indptr + rb4, ptr_bytes, &bars[st], pol_stream);
        if (nnz_bytes) {
            bulk_g2s_hint(sp + TILE_PTR_WORDS, a.indices + a0, nnz_bytes, &bars[st], pol_stream);
            bulk_g2s_hint(sp + TILE_PTR_WORDS + TILE_NNZ_WORDS, a.vals + a0, nnz_bytes, &bars[st], pol_stream);
        }
    };

    __shared__ int s_next[TILE_STAGES];
    int tile = blockIdx.x;
    if (tile < t.n_tiles && threadIdx.x == 0) issue_csr(tile, 0);
    for (unsigned int n = 0; tile < t.n_tiles; ++n) {
        const int st = (int)(n & 1u);
        if (threadIdx.x == 0) {
            const int next = atomicAdd(t.ticket, 1) + (int)gridDim.x;
            s_next[st] = next;
            if (next < t.n_tiles) issue_csr(next, st ^ 1);
        }
        const int4 d = __ldg(t.tiles + tile);
        mbar_wait(&bars[st], (n >> 1) & 1u);
        const int *sp = stage_base + (size_t)st * TILE_STAGE_WORDS;
        const int *s_ptr = sp + (d.x - (d.x & ~3));
        const int a0 = d.z & ~3;
        const int *s_idx = sp + TILE_PTR_WORDS - a0;                    // index with global nnz offsets
        const float *s_val = reinterpret_cast<const float *>(sp + TILE_PTR_WORDS + TILE_NNZ_WORDS) - a0;
        const int n_rows_tile = d.y - d.x;

        for (int lr = warp * RPW + gi; lr < n_rows_tile; lr += (TILE_THREADS / 32) * RPW) {
            const int s = s_ptr[lr];
            const int e = s_ptr[lr + 1];
            if (e - s > a.long_threshold) continue;
            const long long row = (long long)d.x + lr;
            const int own = (w.self != nullptr) ? __ldg(w.self + row) : (int)row;
            float4 av[VPL];
            int4 al[VPL];
#pragma unroll
            for (int i = 0; i < VPL; ++i) { av[i] = sr4_zero<SR>(); al[i] = i4_none(); }
            if (a.add_map != nullptr) {
                const int am = __ldg(a.add_map + row);
                if (am >= 0) {
                    const float4 *ar = reinterpret_cast<const float4 *>(a.add_src) + (long long)am * k4 + gl;
                    const int4 *lr4 = reinterpret_cast<const int4 *>(w.add_lab) + (long long)am * k4 + gl;
#pragma unroll
                    for (int i = 0; i < VPL; ++i)
                        if (gl + i * G < k4) { av[i] = ld_f4_hint(ar + i * G, pol_stream); al[i] = __ldg(lr4 + i * G); }
                }
            }
            int p = s;
            if (EXACT && !t.skip) {
                // unpredicated batches; an entry in the row's own column gets the ⊕ identity and label -1 (a no-op)
                auto batch = [&](auto n_tag) {
                    constexpr int N = decltype(n_tag)::value;
                    float4 x[N][VPL];
#pragma unroll
                    for (int u = 0; u < N; ++u) {
                        const float4 *xr = Xl + (long long)s_idx[p + u] * k4;
#pragma unroll
                        for (int i = 0; i < VPL; ++i) x[u][i] = ldg_f4_hint(xr + i * G, pol_keep);
                    }
#pragma unroll
                    for (int u = 0; u < N; ++u) {
                        const int c = s_idx[p + u];
                        const bool cand = (c != own);
                        const float v = cand ? s_val[p + u] : SR::zero();
#pragma unroll
                        for (int i = 0; i < VPL; ++i) wit4_mac<SR>(av[i], al[i], v, x[u][i], cand ? c : -1);
                    }
                    p += N;
                };
                while (p + UNROLL <= e) batch(std::integral_constant<int, UNROLL>{});
                if constexpr (UNROLL >= 4) { if (e - p >= 2) batch(std::integral_constant<int, 2>{}); }
                if (e - p >= 1) batch(std::integral_constant<int, 1>{});
            }
            // tail (and the general case): predicated batches.  A skipped entry (column -1), an entry in the row's own
            // column or a slot past the row's end is the identity pair (⊕ identity, -1) on zeros: a no-op.
            for (; p < e; p += TAIL) {
                float4 x[TAIL][VPL];
#pragma unroll
                for (int u = 0; u < TAIL; ++u) {
                    const int c = (p + u < e) ? s_idx[p + u] : -1;
                    const float4 *xr = Xl + (long long)c * k4;              // c = -1: address arithmetic only
#pragma unroll
                    for (int i = 0; i < VPL; ++i)
                        x[u][i] = (c >= 0 && gl + i * G < k4) ? ldg_f4_hint(xr + i * G, pol_keep) : f4_zero();
                }
#pragma unroll
                for (int u = 0; u < TAIL; ++u) {
                    const int c = (p + u < e) ? s_idx[p + u] : -1;
                    const bool cand = (c >= 0 && c != own);
                    const float v = cand ? s_val[p + u] : SR::zero();
#pragma unroll
                    for (int i = 0; i < VPL; ++i) wit4_mac<SR>(av[i], al[i], v, x[u][i], cand ? c : -1);
                }
            }
#pragma unroll
            for (int i = 0; i < VPL; ++i) {
                if (gl + i * G < k4) {
                    const long long off = row * k4 + gl + i * G;
                    int4 o = al[i];
                    if (w.dist != nullptr) {
                        const float4 dd = __ldg(reinterpret_cast<const float4 *>(w.dist) + off);
                        o = make_int4(wit_parent<SR>(dd.x, av[i].x, o.x), wit_parent<SR>(dd.y, av[i].y, o.y),
                                      wit_parent<SR>(dd.z, av[i].z, o.z), wit_parent<SR>(dd.w, av[i].w, o.w));
                    }
                    if (a.C != nullptr) st_f4_hint(reinterpret_cast<float4 *>(a.C) + off, av[i], pol_stream);
                    reinterpret_cast<int4 *>(w.lab_out)[off] = o;
                }
            }
        }
        __syncthreads();            // stage `st` may be refilled by the next iteration's copy
        tile = s_next[st];
    }
}

// k not a multiple of 4 or k > 256: warp per row, lanes over columns, scalar accesses
template <class SR>
__global__ void __launch_bounds__(256) k_spmm_generic_wit(WitArgs w) {
    const SpmmArgs &a = w.t.a;
    const int lane = threadIdx.x & 31;
    const long long warps_total = (long long)gridDim.x * (blockDim.x >> 5);
    const long long warp_id = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    for (long long row = warp_id; row < a.n_rows; row += warps_total) {
        const int s = __ldg(a.indptr + row);
        const int e = __ldg(a.indptr + row + 1);
        if (e - s > a.long_threshold) continue;
        const int own = (w.self != nullptr) ? __ldg(w.self + row) : (int)row;
        const int am = (a.add_map != nullptr) ? __ldg(a.add_map + row) : -1;
        for (int c0 = 0; c0 < a.k; c0 += 128) {
            float av[4] = {SR::zero(), SR::zero(), SR::zero(), SR::zero()};
            int al[4] = {-1, -1, -1, -1};
            for (int p = s; p < e; ++p) {
                const int c = __ldg(a.indices + p);
                const float v = __ldg(a.vals + p);
                if (c < 0 || c == own) continue;
                const float *xr = a.X + (long long)c * a.k;
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int col = c0 + lane + 32 * i;
                    if (col < a.k) wit_plus<SR>(av[i], al[i], SR::times(v, __ldg(xr + col)), c);
                }
            }
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int col = c0 + lane + 32 * i;
                if (col < a.k) {
                    const long long off = row * a.k + col;
                    if (am >= 0) wit_plus<SR>(av[i], al[i], a.add_src[(long long)am * a.k + col], w.add_lab[(long long)am * a.k + col]);
                    if (a.C != nullptr) a.C[off] = av[i];
                    w.lab_out[off] = (w.dist != nullptr) ? wit_parent<SR>(w.dist[off], av[i], al[i]) : al[i];
                }
            }
        }
    }
}

// long rows: one CTA per segment ⊕-reduces its entries into a scratch slot (values, then labels), then one CTA per row
// ⊕-reduces the slots and the addend and applies the epilogue (k_spmm_long_partial_sr / k_spmm_long_reduce_sr)
template <class SR>
__global__ void __launch_bounds__(256) k_spmm_long_partial_wit(LongArgs a, const int *__restrict__ self,
                                                               int *__restrict__ lab_scratch) {
    __shared__ float red_wv[LONG_WARPS][LONG_CHUNK];
    __shared__ int red_wl[LONG_WARPS][LONG_CHUNK];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const LongTask t = a.tasks[blockIdx.x];
    const int own = (self != nullptr) ? self[t.row] : t.row;
    for (int c0 = 0; c0 < a.k; c0 += LONG_CHUNK) {
        float av[4] = {SR::zero(), SR::zero(), SR::zero(), SR::zero()};
        int al[4] = {-1, -1, -1, -1};
        for (int p = t.begin + warp; p < t.end; p += LONG_WARPS) {
            const int c = __ldg(a.indices + p);
            const float v = __ldg(a.vals + p);
            if (c < 0 || c == own) continue;
            const float *xr = a.X + (long long)c * a.k;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int col = c0 + lane + 32 * i;
                if (col < a.k) wit_plus<SR>(av[i], al[i], SR::times(v, __ldg(xr + col)), c);
            }
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) { red_wv[warp][lane + 32 * i] = av[i]; red_wl[warp][lane + 32 * i] = al[i]; }
        __syncthreads();
        const int col = c0 + threadIdx.x;
        if (threadIdx.x < LONG_CHUNK && col < a.k) {
            float v = SR::zero();
            int l = -1;
            for (int w = 0; w < LONG_WARPS; ++w) wit_plus<SR>(v, l, red_wv[w][threadIdx.x], red_wl[w][threadIdx.x]);
            a.scratch[(long long)t.slot * a.k + col] = v;
            lab_scratch[(long long)t.slot * a.k + col] = l;
        }
        __syncthreads();
    }
}

template <class SR>
__global__ void __launch_bounds__(128) k_spmm_long_reduce_wit(const int *__restrict__ long_rows,
                                                              const int *__restrict__ long_first,
                                                              const float *__restrict__ scratch,
                                                              const int *__restrict__ lab_scratch, WitArgs w) {
    const SpmmArgs &a = w.t.a;
    const int r = long_rows[blockIdx.x];
    const int am = (a.add_map != nullptr) ? a.add_map[r] : -1;
    const int s0 = long_first[blockIdx.x], s1 = long_first[blockIdx.x + 1];
    const int k = a.k;
    for (int col = threadIdx.x; col < k; col += blockDim.x) {
        float v = SR::zero();
        int l = -1;
        for (int s = s0; s < s1; ++s) wit_plus<SR>(v, l, scratch[(long long)s * k + col], lab_scratch[(long long)s * k + col]);
        if (am >= 0) wit_plus<SR>(v, l, a.add_src[(long long)am * k + col], w.add_lab[(long long)am * k + col]);
        const long long off = (long long)r * k + col;
        if (a.C != nullptr) a.C[off] = v;
        w.lab_out[off] = (w.dist != nullptr) ? wit_parent<SR>(w.dist[off], v, l) : l;
    }
}

template <int G, int VPL, class SR, int TR, int TN>
int launch_tiles_wit_one(arrow_ctx *ctx, const WitArgs &w) {
    return launch_persistent<k_spmm_tiles_wit<G, VPL, SR, TR, TN>, TileCfg<TR, TN>::SMEM_BYTES>(ctx, w, w.t.n_tiles, w.t.ticket);
}

// (lanes per row, float4 per lane): one float4 per lane up to 32 lanes (k <= 128), then two (k <= 256); big tiles as
// launch_tiles picks them (k <= 32)
int launch_tiles_wit_shape(arrow_ctx *ctx, WitArgs &w, const Csr *A, bool min_plus) {
    TileArgs &t = w.t;
    const int k4 = t.a.k4;
    const int vpl = (k4 > 32) ? 2 : 1;
    const int lanes = (k4 + vpl - 1) / vpl;           // <= 32: k4 <= 64
    int g = 1;
    while (g < lanes) g <<= 1;
    const int list = tile_list_for(ctx, t.a.k, 4, k4 <= 8);                  // k <= 32: WIB shapes exist
    const bool big = list == TILE_LIST_BIG;
    t.tiles = A->tiles[list];
    t.n_tiles = A->n_tiles[list];
#define TWI(GG, VV, TR, TN)                                                                              \
    return min_plus ? launch_tiles_wit_one<GG, VV, SrMinPlus, TR, TN>(ctx, w) : launch_tiles_wit_one<GG, VV, SrMaxPlus, TR, TN>(ctx, w)
#define WIB(GG, VV) if (big && g == GG && vpl == VV) TWI(GG, VV, TILE_ROWS_BIG, TILE_NNZ_BIG)
#define WIS(GG, VV) if (g == GG && vpl == VV) TWI(GG, VV, TILE_ROWS, TILE_NNZ)
    WIB(1, 1); WIB(2, 1); WIB(4, 1); WIB(8, 1);
    WIS(1, 1); WIS(2, 1); WIS(4, 1); WIS(8, 1); WIS(16, 1); WIS(32, 1); WIS(32, 2);
#undef WIS
#undef WIB
#undef TWI
    return fail(ctx, ARROW_ERR_UNSUPPORTED, "no witness tile kernel for k4=%d vpl=%d", k4, vpl);
}

// the launches of arrow_spmm_sr_witness; `w` carries the validated fp32 operands
template <class SR>
int spmm_wit(arrow_ctx *ctx, const Csr *A, WitArgs &w, bool min_plus) {
    const SpmmArgs &a = w.t.a;
    const int k = a.k;
    const int lane = ctx->cur_lane;
    cudaStream_t stream = cur_stream(ctx);
    if (k % 4 != 0 || k > 256) {
        const long long ctas = (A->n_rows + 7) / 8;
        auto fn = k_spmm_generic_wit<SR>;
        const int grid = grid_for(ctx, (const void *)fn, 256, 0, ctas);
        fn<<<grid, 256, 0, stream>>>(w);
        ctx->launches++;
    } else if (A->n_tiles[TILE_LIST_SMALL] > 0) {
        w.t.skip = (A->may_skip || ctx->force_skip_path) ? 1 : 0;
        w.t.ticket = ctx->tile_ticket + 2 * lane;
        w.t.l2_hints = ctx->l2_hints_plain;
        w.t.prefetch = 0;
        const int rc = launch_tiles_wit_shape(ctx, w, A, min_plus);
        if (rc != ARROW_OK) return rc;
    }
    CUDA_TRY(ctx, cudaGetLastError());

    if (A->n_long_tasks > 0) {
        const size_t slots = (size_t)A->n_long_tasks * k;
        const int rc = grow_long_scratch(ctx, slots * 8);  // values, then labels
        if (rc != ARROW_OK) return rc;
        LongArgs la;
        la.tasks = A->long_tasks;
        la.indices = a.indices;
        la.vals = a.vals;
        la.X = a.X;
        la.scratch = ctx->long_scratch[lane];
        la.k = k;
        la.X2 = nullptr;
        la.x_split = 0;
        int *lab_scratch = reinterpret_cast<int *>(ctx->long_scratch[lane] + slots);
        k_spmm_long_partial_wit<SR><<<A->n_long_tasks, 256, 0, stream>>>(la, w.self, lab_scratch);
        ctx->launches++;
        k_spmm_long_reduce_wit<SR><<<A->n_long_rows, 128, 0, stream>>>(A->long_rows, A->long_first, la.scratch,
                                                                        lab_scratch, w);
        ctx->launches++;
        CUDA_TRY(ctx, cudaGetLastError());
    }
    return ARROW_OK;
}

}  // namespace

// ------------------------------------------------------------------------------------------------
// personalized PageRank (one GPU, plus-times, float32 or float64).  The walk steps with the engine's own SpMM on a
// values-only copy of every block whose entries are divided by their source's out-weight; the passes here build those
// weights and copies, normalise the restart columns and fold one step into the next iterate.  Every column reduction
// (sigma, dangling mass, residual) runs in float64 over fixed PR_CHUNK-row chunks from row 0: sequential in ascending
// rows inside a chunk, the chunk partials then added in ascending chunk order by one thread per column.  No
// floating-point atomics, so the results depend neither on the grid nor on the schedule.
// ------------------------------------------------------------------------------------------------
namespace {
constexpr int PR_CHUNK = 512;

inline long long pr_chunks(long long n) { return (n + PR_CHUNK - 1) / PR_CHUNK; }

__device__ __forceinline__ double pr_mul(float a, float b) { return (double)__fmul_rn(a, b); }
__device__ __forceinline__ double pr_mul(double a, double b) { return __dmul_rn(a, b); }

// one key per entry of a part, at its (part, entry) slot: the level-0 source u = map(c) of the edge map(c) -> map(r), or
// n_vertices when the entry is not an edge of M (c < 0 or an end at -1); the value goes beside it as float64.  Counts the
// edges whose value is negative, NaN or +-inf (-0 is allowed) with one integer atomic per warp.
template <class T>
__global__ void __launch_bounds__(256) k_pr_out_keys(AdjPart p, const T *__restrict__ vals, int n_vertices,
                                                     int *__restrict__ keys, double *__restrict__ w_out,
                                                     unsigned long long *__restrict__ bad) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    unsigned nbad = 0;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < p.nnz; e += stride) {
        const int c = __ldg(p.indices + e);
        int u = n_vertices;
        if (c >= 0) {
            const int r = last_le(p.indptr, 0, p.n_rows - 1, e);
            const int src = p.map ? __ldg(p.map + c) : c;
            const int dst = p.map ? __ldg(p.map + r) : r;
            if (src >= 0 && dst >= 0) u = src;
        }
        const double a = (double)vals[e];
        keys[e] = u;
        w_out[e] = a;
        if (u < n_vertices && !(a >= 0.0 && a <= 1.7976931348623157e308)) ++nbad;
    }
    for (int o = 16; o > 0; o >>= 1) nbad += __shfl_xor_sync(0xffffffffu, nbad, o);
    if ((threadIdx.x & 31) == 0 && nbad) atomicAdd(bad, (unsigned long long)nbad);
}

__device__ __forceinline__ long long pr_lower_bound(const int *__restrict__ keys, long long m, int want) {
    long long lo = 0, hi = m;
    while (lo < hi) {
        const long long mid = (lo + hi) >> 1;
        if (keys[mid] < want) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

// w[u] = the sequential float64 sum (from +0) of the values of u's entries in (part, entry) order -- the stable sort kept
// it -- and inv[u] = fl_T(1 / w[u]), 0 where w[u] == 0 (dangling).  counts[0] gets the dangling vertices, counts[1] the
// others whose inverse is not finite or 0.
template <class T>
__global__ void __launch_bounds__(256) k_pr_out_sums(const int *__restrict__ keys, const double *__restrict__ vals, long long m,
                                                     long long n, double *__restrict__ w, T *__restrict__ inv,
                                                     unsigned long long *__restrict__ counts) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    unsigned dangling = 0, bad = 0;
    for (long long u = (long long)blockIdx.x * blockDim.x + threadIdx.x; u < n; u += stride) {
        const long long lo = pr_lower_bound(keys, m, (int)u), hi = pr_lower_bound(keys, m, (int)u + 1);
        double acc = 0.0;
        for (long long e = lo; e < hi; ++e) acc = __dadd_rn(acc, vals[e]);
        T q = (T)0;
        if (acc == 0.0) {
            ++dangling;
        } else {
            q = (T)__ddiv_rn(1.0, acc);
            if (!isfinite((double)q) || q == (T)0) ++bad;
        }
        w[u] = acc;
        inv[u] = q;
    }
    for (int o = 16; o > 0; o >>= 1) {
        dangling += __shfl_xor_sync(0xffffffffu, dangling, o);
        bad += __shfl_xor_sync(0xffffffffu, bad, o);
    }
    if ((threadIdx.x & 31) == 0) {
        if (dangling) atomicAdd(counts, (unsigned long long)dangling);
        if (bad) atomicAdd(counts + 1, (unsigned long long)bad);
    }
}

// out[e] = fl_T(a_e * scale[map(c_e)]) (map nullptr: the identity); 0 for an entry whose column is -1 or maps to -1
template <class T>
__global__ void __launch_bounds__(256) k_pr_scale(const int *__restrict__ indices, const T *__restrict__ vals,
                                                  const int *__restrict__ map, const T *__restrict__ scale, T *__restrict__ out,
                                                  long long nnz) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < nnz; e += stride) {
        const int c = __ldg(indices + e);
        const int u = c < 0 ? -1 : (map ? __ldg(map + c) : c);
        out[e] = u < 0 ? (T)0 : (T)pr_mul(vals[e], __ldg(scale + u));
    }
}

// chunk partials of the restart, one thread per (chunk, column), chunk-major so that a warp reads adjacent columns of one
// row: part[s][b] = the sum of X[v, s] over the chunk's rows, part[k + s][b] = 1 where a value is negative, NaN or +-inf
template <class T>
__global__ void __launch_bounds__(256) k_pr_restart_partials(const T *__restrict__ X, long long n, int k, long long nch,
                                                             double *__restrict__ part) {
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < nch * k; t += (long long)gridDim.x * blockDim.x) {
        const long long b = t / k;
        const int s = (int)(t - b * k);
        const long long v1 = min(n, (b + 1) * PR_CHUNK);
        double acc = 0.0;
        bool bad = false;
#pragma unroll 8
        for (long long v = b * PR_CHUNK; v < v1; ++v) {
            const double x = (double)X[v * k + s];
            acc = __dadd_rn(acc, x);
            bad |= !(x >= 0.0 && x <= 1.7976931348623157e308);
        }
        part[(long long)s * nch + b] = acc;
        part[(long long)(k + s) * nch + b] = bad ? 1.0 : 0.0;
    }
}

// S[v, s] = fl_T(X[v, s] / sigma_s) with sigma from the state tile's row 2; part[s][b] = the chunk's dangling mass of S
template <class T>
__global__ void __launch_bounds__(256) k_pr_restart_write(const T *__restrict__ X, const T *__restrict__ inv,
                                                          const double *__restrict__ state, T *__restrict__ S, long long n,
                                                          int k, long long nch, double *__restrict__ part) {
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < nch * k; t += (long long)gridDim.x * blockDim.x) {
        const long long b = t / k;
        const int s = (int)(t - b * k);
        const double sigma = state[2 * k + s];
        const long long v1 = min(n, (b + 1) * PR_CHUNK);
        double m = 0.0;
#pragma unroll 8
        for (long long v = b * PR_CHUNK; v < v1; ++v) {
            const T q = (T)__ddiv_rn((double)X[v * k + s], sigma);
            S[v * k + s] = q;
            if (__ldg(inv + v) == (T)0) m = __dadd_rn(m, (double)q);
        }
        part[(long long)s * nch + b] = m;
    }
}

// one step's update, one thread per (chunk, column): with c = fl(beta + fl(alpha * m_t[s])) (m_t in the state tile's row 0)
// p_{t+1} = fl_T(fl(fl(alpha * Y) + fl(c * S))) over Y in place; part[s][b] = the chunk's dangling mass of p_{t+1},
// part[k + s][b] = its sum of |fl(p_{t+1} - p_t)|.  Separately rounded float64 operations, no contraction.
template <class T>
__global__ void __launch_bounds__(256) k_pr_update(T *__restrict__ Y, const T *__restrict__ P, const T *__restrict__ S,
                                                   const T *__restrict__ inv, const double *__restrict__ state, double alpha,
                                                   double beta, long long n, int k, long long nch, double *__restrict__ part) {
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < nch * k; t += (long long)gridDim.x * blockDim.x) {
        const long long b = t / k;
        const int s = (int)(t - b * k);
        const double c = __dadd_rn(beta, __dmul_rn(alpha, state[s]));
        const long long v1 = min(n, (b + 1) * PR_CHUNK);
        double m = 0.0, r = 0.0;
#pragma unroll 8
        for (long long v = b * PR_CHUNK; v < v1; ++v) {
            const long long i = v * k + s;
            const T q = (T)__dadd_rn(__dmul_rn(alpha, (double)Y[i]), __dmul_rn(c, (double)__ldg(S + i)));
            const double old = (double)__ldg(P + i);
            Y[i] = q;
            r = __dadd_rn(r, fabs(__dsub_rn((double)q, old)));
            if (__ldg(inv + v) == (T)0) m = __dadd_rn(m, (double)q);
        }
        part[(long long)s * nch + b] = m;
        part[(long long)(k + s) * nch + b] = r;
    }
}

// out[q] = part[q][0] + part[q][1] + ... + part[q][nch - 1], left to right from +0: one CTA per row q, which stages the
// row through shared memory and sums it on one thread
__global__ void __launch_bounds__(256) k_pr_chunk_sums(const double *__restrict__ part, long long nch, double *__restrict__ out) {
    constexpr int STAGE = 2048;
    __shared__ double buf[STAGE];
    const double *row = part + (long long)blockIdx.x * nch;
    double acc = 0.0;
    for (long long b0 = 0; b0 < nch; b0 += STAGE) {
        const int len = (int)min((long long)STAGE, nch - b0);
        for (int i = threadIdx.x; i < len; i += blockDim.x) buf[i] = row[b0 + i];
        __syncthreads();
        if (threadIdx.x == 0)
            for (int i = 0; i < len; ++i) acc = __dadd_rn(acc, buf[i]);
        __syncthreads();
    }
    if (threadIdx.x == 0) out[blockIdx.x] = acc;
}

// the tiles of the restart / update passes: x (or y), p and S of one element type T [n x k], inv T [n x 1], scratch float64
// [pr_chunks(n) x 2k], state float64 [4 x k]; the restart has no p (x_buf is then X0)
int pr_tiles(arrow_ctx *ctx, const char *fn, bool restart, int x_buf, int p_buf, int s_buf, int inv_buf, int scratch_buf,
             int state_buf, DenseBuf *t[6]) {
    const int h[6] = {x_buf, p_buf, s_buf, inv_buf, scratch_buf, state_buf};
    const char *name[6] = {restart ? "x" : "y", "p", "s", "inv", "scratch", "state"};
    for (int i = 0; i < 6; ++i) {
        t[i] = nullptr;
        if (i == 1 && restart) continue;
        t[i] = get_dense(ctx, h[i]);
        if (!t[i]) return fail(ctx, ARROW_ERR_HANDLE, "%s: bad dense handle %s=%d", fn, name[i], h[i]);
    }
    const int T = t[0]->dtype;
    if (T != ARROW_F32 && T != ARROW_F64) return fail(ctx, ARROW_ERR_ARG, "%s: %s is a %s tile, expected float32 or float64", fn, name[0], dtype_name(T));
    const long long n = t[0]->rows;
    const int k = t[0]->k;
    const long long want_rows[6] = {n, n, n, n, pr_chunks(n), 4};
    const int want_k[6] = {k, k, k, 1, 2 * k, k};
    for (int i = 0; i < 6; ++i) {
        if (!t[i]) continue;
        const int want = i >= 4 ? ARROW_F64 : T;
        if (t[i]->dtype != want)
            return fail(ctx, ARROW_ERR_ARG, "%s: %s is a %s tile, expected %s", fn, name[i], dtype_name(t[i]->dtype), dtype_name(want));
        if (t[i]->rows != want_rows[i] || t[i]->k != want_k[i])
            return fail(ctx, ARROW_ERR_ARG, "%s: %s is %lld x %d, expected %lld x %d", fn, name[i], (long long)t[i]->rows, t[i]->k,
                        want_rows[i], want_k[i]);
        for (int j = 0; j < i; ++j)
            if (t[j] && (h[j] == h[i] || t[j]->p == t[i]->p)) return fail(ctx, ARROW_ERR_ARG, "%s: %s aliases %s", fn, name[i], name[j]);
    }
    if (ctx->capturing) return fail(ctx, ARROW_ERR_UNSUPPORTED, "%s synchronises: not during graph capture", fn);
    return ARROW_OK;
}

// grid of the chunk passes (grid-stride over (chunk, column) items): ARROW_OPT_SPMM_SM_LIMIT and ARROW_OPT_SPMM_CTAS_PER_SM cap
// it as they cap a SpMM grid; the results do not depend on it
int pr_grid(const arrow_ctx *ctx, long long items) {
    const long long sms = ctx->spmm_sm_limit > 0 ? std::min(ctx->spmm_sm_limit, ctx->sm_count) : ctx->sm_count;
    const long long per_sm = ctx->spmm_ctas_per_sm > 0 ? ctx->spmm_ctas_per_sm : 8;
    return (int)std::max<long long>(1, std::min<long long>((items + 255) / 256, sms * per_sm));
}

// ------------------------------------------------------------------------------------------------
// connected components (one GPU): a lock-free union-find over a parent array (the label tile), in the manner of ECL-CC
// (Jaiganesh and Burtscher, HPDC 2018).  Invariant: parent[x] <= x for every x, with equality exactly for the roots.  It
// holds after the init; a hook CASes a root hi, expected still parent[hi] == hi, to a smaller root lo; path halving stores
// into a vertex that is not a root (so no CAS can target it again) a grandparent, which is below its parent.  A vertex
// never becomes a root again and every store keeps it in its own tree, so trees only merge.  Hence each root is the
// smallest vertex of its tree, and once every entry has joined its two ends, the smallest of its component.
// Termination: a root walk moves to a strictly smaller vertex each round; a union's failed CAS means the larger root gained
// a parent below it, so max(a, b) of the two roots strictly decreases each round.  Every read of parent inside those
// loops is an ld.relaxed.gpu: never served from L1 or kept in a register across rounds.
// ------------------------------------------------------------------------------------------------
constexpr int CC_CHUNK = 256;          // entries of one warp chunk of the hook pass

__device__ __forceinline__ int cc_load(const int *p) {
    int v;
    asm volatile("ld.relaxed.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

__device__ __forceinline__ void cc_store(int *p, int v) {
    asm volatile("st.relaxed.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// the root of v's tree, halving the path: each round either returns or moves v to its grandparent g < parent < v
__device__ __forceinline__ int cc_root(int *parent, int v) {
    for (;;) {
        const int p = cc_load(parent + v);
        if (p == v) return v;
        const int g = cc_load(parent + p);
        if (g == p) return p;
        cc_store(parent + v, g);
        v = g;
    }
}

// joins the trees of u and v: hooks the larger root onto the smaller; on a failed CAS both roots are found again, and
// both lie below the old larger root (the CAS saw its new parent old < hi)
__device__ __forceinline__ void cc_union(int *parent, int u, int v) {
    int a = cc_root(parent, u), b = cc_root(parent, v);
    while (a != b) {
        const int hi = max(a, b), lo = min(a, b);
        const int old = atomicCAS(parent + hi, hi, lo);
        if (old == hi) return;
        a = cc_root(parent, old);
        b = cc_root(parent, lo);
    }
}

__global__ void __launch_bounds__(256) k_cc_init(int *__restrict__ parent, long long n) {
    for (long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x; v < n; v += (long long)gridDim.x * blockDim.x)
        parent[v] = (int)v;
}

// the hook pass over one part: warp-stride over CC_CHUNK-entry chunks, so a long row is spread over many warps.  Lanes 0
// and 1 find the rows of the chunk's first and last entries over the whole block; each entry then searches only the rows
// between them (none for a chunk inside one row).  Entry (r, c) joins map(c) and map(r); c < 0, an end at -1 and u == v
// join nothing.  The value is never read.
__global__ void __launch_bounds__(256) k_cc_hook(AdjPart p, int *parent) {
    const int lane = threadIdx.x & 31;
    const long long warps = ((long long)gridDim.x * blockDim.x) >> 5;
    const long long chunks = (p.nnz + CC_CHUNK - 1) / CC_CHUNK;
    for (long long ch = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; ch < chunks; ch += warps) {
        const long long e0 = ch * CC_CHUNK, e1 = min(p.nnz, e0 + CC_CHUNK);
        int r = 0;
        if (lane < 2) r = last_le(p.indptr, 0, p.n_rows - 1, lane == 0 ? e0 : e1 - 1);
        const int r_lo = __shfl_sync(0xffffffffu, r, 0), r_hi = __shfl_sync(0xffffffffu, r, 1);
        for (long long e = e0 + lane; e < e1; e += 32) {
            const int c = __ldg(p.indices + e);
            if (c < 0) continue;
            const int row = last_le(p.indptr, r_lo, r_hi, e);
            const int u = p.map ? __ldg(p.map + c) : c;
            const int v = p.map ? __ldg(p.map + row) : row;
            if (u >= 0 && v >= 0 && u != v) cc_union(parent, u, v);
        }
    }
}

// labels[v] = root(v) in place, after the hook pass (the roots no longer change).  The walk stores nothing: parent[v] is
// written by v's thread alone, so it ends at the root, and a concurrent walk through v reads its old parent or the root.
// Counts the roots (one integer atomic per warp) and, with sizes, adds each vertex to its label's count.
__global__ void __launch_bounds__(256) k_cc_label(int *parent, long long n, int *__restrict__ sizes,
                                                  unsigned long long *__restrict__ roots) {
    unsigned mine = 0;
    for (long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x; v < n; v += (long long)gridDim.x * blockDim.x) {
        int r = cc_load(parent + v), next;
        while ((next = cc_load(parent + r)) != r) r = next;      // next < r: strictly decreasing
        if (r == (int)v) ++mine;
        else cc_store(parent + v, r);
        if (sizes) atomicAdd(sizes + r, 1);
    }
    for (int o = 16; o > 0; o >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, o);
    if ((threadIdx.x & 31) == 0 && mine) atomicAdd(roots, (unsigned long long)mine);
}

// the (block, row map) pairs of arrow_adj_build and of the passes over the same operator: valid handles, every map covering
// its block's rows and columns and reaching no row past n_vertices, a block under the identity map within n_vertices
int operator_parts(arrow_ctx *ctx, int n_parts, const int *csrs, const int *maps, int64_t n_vertices,
                   std::vector<std::pair<const Csr *, const IdxMap *>> &out) {
    for (int i = 0; i < n_parts; ++i) {
        const Csr *c = get_csr(ctx, csrs[i]);
        if (!c) return fail(ctx, ARROW_ERR_HANDLE, "part %d: bad csr handle %d", i, csrs[i]);
        const IdxMap *m = nullptr;
        if (maps[i] != -1) {
            m = get_map(ctx, maps[i]);
            if (!m) return fail(ctx, ARROW_ERR_HANDLE, "part %d: bad map handle %d", i, maps[i]);
            if (m->n < std::max(c->n_rows, c->n_cols))
                return fail(ctx, ARROW_ERR_ARG, "part %d: the map has %lld entries, the block %lld rows and %lld columns", i,
                            (long long)m->n, (long long)c->n_rows, (long long)c->n_cols);
            if (m->limit > n_vertices)
                return fail(ctx, ARROW_ERR_ARG, "part %d: the map reaches row %lld, there are %lld vertices", i,
                            (long long)m->limit, (long long)n_vertices);
        } else if (c->n_rows > n_vertices || c->n_cols > n_vertices) {
            return fail(ctx, ARROW_ERR_ARG, "part %d: a %lld x %lld block with the identity map exceeds %lld vertices", i,
                        (long long)c->n_rows, (long long)c->n_cols, (long long)n_vertices);
        }
        out.emplace_back(c, m);
    }
    return ARROW_OK;
}
}  // namespace

// ================================================================================================
// C ABI
// ================================================================================================
extern "C" {

int arrow_b200_abi_version(void) { return ARROW_ABI_VERSION; }

const char *arrow_last_error(const arrow_ctx *ctx) { return ctx ? ctx->err.c_str() : g_create_error.c_str(); }

int arrow_ctx_create(int device, void *stream, arrow_ctx **out) {
    if (!out) return fail(nullptr, ARROW_ERR_ARG, "out is null");
    *out = nullptr;
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0)
        return fail(nullptr, ARROW_ERR_CUDA, "no CUDA device available (%s); libarrow_b200 has no CPU fallback",
                    cudaGetErrorString(e));
    if (device < 0 || device >= n) return fail(nullptr, ARROW_ERR_ARG, "device %d out of range [0,%d)", device, n);
    e = cudaSetDevice(device);
    if (e != cudaSuccess) return fail(nullptr, ARROW_ERR_CUDA, "cudaSetDevice: %s", cudaGetErrorString(e));
    arrow_ctx *ctx = new arrow_ctx();
    ctx->device = device;
    cudaDeviceProp prop;
    e = cudaGetDeviceProperties(&prop, device);
    if (e != cudaSuccess) {
        delete ctx;
        return fail(nullptr, ARROW_ERR_CUDA, "cudaGetDeviceProperties: %s", cudaGetErrorString(e));
    }
    ctx->sm_count = prop.multiProcessorCount;
    if (prop.l2CacheSize > 0) ctx->l2_bytes = prop.l2CacheSize;
    if (stream) {
        ctx->stream = (cudaStream_t)stream;
    } else {
        e = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking);
        if (e != cudaSuccess) {
            delete ctx;
            return fail(nullptr, ARROW_ERR_CUDA, "cudaStreamCreate: %s", cudaGetErrorString(e));
        }
        ctx->own_stream = true;
    }
    e = cudaMalloc(&ctx->dev_status, sizeof(int));
    if (e == cudaSuccess) e = cudaMemset(ctx->dev_status, 0, sizeof(int));
    if (e == cudaSuccess) e = cudaMalloc(&ctx->barrier_epoch, ARROW_N_LANES * sizeof(unsigned int));
    if (e == cudaSuccess) e = cudaMemset(ctx->barrier_epoch, 0, ARROW_N_LANES * sizeof(unsigned int));
    if (e == cudaSuccess) e = cudaMalloc(&ctx->tile_ticket, 2 * ARROW_N_LANES * sizeof(int));
    if (e == cudaSuccess) e = cudaMemset(ctx->tile_ticket, 0, 2 * ARROW_N_LANES * sizeof(int));
    if (e != cudaSuccess) {
        if (ctx->dev_status) cudaFree(ctx->dev_status);
        if (ctx->barrier_epoch) cudaFree(ctx->barrier_epoch);
        if (ctx->tile_ticket) cudaFree(ctx->tile_ticket);
        delete ctx;
        return fail(nullptr, ARROW_ERR_CUDA, "context state alloc: %s", cudaGetErrorString(e));
    }
    ctx->clock_khz = prop.clockRate > 0 ? prop.clockRate : 2000000;
    *out = ctx;
    return ARROW_OK;
}

void arrow_ctx_destroy(arrow_ctx *ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    for (auto &d : ctx->dense)
        if (d.live) {
            if (d.owned) cudaFree(d.p);
            else if (d.ipc) cudaIpcCloseMemHandle(d.ipc_base);
        }
    for (auto &c : ctx->csrs)
        if (c.live) csr_release(c);
    for (auto &m : ctx->maps)
        if (m.live) cudaFree(m.p);
    for (auto &a : ctx->adjs)
        if (a.live) adj_release(a);
    for (auto &t : ctx->timers) {
        if (t.a) cudaEventDestroy(t.a);
        if (t.b) cudaEventDestroy(t.b);
    }
    for (int l = 0; l < ARROW_N_LANES; ++l)
        if (ctx->long_scratch[l]) cudaFree(ctx->long_scratch[l]);
    for (auto &pt : ctx->ptrtabs)
        if (pt.live) cudaFree(pt.p);
    for (auto g : ctx->graphs)
        if (g) cudaGraphExecDestroy(g);
    if (ctx->flush_buf) cudaFree(ctx->flush_buf);
    if (ctx->dev_status) cudaFree(ctx->dev_status);
    if (ctx->barrier_epoch) cudaFree(ctx->barrier_epoch);
    if (ctx->tile_ticket) cudaFree(ctx->tile_ticket);
    for (int l = 1; l < ARROW_N_LANES; ++l)
        if (ctx->lanes[l]) { cudaStreamSynchronize(ctx->lanes[l]); cudaStreamDestroy(ctx->lanes[l]); }
    for (int l = 0; l < ARROW_N_LANES; ++l)
        if (ctx->lane_events[l]) cudaEventDestroy(ctx->lane_events[l]);
    for (int e = 0; e < ARROW_MAX_EVENTS; ++e)
        if (ctx->user_events[e]) cudaEventDestroy(ctx->user_events[e]);
    if (ctx->own_stream) cudaStreamDestroy(ctx->stream);
    delete ctx;
}

int arrow_sync(arrow_ctx *ctx) {
    CHECK_CTX(ctx);
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    int st = 0;
    CUDA_TRY(ctx, cudaMemcpy(&st, ctx->dev_status, sizeof(int), cudaMemcpyDeviceToHost));
    if (st != 0) {
        ctx->poisoned = true;
        return fail(ctx, ARROW_ERR_CUDA, "device-side failure flag %d: a peer barrier timed out after %lld ms; the context is "
                    "poisoned (results after the time-out are racy) -- destroy it", st, ctx->barrier_timeout_ms);
    }
    return ARROW_OK;
}

int arrow_device_info(arrow_ctx *ctx, int *sm_count, int64_t *free_bytes, int64_t *total_bytes) {
    CHECK_CTX(ctx);
    size_t f = 0, t = 0;
    CUDA_TRY(ctx, cudaMemGetInfo(&f, &t));
    if (sm_count) *sm_count = ctx->sm_count;
    if (free_bytes) *free_bytes = (int64_t)f;
    if (total_bytes) *total_bytes = (int64_t)t;
    return ARROW_OK;
}

int arrow_set_tuning(arrow_ctx *ctx, int long_row_threshold, int long_row_segment) {
    CHECK_CTX(ctx);
    if (long_row_threshold < 1 || long_row_segment < 32 || long_row_threshold > TILE_NNZ - 8)
        return fail(ctx, ARROW_ERR_ARG, "bad tuning values (threshold must be in [1, %d])", TILE_NNZ - 8);
    ctx->long_threshold = long_row_threshold;
    ctx->long_segment = long_row_segment;
    return ARROW_OK;
}

int arrow_set_option(arrow_ctx *ctx, int option, int value) {
    CHECK_CTX(ctx);
    switch (option) {
        case ARROW_OPT_L2_HINTS_PLAIN: ctx->l2_hints_plain = value & 3; return ARROW_OK;
        case ARROW_OPT_L2_HINTS_FUSED: ctx->l2_hints_fused = value & 3; return ARROW_OK;
        case ARROW_OPT_BIG_TILES: ctx->big_tiles = value ? 1 : 0; return ARROW_OK;
        case ARROW_OPT_TILE_ROWS:
            if (value != 0 && value != 16 && value != 32 && value != 64 && value != 128)
                return fail(ctx, ARROW_ERR_ARG, "tile rows are 0 (automatic), 16, 32, 64 or 128, not %d", value);
            ctx->tile_rows = value;
            return ARROW_OK;
        case ARROW_OPT_SPMM_CTAS_PER_SM: ctx->spmm_ctas_per_sm = value < 0 ? 0 : value; return ARROW_OK;
        case ARROW_OPT_PREFETCH: ctx->prefetch_plain = value & 0xF; ctx->prefetch_fused = (value >> 4) & 0xF;
            if (ctx->prefetch_plain > 1 || ctx->prefetch_fused > 1) { ctx->prefetch_plain = ctx->prefetch_fused = 0; return fail(ctx, ARROW_ERR_ARG, "prefetch modes are 0..1 per nibble"); }
            return ARROW_OK;
        case ARROW_OPT_ROWS_PER_GROUP: ctx->rows_per_group = (value == 1 || value == 2) ? value : 0; return ARROW_OK;
        case ARROW_OPT_SMEM_CARVEOUT: ctx->smem_carveout = value; return ARROW_OK;
        case ARROW_OPT_FORCE_PREDICATED: ctx->force_skip_path = value ? 1 : 0; return ARROW_OK;
        case ARROW_OPT_TILE_KERNEL: ctx->tile_kernel = value ? 1 : 0; return ARROW_OK;
        case ARROW_OPT_SPMM_SM_LIMIT: ctx->spmm_sm_limit = value < 0 ? 0 : value; return ARROW_OK;
        case ARROW_OPT_PUSH_CTAS: ctx->push_ctas = value < 0 ? 0 : value; return ARROW_OK;
        case ARROW_OPT_PUSH_INTERLEAVE: ctx->push_interleave = value ? 1 : 0; return ARROW_OK;
        case ARROW_OPT_BARRIER_TIMEOUT_MS: ctx->barrier_timeout_ms = value < 1 ? 1 : value; return ARROW_OK;
        default: return fail(ctx, ARROW_ERR_ARG, "unknown option %d", option);
    }
}

int arrow_tile_rows_rule(int k, int elem_bytes, int64_t l2_bytes, int resident_ctas, int big_ok) {
    if (k < 1 || (elem_bytes != 4 && elem_bytes != 8) || l2_bytes < 1 || resident_ctas < 1) return ARROW_ERR_ARG;
    return TILE_LISTS[tile_list_rule(k, elem_bytes, l2_bytes, resident_ctas, big_ok != 0)].rows;
}

int arrow_tile_rows(arrow_ctx *ctx, int k, int dtype, int *rows) {
    CHECK_CTX(ctx);
    if (!rows || k < 1 || (dtype != ARROW_F32 && dtype != ARROW_F64)) return fail(ctx, ARROW_ERR_ARG, "bad tile-rows query");
    const bool f64 = dtype == ARROW_F64;
    *rows = TILE_LISTS[tile_list_for(ctx, k, f64 ? 8 : 4, !f64 && k <= 32)].rows;
    return ARROW_OK;
}

// ---- sparse -------------------------------------------------------------------------------------
static int build_long_rows(arrow_ctx *ctx, Csr &c, const std::vector<int> &h_indptr) {
    // host pass over the (rebased) row pointer: rows above the threshold become segment tasks
    std::vector<LongTask> tasks;
    std::vector<int> rows, first;
    int64_t mx = 0;
    const int thr = ctx->long_threshold, seg = ctx->long_segment;
    for (int64_t r = 0; r < c.n_rows; ++r) {
        const int len = h_indptr[r + 1] - h_indptr[r];
        mx = std::max<int64_t>(mx, len);
        if (len > thr) {
            rows.push_back((int)r);
            first.push_back((int)tasks.size());
            for (int b = h_indptr[r]; b < h_indptr[r + 1]; b += seg)
                tasks.push_back(LongTask{(int)r, b, std::min(b + seg, h_indptr[r + 1]), (int)tasks.size()});
        }
    }
    first.push_back((int)tasks.size());
    // row tiles for k_spmm_tiles: contiguous rows, <= rows_cap rows and <= nnz_cap entries, cut around long rows
    auto build_tiles = [&](int rows_cap, int nnz_cap, int4 **out, int *n_out) -> int {
        std::vector<int4> tiles;
        int64_t r = 0;
        while (r < c.n_rows) {
            const int len0 = h_indptr[r + 1] - h_indptr[r];
            if (len0 > thr) { ++r; continue; }                     // long rows are not tiled
            int64_t e = r;
            while (e < c.n_rows && e - r < rows_cap) {
                const int len = h_indptr[e + 1] - h_indptr[e];
                if (len > thr) break;
                if (h_indptr[e + 1] - h_indptr[r] > nnz_cap - 4 && e > r) break;
                ++e;
            }
            if (e == r) ++e;                                       // a single row may pass nnz_cap but fits the kernels: thr <= TILE_NNZ - 8
            tiles.push_back(make_int4((int)r, (int)e, h_indptr[r], h_indptr[e]));
            r = e;
        }
        *n_out = (int)tiles.size();
        if (!tiles.empty()) {
            CUDA_TRY(ctx, cudaMalloc(out, tiles.size() * sizeof(int4)));
            CUDA_TRY(ctx, cudaMemcpy(*out, tiles.data(), tiles.size() * sizeof(int4), cudaMemcpyHostToDevice));
        }
        return ARROW_OK;
    };
    for (int i = 0; i < N_TILE_LISTS; ++i) {
        const int rc = build_tiles(TILE_LISTS[i].rows, TILE_LISTS[i].nnz, &c.tiles[i], &c.n_tiles[i]);
        if (rc != ARROW_OK) return rc;
    }
    c.max_row_nnz = mx;
    c.long_threshold = thr;
    c.n_long_rows = (int)rows.size();
    c.n_long_tasks = (int)tasks.size();
    c.owns_long = true;
    if (!rows.empty()) {
        CUDA_TRY(ctx, cudaMalloc(&c.long_tasks, tasks.size() * sizeof(LongTask)));
        CUDA_TRY(ctx, cudaMalloc(&c.long_rows, rows.size() * sizeof(int)));
        CUDA_TRY(ctx, cudaMalloc(&c.long_first, first.size() * sizeof(int)));
        CUDA_TRY(ctx, cudaMemcpy(c.long_tasks, tasks.data(), tasks.size() * sizeof(LongTask), cudaMemcpyHostToDevice));
        CUDA_TRY(ctx, cudaMemcpy(c.long_rows, rows.data(), rows.size() * sizeof(int), cudaMemcpyHostToDevice));
        CUDA_TRY(ctx, cudaMemcpy(c.long_first, first.data(), first.size() * sizeof(int), cudaMemcpyHostToDevice));
    }
    return ARROW_OK;
}

// device side of arrow_csr_upload; on failure the caller releases whatever `c` already owns
static int csr_fill(arrow_ctx *ctx, Csr &c, int64_t n_rows, int64_t n_cols, int64_t nnz, const std::vector<int> &h_indptr,
                    const void *indices, int indices_bytes, const void *data, int dtype) {
    const size_t esize = dtype_size(dtype);
    c.dtype = dtype;
    c.n_rows = n_rows;
    c.n_cols = n_cols;
    c.nnz = nnz;
    c.owns_indptr = c.owns_indices = c.owns_vals = c.owns_long = true;     // every array below belongs to this block
    CUDA_TRY(ctx, cudaMalloc(&c.indptr, ((size_t)n_rows + 1 + 8) * sizeof(int)));
    CUDA_TRY(ctx, cudaMemsetAsync(c.indptr, 0, ((size_t)n_rows + 1 + 8) * sizeof(int), ctx->stream));
    CUDA_TRY(ctx, cudaMemcpyAsync(c.indptr, h_indptr.data(), ((size_t)n_rows + 1) * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
    const size_t nz = (size_t)nnz + 8;                       // slack: bulk copies round up to 16 bytes
    CUDA_TRY(ctx, cudaMalloc(&c.indices, nz * sizeof(int)));
    CUDA_TRY(ctx, cudaMalloc(&c.vals, nz * esize));
    CUDA_TRY(ctx, cudaMemsetAsync(c.indices, 0, nz * sizeof(int), ctx->stream));
    CUDA_TRY(ctx, cudaMemsetAsync(c.vals, 0, nz * esize, ctx->stream));
    DevTmp wide, bad;
    int hbad = 0;
    if (nnz > 0) {
        CUDA_TRY(ctx, cudaMalloc(&bad.p, sizeof(int)));
        CUDA_TRY(ctx, cudaMemsetAsync(bad.p, 0, sizeof(int), ctx->stream));
        if (indices_bytes == 4) {
            CUDA_TRY(ctx, cudaMemcpyAsync(c.indices, indices, (size_t)nnz * 4, cudaMemcpyHostToDevice, ctx->stream));
        } else {
            CUDA_TRY(ctx, cudaMalloc(&wide.p, (size_t)nnz * 8));
            CUDA_TRY(ctx, cudaMemcpyAsync(wide.p, indices, (size_t)nnz * 8, cudaMemcpyHostToDevice, ctx->stream));
            k_to_i32<long long><<<ctx->sm_count * 8, 256, 0, ctx->stream>>>((const long long *)wide.p, c.indices, nnz, 0, (int *)bad.p);
            ctx->launches++;
        }
        // a column outside [0, n_cols) would read outside the X tile: reject the block instead
        k_check_cols<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(c.indices, nnz, n_cols, (int *)bad.p);
        ctx->launches++;
        CUDA_TRY(ctx, cudaMemcpyAsync(&hbad, bad.p, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
        if (data) {
            CUDA_TRY(ctx, cudaMemcpyAsync(c.vals, data, (size_t)nnz * esize, cudaMemcpyHostToDevice, ctx->stream));
        } else if (dtype == ARROW_F64) {
            k_fill<double><<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(reinterpret_cast<double *>(c.vals), 1.0, nnz);
            ctx->launches++;
        } else {
            k_fill<float><<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(c.vals, 1.0f, nnz);
            ctx->launches++;
        }
    }
    const int rc = build_long_rows(ctx, c, h_indptr);
    if (rc != ARROW_OK) return rc;
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));      // the host staging arrays may go out of scope now
    CUDA_TRY(ctx, cudaGetLastError());
    if (hbad) return fail(ctx, ARROW_ERR_RANGE, "a column index lies outside [0, %lld)", (long long)n_cols);
    return ARROW_OK;
}

static int csr_upload(arrow_ctx *ctx, int64_t n_rows, int64_t n_cols, int64_t nnz, const void *indptr, int indptr_bytes,
                      const void *indices, int indices_bytes, const void *data, int dtype, int *csr_out) {
    CHECK_CTX(ctx);
    if (!csr_out || !indptr || (nnz > 0 && !indices)) return fail(ctx, ARROW_ERR_ARG, "null pointer argument");
    if (n_rows < 0 || n_cols < 0 || nnz < 0) return fail(ctx, ARROW_ERR_ARG, "negative size");
    if ((indptr_bytes != 4 && indptr_bytes != 8) || (indices_bytes != 4 && indices_bytes != 8))
        return fail(ctx, ARROW_ERR_ARG, "index width must be 4 or 8 bytes");
    if (nnz > 2147483647LL || n_rows >= 2147483647LL || n_cols > 2147483647LL)
        return fail(ctx, ARROW_ERR_RANGE, "block exceeds the int32 device layout (rows=%lld cols=%lld nnz=%lld); shard it",
                    (long long)n_rows, (long long)n_cols, (long long)nnz);
    // host view of the row pointer, rebased
    std::vector<int> h_indptr((size_t)n_rows + 1);
    int64_t base = 0;
    if (indptr_bytes == 8) {
        const int64_t *ip = (const int64_t *)indptr;
        base = ip[0];
        for (int64_t r = 0; r <= n_rows; ++r) {
            const int64_t v = ip[r] - base;
            if (v < 0 || v > nnz || (r > 0 && v < h_indptr[r - 1]))
                return fail(ctx, ARROW_ERR_ARG, "indptr is not a non-decreasing sequence inside [0, nnz] at row %lld", (long long)r);
            h_indptr[r] = (int)v;
        }
    } else {
        const int32_t *ip = (const int32_t *)indptr;
        base = ip[0];
        for (int64_t r = 0; r <= n_rows; ++r) {
            const int64_t v = (int64_t)ip[r] - base;
            if (v < 0 || v > nnz || (r > 0 && v < h_indptr[r - 1]))
                return fail(ctx, ARROW_ERR_ARG, "indptr is not a non-decreasing sequence inside [0, nnz] at row %lld", (long long)r);
            h_indptr[r] = (int)v;
        }
    }
    if (h_indptr[n_rows] != nnz)
        return fail(ctx, ARROW_ERR_ARG, "indptr[n_rows]-indptr[0] = %d but nnz = %lld", h_indptr[n_rows], (long long)nnz);

    Csr c;
    const int rc = csr_fill(ctx, c, n_rows, n_cols, nnz, h_indptr, indices, indices_bytes, data, dtype);
    if (rc != ARROW_OK) {
        cudaStreamSynchronize(ctx->stream);                  // nothing may still write into what is released next
        cudaGetLastError();
        csr_release(c);
        return rc;
    }
    c.live = true;
    const int h = new_slot(ctx->csrs);
    ctx->csrs[h] = c;
    *csr_out = h;
    return ARROW_OK;
}

int arrow_csr_upload(arrow_ctx *ctx, int64_t n_rows, int64_t n_cols, int64_t nnz, const void *indptr, int indptr_bytes,
                     const void *indices, int indices_bytes, const float *data, int *csr_out) {
    return csr_upload(ctx, n_rows, n_cols, nnz, indptr, indptr_bytes, indices, indices_bytes, data, ARROW_F32, csr_out);
}

int arrow_csr_upload_f64(arrow_ctx *ctx, int64_t n_rows, int64_t n_cols, int64_t nnz, const void *indptr, int indptr_bytes,
                         const void *indices, int indices_bytes, const double *data, int *csr_out) {
    return csr_upload(ctx, n_rows, n_cols, nnz, indptr, indptr_bytes, indices, indices_bytes, data, ARROW_F64, csr_out);
}

int arrow_csr_free(arrow_ctx *ctx, int csr) {
    CHECK_CTX(ctx);
    Csr *c = get_csr(ctx, csr);
    if (!c) return fail(ctx, ARROW_ERR_HANDLE, "bad csr handle %d", csr);
    if (c->children > 0)
        return fail(ctx, ARROW_ERR_ARG, "csr %d still backs %d remapped block(s); free those first", csr, c->children);
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    if (Csr *parent = get_csr(ctx, c->parent)) parent->children--;
    csr_release(*c);
    return ARROW_OK;
}

int arrow_csr_info(arrow_ctx *ctx, int csr, int64_t *n_rows, int64_t *n_cols, int64_t *nnz, int64_t *max_row_nnz,
                   int64_t *n_long_rows) {
    CHECK_CTX(ctx);
    Csr *c = get_csr(ctx, csr);
    if (!c) return fail(ctx, ARROW_ERR_HANDLE, "bad csr handle %d", csr);
    if (n_rows) *n_rows = c->n_rows;
    if (n_cols) *n_cols = c->n_cols;
    if (nnz) *nnz = c->nnz;
    if (max_row_nnz) *max_row_nnz = c->max_row_nnz;
    if (n_long_rows) *n_long_rows = c->n_long_rows;
    return ARROW_OK;
}

int arrow_csr_remap_columns(arrow_ctx *ctx, int csr, int map, int64_t new_n_cols, int *csr_out) {
    CHECK_CTX(ctx);
    Csr *c = get_csr(ctx, csr);
    IdxMap *m = get_map(ctx, map);
    if (!c) return fail(ctx, ARROW_ERR_HANDLE, "bad csr handle %d", csr);
    if (!m) return fail(ctx, ARROW_ERR_HANDLE, "bad map handle %d", map);
    if (!csr_out) return fail(ctx, ARROW_ERR_ARG, "csr_out is null");
    if (new_n_cols < 0 || new_n_cols > 2147483647LL || m->limit > new_n_cols)
        return fail(ctx, ARROW_ERR_ARG, "map reaches column %lld but the remapped block has %lld columns", (long long)m->limit, (long long)new_n_cols);
    if (c->parent >= 0) return fail(ctx, ARROW_ERR_ARG, "csr %d is itself a remapped copy; remap its source", csr);
    Csr d = *c;
    d.owns_indptr = d.owns_vals = d.owns_long = false;      // shared with the source block
    d.owns_indices = true;
    d.indices = nullptr;
    d.n_cols = new_n_cols;
    d.parent = csr;
    d.children = 0;
    CUDA_TRY(ctx, cudaMalloc(&d.indices, ((size_t)c->nnz + 8) * sizeof(int)));
    cudaError_t e = cudaMemsetAsync(d.indices, 0, ((size_t)c->nnz + 8) * sizeof(int), ctx->stream);
    int h_invalid = 0;
    if (e == cudaSuccess && c->nnz > 0) {
        DevTmp flag;
        e = cudaMalloc(&flag.p, sizeof(int));
        if (e == cudaSuccess) e = cudaMemsetAsync(flag.p, 0, sizeof(int), ctx->stream);
        if (e == cudaSuccess) {
            k_remap<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(c->indices, m->p, m->n, d.indices, c->nnz, (int *)flag.p);
            ctx->launches++;
            e = cudaGetLastError();
        }
        if (e == cudaSuccess) e = cudaMemcpyAsync(&h_invalid, flag.p, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    }
    if (e != cudaSuccess) {
        cudaFree(d.indices);
        return fail(ctx, ARROW_ERR_CUDA, "column remap failed: %s", cudaGetErrorString(e));
    }
    // entries whose image is invalid are skipped by the kernels (predicated gathers); when every entry maps to a valid
    // column -- always the case on the fused path -- the copy runs the unpredicated batches like its source
    d.may_skip = c->may_skip || h_invalid != 0;
    const int h = new_slot(ctx->csrs);       // may grow the table: `c` is not used past this point
    ctx->csrs[h] = d;
    ctx->csrs[csr].children++;
    *csr_out = h;
    return ARROW_OK;
}

// ---- maps ---------------------------------------------------------------------------------------
int arrow_map_upload(arrow_ctx *ctx, const int64_t *map, int64_t n, int64_t limit, int *map_out) {
    CHECK_CTX(ctx);
    if (!map_out || (n > 0 && !map)) return fail(ctx, ARROW_ERR_ARG, "null pointer argument");
    if (n < 0 || limit < 0 || limit > 2147483647LL || n > 2147483647LL)
        return fail(ctx, ARROW_ERR_RANGE, "map size/limit exceed the int32 device layout");
    IdxMap m;
    m.n = n;
    m.limit = limit;
    CUDA_TRY(ctx, cudaMalloc(&m.p, (size_t)std::max<int64_t>(n, 1) * sizeof(int)));
    cudaError_t e = cudaSuccess;
    if (n > 0) {
        DevTmp wide;
        e = cudaMalloc(&wide.p, (size_t)n * 8);
        if (e == cudaSuccess) e = cudaMemcpyAsync(wide.p, map, (size_t)n * 8, cudaMemcpyHostToDevice, ctx->stream);
        if (e == cudaSuccess) {
            k_map_from_i64<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>((const long long *)wide.p, m.p, n, limit);
            ctx->launches++;
            e = cudaStreamSynchronize(ctx->stream);
        }
    }
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e != cudaSuccess) {
        cudaGetLastError();
        cudaFree(m.p);
        return fail(ctx, ARROW_ERR_CUDA, "map upload failed: %s", cudaGetErrorString(e));
    }
    m.live = true;
    const int h = new_slot(ctx->maps);
    ctx->maps[h] = m;
    *map_out = h;
    return ARROW_OK;
}

int arrow_map_free(arrow_ctx *ctx, int map) {
    CHECK_CTX(ctx);
    IdxMap *m = get_map(ctx, map);
    if (!m) return fail(ctx, ARROW_ERR_HANDLE, "bad map handle %d", map);
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    cudaFree(m->p);
    *m = IdxMap();
    return ARROW_OK;
}

int arrow_map_compose(arrow_ctx *ctx, int inner, int outer, int *map_out) {
    CHECK_CTX(ctx);
    IdxMap *a = get_map(ctx, inner), *b = get_map(ctx, outer);
    if (!a || !b) return fail(ctx, ARROW_ERR_HANDLE, "bad map handle");
    if (!map_out) return fail(ctx, ARROW_ERR_ARG, "map_out is null");
    IdxMap m;
    m.n = a->n;
    m.limit = b->limit;
    CUDA_TRY(ctx, cudaMalloc(&m.p, (size_t)std::max<int64_t>(m.n, 1) * sizeof(int)));
    if (m.n > 0) {
        k_remap<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(a->p, b->p, b->n, m.p, m.n, nullptr);
        ctx->launches++;
    }
    if (cudaError_t e = cudaGetLastError(); e != cudaSuccess) {
        cudaFree(m.p);
        return fail(ctx, ARROW_ERR_CUDA, "map compose failed: %s", cudaGetErrorString(e));
    }
    m.live = true;
    const int h = new_slot(ctx->maps);
    ctx->maps[h] = m;
    *map_out = h;
    return ARROW_OK;
}

int arrow_map_invert(arrow_ctx *ctx, int map, int64_t n_out, int *map_out) {
    CHECK_CTX(ctx);
    IdxMap *a = get_map(ctx, map);
    if (!a) return fail(ctx, ARROW_ERR_HANDLE, "bad map handle %d", map);
    if (!map_out || n_out < 0 || n_out > 2147483647LL) return fail(ctx, ARROW_ERR_ARG, "bad argument");
    IdxMap m;
    m.n = n_out;
    m.limit = a->n;
    CUDA_TRY(ctx, cudaMalloc(&m.p, (size_t)std::max<int64_t>(n_out, 1) * sizeof(int)));
    if (n_out > 0) {
        k_fill<int><<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(m.p, -1, n_out);
        ctx->launches++;
    }
    if (a->n > 0) {
        k_map_invert<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(a->p, a->n, m.p, n_out);
        ctx->launches++;
    }
    if (cudaError_t e = cudaGetLastError(); e != cudaSuccess) {
        cudaFree(m.p);
        return fail(ctx, ARROW_ERR_CUDA, "map invert failed: %s", cudaGetErrorString(e));
    }
    m.live = true;
    const int h = new_slot(ctx->maps);
    ctx->maps[h] = m;
    *map_out = h;
    return ARROW_OK;
}

int arrow_map_d2h(arrow_ctx *ctx, int map, int32_t *host, int64_t n) {
    CHECK_CTX(ctx);
    IdxMap *a = get_map(ctx, map);
    if (!a) return fail(ctx, ARROW_ERR_HANDLE, "bad map handle %d", map);
    if (!host || n < 0 || n > a->n) return fail(ctx, ARROW_ERR_ARG, "bad host buffer / length");
    CUDA_TRY(ctx, cudaMemcpyAsync(host, a->p, (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    return ARROW_OK;
}

// ---- dense --------------------------------------------------------------------------------------
int arrow_dense_alloc_dtype(arrow_ctx *ctx, int64_t rows, int k, int dtype, int *buf_out) {
    CHECK_CTX(ctx);
    if (!buf_out || rows < 0 || k < 1) return fail(ctx, ARROW_ERR_ARG, "bad dense shape %lld x %d", (long long)rows, k);
    if (dtype != ARROW_F32 && dtype != ARROW_F64 && dtype != ARROW_I32 && dtype != ARROW_B1)
        return fail(ctx, ARROW_ERR_ARG, "unknown dtype %d", dtype);
    DenseBuf d;
    d.rows = rows;
    d.k = k;
    d.dtype = dtype;
    const size_t bytes = std::max<size_t>((size_t)rows * row_bytes(dtype, k), 16);
    cudaError_t e = cudaMalloc(&d.p, bytes);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return fail(ctx, ARROW_ERR_NOMEM, "cudaMalloc(%zu bytes) for a %lld x %d tile: %s", bytes, (long long)rows, k,
                    cudaGetErrorString(e));
    }
    CUDA_TRY(ctx, cudaMemsetAsync(d.p, 0, bytes, ctx->stream));
    d.owned = true;
    d.live = true;
    const int h = new_slot(ctx->dense);
    ctx->dense[h] = d;
    *buf_out = h;
    return ARROW_OK;
}

int arrow_dense_alloc(arrow_ctx *ctx, int64_t rows, int k, int *buf_out) {
    return arrow_dense_alloc_dtype(ctx, rows, k, ARROW_F32, buf_out);
}

int arrow_dense_dtype(arrow_ctx *ctx, int buf, int *dtype) {
    CHECK_CTX(ctx);
    DenseBuf *d = get_dense(ctx, buf);
    if (!d) return fail(ctx, ARROW_ERR_HANDLE, "bad dense handle %d", buf);
    if (!dtype) return fail(ctx, ARROW_ERR_ARG, "dtype is null");
    *dtype = d->dtype;
    return ARROW_OK;
}

int arrow_dense_free(arrow_ctx *ctx, int buf) {
    CHECK_CTX(ctx);
    DenseBuf *d = get_dense(ctx, buf);
    if (!d) return fail(ctx, ARROW_ERR_HANDLE, "bad dense handle %d", buf);
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    if (d->owned) cudaFree(d->p);
    else if (d->ipc) cudaIpcCloseMemHandle(d->ipc_base);
    *d = DenseBuf();
    return ARROW_OK;
}

int arrow_dense_fill(arrow_ctx *ctx, int buf, float value) {
    CHECK_CTX(ctx);
    DenseBuf *d = get_dense(ctx, buf);
    if (!d) return fail(ctx, ARROW_ERR_HANDLE, "bad dense handle %d", buf);
    REFUSE_I32(ctx, d, "arrow_dense_fill");
    if (d->dtype == ARROW_B1 && value != 0.f) return fail(ctx, ARROW_ERR_ARG, "a bit tile is filled with 0 only");
    const long long n = (long long)d->rows * d->k;
    if (n == 0) return ARROW_OK;
    if (value == 0.f) {
        CUDA_TRY(ctx, cudaMemsetAsync(d->p, 0, (size_t)d->rows * row_bytes(d->dtype, d->k), ctx->stream));
    } else if (d->dtype == ARROW_F64) {
        k_fill<double><<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(reinterpret_cast<double *>(d->p), (double)value, n);
        ctx->launches++;
        CUDA_TRY(ctx, cudaGetLastError());
    } else {
        k_fill<float><<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(d->p, value, n);
        ctx->launches++;
        CUDA_TRY(ctx, cudaGetLastError());
    }
    return ARROW_OK;
}

int arrow_dense_h2d(arrow_ctx *ctx, int buf, int64_t row0, int64_t rows, const void *host) {
    CHECK_CTX(ctx);
    DenseBuf *d = get_dense(ctx, buf);
    if (!d) return fail(ctx, ARROW_ERR_HANDLE, "bad dense handle %d", buf);
    if (!host || row0 < 0 || rows < 0 || row0 + rows > d->rows)
        return fail(ctx, ARROW_ERR_ARG, "h2d rows [%lld,%lld) outside tile of %lld rows", (long long)row0, (long long)(row0 + rows), (long long)d->rows);
    if (rows == 0) return ARROW_OK;
    CUDA_TRY(ctx, cudaMemcpyAsync(dense_row(d, row0), host, (size_t)rows * row_bytes(d->dtype, d->k), cudaMemcpyHostToDevice, ctx->stream));
    return ARROW_OK;
}

int arrow_dense_d2h(arrow_ctx *ctx, int buf, int64_t row0, int64_t rows, void *host) {
    CHECK_CTX(ctx);
    DenseBuf *d = get_dense(ctx, buf);
    if (!d) return fail(ctx, ARROW_ERR_HANDLE, "bad dense handle %d", buf);
    if (!host || row0 < 0 || rows < 0 || row0 + rows > d->rows)
        return fail(ctx, ARROW_ERR_ARG, "d2h rows [%lld,%lld) outside tile of %lld rows", (long long)row0, (long long)(row0 + rows), (long long)d->rows);
    if (rows == 0) return ARROW_OK;
    CUDA_TRY(ctx, cudaMemcpyAsync(host, dense_row(d, row0), (size_t)rows * row_bytes(d->dtype, d->k), cudaMemcpyDeviceToHost, ctx->stream));
    return ARROW_OK;
}

int arrow_dense_copy(arrow_ctx *ctx, int dst, int64_t dst_row0, int src, int64_t src_row0, int64_t rows) {
    CHECK_CTX(ctx);
    DenseBuf *a = get_dense(ctx, dst), *b = get_dense(ctx, src);
    if (!a || !b) return fail(ctx, ARROW_ERR_HANDLE, "bad dense handle");
    if (a->k != b->k) return fail(ctx, ARROW_ERR_ARG, "feature width mismatch %d vs %d", a->k, b->k);
    if (a->dtype != b->dtype) return fail(ctx, ARROW_ERR_ARG, "dtype mismatch: %s vs %s", dtype_name(a->dtype), dtype_name(b->dtype));
    if (rows < 0 || dst_row0 < 0 || src_row0 < 0 || dst_row0 + rows > a->rows || src_row0 + rows > b->rows)
        return fail(ctx, ARROW_ERR_ARG, "copy range outside tiles");
    if (rows == 0) return ARROW_OK;
    CUDA_TRY(ctx, cudaMemcpyAsync(dense_row(a, dst_row0), dense_row(b, src_row0), (size_t)rows * row_bytes(a->dtype, a->k),
                                  cudaMemcpyDeviceToDevice, cur_stream(ctx)));
    return ARROW_OK;
}

int arrow_dense_ptr(arrow_ctx *ctx, int buf, void **device_ptr, int64_t *rows, int *k) {
    CHECK_CTX(ctx);
    DenseBuf *d = get_dense(ctx, buf);
    if (!d) return fail(ctx, ARROW_ERR_HANDLE, "bad dense handle %d", buf);
    if (device_ptr) *device_ptr = d->p;
    if (rows) *rows = d->rows;
    if (k) *k = d->k;
    return ARROW_OK;
}

int arrow_dense_wrap(arrow_ctx *ctx, void *device_ptr, int64_t rows, int k, int *buf_out) {
    CHECK_CTX(ctx);
    if (!device_ptr || !buf_out || rows < 0 || k < 1) return fail(ctx, ARROW_ERR_ARG, "bad wrap arguments");
    // the vector kernels load and store float4 rows (and cp.async.bulk moves 16-byte units) when k % 4 == 0
    const uintptr_t align = (k % 4 == 0) ? 16 : 4;
    if ((uintptr_t)device_ptr % align != 0)
        return fail(ctx, ARROW_ERR_ARG, "wrapped pointer %p is not %d-byte aligned (k = %d)", device_ptr, (int)align, k);
    DenseBuf d;
    d.p = (float *)device_ptr;
    d.rows = rows;
    d.k = k;
    d.live = true;
    const int h = new_slot(ctx->dense);
    ctx->dense[h] = d;
    *buf_out = h;
    return ARROW_OK;
}

int arrow_host_alloc(size_t bytes, void **ptr) {
    if (!ptr) return ARROW_ERR_ARG;
    cudaError_t e = cudaMallocHost(ptr, std::max<size_t>(bytes, 16));
    if (e != cudaSuccess) {
        cudaGetLastError();
        return fail(nullptr, ARROW_ERR_NOMEM, "cudaMallocHost(%zu): %s", bytes, cudaGetErrorString(e));
    }
    return ARROW_OK;
}

int arrow_host_free(void *ptr) {
    if (!ptr) return ARROW_OK;
    size_t len = 0;
    {
        std::lock_guard<std::mutex> lk(g_numa_mu);
        auto it = g_numa_allocs.find(ptr);
        if (it != g_numa_allocs.end()) { len = it->second; g_numa_allocs.erase(it); }
    }
    if (len) {
        const bool ok = cudaHostUnregister(ptr) == cudaSuccess;
        munmap(ptr, len);
        return ok ? ARROW_OK : ARROW_ERR_CUDA;
    }
    return cudaFreeHost(ptr) == cudaSuccess ? ARROW_OK : ARROW_ERR_CUDA;
}

// ---- hot path -----------------------------------------------------------------------------------
struct SpmmCall {
    int csr = -1, x_buf = -1, c_buf = -1;
    int rowmap = -1, flags = 0, variant = ARROW_VARIANT_AUTO;
    int add_buf = -1, add_map = -1;
    int x2_buf = -1;
    int64_t x_split = 0;
    int out_table = -1;
};
static int spmm_impl(arrow_ctx *ctx, const SpmmCall &q);

#define CHECK_POISON(ctx)                                                                                     \
    do {                                                                                                      \
        if ((ctx)->poisoned) return fail((ctx), ARROW_ERR_CUDA, "context is poisoned by a peer-barrier time-out"); \
    } while (0)

int arrow_spmm(arrow_ctx *ctx, int csr, int x_buf, int c_buf, int rowmap, int flags, int variant) {
    SpmmCall q;
    q.csr = csr; q.x_buf = x_buf; q.c_buf = c_buf; q.rowmap = rowmap; q.flags = flags; q.variant = variant;
    return spmm_impl(ctx, q);
}

int arrow_spmm_add(arrow_ctx *ctx, int csr, int x_buf, int c_buf, int add_buf, int add_map, int variant) {
    SpmmCall q;
    q.csr = csr; q.x_buf = x_buf; q.c_buf = c_buf; q.variant = variant; q.add_buf = add_buf; q.add_map = add_map;
    return spmm_impl(ctx, q);
}

int arrow_spmm_ex(arrow_ctx *ctx, int csr, int x_buf, int x2_buf, int64_t x_split, int c_buf, int out_table,
                  int add_buf, int add_map, int variant) {
    SpmmCall q;
    q.csr = csr; q.x_buf = x_buf; q.x2_buf = x2_buf; q.x_split = x_split; q.c_buf = c_buf; q.out_table = out_table;
    q.add_buf = add_buf; q.add_map = add_map; q.variant = variant;
    return spmm_impl(ctx, q);
}

static int spmm_impl(arrow_ctx *ctx, const SpmmCall &q) {
    CHECK_CTX(ctx);
    CHECK_POISON(ctx);
    Csr *A = get_csr(ctx, q.csr);
    DenseBuf *X = get_dense(ctx, q.x_buf);
    DenseBuf *C = q.c_buf >= 0 ? get_dense(ctx, q.c_buf) : nullptr;
    if (!A) return fail(ctx, ARROW_ERR_HANDLE, "bad csr handle %d", q.csr);
    if (!X) return fail(ctx, ARROW_ERR_HANDLE, "bad dense handle (x=%d)", q.x_buf);
    // every operand of a launch has the block's precision
    if (X->dtype != A->dtype || (C && C->dtype != A->dtype))
        return fail(ctx, ARROW_ERR_ARG, "mixed precision: the block is %s, X is %s, C is %s", dtype_name(A->dtype),
                    dtype_name(X->dtype), C ? dtype_name(C->dtype) : "-");
    PtrTable *OT = nullptr;
    if (q.out_table >= 0) {
        if (q.out_table >= (int)ctx->ptrtabs.size() || !ctx->ptrtabs[q.out_table].live)
            return fail(ctx, ARROW_ERR_HANDLE, "bad pointer table handle %d", q.out_table);
        OT = &ctx->ptrtabs[q.out_table];
        if (OT->n < A->n_rows) return fail(ctx, ARROW_ERR_ARG, "pointer table has %lld entries, block has %lld rows", (long long)OT->n, (long long)A->n_rows);
        if (OT->k != X->k) return fail(ctx, ARROW_ERR_ARG, "pointer table was built for %d feature columns, X has %d", OT->k, X->k);
        if (q.rowmap >= 0 || (q.flags & ARROW_ACCUMULATE)) return fail(ctx, ARROW_ERR_ARG, "a pointer table excludes rowmap / accumulate");
    } else if (!C) {
        return fail(ctx, ARROW_ERR_HANDLE, "bad dense handle (c=%d)", q.c_buf);
    }
    if (C) {
        if (X->k != C->k) return fail(ctx, ARROW_ERR_ARG, "X has %d feature columns, C has %d", X->k, C->k);
        if (X->p == C->p) return fail(ctx, ARROW_ERR_ARG, "X and C must not alias");
    }
    DenseBuf *X2 = nullptr;
    if (q.x2_buf >= 0) {
        X2 = get_dense(ctx, q.x2_buf);
        if (!X2) return fail(ctx, ARROW_ERR_HANDLE, "bad dense handle (x2=%d)", q.x2_buf);
        if (X2->dtype != A->dtype) return fail(ctx, ARROW_ERR_ARG, "mixed precision: the block is %s, X2 is %s", dtype_name(A->dtype), dtype_name(X2->dtype));
        if (X2->k != X->k) return fail(ctx, ARROW_ERR_ARG, "X2 has %d feature columns, X has %d", X2->k, X->k);
        if (q.x_split < 0 || q.x_split > X->rows || q.x_split > A->n_cols)
            return fail(ctx, ARROW_ERR_ARG, "x_split %lld outside X (%lld rows) / the block's %lld columns", (long long)q.x_split, (long long)X->rows, (long long)A->n_cols);
        if (X2->rows < A->n_cols - q.x_split)
            return fail(ctx, ARROW_ERR_ARG, "X2 has %lld rows, columns beyond the split need %lld", (long long)X2->rows, (long long)(A->n_cols - q.x_split));
        if (C && X2->p == C->p) return fail(ctx, ARROW_ERR_ARG, "X2 and C must not alias");
    } else if (X->rows < A->n_cols) {
        return fail(ctx, ARROW_ERR_ARG, "X has %lld rows, block has %lld columns", (long long)X->rows, (long long)A->n_cols);
    }
    IdxMap *rm = nullptr;
    if (q.rowmap >= 0) {
        rm = get_map(ctx, q.rowmap);
        if (!rm) return fail(ctx, ARROW_ERR_HANDLE, "bad rowmap handle %d", q.rowmap);
        if (rm->n < A->n_rows) return fail(ctx, ARROW_ERR_ARG, "rowmap has %lld entries, block has %lld rows", (long long)rm->n, (long long)A->n_rows);
        if (rm->limit > C->rows) return fail(ctx, ARROW_ERR_ARG, "rowmap reaches row %lld, C has %lld rows", (long long)rm->limit, (long long)C->rows);
    } else if (C && !OT && C->rows < A->n_rows) {
        return fail(ctx, ARROW_ERR_ARG, "C has %lld rows, block has %lld rows", (long long)C->rows, (long long)A->n_rows);
    }
    if (A->n_rows == 0) return ARROW_OK;
    const bool acc = (q.flags & ARROW_ACCUMULATE) != 0;
    const int k = X->k;
    const int lane = ctx->cur_lane;
    SpmmArgs a;
    a.indptr = A->indptr;
    a.indices = A->indices;
    a.vals = A->vals;
    a.X = X->p;
    a.C = C ? C->p : nullptr;
    a.rowmap = rm ? rm->p : nullptr;
    a.n_rows = A->n_rows;
    a.k = k;
    a.k4 = k / 4;
    a.long_threshold = A->long_threshold;
    a.add_src = nullptr;
    a.add_map = nullptr;
    a.X2 = X2 ? X2->p : nullptr;
    a.x_split = X2 ? (int)q.x_split : 0;
    a.out_ptr = OT ? OT->p : nullptr;
    if (q.add_buf >= 0 || q.add_map >= 0) {
        DenseBuf *S = get_dense(ctx, q.add_buf);
        IdxMap *am = get_map(ctx, q.add_map);
        if (!S || !am) return fail(ctx, ARROW_ERR_HANDLE, "bad addend handles (buf=%d map=%d)", q.add_buf, q.add_map);
        if (S->k != k) return fail(ctx, ARROW_ERR_ARG, "addend has %d feature columns, expected %d", S->k, k);
        if (S->dtype != A->dtype) return fail(ctx, ARROW_ERR_ARG, "mixed precision: the block is %s, the addend is %s", dtype_name(A->dtype), dtype_name(S->dtype));
        if (am->n < A->n_rows) return fail(ctx, ARROW_ERR_ARG, "addend map has %lld entries, block has %lld rows", (long long)am->n, (long long)A->n_rows);
        if (am->limit > S->rows) return fail(ctx, ARROW_ERR_ARG, "addend map reaches row %lld, addend tile has %lld rows", (long long)am->limit, (long long)S->rows);
        if (C && S->p == C->p) return fail(ctx, ARROW_ERR_ARG, "addend and C must not alias");
        a.add_src = S->p;
        a.add_map = am->p;
    }
    if (A->dtype == ARROW_F64) {
        // float64 runs the one-GPU product: no two-part operand, no pointer table, no kernel override
        if (X2 || OT) return fail(ctx, ARROW_ERR_UNSUPPORTED, "float64 has no two-part X operand or pointer-table epilogue (one GPU only)");
        if (q.variant != ARROW_VARIANT_AUTO && q.variant != ARROW_VARIANT_TILES)
            return fail(ctx, ARROW_ERR_UNSUPPORTED, "float64 has no kernel variant override (variant %d)", q.variant);
        return spmm_f64(ctx, A, a, rm != nullptr, acc);
    }
    int variant = q.variant;
    if (variant == ARROW_VARIANT_AUTO) variant = pick_variant(k);
    const int vpl_req = (variant >> 4) & 0xF;          // optional float4-per-lane override (tile kernel)
    const int rpg_req = (variant >> 8) & 0x3;          // optional rows-per-group override (tile kernel, k <= 32)
    variant &= 0xF;
    // the epilogue gather-add, the dual X base and the row-pointer epilogue live in the tile / generic / long kernels
    if ((a.add_map != nullptr || X2 || OT) && variant != 3) variant = 3;
    if (variant < 0 || variant > 3) return fail(ctx, ARROW_ERR_ARG, "unknown variant %d", variant);
    const bool fused_launch = rm != nullptr || acc || OT != nullptr || X2 != nullptr || a.add_map != nullptr;

    const bool vec_ok = (k % 4 == 0) && k <= 256;
    if (!vec_ok) {
        launch_generic<PlusTimes<float>>(ctx, a, rm != nullptr, acc);
    } else if (variant == 3) {
        if (A->n_tiles[TILE_LIST_SMALL] > 0) {
            TileArgs t;
            t.a = a;
            t.skip = (A->may_skip || ctx->force_skip_path) ? 1 : 0;
            t.ticket = ctx->tile_ticket + 2 * lane;
            t.l2_hints = (rm != nullptr || acc) ? ctx->l2_hints_fused : ctx->l2_hints_plain;
            t.prefetch = fused_launch ? ctx->prefetch_fused : ctx->prefetch_plain;
            TileLaunch L;
            L.out_mode = OT ? OUT_ROWPTR : (rm ? OUT_ROWMAP : OUT_IDENTITY);
            L.acc = acc;
            L.dualx = X2 != nullptr;
            L.vpl_req = vpl_req;
            L.rpg_req = rpg_req;
            int rc = launch_tiles(ctx, t, A, L);
            if (rc != ARROW_OK) return rc;
        }
    } else if (variant == ARROW_VARIANT_TMA && k >= 32 && k <= 128) {
        if (a.k4 <= 32) launch_tma<1>(ctx, a, rm != nullptr, acc);
        else launch_tma<2>(ctx, a, rm != nullptr, acc);
    } else {
        if (variant == ARROW_VARIANT_TMA) variant = ARROW_VARIANT_SHFL;
        const int k4 = a.k4;
        if (k4 <= 1) launch_vec<1, 1>(ctx, a, rm != nullptr, acc, variant);
        else if (k4 <= 2) launch_vec<2, 1>(ctx, a, rm != nullptr, acc, variant);
        else if (k4 <= 4) launch_vec<4, 1>(ctx, a, rm != nullptr, acc, variant);
        else if (k4 <= 8) launch_vec<8, 1>(ctx, a, rm != nullptr, acc, variant);
        else if (k4 <= 16) launch_vec<16, 1>(ctx, a, rm != nullptr, acc, variant);
        else if (k4 <= 32) launch_vec<32, 1>(ctx, a, rm != nullptr, acc, variant);
        else launch_vec<32, 2>(ctx, a, rm != nullptr, acc, variant);
    }
    CUDA_TRY(ctx, cudaGetLastError());
    return launch_long_rows<PlusTimes<float>>(ctx, A, a, rm != nullptr, acc);
}

// ---- pointer tables -------------------------------------------------------------------------------
int arrow_ptrtable_upload(arrow_ctx *ctx, const int *bufs, int n_bufs, const int32_t *which, const int64_t *row, int64_t n,
                          int *table_out) {
    CHECK_CTX(ctx);
    if (!table_out || n < 0 || n_bufs < 1 || n_bufs > 64 || !bufs || (n > 0 && (!which || !row)))
        return fail(ctx, ARROW_ERR_ARG, "bad pointer table arguments");
    unsigned long long bases[64];
    int64_t rows_of[64];
    int k = 0;
    for (int b = 0; b < n_bufs; ++b) {
        DenseBuf *d = get_dense(ctx, bufs[b]);
        if (!d) return fail(ctx, ARROW_ERR_HANDLE, "bad dense handle %d", bufs[b]);
        if (b == 0) k = d->k;
        else if (d->k != k) return fail(ctx, ARROW_ERR_ARG, "tiles of a pointer table must share the feature width");
        REFUSE_I32(ctx, d, "arrow_ptrtable_upload");
        REFUSE_B1(ctx, d, "arrow_ptrtable_upload");
        if (d->dtype != ARROW_F32) return fail(ctx, ARROW_ERR_UNSUPPORTED, "pointer tables are float32 only");
        bases[b] = (unsigned long long)d->p;
        rows_of[b] = d->rows;
    }
    for (int64_t i = 0; i < n; ++i) {
        const int w = which[i];
        if (w >= n_bufs) return fail(ctx, ARROW_ERR_ARG, "row %lld refers to tile %d of %d", (long long)i, w, n_bufs);
        if (w >= 0 && (row[i] < 0 || row[i] >= rows_of[w]))
            return fail(ctx, ARROW_ERR_ARG, "row %lld points at row %lld of a %lld-row tile", (long long)i, (long long)row[i], (long long)rows_of[w]);
    }
    PtrTable t;
    t.n = n;
    t.k = k;
    CUDA_TRY(ctx, cudaMalloc(&t.p, (size_t)std::max<int64_t>(n, 1) * sizeof(float *)));
    cudaError_t e = cudaSuccess;
    if (n > 0) {
        DevTmp dw, dr, db;
        e = cudaMalloc(&dw.p, (size_t)n * 4);
        if (e == cudaSuccess) e = cudaMalloc(&dr.p, (size_t)n * 8);
        if (e == cudaSuccess) e = cudaMalloc(&db.p, sizeof bases);
        if (e == cudaSuccess) e = cudaMemcpyAsync(dw.p, which, (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream);
        if (e == cudaSuccess) e = cudaMemcpyAsync(dr.p, row, (size_t)n * 8, cudaMemcpyHostToDevice, ctx->stream);
        if (e == cudaSuccess) e = cudaMemcpyAsync(db.p, bases, sizeof bases, cudaMemcpyHostToDevice, ctx->stream);
        if (e == cudaSuccess) {
            k_fill_ptr_table<<<ctx->sm_count * 4, 256, 0, ctx->stream>>>(t.p, (const int *)dw.p, (const long long *)dr.p,
                                                                         (const unsigned long long *)db.p, n, k);
            ctx->launches++;
            e = cudaStreamSynchronize(ctx->stream);
        }
        if (e == cudaSuccess) e = cudaGetLastError();
    }
    if (e != cudaSuccess) {
        cudaGetLastError();
        cudaFree(t.p);
        return fail(ctx, ARROW_ERR_CUDA, "pointer table upload failed: %s", cudaGetErrorString(e));
    }
    t.live = true;
    int h = -1;
    for (size_t i = 0; i < ctx->ptrtabs.size(); ++i)
        if (!ctx->ptrtabs[i].live) { h = (int)i; break; }
    if (h < 0) { ctx->ptrtabs.emplace_back(); h = (int)ctx->ptrtabs.size() - 1; }
    ctx->ptrtabs[h] = t;
    *table_out = h;
    return ARROW_OK;
}

int arrow_ptrtable_free(arrow_ctx *ctx, int table) {
    CHECK_CTX(ctx);
    if (table < 0 || table >= (int)ctx->ptrtabs.size() || !ctx->ptrtabs[table].live)
        return fail(ctx, ARROW_ERR_HANDLE, "bad pointer table handle %d", table);
    CUDA_TRY(ctx, cudaDeviceSynchronize());
    cudaFree(ctx->ptrtabs[table].p);
    ctx->ptrtabs[table] = PtrTable();
    return ARROW_OK;
}

static int gather_common(arrow_ctx *ctx, DenseBuf *D, const float *src, const MultiSrc &ms, bool multi, IdxMap *m, bool acc) {
    CHECK_POISON(ctx);
    const long long n_rows = m->n;
    if (n_rows == 0) return ARROW_OK;
    const int k = D->k;
    const bool f64 = D->dtype == ARROW_F64;
    const bool bits = D->dtype == ARROW_B1;                  // whole rows of words, moved as float4 loads / stores (no arithmetic)
    const bool vec = bits ? bit_row_words(k) % 4 == 0 : (f64 ? (k % 2 == 0) : (k % 4 == 0));        // 16-byte vectors: float4 / double2
    const int vpr = bits ? (vec ? bit_row_words(k) / 4 : bit_row_words(k)) : (vec ? (f64 ? k / 2 : k / 4) : k);
    int g = 1;
    while (g < vpr && g < 32) g <<= 1;                       // lanes per row
    if (g > 8 && vpr <= 32) g = 8;                           // 8 lanes x 4 vectors cover k <= 128 in one pass
    const int threads = 256;
    const long long rows_per_cta = (threads / 32) * (32 / g);
    int grid = (int)std::min<long long>((n_rows + rows_per_cta - 1) / rows_per_cta, (long long)ctx->sm_count * 8);
    grid = std::max(grid, 1);
#define LAUNCH_GA(VT, GG, ACCV, MULTIV)                                                                          \
    k_gather_rows<VT, GG, ACCV, MULTIV><<<grid, threads, 0, cur_stream(ctx)>>>(reinterpret_cast<VT *>(D->p),     \
                                                                           reinterpret_cast<const VT *>(src), ms, m->p, n_rows, vpr)
#define DISPATCH_G(VT, ACCV, MULTIV)                                                                             \
    do {                                                                                                         \
        switch (g) {                                                                                             \
            case 1: LAUNCH_GA(VT, 1, ACCV, MULTIV); break;                                                       \
            case 2: LAUNCH_GA(VT, 2, ACCV, MULTIV); break;                                                       \
            case 4: LAUNCH_GA(VT, 4, ACCV, MULTIV); break;                                                       \
            case 8: LAUNCH_GA(VT, 8, ACCV, MULTIV); break;                                                       \
            case 16: LAUNCH_GA(VT, 16, ACCV, MULTIV); break;                                                     \
            default: LAUNCH_GA(VT, 32, ACCV, MULTIV); break;                                                     \
        }                                                                                                        \
    } while (0)
    if (f64) {                                                // one GPU: no multi-source gather
        if (vec) { if (acc) DISPATCH_G(double2, true, false); else DISPATCH_G(double2, false, false); }
        else     { if (acc) DISPATCH_G(double, true, false); else DISPATCH_G(double, false, false); }
    } else if (vec) {
        if (multi) { if (acc) DISPATCH_G(float4, true, true); else DISPATCH_G(float4, false, true); }
        else       { if (acc) DISPATCH_G(float4, true, false); else DISPATCH_G(float4, false, false); }
    } else {
        if (multi) { if (acc) DISPATCH_G(float, true, true); else DISPATCH_G(float, false, true); }
        else       { if (acc) DISPATCH_G(float, true, false); else DISPATCH_G(float, false, false); }
    }
#undef DISPATCH_G
#undef LAUNCH_GA
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
    return ARROW_OK;
}

int arrow_gather_rows(arrow_ctx *ctx, int dst_buf, int src_buf, int map, int flags) {
    CHECK_CTX(ctx);
    DenseBuf *D = get_dense(ctx, dst_buf), *S = get_dense(ctx, src_buf);
    IdxMap *m = get_map(ctx, map);
    if (!D || !S) return fail(ctx, ARROW_ERR_HANDLE, "bad dense handle (dst=%d src=%d)", dst_buf, src_buf);
    if (!m) return fail(ctx, ARROW_ERR_HANDLE, "bad map handle %d", map);
    if (D->k != S->k) return fail(ctx, ARROW_ERR_ARG, "feature width mismatch %d vs %d", D->k, S->k);
    if (D->dtype != S->dtype) return fail(ctx, ARROW_ERR_ARG, "dtype mismatch: destination %s, source %s", dtype_name(D->dtype), dtype_name(S->dtype));
    REFUSE_I32(ctx, D, "arrow_gather_rows");
    if (D->dtype == ARROW_B1 && (flags & ARROW_ACCUMULATE))
        return fail(ctx, ARROW_ERR_ARG, "arrow_gather_rows: bits do not accumulate (arrow_gather_rows_sr with ARROW_SR_OR_AND ORs them)");
    if (D->p == S->p) return fail(ctx, ARROW_ERR_ARG, "gather source and destination must not alias");
    if (m->n > D->rows) return fail(ctx, ARROW_ERR_ARG, "map has %lld entries, destination has %lld rows", (long long)m->n, (long long)D->rows);
    if (m->limit > S->rows) return fail(ctx, ARROW_ERR_ARG, "map reaches row %lld, source has %lld rows", (long long)m->limit, (long long)S->rows);
    MultiSrc ms;
    memset(&ms, 0, sizeof ms);
    return gather_common(ctx, D, S->p, ms, false, m, (flags & ARROW_ACCUMULATE) != 0);
}

// ---- semirings ------------------------------------------------------------------------------------
int arrow_spmm_sr(arrow_ctx *ctx, int csr, int x_buf, int c_buf, int add_buf, int add_map, int semiring) {
    CHECK_CTX(ctx);
    if (semiring == ARROW_SR_PLUS_TIMES) {
        if (add_buf < 0 && add_map < 0) return arrow_spmm(ctx, csr, x_buf, c_buf, -1, 0, ARROW_VARIANT_AUTO);
        return arrow_spmm_add(ctx, csr, x_buf, c_buf, add_buf, add_map, ARROW_VARIANT_AUTO);
    }
    if (!fp32_semiring(semiring) && semiring != ARROW_SR_OR_AND) return fail(ctx, ARROW_ERR_ARG, "unknown semiring %d", semiring);
    CHECK_POISON(ctx);
    Csr *A = get_csr(ctx, csr);
    DenseBuf *X = get_dense(ctx, x_buf);
    DenseBuf *C = get_dense(ctx, c_buf);
    if (!A) return fail(ctx, ARROW_ERR_HANDLE, "bad csr handle %d", csr);
    if (!X || !C) return fail(ctx, ARROW_ERR_HANDLE, "bad dense handle (x=%d c=%d)", x_buf, c_buf);
    // (or, and) reads the block's structure only: its operands are bit tiles whatever the block's value type
    const int op_dtype = semiring == ARROW_SR_OR_AND ? ARROW_B1 : A->dtype;
    if (semiring == ARROW_SR_OR_AND && (X->dtype != ARROW_B1 || C->dtype != ARROW_B1))
        return fail(ctx, ARROW_ERR_ARG, "(or, and) runs on bit tiles: X is %s, C is %s", dtype_name(X->dtype), dtype_name(C->dtype));
    if (X->dtype != op_dtype || C->dtype != op_dtype)
        return fail(ctx, ARROW_ERR_ARG, "mixed precision: the block is %s, X is %s, C is %s", dtype_name(A->dtype),
                    dtype_name(X->dtype), dtype_name(C->dtype));
    if (X->k != C->k) return fail(ctx, ARROW_ERR_ARG, "X has %d feature columns, C has %d", X->k, C->k);
    if (X->p == C->p) return fail(ctx, ARROW_ERR_ARG, "X and C must not alias");
    if (X->rows < A->n_cols) return fail(ctx, ARROW_ERR_ARG, "X has %lld rows, block has %lld columns", (long long)X->rows, (long long)A->n_cols);
    if (C->rows < A->n_rows) return fail(ctx, ARROW_ERR_ARG, "C has %lld rows, block has %lld rows", (long long)C->rows, (long long)A->n_rows);
    const int k = X->k;
    SpmmArgs a;
    memset(&a, 0, sizeof a);
    if (add_buf >= 0 || add_map >= 0) {
        DenseBuf *S = get_dense(ctx, add_buf);
        IdxMap *am = get_map(ctx, add_map);
        if (!S || !am) return fail(ctx, ARROW_ERR_HANDLE, "bad addend handles (buf=%d map=%d)", add_buf, add_map);
        if (S->k != k) return fail(ctx, ARROW_ERR_ARG, "addend has %d feature columns, expected %d", S->k, k);
        if (S->dtype != op_dtype) return fail(ctx, ARROW_ERR_ARG, "mixed precision: the operands are %s, the addend is %s", dtype_name(op_dtype), dtype_name(S->dtype));
        if (am->n < A->n_rows) return fail(ctx, ARROW_ERR_ARG, "addend map has %lld entries, block has %lld rows", (long long)am->n, (long long)A->n_rows);
        if (am->limit > S->rows) return fail(ctx, ARROW_ERR_ARG, "addend map reaches row %lld, addend tile has %lld rows", (long long)am->limit, (long long)S->rows);
        if (S->p == C->p) return fail(ctx, ARROW_ERR_ARG, "addend and C must not alias");
        a.add_src = S->p;
        a.add_map = am->p;
    }
    if (semiring == ARROW_SR_OR_AND) {
        if (k > BITS_MAX_K) return fail(ctx, ARROW_ERR_UNSUPPORTED, "(or, and) covers k <= %d columns, X has %d", BITS_MAX_K, k);
        if (A->n_rows == 0) return ARROW_OK;
        a.indptr = A->indptr;
        a.indices = A->indices;
        a.X = X->p;
        a.C = C->p;
        a.n_rows = A->n_rows;
        a.k = bit_row_words(k);                   // the bit kernels count in words
        a.k4 = a.k / 4;
        a.long_threshold = A->long_threshold;
        return spmm_bits(ctx, A, a);
    }
    if (A->dtype != ARROW_F32) return fail(ctx, ARROW_ERR_UNSUPPORTED, "the (min, +) / (max, +) / (max, min) / (min, max) semirings are float32 only");
    if (A->n_rows == 0) return ARROW_OK;
    a.indptr = A->indptr;
    a.indices = A->indices;
    a.vals = A->vals;
    a.X = X->p;
    a.C = C->p;
    a.n_rows = A->n_rows;
    a.k = k;
    a.k4 = k / 4;
    a.long_threshold = A->long_threshold;
    if (semiring == ARROW_SR_MIN_PLUS) return spmm_sr<SrMinPlus>(ctx, A, a);
    if (semiring == ARROW_SR_MAX_PLUS) return spmm_sr<SrMaxPlus>(ctx, A, a);
    if (semiring == ARROW_SR_MAX_MIN) return spmm_sr<SrMaxMin>(ctx, A, a);
    return spmm_sr<SrMinMax>(ctx, A, a);
}

int arrow_gather_rows_sr(arrow_ctx *ctx, int dst_buf, int src_buf, int map, int semiring) {
    CHECK_CTX(ctx);
    if (semiring == ARROW_SR_PLUS_TIMES) return arrow_gather_rows(ctx, dst_buf, src_buf, map, ARROW_ACCUMULATE);
    if (!fp32_semiring(semiring) && semiring != ARROW_SR_OR_AND) return fail(ctx, ARROW_ERR_ARG, "unknown semiring %d", semiring);
    CHECK_POISON(ctx);
    DenseBuf *D = get_dense(ctx, dst_buf), *S = get_dense(ctx, src_buf);
    IdxMap *m = get_map(ctx, map);
    if (!D || !S) return fail(ctx, ARROW_ERR_HANDLE, "bad dense handle (dst=%d src=%d)", dst_buf, src_buf);
    if (!m) return fail(ctx, ARROW_ERR_HANDLE, "bad map handle %d", map);
    if (D->k != S->k) return fail(ctx, ARROW_ERR_ARG, "feature width mismatch %d vs %d", D->k, S->k);
    if (D->dtype != S->dtype) return fail(ctx, ARROW_ERR_ARG, "dtype mismatch: destination %s, source %s", dtype_name(D->dtype), dtype_name(S->dtype));
    REFUSE_I32(ctx, D, "arrow_gather_rows_sr");
    if (D->p == S->p) return fail(ctx, ARROW_ERR_ARG, "gather source and destination must not alias");
    if (m->n > D->rows) return fail(ctx, ARROW_ERR_ARG, "map has %lld entries, destination has %lld rows", (long long)m->n, (long long)D->rows);
    if (m->limit > S->rows) return fail(ctx, ARROW_ERR_ARG, "map reaches row %lld, source has %lld rows", (long long)m->limit, (long long)S->rows);
    if ((semiring == ARROW_SR_OR_AND) != (D->dtype == ARROW_B1))
        return fail(ctx, ARROW_ERR_ARG, "(or, and) runs on bit tiles and only there: semiring %d, tiles of %s", semiring, dtype_name(D->dtype));
    if (semiring == ARROW_SR_OR_AND) return gather_rows_or(ctx, D, S, m);
    if (D->dtype != ARROW_F32) return fail(ctx, ARROW_ERR_UNSUPPORTED, "the (min, +) / (max, +) / (max, min) / (min, max) semirings are float32 only");
    if (semiring == ARROW_SR_MIN_PLUS) return gather_rows_sr<SrMinPlus>(ctx, D, S, m);
    if (semiring == ARROW_SR_MAX_PLUS) return gather_rows_sr<SrMaxPlus>(ctx, D, S, m);
    if (semiring == ARROW_SR_MAX_MIN) return gather_rows_sr<SrMaxMin>(ctx, D, S, m);
    return gather_rows_sr<SrMinMax>(ctx, D, S, m);
}

// ---- predecessors ---------------------------------------------------------------------------------
int arrow_spmm_sr_witness(arrow_ctx *ctx, int csr, int x_buf, int row_labels, int val_out, int lab_out, int add_val,
                          int add_lab, int add_map, int dist_buf, int semiring) {
    CHECK_CTX(ctx);
    if (semiring == ARROW_SR_PLUS_TIMES)
        return fail(ctx, ARROW_ERR_UNSUPPORTED, "predecessors exist in the (min, +) / (max, +) semirings only");
    if (semiring == ARROW_SR_MAX_MIN || semiring == ARROW_SR_MIN_MAX)
        return fail(ctx, ARROW_ERR_UNSUPPORTED, "the witness rule makes cycles in the bottleneck semirings: use arrow_sr_tree_parents");
    if (semiring != ARROW_SR_MIN_PLUS && semiring != ARROW_SR_MAX_PLUS)
        return fail(ctx, ARROW_ERR_ARG, "unknown semiring %d", semiring);
    CHECK_POISON(ctx);
    Csr *A = get_csr(ctx, csr);
    DenseBuf *X = get_dense(ctx, x_buf);
    DenseBuf *L = get_dense(ctx, lab_out);
    DenseBuf *V = val_out >= 0 ? get_dense(ctx, val_out) : nullptr;
    DenseBuf *D = dist_buf >= 0 ? get_dense(ctx, dist_buf) : nullptr;
    if (!A) return fail(ctx, ARROW_ERR_HANDLE, "bad csr handle %d", csr);
    if (!X || !L) return fail(ctx, ARROW_ERR_HANDLE, "bad dense handle (x=%d lab_out=%d)", x_buf, lab_out);
    if (val_out >= 0 && !V) return fail(ctx, ARROW_ERR_HANDLE, "bad dense handle (val_out=%d)", val_out);
    if (dist_buf >= 0 && !D) return fail(ctx, ARROW_ERR_HANDLE, "bad dense handle (dist=%d)", dist_buf);
    if (!V && !D) return fail(ctx, ARROW_ERR_ARG, "the pair epilogue (dist_buf < 0) needs a value tile");
    if (X->dtype != A->dtype || (V && V->dtype != A->dtype) || (D && D->dtype != A->dtype))
        return fail(ctx, ARROW_ERR_ARG, "mixed precision: the block is %s, X is %s, val_out is %s, dist is %s", dtype_name(A->dtype),
                    dtype_name(X->dtype), V ? dtype_name(V->dtype) : "-", D ? dtype_name(D->dtype) : "-");
    if (L->dtype != ARROW_I32) return fail(ctx, ARROW_ERR_ARG, "lab_out is %s, labels are int32", dtype_name(L->dtype));
    const int k = X->k;
    if (L->k != k || (V && V->k != k) || (D && D->k != k))
        return fail(ctx, ARROW_ERR_ARG, "X has %d feature columns, lab_out %d, val_out %d, dist %d", k, L->k, V ? V->k : -1, D ? D->k : -1);
    if (X->rows < A->n_cols) return fail(ctx, ARROW_ERR_ARG, "X has %lld rows, block has %lld columns", (long long)X->rows, (long long)A->n_cols);
    if (L->rows < A->n_rows || (V && V->rows < A->n_rows) || (D && D->rows < A->n_rows))
        return fail(ctx, ARROW_ERR_ARG, "an output or dist tile has fewer rows than the block (%lld)", (long long)A->n_rows);
    IdxMap *self = nullptr;
    if (row_labels >= 0) {
        self = get_map(ctx, row_labels);
        if (!self) return fail(ctx, ARROW_ERR_HANDLE, "bad row label map %d", row_labels);
        if (self->n < A->n_rows) return fail(ctx, ARROW_ERR_ARG, "row label map has %lld entries, block has %lld rows", (long long)self->n, (long long)A->n_rows);
    }
    DenseBuf *SV = nullptr, *SL = nullptr;
    IdxMap *am = nullptr;
    if (add_val >= 0 || add_lab >= 0 || add_map >= 0) {
        SV = get_dense(ctx, add_val);
        SL = get_dense(ctx, add_lab);
        am = get_map(ctx, add_map);
        if (!SV || !SL || !am) return fail(ctx, ARROW_ERR_HANDLE, "bad addend handles (val=%d lab=%d map=%d)", add_val, add_lab, add_map);
        if (SV->dtype != A->dtype) return fail(ctx, ARROW_ERR_ARG, "mixed precision: the block is %s, the addend is %s", dtype_name(A->dtype), dtype_name(SV->dtype));
        if (SL->dtype != ARROW_I32) return fail(ctx, ARROW_ERR_ARG, "the addend's labels are %s, labels are int32", dtype_name(SL->dtype));
        if (SV->k != k || SL->k != k) return fail(ctx, ARROW_ERR_ARG, "addend has %d / %d feature columns, expected %d", SV->k, SL->k, k);
        if (am->n < A->n_rows) return fail(ctx, ARROW_ERR_ARG, "addend map has %lld entries, block has %lld rows", (long long)am->n, (long long)A->n_rows);
        if (am->limit > SV->rows || am->limit > SL->rows)
            return fail(ctx, ARROW_ERR_ARG, "addend map reaches row %lld, addend tiles have %lld / %lld rows", (long long)am->limit, (long long)SV->rows, (long long)SL->rows);
    }
    // the outputs alias nothing the launch reads, nor each other
    const void *outs[2] = {V ? (const void *)V->p : nullptr, (const void *)L->p};
    const void *ins[4] = {X->p, SV ? (const void *)SV->p : nullptr, SL ? (const void *)SL->p : nullptr, D ? (const void *)D->p : nullptr};
    if (outs[0] == outs[1]) return fail(ctx, ARROW_ERR_ARG, "val_out and lab_out must not alias");
    for (const void *o : outs)
        for (const void *i : ins)
            if (o != nullptr && o == i) return fail(ctx, ARROW_ERR_ARG, "an output tile aliases an input tile");
    if (A->dtype != ARROW_F32) return fail(ctx, ARROW_ERR_UNSUPPORTED, "predecessors of the (min, +) / (max, +) semirings are float32 only");
    if (A->n_rows == 0) return ARROW_OK;
    WitArgs w;
    memset(&w, 0, sizeof w);
    SpmmArgs &a = w.t.a;
    a.indptr = A->indptr;
    a.indices = A->indices;
    a.vals = A->vals;
    a.X = X->p;
    a.C = V ? V->p : nullptr;
    a.n_rows = A->n_rows;
    a.k = k;
    a.k4 = k / 4;
    a.long_threshold = A->long_threshold;
    a.add_src = SV ? SV->p : nullptr;
    a.add_map = am ? am->p : nullptr;
    w.self = self ? self->p : nullptr;
    w.lab_out = reinterpret_cast<int *>(L->p);
    w.add_lab = SL ? reinterpret_cast<const int *>(SL->p) : nullptr;
    w.dist = D ? D->p : nullptr;
    if (semiring == ARROW_SR_MIN_PLUS) return spmm_wit<SrMinPlus>(ctx, A, w, true);
    return spmm_wit<SrMaxPlus>(ctx, A, w, false);
}

int arrow_dense_count_diff(arrow_ctx *ctx, int a, int b, int64_t *rows_changed) {
    CHECK_CTX(ctx);
    CHECK_POISON(ctx);
    DenseBuf *A = get_dense(ctx, a), *B = get_dense(ctx, b);
    if (!A || !B) return fail(ctx, ARROW_ERR_HANDLE, "bad dense handle (a=%d b=%d)", a, b);
    if (!rows_changed) return fail(ctx, ARROW_ERR_ARG, "null rows_changed");
    REFUSE_I32(ctx, A, "arrow_dense_count_diff");
    REFUSE_I32(ctx, B, "arrow_dense_count_diff");
    if (A->rows != B->rows || A->k != B->k || A->dtype != B->dtype)
        return fail(ctx, ARROW_ERR_ARG, "tiles differ in shape or type: %lld x %d %s vs %lld x %d %s", (long long)A->rows, A->k,
                    dtype_name(A->dtype), (long long)B->rows, B->k, dtype_name(B->dtype));
    *rows_changed = 0;
    if (A->rows == 0 || A->k == 0) return ARROW_OK;
    cudaStream_t stream = cur_stream(ctx);
    DevTmp cnt;
    CUDA_TRY(ctx, cudaMalloc(&cnt.p, sizeof(unsigned long long)));
    CUDA_TRY(ctx, cudaMemsetAsync(cnt.p, 0, sizeof(unsigned long long), stream));
    const int grid = (int)std::min<long long>((A->rows + 7) / 8, (long long)ctx->sm_count * 8);
    unsigned long long *c = reinterpret_cast<unsigned long long *>(cnt.p);
    if (A->dtype == ARROW_B1)
        k_count_diff_bits<<<grid, 256, 0, stream>>>(reinterpret_cast<const unsigned int *>(A->p), reinterpret_cast<const unsigned int *>(B->p),
                                                    A->rows, A->k, bit_row_words(A->k), c);
    else if (A->dtype == ARROW_F64)
        k_count_diff<double><<<grid, 256, 0, stream>>>(reinterpret_cast<const double *>(A->p), reinterpret_cast<const double *>(B->p), A->rows, A->k, c);
    else
        k_count_diff<float><<<grid, 256, 0, stream>>>(A->p, B->p, A->rows, A->k, c);
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
    unsigned long long h = 0;
    CUDA_TRY(ctx, cudaMemcpyAsync(&h, cnt.p, sizeof h, cudaMemcpyDeviceToHost, stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(stream));
    *rows_changed = (int64_t)h;
    return ARROW_OK;
}

int arrow_dense_count_diff_bits(arrow_ctx *ctx, int a, int b, int64_t *rows_changed) {
    CHECK_CTX(ctx);
    CHECK_POISON(ctx);
    DenseBuf *A = get_dense(ctx, a), *B = get_dense(ctx, b);
    if (!A || !B) return fail(ctx, ARROW_ERR_HANDLE, "bad dense handle (a=%d b=%d)", a, b);
    if (!rows_changed) return fail(ctx, ARROW_ERR_ARG, "null rows_changed");
    if (A->dtype != ARROW_F32 || B->dtype != ARROW_F32 || A->rows != B->rows || A->k != B->k)
        return fail(ctx, ARROW_ERR_ARG, "two fp32 tiles of one shape: %lld x %d %s vs %lld x %d %s", (long long)A->rows, A->k,
                    dtype_name(A->dtype), (long long)B->rows, B->k, dtype_name(B->dtype));
    *rows_changed = 0;
    if (A->rows == 0 || A->k == 0) return ARROW_OK;
    cudaStream_t stream = cur_stream(ctx);
    DevTmp cnt;
    CUDA_TRY(ctx, cudaMalloc(&cnt.p, sizeof(unsigned long long)));
    CUDA_TRY(ctx, cudaMemsetAsync(cnt.p, 0, sizeof(unsigned long long), stream));
    const int grid = (int)std::min<long long>((A->rows + 7) / 8, (long long)ctx->sm_count * 8);
    // a row of k fp32 elements read as k words of 32 bits each: the bit-tile comparison over all 32 k bits
    k_count_diff_bits<<<grid, 256, 0, stream>>>(reinterpret_cast<const unsigned int *>(A->p), reinterpret_cast<const unsigned int *>(B->p),
                                                A->rows, 32 * A->k, A->k, reinterpret_cast<unsigned long long *>(cnt.p));
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
    unsigned long long h = 0;
    CUDA_TRY(ctx, cudaMemcpyAsync(&h, cnt.p, sizeof h, cudaMemcpyDeviceToHost, stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(stream));
    *rows_changed = (int64_t)h;
    return ARROW_OK;
}

int arrow_bits_mark_new(arrow_ctx *ctx, int new_buf, int old_buf, int dist_buf, int level, int64_t *n_new) {
    CHECK_CTX(ctx);
    CHECK_POISON(ctx);
    DenseBuf *N = get_dense(ctx, new_buf), *O = get_dense(ctx, old_buf), *D = get_dense(ctx, dist_buf);
    if (!N || !O || !D) return fail(ctx, ARROW_ERR_HANDLE, "bad dense handle (new=%d old=%d dist=%d)", new_buf, old_buf, dist_buf);
    if (!n_new) return fail(ctx, ARROW_ERR_ARG, "null n_new");
    if (N->dtype != ARROW_B1 || O->dtype != ARROW_B1 || D->dtype != ARROW_I32)
        return fail(ctx, ARROW_ERR_ARG, "new / old are bit tiles and dist an int32 tile: got %s / %s / %s", dtype_name(N->dtype),
                    dtype_name(O->dtype), dtype_name(D->dtype));
    if (N->rows != O->rows || N->k != O->k || D->rows != N->rows || D->k != N->k)
        return fail(ctx, ARROW_ERR_ARG, "tiles differ in shape: new %lld x %d, old %lld x %d, dist %lld x %d", (long long)N->rows, N->k,
                    (long long)O->rows, O->k, (long long)D->rows, D->k);
    *n_new = 0;
    if (N->rows == 0) return ARROW_OK;
    cudaStream_t stream = cur_stream(ctx);
    DevTmp cnt;
    CUDA_TRY(ctx, cudaMalloc(&cnt.p, sizeof(unsigned long long)));
    CUDA_TRY(ctx, cudaMemsetAsync(cnt.p, 0, sizeof(unsigned long long), stream));
    const long long items = N->rows * (long long)((N->k + 31) / 32);
    const int grid = (int)std::max<long long>(1, std::min<long long>((items + 255) / 256, (long long)ctx->sm_count * 8));
    k_bits_mark_new<<<grid, 256, 0, stream>>>(reinterpret_cast<const unsigned int *>(N->p), reinterpret_cast<const unsigned int *>(O->p),
                                              reinterpret_cast<int *>(D->p), N->rows, N->k, bit_row_words(N->k), level,
                                              reinterpret_cast<unsigned long long *>(cnt.p));
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
    unsigned long long h = 0;
    CUDA_TRY(ctx, cudaMemcpyAsync(&h, cnt.p, sizeof h, cudaMemcpyDeviceToHost, stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(stream));
    *n_new = (int64_t)h;
    return ARROW_OK;
}

namespace {
// arrow_adj_build (weighted false), arrow_adj_build_weighted, arrow_adj_build_in (incoming) and arrow_adj_build_loopfree
// (weighted and loop-free, either direction): one validation, one edge pass, one sort
int adj_build(arrow_ctx *ctx, int n_parts, const int *csrs, const int *maps, int64_t n_vertices, bool weighted, bool incoming,
              bool loopfree, int *adj_out) {
    const char *fn = loopfree ? "arrow_adj_build_loopfree" : weighted ? "arrow_adj_build_weighted"
                                                          : incoming ? "arrow_adj_build_in" : "arrow_adj_build";
    if (!adj_out || n_parts < 0 || (n_parts > 0 && (!csrs || !maps)) || n_vertices < 0)
        return fail(ctx, ARROW_ERR_ARG, "bad arguments (n_parts=%d, n_vertices=%lld)", n_parts, (long long)n_vertices);
    if (n_vertices > 2147483646LL) return fail(ctx, ARROW_ERR_RANGE, "%lld vertices exceed the int32 device layout", (long long)n_vertices);
    if (ctx->capturing) return fail(ctx, ARROW_ERR_UNSUPPORTED, "%s allocates and synchronises: not during graph capture", fn);
    std::vector<std::pair<const Csr *, const IdxMap *>> blocks;
    if (const int rc = operator_parts(ctx, n_parts, csrs, maps, n_vertices, blocks)) return rc;
    std::vector<AdjPart> parts;
    std::vector<const float *> weights;                       // the entries' values of each part (weighted only)
    for (int i = 0; i < n_parts; ++i) {
        const Csr *c = blocks[i].first;
        const IdxMap *m = blocks[i].second;
        if (weighted && c->dtype != ARROW_F32)
            return fail(ctx, ARROW_ERR_UNSUPPORTED, "part %d: %s carries fp32 weights, the block is %s", i, fn,
                        dtype_name(c->dtype));
        if (weighted && c->nnz > 0 && !c->vals)
            return fail(ctx, ARROW_ERR_ARG, "part %d: the block has no values to carry as weights", i);
        if (c->nnz > 0) {
            parts.push_back(AdjPart{c->indptr, c->indices, m ? m->p : nullptr, (long long)c->nnz, (int)c->n_rows});
            weights.push_back(c->vals);
        }
    }
    cudaStream_t s = ctx->stream;
    auto edge_grid = [&](long long nnz) { return (int)std::min<long long>((nnz + 255) / 256, (long long)ctx->sm_count * 8); };
    DevTmp cnt;
    unsigned long long m = 0;
    CUDA_TRY(ctx, cudaMalloc(&cnt.p, sizeof(unsigned long long)));
    unsigned long long *count = reinterpret_cast<unsigned long long *>(cnt.p);
    CUDA_TRY(ctx, cudaMemsetAsync(count, 0, sizeof m, s));
    for (const AdjPart &p : parts) {
        if (loopfree && incoming) k_adj_edges<true, true, false><<<edge_grid(p.nnz), 256, 0, s>>>(p, count, nullptr);
        else if (loopfree) k_adj_edges<true, false, false><<<edge_grid(p.nnz), 256, 0, s>>>(p, count, nullptr);
        else if (weighted) k_adj_edges<true><<<edge_grid(p.nnz), 256, 0, s>>>(p, count, nullptr);
        else if (incoming) k_adj_edges<false, true><<<edge_grid(p.nnz), 256, 0, s>>>(p, count, nullptr);
        else k_adj_edges<false><<<edge_grid(p.nnz), 256, 0, s>>>(p, count, nullptr);
        ctx->launches++;
    }
    CUDA_TRY(ctx, cudaGetLastError());
    CUDA_TRY(ctx, cudaMemcpyAsync(&m, count, sizeof m, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(ctx, cudaStreamSynchronize(s));
    if (m > 2147483647ULL) return fail(ctx, ARROW_ERR_RANGE, "%llu edges exceed the int32 device layout", m);

    Adj a;
    a.n = n_vertices;
    a.m = (int64_t)m;
    a.weighted = weighted;
    a.incoming = incoming;
    a.loopfree = loopfree;
    cudaError_t e = cudaMalloc(&a.indptr, (size_t)(n_vertices + 1) * 4);
    if (e == cudaSuccess) e = cudaMalloc(&a.indices, (size_t)std::max<unsigned long long>(m, 1) * 4);
    if (e == cudaSuccess && weighted) e = cudaMalloc(&a.values, (size_t)std::max<unsigned long long>(m, 1) * 4);
    if (e == cudaSuccess && !incoming) e = cudaMalloc(&a.front_rows, (size_t)std::max<int64_t>(n_vertices, 1) * 4);
    if (e == cudaSuccess && !incoming) e = cudaMalloc(&a.front_off, (size_t)std::max<int64_t>(n_vertices, 1) * 4);
    // build scratch: 16 bytes per edge (24 weighted) and the sort's temporary storage
    DevTmp keys, alt, wk, walt, temp;
    const unsigned long long *sorted = nullptr;
    if (e == cudaSuccess && m > 0) {
        e = cudaMalloc(&keys.p, (size_t)m * 8);
        if (e == cudaSuccess) e = cudaMalloc(&alt.p, (size_t)m * 8);
        if (e == cudaSuccess && weighted) e = cudaMalloc(&wk.p, (size_t)m * 4);
        if (e == cudaSuccess && weighted) e = cudaMalloc(&walt.p, (size_t)m * 4);
        if (e == cudaSuccess) e = cudaMemsetAsync(count, 0, sizeof m, s);
        if (e == cudaSuccess) {
            unsigned long long *kp = reinterpret_cast<unsigned long long *>(keys.p);
            for (size_t i = 0; i < parts.size(); ++i) {
                const AdjPart &p = parts[i];
                float *w_out = reinterpret_cast<float *>(wk.p);
                if (loopfree && incoming)
                    k_adj_edges<true, true, false><<<edge_grid(p.nnz), 256, 0, s>>>(p, count, kp, weights[i], w_out);
                else if (loopfree)
                    k_adj_edges<true, false, false><<<edge_grid(p.nnz), 256, 0, s>>>(p, count, kp, weights[i], w_out);
                else if (weighted)
                    k_adj_edges<true><<<edge_grid(p.nnz), 256, 0, s>>>(p, count, kp, weights[i], w_out);
                else if (incoming)
                    k_adj_edges<false, true><<<edge_grid(p.nnz), 256, 0, s>>>(p, count, kp);
                else
                    k_adj_edges<false><<<edge_grid(p.nnz), 256, 0, s>>>(p, count, kp);
                ctx->launches++;
            }
            e = cudaGetLastError();
        }
        int end_bit = 33;                                     // keys are (u << 32) | v with u < n_vertices (in: v, u)
        while (end_bit < 64 && (1LL << (end_bit - 32)) < n_vertices) ++end_bit;
        cub::DoubleBuffer<unsigned long long> db(reinterpret_cast<unsigned long long *>(keys.p),
                                                 reinterpret_cast<unsigned long long *>(alt.p));
        cub::DoubleBuffer<float> dw(reinterpret_cast<float *>(wk.p), reinterpret_cast<float *>(walt.p));
        size_t temp_bytes = 0;
        if (weighted) {                                       // duplicates of (u, v) may leave in any order
            if (e == cudaSuccess) e = cub::DeviceRadixSort::SortPairs(nullptr, temp_bytes, db, dw, (int)m, 0, end_bit, s);
            if (e == cudaSuccess) e = cudaMalloc(&temp.p, std::max<size_t>(temp_bytes, 1));
            if (e == cudaSuccess) e = cub::DeviceRadixSort::SortPairs(temp.p, temp_bytes, db, dw, (int)m, 0, end_bit, s);
            if (e == cudaSuccess) e = cudaMemcpyAsync(a.values, dw.Current(), (size_t)m * 4, cudaMemcpyDeviceToDevice, s);
        } else {
            if (e == cudaSuccess) e = cub::DeviceRadixSort::SortKeys(nullptr, temp_bytes, db, (int)m, 0, end_bit, s);
            if (e == cudaSuccess) e = cudaMalloc(&temp.p, std::max<size_t>(temp_bytes, 1));
            if (e == cudaSuccess) e = cub::DeviceRadixSort::SortKeys(temp.p, temp_bytes, db, (int)m, 0, end_bit, s);
        }
        sorted = db.Current();
    }
    if (e == cudaSuccess) {
        const long long work = std::max<long long>((long long)m, n_vertices + 1);
        k_adj_csr<<<edge_grid(work), 256, 0, s>>>(sorted, (long long)m, n_vertices, a.indptr, a.indices);
        ctx->launches++;
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e == cudaSuccess && (incoming || loopfree)) e = build_segs(a);   // the segments of the long lists
    if (e != cudaSuccess) {
        cudaGetLastError();
        adj_release(a);
        return fail(ctx, e == cudaErrorMemoryAllocation ? ARROW_ERR_NOMEM : ARROW_ERR_CUDA, "adjacency build failed: %s",
                    cudaGetErrorString(e));
    }
    a.live = true;
    const int h = new_slot(ctx->adjs);
    ctx->adjs[h] = a;
    *adj_out = h;
    return ARROW_OK;
}
}  // namespace

int arrow_adj_build(arrow_ctx *ctx, int n_parts, const int *csrs, const int *maps, int64_t n_vertices, int *adj_out) {
    CHECK_CTX(ctx);
    CHECK_POISON(ctx);
    return adj_build(ctx, n_parts, csrs, maps, n_vertices, false, false, false, adj_out);
}

int arrow_adj_build_in(arrow_ctx *ctx, int n_parts, const int *csrs, const int *maps, int64_t n_vertices, int *adj_out) {
    CHECK_CTX(ctx);
    CHECK_POISON(ctx);
    return adj_build(ctx, n_parts, csrs, maps, n_vertices, false, true, false, adj_out);
}

int arrow_adj_build_weighted(arrow_ctx *ctx, int n_parts, const int *csrs, const int *maps, int64_t n_vertices,
                             int *adj_out) {
    CHECK_CTX(ctx);
    CHECK_POISON(ctx);
    return adj_build(ctx, n_parts, csrs, maps, n_vertices, true, false, false, adj_out);
}

int arrow_adj_build_loopfree(arrow_ctx *ctx, int n_parts, const int *csrs, const int *maps, int64_t n_vertices, int incoming,
                             int *adj_out) {
    CHECK_CTX(ctx);
    CHECK_POISON(ctx);
    return adj_build(ctx, n_parts, csrs, maps, n_vertices, true, incoming != 0, true, adj_out);
}

int arrow_adj_values_d2h(arrow_ctx *ctx, int adj, float *values) {
    CHECK_CTX(ctx);
    const Adj *a = get_adj(ctx, adj);
    if (!a) return fail(ctx, ARROW_ERR_HANDLE, "bad adjacency handle %d", adj);
    if (a->incoming) return fail(ctx, ARROW_ERR_ARG, "adjacency %d is an in-adjacency (arrow_adj_build_in)", adj);
    if (!a->weighted) return fail(ctx, ARROW_ERR_ARG, "the adjacency carries no weights (built by arrow_adj_build)");
    if (a->m > 0 && !values) return fail(ctx, ARROW_ERR_ARG, "null host buffer");
    if (a->m > 0) CUDA_TRY(ctx, cudaMemcpyAsync(values, a->values, (size_t)a->m * 4, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    return ARROW_OK;
}

int arrow_adj_free(arrow_ctx *ctx, int adj) {
    CHECK_CTX(ctx);
    Adj *a = get_adj(ctx, adj);
    if (!a) return fail(ctx, ARROW_ERR_HANDLE, "bad adjacency handle %d", adj);
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    adj_release(*a);
    return ARROW_OK;
}

int arrow_adj_info(arrow_ctx *ctx, int adj, int64_t *n_vertices, int64_t *n_edges) {
    CHECK_CTX(ctx);
    const Adj *a = get_adj(ctx, adj);
    if (!a) return fail(ctx, ARROW_ERR_HANDLE, "bad adjacency handle %d", adj);
    if (n_vertices) *n_vertices = a->n;
    if (n_edges) *n_edges = a->m;
    return ARROW_OK;
}

int arrow_adj_d2h(arrow_ctx *ctx, int adj, int32_t *indptr, int32_t *indices) {
    CHECK_CTX(ctx);
    const Adj *a = get_adj(ctx, adj);
    if (!a) return fail(ctx, ARROW_ERR_HANDLE, "bad adjacency handle %d", adj);
    if (!indptr || (a->m > 0 && !indices)) return fail(ctx, ARROW_ERR_ARG, "null host buffer");
    CUDA_TRY(ctx, cudaMemcpyAsync(indptr, a->indptr, (size_t)(a->n + 1) * 4, cudaMemcpyDeviceToHost, ctx->stream));
    if (a->m > 0) CUDA_TRY(ctx, cudaMemcpyAsync(indices, a->indices, (size_t)a->m * 4, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    return ARROW_OK;
}

int arrow_bits_mark_frontier(arrow_ctx *ctx, int adj, int new_buf, int old_buf, int dist_buf, int level, int64_t *n_new,
                             int64_t *frontier_rows, int64_t *frontier_edges) {
    CHECK_CTX(ctx);
    CHECK_POISON(ctx);
    Adj *a = get_adj(ctx, adj);
    if (!a) return fail(ctx, ARROW_ERR_HANDLE, "bad adjacency handle %d", adj);
    if (a->incoming) return fail(ctx, ARROW_ERR_ARG, "adjacency %d is an in-adjacency (arrow_adj_build_in)", adj);
    DenseBuf *N = get_dense(ctx, new_buf), *O = get_dense(ctx, old_buf), *D = get_dense(ctx, dist_buf);
    if (!N || !O || !D) return fail(ctx, ARROW_ERR_HANDLE, "bad dense handle (new=%d old=%d dist=%d)", new_buf, old_buf, dist_buf);
    if (!n_new || !frontier_rows || !frontier_edges) return fail(ctx, ARROW_ERR_ARG, "null output");
    if (N->dtype != ARROW_B1 || O->dtype != ARROW_B1 || D->dtype != ARROW_I32)
        return fail(ctx, ARROW_ERR_ARG, "new / old are bit tiles and dist an int32 tile: got %s / %s / %s", dtype_name(N->dtype),
                    dtype_name(O->dtype), dtype_name(D->dtype));
    if (N->rows != O->rows || N->k != O->k || D->rows != N->rows || D->k != N->k || N->rows != a->n)
        return fail(ctx, ARROW_ERR_ARG, "tiles differ in shape: new %lld x %d, old %lld x %d, dist %lld x %d, adjacency %lld rows",
                    (long long)N->rows, N->k, (long long)O->rows, O->k, (long long)D->rows, D->k, (long long)a->n);
    *n_new = *frontier_rows = *frontier_edges = 0;
    a->tag = -1;                                              // the record is rewritten below
    cudaStream_t stream = cur_stream(ctx);
    unsigned long long h[2] = {0, 0};                         // fresh bits, (frontier rows << 32) | frontier edges
    if (N->rows > 0) {
        DevTmp cnt;
        CUDA_TRY(ctx, cudaMalloc(&cnt.p, sizeof h));
        CUDA_TRY(ctx, cudaMemsetAsync(cnt.p, 0, sizeof h, stream));
        const int grid = (int)std::max<long long>(1, std::min<long long>((N->rows + MARK_THREADS - 1) / MARK_THREADS,
                                                                         (long long)ctx->sm_count * 8));
        k_bits_mark_frontier<<<grid, MARK_THREADS, 0, stream>>>(reinterpret_cast<const unsigned int *>(N->p),
                                                                reinterpret_cast<const unsigned int *>(O->p),
                                                                reinterpret_cast<int *>(D->p), N->rows, N->k, bit_row_words(N->k),
                                                                level, a->indptr, a->front_rows, a->front_off,
                                                                reinterpret_cast<unsigned long long *>(cnt.p));
        ctx->launches++;
        CUDA_TRY(ctx, cudaGetLastError());
        CUDA_TRY(ctx, cudaMemcpyAsync(h, cnt.p, sizeof h, cudaMemcpyDeviceToHost, stream));
        CUDA_TRY(ctx, cudaStreamSynchronize(stream));
    }
    a->n_front = (int64_t)(h[1] >> 32);
    a->front_edges = (int64_t)(h[1] & 0xffffffffULL);
    a->tag = new_buf;
    a->tag_p = N->p;
    a->tag_k = N->k;
    *n_new = (int64_t)h[0];
    *frontier_rows = a->n_front;
    *frontier_edges = a->front_edges;
    return ARROW_OK;
}

int arrow_bits_push_frontier(arrow_ctx *ctx, int adj, int x_buf, int out_buf) {
    CHECK_CTX(ctx);
    CHECK_POISON(ctx);
    const Adj *a = get_adj(ctx, adj);
    if (!a) return fail(ctx, ARROW_ERR_HANDLE, "bad adjacency handle %d", adj);
    if (a->incoming) return fail(ctx, ARROW_ERR_ARG, "adjacency %d is an in-adjacency (arrow_adj_build_in)", adj);
    DenseBuf *X = get_dense(ctx, x_buf), *O = get_dense(ctx, out_buf);
    if (!X || !O) return fail(ctx, ARROW_ERR_HANDLE, "bad dense handle (x=%d out=%d)", x_buf, out_buf);
    if (X->dtype != ARROW_B1 || O->dtype != ARROW_B1)
        return fail(ctx, ARROW_ERR_ARG, "x / out are bit tiles: got %s / %s", dtype_name(X->dtype), dtype_name(O->dtype));
    if (a->tag < 0) return fail(ctx, ARROW_ERR_ARG, "no frontier record: run arrow_bits_mark_frontier on the adjacency first");
    if (x_buf != a->tag || X->p != a->tag_p || X->k != a->tag_k)
        return fail(ctx, ARROW_ERR_ARG, "x (tile %d) is not the tile of the last arrow_bits_mark_frontier (tile %d)", x_buf, a->tag);
    if (x_buf == out_buf || X->p == O->p) return fail(ctx, ARROW_ERR_ARG, "out aliases x");
    if (X->rows != a->n || O->rows != X->rows || O->k != X->k)
        return fail(ctx, ARROW_ERR_ARG, "shape: x %lld x %d, out %lld x %d, adjacency %lld rows", (long long)X->rows, X->k,
                    (long long)O->rows, O->k, (long long)a->n);
    if (X->k > BITS_MAX_K) return fail(ctx, ARROW_ERR_UNSUPPORTED, "k=%d > %d", X->k, BITS_MAX_K);
    cudaStream_t stream = cur_stream(ctx);
    if (X->rows == 0) return ARROW_OK;
    CUDA_TRY(ctx, cudaMemcpyAsync(O->p, X->p, (size_t)X->rows * row_bytes(ARROW_B1, X->k), cudaMemcpyDeviceToDevice, stream));
    if (a->front_edges == 0) return ARROW_OK;
    const int words = bit_row_words(X->k);
    const int row_vecs = words == 1 ? 1 : words / 4;
    const int vecs = words == 1 ? 1 : ((X->k + 31) / 32 + 3) / 4;         // the vectors that hold columns < k
    const long long items = a->front_edges * vecs;
    const long long chunks = (items + (long long)PUSH_THREADS * PUSH_ITEMS - 1) / ((long long)PUSH_THREADS * PUSH_ITEMS);
    const int per_sm = ctx->spmm_ctas_per_sm > 0 ? std::min(ctx->spmm_ctas_per_sm, 8) : 8;
    const int sms = ctx->spmm_sm_limit > 0 ? std::min(ctx->sm_count, ctx->spmm_sm_limit) : ctx->sm_count;
    const int grid = (int)std::min<long long>(chunks, (long long)per_sm * sms);
    unsigned *out = reinterpret_cast<unsigned *>(O->p);
    if (words == 1)
        k_bits_push<unsigned><<<grid, PUSH_THREADS, 0, stream>>>(reinterpret_cast<const unsigned *>(X->p), out, a->indptr,
                                                                 a->indices, a->front_rows, a->front_off, (int)a->n_front,
                                                                 items, vecs, row_vecs);
    else
        k_bits_push<uint4><<<grid, PUSH_THREADS, 0, stream>>>(reinterpret_cast<const uint4 *>(X->p), out, a->indptr,
                                                              a->indices, a->front_rows, a->front_off, (int)a->n_front,
                                                              items, vecs, row_vecs);
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
    return ARROW_OK;
}

int arrow_bits_parents(arrow_ctx *ctx, int in_adj, int adj, int new_buf, int old_buf, int parent_buf, int64_t *edges_scanned) {
    CHECK_CTX(ctx);
    CHECK_POISON(ctx);
    const Adj *in = get_adj(ctx, in_adj), *a = get_adj(ctx, adj);
    if (!in || !a) return fail(ctx, ARROW_ERR_HANDLE, "bad adjacency handle (in=%d adj=%d)", in_adj, adj);
    DenseBuf *N = get_dense(ctx, new_buf), *O = get_dense(ctx, old_buf), *P = get_dense(ctx, parent_buf);
    if (!N || !O || !P) return fail(ctx, ARROW_ERR_HANDLE, "bad dense handle (new=%d old=%d parent=%d)", new_buf, old_buf, parent_buf);
    if (!in->incoming || a->incoming)
        return fail(ctx, ARROW_ERR_ARG, "in_adj is the in-adjacency (arrow_adj_build_in) and adj the push adjacency");
    if (in->n != a->n)
        return fail(ctx, ARROW_ERR_ARG, "the adjacencies differ in vertices: in %lld, push %lld", (long long)in->n, (long long)a->n);
    if (N->dtype != ARROW_B1 || O->dtype != ARROW_B1 || P->dtype != ARROW_I32)
        return fail(ctx, ARROW_ERR_ARG, "new / old are bit tiles and parent an int32 tile: got %s / %s / %s", dtype_name(N->dtype),
                    dtype_name(O->dtype), dtype_name(P->dtype));
    if (N->rows != a->n || O->rows != N->rows || P->rows != N->rows || O->k != N->k || P->k != N->k)
        return fail(ctx, ARROW_ERR_ARG, "shape: new %lld x %d, old %lld x %d, parent %lld x %d, adjacency %lld rows",
                    (long long)N->rows, N->k, (long long)O->rows, O->k, (long long)P->rows, P->k, (long long)a->n);
    if (new_buf == old_buf || N->p == O->p) return fail(ctx, ARROW_ERR_ARG, "old aliases new");
    if (a->tag < 0) return fail(ctx, ARROW_ERR_ARG, "no frontier record: run arrow_bits_mark_frontier on the adjacency first");
    if (new_buf != a->tag || N->p != a->tag_p || N->k != a->tag_k)
        return fail(ctx, ARROW_ERR_ARG, "new (tile %d) is not the tile of the last arrow_bits_mark_frontier (tile %d)", new_buf, a->tag);
    if (N->k > BITS_MAX_K) return fail(ctx, ARROW_ERR_UNSUPPORTED, "k=%d > %d", N->k, BITS_MAX_K);
    if (edges_scanned) *edges_scanned = 0;
    if (N->rows == 0 || N->k == 0 || a->n_front == 0) return ARROW_OK;
    const int words = bit_row_words(N->k);
    ParentArgs p{};
    p.nw = N->p;
    p.old = O->p;
    p.parent = reinterpret_cast<int *>(P->p);
    p.in_ptr = in->indptr;
    p.in_idx = in->indices;
    p.k = N->k;
    p.row_vecs = words == 1 ? 1 : words / 4;
    p.vecs = words == 1 ? 1 : ((N->k + 31) / 32 + 3) / 4;
    DevTmp cnt;
    if (edges_scanned) {
        CUDA_TRY(ctx, cudaMalloc(&cnt.p, sizeof(unsigned long long)));
        CUDA_TRY(ctx, cudaMemsetAsync(cnt.p, 0, sizeof(unsigned long long), cur_stream(ctx)));
        p.scanned = reinterpret_cast<unsigned long long *>(cnt.p);
    }
    const int rc = bits_parents(ctx, p, in, a);
    if (rc != ARROW_OK) return rc;
    if (edges_scanned) {
        unsigned long long h = 0;
        CUDA_TRY(ctx, cudaMemcpyAsync(&h, cnt.p, sizeof h, cudaMemcpyDeviceToHost, cur_stream(ctx)));
        CUDA_TRY(ctx, cudaStreamSynchronize(cur_stream(ctx)));
        *edges_scanned = (int64_t)h;
    }
    return ARROW_OK;
}

namespace {
// grows the adjacency's history to hold `need` rows, keeping the rows it holds (stream-ordered); it doubles, from 1024
int hist_reserve(arrow_ctx *ctx, Adj *a, int64_t need) {
    if (need <= a->hist_cap) return ARROW_OK;
    const int64_t at = a->hist_off.empty() ? 0 : a->hist_off.back();
    const int64_t cap = std::max<int64_t>({need, 2 * a->hist_cap, 1024});
    int *grown = nullptr;
    CUDA_TRY(ctx, cudaMalloc(&grown, (size_t)cap * 4));
    if (at > 0) {
        const cudaError_t e = cudaMemcpyAsync(grown, a->hist, (size_t)at * 4, cudaMemcpyDeviceToDevice, cur_stream(ctx));
        if (e != cudaSuccess) {
            cudaFree(grown);
            return fail(ctx, ARROW_ERR_CUDA, "history copy: %s", cudaGetErrorString(e));
        }
    }
    cudaFree(a->hist);                                        // waits for the copy
    a->hist = grown;
    a->hist_cap = cap;
    return ARROW_OK;
}
// reads back the optional edge counter of a path-count / dependency pass (synchronises)
int read_scanned(arrow_ctx *ctx, const DevTmp &cnt, int64_t *edges_scanned) {
    if (!edges_scanned) return ARROW_OK;
    unsigned long long h = 0;
    CUDA_TRY(ctx, cudaMemcpyAsync(&h, cnt.p, sizeof h, cudaMemcpyDeviceToHost, cur_stream(ctx)));
    CUDA_TRY(ctx, cudaStreamSynchronize(cur_stream(ctx)));
    *edges_scanned = (int64_t)h;
    return ARROW_OK;
}
int alloc_scanned(arrow_ctx *ctx, DevTmp &cnt, int64_t *edges_scanned, PathArgs &p) {
    if (!edges_scanned) return ARROW_OK;
    *edges_scanned = 0;
    CUDA_TRY(ctx, cudaMalloc(&cnt.p, sizeof(unsigned long long)));
    CUDA_TRY(ctx, cudaMemsetAsync(cnt.p, 0, sizeof(unsigned long long), cur_stream(ctx)));
    p.scanned = reinterpret_cast<unsigned long long *>(cnt.p);
    return ARROW_OK;
}
}  // namespace

int arrow_bits_path_counts(arrow_ctx *ctx, int in_adj, int adj, int new_buf, int old_buf, int sigma_buf, int64_t *edges_scanned) {
    CHECK_CTX(ctx);
    CHECK_POISON(ctx);
    Adj *in = get_adj(ctx, in_adj);
    const Adj *a = get_adj(ctx, adj);
    if (!in || !a) return fail(ctx, ARROW_ERR_HANDLE, "bad adjacency handle (in=%d adj=%d)", in_adj, adj);
    DenseBuf *N = get_dense(ctx, new_buf), *O = get_dense(ctx, old_buf), *S = get_dense(ctx, sigma_buf);
    if (!N || !O || !S) return fail(ctx, ARROW_ERR_HANDLE, "bad dense handle (new=%d old=%d sigma=%d)", new_buf, old_buf, sigma_buf);
    if (!in->incoming || a->incoming)
        return fail(ctx, ARROW_ERR_ARG, "in_adj is the in-adjacency (arrow_adj_build_in) and adj the push adjacency");
    if (in->n != a->n)
        return fail(ctx, ARROW_ERR_ARG, "the adjacencies differ in vertices: in %lld, push %lld", (long long)in->n, (long long)a->n);
    if (N->dtype != ARROW_B1 || O->dtype != ARROW_B1 || S->dtype != ARROW_F64)
        return fail(ctx, ARROW_ERR_ARG, "new / old are bit tiles and sigma a float64 tile: got %s / %s / %s", dtype_name(N->dtype),
                    dtype_name(O->dtype), dtype_name(S->dtype));
    if (N->rows != a->n || O->rows != N->rows || S->rows != N->rows || O->k != N->k || S->k != N->k)
        return fail(ctx, ARROW_ERR_ARG, "shape: new %lld x %d, old %lld x %d, sigma %lld x %d, adjacency %lld rows",
                    (long long)N->rows, N->k, (long long)O->rows, O->k, (long long)S->rows, S->k, (long long)a->n);
    if (new_buf == old_buf || N->p == O->p) return fail(ctx, ARROW_ERR_ARG, "old aliases new");
    if (a->tag < 0) return fail(ctx, ARROW_ERR_ARG, "no frontier record: run arrow_bits_mark_frontier on the adjacency first");
    if (new_buf != a->tag || N->p != a->tag_p || N->k != a->tag_k)
        return fail(ctx, ARROW_ERR_ARG, "new (tile %d) is not the tile of the last arrow_bits_mark_frontier (tile %d)", new_buf, a->tag);
    if (N->k > BITS_MAX_K) return fail(ctx, ARROW_ERR_UNSUPPORTED, "k=%d > %d", N->k, BITS_MAX_K);
    PathArgs p{};
    DevTmp cnt;
    if (const int rc = alloc_scanned(ctx, cnt, edges_scanned, p)) return rc;
    if (N->rows == 0 || N->k == 0 || a->n_front == 0) return read_scanned(ctx, cnt, edges_scanned);
    p.nw = reinterpret_cast<const unsigned *>(N->p);
    p.old = reinterpret_cast<const unsigned *>(O->p);
    p.sigma = reinterpret_cast<double *>(S->p);
    p.ptr = in->indptr;
    p.idx = in->indices;
    p.rows = a->front_rows;
    p.k = N->k;
    p.words = bit_row_words(N->k);
    p.used = (N->k + 31) / 32;
    if (const int rc = launch_paths(ctx, p, in, a->n_front, false)) return rc;
    return read_scanned(ctx, cnt, edges_scanned);
}

int arrow_adj_keep_record(arrow_ctx *ctx, int adj, int level) {
    CHECK_CTX(ctx);
    CHECK_POISON(ctx);
    Adj *a = get_adj(ctx, adj);
    if (!a) return fail(ctx, ARROW_ERR_HANDLE, "bad adjacency handle %d", adj);
    if (a->incoming) return fail(ctx, ARROW_ERR_ARG, "adjacency %d is an in-adjacency (arrow_adj_build_in)", adj);
    if (a->tag < 0) return fail(ctx, ARROW_ERR_ARG, "no frontier record: run arrow_bits_mark_frontier on the adjacency first");
    const int kept = a->hist_off.empty() ? 0 : (int)a->hist_off.size() - 1;
    if (level != 0 && level != kept)
        return fail(ctx, ARROW_ERR_ARG, "level %d: the history holds levels 0..%d, the next one kept is %d (or 0 to restart)", level,
                    kept - 1, kept);
    if (level == 0) a->hist_off.assign(1, 0);
    a->wp_tag_p = nullptr;                                    // the history no longer holds arrow_wpaths_counts' rounds
    const int64_t at = a->hist_off.back(), need = at + a->n_front;
    if (const int rc = hist_reserve(ctx, a, need)) return rc;
    if (a->n_front > 0)
        CUDA_TRY(ctx, cudaMemcpyAsync(a->hist + at, a->front_rows, (size_t)a->n_front * 4, cudaMemcpyDeviceToDevice, cur_stream(ctx)));
    a->hist_off.push_back(need);
    return ARROW_OK;
}

int arrow_bits_dependencies(arrow_ctx *ctx, int adj, int level, int dist_buf, int sigma_buf, int delta_buf, int64_t *edges_scanned) {
    CHECK_CTX(ctx);
    CHECK_POISON(ctx);
    Adj *a = get_adj(ctx, adj);
    if (!a) return fail(ctx, ARROW_ERR_HANDLE, "bad adjacency handle %d", adj);
    if (a->incoming) return fail(ctx, ARROW_ERR_ARG, "adjacency %d is an in-adjacency (arrow_adj_build_in)", adj);
    if (a->weighted) return fail(ctx, ARROW_ERR_ARG, "adjacency %d is weighted (it keeps the edges u == v)", adj);
    DenseBuf *D = get_dense(ctx, dist_buf), *S = get_dense(ctx, sigma_buf), *T = get_dense(ctx, delta_buf);
    if (!D || !S || !T) return fail(ctx, ARROW_ERR_HANDLE, "bad dense handle (dist=%d sigma=%d delta=%d)", dist_buf, sigma_buf, delta_buf);
    if (D->dtype != ARROW_I32 || S->dtype != ARROW_F64 || T->dtype != ARROW_F64)
        return fail(ctx, ARROW_ERR_ARG, "dist is an int32 tile and sigma / delta float64 tiles: got %s / %s / %s", dtype_name(D->dtype),
                    dtype_name(S->dtype), dtype_name(T->dtype));
    if (D->rows != a->n || S->rows != D->rows || T->rows != D->rows || S->k != D->k || T->k != D->k)
        return fail(ctx, ARROW_ERR_ARG, "shape: dist %lld x %d, sigma %lld x %d, delta %lld x %d, adjacency %lld rows",
                    (long long)D->rows, D->k, (long long)S->rows, S->k, (long long)T->rows, T->k, (long long)a->n);
    if (sigma_buf == delta_buf || S->p == T->p) return fail(ctx, ARROW_ERR_ARG, "delta aliases sigma");
    const int kept = a->hist_off.empty() ? 0 : (int)a->hist_off.size() - 1;
    if (level < 1 || level >= kept)
        return fail(ctx, ARROW_ERR_ARG, "level %d: the history holds levels 0..%d (arrow_adj_keep_record), the sweep runs 1..%d", level,
                    kept - 1, kept - 1);
    PathArgs p{};
    DevTmp cnt;
    if (const int rc = alloc_scanned(ctx, cnt, edges_scanned, p)) return rc;
    const int64_t n_rows = a->hist_off[level + 1] - a->hist_off[level];
    if (D->k == 0 || n_rows == 0) return read_scanned(ctx, cnt, edges_scanned);
    if (!a->has_segs) CUDA_TRY(ctx, build_segs(*a));         // the segments of the long out-lists, on first use
    p.dist = reinterpret_cast<const int *>(D->p);
    p.sigma = reinterpret_cast<double *>(S->p);
    p.delta = reinterpret_cast<double *>(T->p);
    p.ptr = a->indptr;
    p.idx = a->indices;
    p.rows = a->hist + a->hist_off[level];
    p.k = D->k;
    p.used = (D->k + 31) / 32;
    p.level = level;
    if (const int rc = launch_paths(ctx, p, a, n_rows, true)) return rc;
    return read_scanned(ctx, cnt, edges_scanned);
}

int arrow_bits_fill_f64(arrow_ctx *ctx, int new_buf, int old_buf, int out_buf, double value) {
    CHECK_CTX(ctx);
    CHECK_POISON(ctx);
    DenseBuf *N = get_dense(ctx, new_buf), *O = get_dense(ctx, old_buf), *X = get_dense(ctx, out_buf);
    if (!N || !O || !X) return fail(ctx, ARROW_ERR_HANDLE, "bad dense handle (new=%d old=%d out=%d)", new_buf, old_buf, out_buf);
    if (N->dtype != ARROW_B1 || O->dtype != ARROW_B1 || X->dtype != ARROW_F64)
        return fail(ctx, ARROW_ERR_ARG, "new / old are bit tiles and out a float64 tile: got %s / %s / %s", dtype_name(N->dtype),
                    dtype_name(O->dtype), dtype_name(X->dtype));
    if (N->rows != O->rows || N->k != O->k || X->rows != N->rows || X->k != N->k)
        return fail(ctx, ARROW_ERR_ARG, "tiles differ in shape: new %lld x %d, old %lld x %d, out %lld x %d", (long long)N->rows, N->k,
                    (long long)O->rows, O->k, (long long)X->rows, X->k);
    const long long items = N->rows * (long long)((N->k + 31) / 32);
    if (items == 0) return ARROW_OK;
    const int grid = (int)std::min<long long>((items + 255) / 256, (long long)ctx->sm_count * 8);
    k_bits_fill_f64<<<grid, 256, 0, cur_stream(ctx)>>>(reinterpret_cast<const unsigned *>(N->p), reinterpret_cast<const unsigned *>(O->p),
                                                       reinterpret_cast<double *>(X->p), N->rows, N->k, bit_row_words(N->k), value);
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
    return ARROW_OK;
}

int arrow_dense_row_sum(arrow_ctx *ctx, int in_buf, int out_buf) {
    CHECK_CTX(ctx);
    CHECK_POISON(ctx);
    DenseBuf *X = get_dense(ctx, in_buf), *Y = get_dense(ctx, out_buf);
    if (!X || !Y) return fail(ctx, ARROW_ERR_HANDLE, "bad dense handle (in=%d out=%d)", in_buf, out_buf);
    if (X->dtype != ARROW_F64 || Y->dtype != ARROW_F64)
        return fail(ctx, ARROW_ERR_ARG, "in / out are float64 tiles: got %s / %s", dtype_name(X->dtype), dtype_name(Y->dtype));
    if (Y->rows != X->rows || Y->k != 1)
        return fail(ctx, ARROW_ERR_ARG, "out is %lld x %d, expected %lld x 1", (long long)Y->rows, Y->k, (long long)X->rows);
    if (in_buf == out_buf || X->p == Y->p) return fail(ctx, ARROW_ERR_ARG, "out aliases in");
    if (X->rows == 0) return ARROW_OK;
    const int grid = (int)std::min<long long>((X->rows + 255) / 256, (long long)ctx->sm_count * 8);
    k_row_sum_f64<<<grid, 256, 0, cur_stream(ctx)>>>(reinterpret_cast<const double *>(X->p), reinterpret_cast<double *>(Y->p), X->rows, X->k);
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
    return ARROW_OK;
}

namespace {
// the tiles of the weighted path calls: x0 / dist float32, state int32, sigma (and delta) float64, all n x k; k >= 1
int wpaths_tiles(arrow_ctx *ctx, const Adj *a, int x0_buf, int dist_buf, int state_buf, int sigma_buf, int delta_buf,
                 DenseBuf *t[5]) {
    const int h[5] = {x0_buf, dist_buf, state_buf, sigma_buf, delta_buf};
    const int want[5] = {ARROW_F32, ARROW_F32, ARROW_I32, ARROW_F64, ARROW_F64};
    const char *name[5] = {"x0", "dist", "state", "sigma", "delta"};
    const int n_tiles = delta_buf < 0 ? 4 : 5;
    for (int i = 0; i < n_tiles; ++i) {
        t[i] = get_dense(ctx, h[i]);
        if (!t[i]) return fail(ctx, ARROW_ERR_HANDLE, "bad dense handle %s=%d", name[i], h[i]);
        if (t[i]->dtype != want[i])
            return fail(ctx, ARROW_ERR_ARG, "%s is a %s tile, expected %s", name[i], dtype_name(t[i]->dtype), dtype_name(want[i]));
        if (t[i]->rows != a->n || t[i]->k != t[0]->k)
            return fail(ctx, ARROW_ERR_ARG, "shape: %s %lld x %d, x0 %lld x %d, adjacency %lld rows", name[i], (long long)t[i]->rows,
                        t[i]->k, (long long)t[0]->rows, t[0]->k, (long long)a->n);
        for (int j = 0; j < i; ++j)
            if (h[j] == h[i] || t[j]->p == t[i]->p) return fail(ctx, ARROW_ERR_ARG, "%s aliases %s", name[i], name[j]);
    }
    if (t[0]->k > BITS_MAX_K) return fail(ctx, ARROW_ERR_UNSUPPORTED, "k=%d > %d", t[0]->k, BITS_MAX_K);
    if (a->n * (long long)((t[0]->k + 31) / 32) > INT_MAX)
        return fail(ctx, ARROW_ERR_RANGE, "%lld rows x %d words exceed the int32 item count", (long long)a->n, (t[0]->k + 31) / 32);
    return ARROW_OK;
}

WPathArgs wpaths_args(DenseBuf *const t[5], const Adj *lists) {
    WPathArgs w{};
    w.p.ptr = lists->indptr;
    w.p.idx = lists->indices;
    w.wt = lists->values;
    w.D = t[1]->p;
    w.x0 = t[0]->p;
    w.state = reinterpret_cast<int *>(t[2]->p);
    w.p.sigma = reinterpret_cast<double *>(t[3]->p);
    w.p.k = t[0]->k;
    w.p.used = (t[0]->k + 31) / 32;
    return w;
}
}  // namespace

int arrow_wpaths_counts(arrow_ctx *ctx, int in_adj, int out_adj, int x0_buf, int dist_buf, int state_buf, int sigma_buf,
                        int64_t *rounds, int64_t *entries_read) {
    CHECK_CTX(ctx);
    CHECK_POISON(ctx);
    Adj *in = get_adj(ctx, in_adj), *out = get_adj(ctx, out_adj);
    if (!in || !out) return fail(ctx, ARROW_ERR_HANDLE, "bad adjacency handle (in=%d out=%d)", in_adj, out_adj);
    if (!in->loopfree || !in->incoming || !out->loopfree || out->incoming)
        return fail(ctx, ARROW_ERR_ARG, "in_adj / out_adj are the loop-free in- and out-adjacencies (arrow_adj_build_loopfree)");
    if (in->n != out->n)
        return fail(ctx, ARROW_ERR_ARG, "the adjacencies differ in vertices: in %lld, out %lld", (long long)in->n, (long long)out->n);
    if (ctx->capturing) return fail(ctx, ARROW_ERR_UNSUPPORTED, "arrow_wpaths_counts synchronises: not during graph capture");
    DenseBuf *t[5];
    if (const int rc = wpaths_tiles(ctx, out, x0_buf, dist_buf, state_buf, sigma_buf, -1, t)) return rc;
    cudaStream_t s = cur_stream(ctx);
    out->wp_tag_p = nullptr;
    out->hist_off.assign(1, 0);
    if (rounds) *rounds = 0;
    if (entries_read) *entries_read = 0;
    const int64_t n = out->n;
    if (n == 0 || t[0]->k == 0) {
        out->wp_tag_p = t[2]->p;
        out->wp_tag_k = t[2]->k;
        return ARROW_OK;
    }
    DevTmp mark, cnt;                                         // the rows' last round; {cursor, entries read}
    CUDA_TRY(ctx, cudaMalloc(&mark.p, (size_t)n * 4));
    CUDA_TRY(ctx, cudaMalloc(&cnt.p, 2 * sizeof(unsigned long long)));
    CUDA_TRY(ctx, cudaMemsetAsync(mark.p, 0xff, (size_t)n * 4, s));
    CUDA_TRY(ctx, cudaMemsetAsync(cnt.p, 0, 2 * sizeof(unsigned long long), s));
    unsigned long long *cursor = reinterpret_cast<unsigned long long *>(cnt.p);
    WPathArgs w = wpaths_args(t, in);
    w.mark = reinterpret_cast<int *>(mark.p);
    w.cursor = cursor;
    w.p.scanned = entries_read ? cursor + 1 : nullptr;
    // runs a pass over `items` items, rows from history offset rows_at, that lists at most n rows at the end of the
    // history, and keeps them as the next round (synchronises)
    auto list_round = [&](auto kernel, int items, int64_t rows_at) -> int {
        const int64_t at = out->hist_off.back();
        if (const int rc = hist_reserve(ctx, out, at + n)) return rc;
        w.p.rows = out->hist + rows_at;
        w.next = out->hist + at;
        w.p.n_items = items;
        CUDA_TRY(ctx, cudaMemsetAsync(cursor, 0, sizeof(unsigned long long), s));
        kernel<<<path_grid(ctx, items), 256, 0, s>>>(w);
        ctx->launches++;
        CUDA_TRY(ctx, cudaGetLastError());
        unsigned long long listed = 0;
        CUDA_TRY(ctx, cudaMemcpyAsync(&listed, cursor, sizeof listed, cudaMemcpyDeviceToHost, s));
        CUDA_TRY(ctx, cudaStreamSynchronize(s));
        out->hist_off.push_back(at + (int64_t)listed);
        return ARROW_OK;
    };
    w.p.level = 0;
    if (const int rc = list_round(k_wpaths<WP_PENDING>, (int)(n * w.p.used), 0)) return rc;
    for (int r = 0; out->hist_off[r + 1] > out->hist_off[r]; ++r) {
        const long long n_rows = out->hist_off[r + 1] - out->hist_off[r];
        w.p.level = r;
        w.p.rows = out->hist + out->hist_off[r];
        if (r > 0) {                                          // round 0's counts are the pending pass's
            WPathArgs c = w;
            c.p.ptr = in->indptr;
            c.p.idx = in->indices;
            c.wt = in->values;
            const int rc = launch_seg_passes(ctx, c.p, in, n_rows, [&](int grid, const PathArgs &q) {
                c.p = q;
                k_wpaths<WP_COUNTS><<<grid, 256, 0, s>>>(c);
            });
            if (rc) return rc;
        }
        w.p.ptr = out->indptr;
        w.p.idx = out->indices;
        w.wt = out->values;
        if (const int rc = list_round(k_wpaths<WP_RELEASE>, (int)(n_rows * w.p.used), out->hist_off[r])) return rc;
    }
    out->hist_off.pop_back();                                 // the empty round that ended the loop
    out->wp_tag_p = t[2]->p;
    out->wp_tag_k = t[2]->k;
    if (rounds) *rounds = (int64_t)out->hist_off.size() - 1;
    if (entries_read) {
        unsigned long long h = 0;
        CUDA_TRY(ctx, cudaMemcpyAsync(&h, cursor + 1, sizeof h, cudaMemcpyDeviceToHost, s));
        CUDA_TRY(ctx, cudaStreamSynchronize(s));
        *entries_read = (int64_t)h;
    }
    return ARROW_OK;
}

int arrow_wpaths_dependencies(arrow_ctx *ctx, int out_adj, int x0_buf, int dist_buf, int state_buf, int sigma_buf, int delta_buf,
                              int64_t *entries_read) {
    CHECK_CTX(ctx);
    CHECK_POISON(ctx);
    Adj *out = get_adj(ctx, out_adj);
    if (!out) return fail(ctx, ARROW_ERR_HANDLE, "bad adjacency handle %d", out_adj);
    if (!out->loopfree || out->incoming)
        return fail(ctx, ARROW_ERR_ARG, "out_adj is the loop-free out-adjacency (arrow_adj_build_loopfree)");
    DenseBuf *t[5];
    if (const int rc = wpaths_tiles(ctx, out, x0_buf, dist_buf, state_buf, sigma_buf, delta_buf, t)) return rc;
    if (!out->wp_tag_p || out->wp_tag_p != t[2]->p || out->wp_tag_k != t[2]->k)
        return fail(ctx, ARROW_ERR_ARG, "the adjacency holds no rounds of arrow_wpaths_counts for state tile %d", state_buf);
    PathArgs scan{};
    DevTmp cnt;
    if (const int rc = alloc_scanned(ctx, cnt, entries_read, scan)) return rc;
    WPathArgs w = wpaths_args(t, out);
    w.p.delta = reinterpret_cast<double *>(t[4]->p);
    w.p.scanned = scan.scanned;
    cudaStream_t s = cur_stream(ctx);
    for (int r = (int)out->hist_off.size() - 2; r >= 0; --r) {
        w.p.level = r;
        w.p.rows = out->hist + out->hist_off[r];
        const int rc = launch_seg_passes(ctx, w.p, out, out->hist_off[r + 1] - out->hist_off[r], [&](int grid, const PathArgs &q) {
            WPathArgs d = w;
            d.p = q;
            k_wpaths<WP_DEPENDENCIES><<<grid, 256, 0, s>>>(d);
        });
        if (rc) return rc;
    }
    return read_scanned(ctx, cnt, entries_read);
}

namespace {
// arrow_sr_mark_frontier, and with steps_buf >= 0 arrow_sr_mark_frontier_steps
int sr_mark_frontier(arrow_ctx *ctx, int adj, int new_buf, int old_buf, int steps_buf, int level, int64_t *rows_changed,
                     int64_t *frontier_rows, int64_t *frontier_edges) {
    Adj *a = get_adj(ctx, adj);
    if (!a) return fail(ctx, ARROW_ERR_HANDLE, "bad adjacency handle %d", adj);
    if (a->incoming) return fail(ctx, ARROW_ERR_ARG, "adjacency %d is an in-adjacency (arrow_adj_build_in)", adj);
    DenseBuf *N = get_dense(ctx, new_buf), *O = get_dense(ctx, old_buf);
    if (!N || !O) return fail(ctx, ARROW_ERR_HANDLE, "bad dense handle (new=%d old=%d)", new_buf, old_buf);
    if (!rows_changed || !frontier_rows || !frontier_edges) return fail(ctx, ARROW_ERR_ARG, "null output");
    if (N->dtype != ARROW_F32 || O->dtype != ARROW_F32)
        return fail(ctx, ARROW_ERR_ARG, "new / old are fp32 tiles: got %s / %s", dtype_name(N->dtype), dtype_name(O->dtype));
    if (N->rows != O->rows || N->k != O->k || N->rows != a->n)
        return fail(ctx, ARROW_ERR_ARG, "tiles differ in shape: new %lld x %d, old %lld x %d, adjacency %lld rows",
                    (long long)N->rows, N->k, (long long)O->rows, O->k, (long long)a->n);
    DenseBuf *S = nullptr;
    if (steps_buf >= 0) {
        S = get_dense(ctx, steps_buf);
        if (!S) return fail(ctx, ARROW_ERR_HANDLE, "bad dense handle (steps=%d)", steps_buf);
        if (S->dtype != ARROW_I32 || S->rows != N->rows || S->k != N->k)
            return fail(ctx, ARROW_ERR_ARG, "steps is an int32 tile of new's shape (%lld x %d): got %s %lld x %d", (long long)N->rows,
                        N->k, dtype_name(S->dtype), (long long)S->rows, S->k);
        if (S->p == N->p || S->p == O->p) return fail(ctx, ARROW_ERR_ARG, "steps aliases new or old");
        if (level < 0) return fail(ctx, ARROW_ERR_ARG, "level %d < 0", level);
    }
    *rows_changed = *frontier_rows = *frontier_edges = 0;
    a->tag = -1;                                              // the record is rewritten below
    cudaStream_t stream = cur_stream(ctx);
    unsigned long long h[2] = {0, 0};                         // rows changed, (frontier rows << 32) | frontier edges
    if (N->rows > 0 && N->k > 0) {
        DevTmp cnt;
        CUDA_TRY(ctx, cudaMalloc(&cnt.p, sizeof h));
        CUDA_TRY(ctx, cudaMemsetAsync(cnt.p, 0, sizeof h, stream));
        const int grid = (int)std::min<long long>((N->rows + MARK_THREADS - 1) / MARK_THREADS, (long long)ctx->sm_count * 8);
        unsigned long long *counts = reinterpret_cast<unsigned long long *>(cnt.p);
        if (S)
            k_sr_mark_frontier<true><<<grid, MARK_THREADS, 0, stream>>>(N->p, O->p, N->rows, N->k, a->indptr, a->front_rows,
                                                                        a->front_off, counts, reinterpret_cast<int *>(S->p), level);
        else
            k_sr_mark_frontier<false><<<grid, MARK_THREADS, 0, stream>>>(N->p, O->p, N->rows, N->k, a->indptr, a->front_rows,
                                                                         a->front_off, counts, nullptr, 0);
        ctx->launches++;
        CUDA_TRY(ctx, cudaGetLastError());
        CUDA_TRY(ctx, cudaMemcpyAsync(h, cnt.p, sizeof h, cudaMemcpyDeviceToHost, stream));
        CUDA_TRY(ctx, cudaStreamSynchronize(stream));
    }
    a->n_front = (int64_t)(h[1] >> 32);
    a->front_edges = (int64_t)(h[1] & 0xffffffffULL);
    a->tag = new_buf;
    a->tag_p = N->p;
    a->tag_k = N->k;
    *rows_changed = (int64_t)h[0];
    *frontier_rows = a->n_front;
    *frontier_edges = a->front_edges;
    return ARROW_OK;
}
}  // namespace

int arrow_sr_mark_frontier(arrow_ctx *ctx, int adj, int new_buf, int old_buf, int64_t *rows_changed, int64_t *frontier_rows,
                           int64_t *frontier_edges) {
    CHECK_CTX(ctx);
    CHECK_POISON(ctx);
    return sr_mark_frontier(ctx, adj, new_buf, old_buf, -1, 0, rows_changed, frontier_rows, frontier_edges);
}

int arrow_sr_mark_frontier_steps(arrow_ctx *ctx, int adj, int new_buf, int old_buf, int steps_buf, int level,
                                 int64_t *rows_changed, int64_t *frontier_rows, int64_t *frontier_edges) {
    CHECK_CTX(ctx);
    CHECK_POISON(ctx);
    if (steps_buf < 0) return fail(ctx, ARROW_ERR_HANDLE, "bad dense handle (steps=%d)", steps_buf);
    return sr_mark_frontier(ctx, adj, new_buf, old_buf, steps_buf, level, rows_changed, frontier_rows, frontier_edges);
}

int arrow_sr_push_frontier(arrow_ctx *ctx, int adj, int x_buf, int out_buf, int semiring) {
    CHECK_CTX(ctx);
    CHECK_POISON(ctx);
    if (semiring == ARROW_SR_PLUS_TIMES || semiring == ARROW_SR_OR_AND)
        return fail(ctx, ARROW_ERR_UNSUPPORTED, "arrow_sr_push_frontier runs the fp32 semirings, not semiring %d", semiring);
    if (!fp32_semiring(semiring)) return fail(ctx, ARROW_ERR_ARG, "unknown semiring %d", semiring);
    const Adj *a = get_adj(ctx, adj);
    if (!a) return fail(ctx, ARROW_ERR_HANDLE, "bad adjacency handle %d", adj);
    if (a->incoming) return fail(ctx, ARROW_ERR_ARG, "adjacency %d is an in-adjacency (arrow_adj_build_in)", adj);
    DenseBuf *X = get_dense(ctx, x_buf), *O = get_dense(ctx, out_buf);
    if (!X || !O) return fail(ctx, ARROW_ERR_HANDLE, "bad dense handle (x=%d out=%d)", x_buf, out_buf);
    if (X->dtype != ARROW_F32 || O->dtype != ARROW_F32)
        return fail(ctx, ARROW_ERR_ARG, "x / out are fp32 tiles: got %s / %s", dtype_name(X->dtype), dtype_name(O->dtype));
    if (!a->weighted) return fail(ctx, ARROW_ERR_ARG, "the adjacency carries no weights: build it with arrow_adj_build_weighted");
    if (a->tag < 0) return fail(ctx, ARROW_ERR_ARG, "no frontier record: run arrow_sr_mark_frontier on the adjacency first");
    if (x_buf != a->tag || X->p != a->tag_p || X->k != a->tag_k)
        return fail(ctx, ARROW_ERR_ARG, "x (tile %d) is not the tile of the last arrow_sr_mark_frontier (tile %d)", x_buf, a->tag);
    if (x_buf == out_buf || X->p == O->p) return fail(ctx, ARROW_ERR_ARG, "out aliases x");
    if (X->rows != a->n || O->rows != X->rows || O->k != X->k)
        return fail(ctx, ARROW_ERR_ARG, "shape: x %lld x %d, out %lld x %d, adjacency %lld rows", (long long)X->rows, X->k,
                    (long long)O->rows, O->k, (long long)a->n);
    cudaStream_t stream = cur_stream(ctx);
    const long long n = (long long)X->rows * X->k;
    if (n == 0) return ARROW_OK;
    const bool mn = semiring == ARROW_SR_MIN_PLUS;
    {                                                         // out = canon(x), float4 groups and a scalar tail
        const bool aligned = (((uintptr_t)X->p | (uintptr_t)O->p) & 15) == 0;     // a wrapped tile with k % 4 != 0 may not be
        const long long n4 = aligned ? n / 4 : 0;
        const int grid = (int)std::max<long long>(1, std::min<long long>((n4 + 255) / 256, (long long)ctx->sm_count * 8));
        const float4 *x4 = reinterpret_cast<const float4 *>(X->p);
        float4 *o4 = reinterpret_cast<float4 *>(O->p);
        if (mn) k_sr_canon<SrMinPlus><<<grid, 256, 0, stream>>>(x4, o4, n4, X->p, O->p, n);
        else if (semiring == ARROW_SR_MAX_PLUS) k_sr_canon<SrMaxPlus><<<grid, 256, 0, stream>>>(x4, o4, n4, X->p, O->p, n);
        else if (semiring == ARROW_SR_MAX_MIN) k_sr_canon<SrMaxMin><<<grid, 256, 0, stream>>>(x4, o4, n4, X->p, O->p, n);
        else k_sr_canon<SrMinMax><<<grid, 256, 0, stream>>>(x4, o4, n4, X->p, O->p, n);
        ctx->launches++;
        CUDA_TRY(ctx, cudaGetLastError());
    }
    if (a->front_edges == 0) return ARROW_OK;
    const bool v4 = X->k % 4 == 0;
    const int vecs = v4 ? X->k / 4 : X->k;
    const long long items = a->front_edges * vecs;
    const long long chunks = (items + (long long)PUSH_THREADS * PUSH_ITEMS - 1) / ((long long)PUSH_THREADS * PUSH_ITEMS);
    const int per_sm = ctx->spmm_ctas_per_sm > 0 ? std::min(ctx->spmm_ctas_per_sm, 8) : 8;
    const int sms = ctx->spmm_sm_limit > 0 ? std::min(ctx->sm_count, ctx->spmm_sm_limit) : ctx->sm_count;
    const int grid = (int)std::min<long long>(chunks, (long long)per_sm * sms);
    if (semiring == ARROW_SR_MAX_MIN) launch_bottleneck_push<SrMaxMin>(stream, grid, a, X, O, items, vecs);
    if (semiring == ARROW_SR_MIN_MAX) launch_bottleneck_push<SrMinMax>(stream, grid, a, X, O, items, vecs);
    if (semiring == ARROW_SR_MAX_MIN || semiring == ARROW_SR_MIN_MAX) {
        ctx->launches++;
        CUDA_TRY(ctx, cudaGetLastError());
        return ARROW_OK;
    }
    const float4 *x4 = reinterpret_cast<const float4 *>(X->p);
#define SRP(SR, V, XP) k_sr_push<SR, V><<<grid, PUSH_THREADS, 0, stream>>>(XP, O->p, a->indptr, a->indices, a->values, \
                                                                       a->front_rows, a->front_off, (int)a->n_front, items, vecs)
    if (mn && v4) SRP(SrMinPlus, float4, x4);
    else if (mn) SRP(SrMinPlus, float, X->p);
    else if (v4) SRP(SrMaxPlus, float4, x4);
    else SRP(SrMaxPlus, float, X->p);
#undef SRP
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
    return ARROW_OK;
}

int arrow_sr_tree_parents(arrow_ctx *ctx, int in_adj, int dist_buf, int steps_buf, int parent_buf, int semiring,
                          int64_t *entries_read) {
    CHECK_CTX(ctx);
    CHECK_POISON(ctx);
    if (semiring == ARROW_SR_PLUS_TIMES || semiring == ARROW_SR_MIN_PLUS || semiring == ARROW_SR_MAX_PLUS || semiring == ARROW_SR_OR_AND)
        return fail(ctx, ARROW_ERR_UNSUPPORTED, "arrow_sr_tree_parents runs max-min and min-max, not semiring %d", semiring);
    if (semiring != ARROW_SR_MAX_MIN && semiring != ARROW_SR_MIN_MAX) return fail(ctx, ARROW_ERR_ARG, "unknown semiring %d", semiring);
    Adj *in = get_adj(ctx, in_adj);
    if (!in) return fail(ctx, ARROW_ERR_HANDLE, "bad adjacency handle %d", in_adj);
    if (!in->loopfree || !in->incoming)
        return fail(ctx, ARROW_ERR_ARG, "in_adj is the loop-free in-adjacency (arrow_adj_build_loopfree, incoming)");
    DenseBuf *D = get_dense(ctx, dist_buf), *T = get_dense(ctx, steps_buf), *P = get_dense(ctx, parent_buf);
    if (!D || !T || !P) return fail(ctx, ARROW_ERR_HANDLE, "bad dense handle (dist=%d steps=%d parent=%d)", dist_buf, steps_buf, parent_buf);
    if (D->dtype != ARROW_F32 || T->dtype != ARROW_I32 || P->dtype != ARROW_I32)
        return fail(ctx, ARROW_ERR_ARG, "dist is fp32, steps and parent int32: got %s / %s / %s", dtype_name(D->dtype),
                    dtype_name(T->dtype), dtype_name(P->dtype));
    if (D->rows != in->n || T->rows != in->n || P->rows != in->n || T->k != D->k || P->k != D->k)
        return fail(ctx, ARROW_ERR_ARG, "shape: dist %lld x %d, steps %lld x %d, parent %lld x %d, adjacency %lld rows",
                    (long long)D->rows, D->k, (long long)T->rows, T->k, (long long)P->rows, P->k, (long long)in->n);
    if (P->p == D->p || P->p == T->p) return fail(ctx, ARROW_ERR_ARG, "parent aliases dist or steps");
    TreeArgs t{};
    DevTmp cnt;
    if (const int rc = alloc_scanned(ctx, cnt, entries_read, t.p)) return rc;
    const long long n = in->n;
    const int k = D->k;
    if (n == 0 || k == 0) return read_scanned(ctx, cnt, entries_read);
    cudaStream_t s = cur_stream(ctx);
    // -1 everywhere: the row pass stores the hits of the short lists, the segment pass folds those of the long ones
    CUDA_TRY(ctx, cudaMemsetAsync(P->p, 0xff, (size_t)n * k * 4, s));
    t.p.ptr = in->indptr;
    t.p.idx = in->indices;
    t.p.k = k;
    t.p.used = (k + 31) / 32;
    t.wt = in->values;
    t.D = D->p;
    t.T = reinterpret_cast<const int *>(T->p);
    t.parent = reinterpret_cast<int *>(P->p);
    // launch_seg_passes runs the segment pass first (when there are segments), then the row pass over every row
    bool first = true;
    const int rc = launch_seg_passes(ctx, t.p, in, n, [&](int grid, const PathArgs &q) {
        TreeArgs a = t;
        a.p = q;
        a.seg_pass = first && in->n_segs > 0;
        first = false;
        if (semiring == ARROW_SR_MAX_MIN) k_sr_tree<SrMaxMin><<<grid, 256, 0, s>>>(a);
        else k_sr_tree<SrMinMax><<<grid, 256, 0, s>>>(a);
    }, false);                                                // the hits fold into P: no segment partials
    if (rc) return rc;
    return read_scanned(ctx, cnt, entries_read);
}

int arrow_out_weights(arrow_ctx *ctx, int n_parts, const int *csrs, const int *maps, int64_t n_vertices, int w_buf, int inv_buf,
                      int64_t *bad_entries, int64_t *dangling, int64_t *bad_inverses) {
    CHECK_CTX(ctx);
    CHECK_POISON(ctx);
    if (n_parts < 0 || (n_parts > 0 && (!csrs || !maps)) || n_vertices < 0)
        return fail(ctx, ARROW_ERR_ARG, "bad arguments (n_parts=%d, n_vertices=%lld)", n_parts, (long long)n_vertices);
    if (n_vertices > 2147483646LL) return fail(ctx, ARROW_ERR_RANGE, "%lld vertices exceed the int32 device layout", (long long)n_vertices);
    if (ctx->capturing) return fail(ctx, ARROW_ERR_UNSUPPORTED, "arrow_out_weights allocates and synchronises: not during graph capture");
    DenseBuf *W = get_dense(ctx, w_buf), *I = get_dense(ctx, inv_buf);
    if (!W || !I) return fail(ctx, ARROW_ERR_HANDLE, "bad dense handle (w=%d inv=%d)", w_buf, inv_buf);
    int T = -1;
    std::vector<std::pair<const Csr *, const IdxMap *>> blocks;
    if (const int rc = operator_parts(ctx, n_parts, csrs, maps, n_vertices, blocks)) return rc;
    std::vector<AdjPart> parts;
    std::vector<const void *> vals;
    long long m = 0;
    for (int i = 0; i < n_parts; ++i) {
        const Csr *c = blocks[i].first;
        const IdxMap *mp = blocks[i].second;
        if (T >= 0 && c->dtype != T) return fail(ctx, ARROW_ERR_ARG, "part %d is %s, part 0 %s", i, dtype_name(c->dtype), dtype_name(T));
        T = c->dtype;
        if (c->nnz > 0 && !c->vals) return fail(ctx, ARROW_ERR_ARG, "part %d: the block has no values", i);
        if (c->nnz > 0) {
            parts.push_back(AdjPart{c->indptr, c->indices, mp ? mp->p : nullptr, (long long)c->nnz, (int)c->n_rows});
            vals.push_back(c->vals);
            m += c->nnz;
        }
    }
    if (T < 0) T = I->dtype;
    if (W->dtype != ARROW_F64 || I->dtype != T || W->rows != n_vertices || I->rows != n_vertices || W->k != 1 || I->k != 1)
        return fail(ctx, ARROW_ERR_ARG, "w is float64 and inv %s, both %lld x 1: got %s %lld x %d and %s %lld x %d", dtype_name(T),
                    (long long)n_vertices, dtype_name(W->dtype), (long long)W->rows, W->k, dtype_name(I->dtype), (long long)I->rows, I->k);
    if (T != ARROW_F32 && T != ARROW_F64) return fail(ctx, ARROW_ERR_ARG, "inv is a %s tile, expected float32 or float64", dtype_name(T));
    if (W->p == I->p) return fail(ctx, ARROW_ERR_ARG, "inv aliases w");
    if (m > 2147483647LL) return fail(ctx, ARROW_ERR_RANGE, "%lld entries exceed the int32 sort layout", m);
    cudaStream_t s = ctx->stream;
    auto grid = [&](long long items) { return (int)std::max<long long>(1, std::min<long long>((items + 255) / 256, (long long)ctx->sm_count * 8)); };
    // 24 bytes per entry (key and float64 value, twice) and the sort's temporary storage
    DevTmp cnt, keys, alt, wv, walt, temp;
    unsigned long long h_cnt[3] = {0, 0, 0};
    cudaError_t e = cudaMalloc(&cnt.p, sizeof h_cnt);
    if (e == cudaSuccess) e = cudaMemsetAsync(cnt.p, 0, sizeof h_cnt, s);
    unsigned long long *dc = reinterpret_cast<unsigned long long *>(cnt.p);
    if (e == cudaSuccess && m > 0) {
        e = cudaMalloc(&keys.p, (size_t)m * 4);
        if (e == cudaSuccess) e = cudaMalloc(&alt.p, (size_t)m * 4);
        if (e == cudaSuccess) e = cudaMalloc(&wv.p, (size_t)m * 8);
        if (e == cudaSuccess) e = cudaMalloc(&walt.p, (size_t)m * 8);
        long long off = 0;
        for (size_t i = 0; e == cudaSuccess && i < parts.size(); ++i) {
            int *kp = reinterpret_cast<int *>(keys.p) + off;
            double *vp = reinterpret_cast<double *>(wv.p) + off;
            if (T == ARROW_F64)
                k_pr_out_keys<double><<<grid(parts[i].nnz), 256, 0, s>>>(parts[i], (const double *)vals[i], (int)n_vertices, kp, vp, dc + 2);
            else
                k_pr_out_keys<float><<<grid(parts[i].nnz), 256, 0, s>>>(parts[i], (const float *)vals[i], (int)n_vertices, kp, vp, dc + 2);
            ctx->launches++;
            off += parts[i].nnz;
            e = cudaGetLastError();
        }
        int end_bit = 1;                                          // keys lie in [0, n_vertices]
        while ((1LL << end_bit) <= n_vertices) ++end_bit;
        cub::DoubleBuffer<int> db(reinterpret_cast<int *>(keys.p), reinterpret_cast<int *>(alt.p));
        cub::DoubleBuffer<double> dv(reinterpret_cast<double *>(wv.p), reinterpret_cast<double *>(walt.p));
        size_t temp_bytes = 0;
        if (e == cudaSuccess) e = cub::DeviceRadixSort::SortPairs(nullptr, temp_bytes, db, dv, (int)m, 0, end_bit, s);
        if (e == cudaSuccess) e = cudaMalloc(&temp.p, std::max<size_t>(temp_bytes, 1));
        if (e == cudaSuccess) e = cub::DeviceRadixSort::SortPairs(temp.p, temp_bytes, db, dv, (int)m, 0, end_bit, s);
        if (e == cudaSuccess && n_vertices > 0) {
            if (T == ARROW_F64)
                k_pr_out_sums<double><<<grid(n_vertices), 256, 0, s>>>(db.Current(), dv.Current(), m, n_vertices, (double *)W->p,
                                                                       (double *)I->p, dc);
            else
                k_pr_out_sums<float><<<grid(n_vertices), 256, 0, s>>>(db.Current(), dv.Current(), m, n_vertices, (double *)W->p,
                                                                      I->p, dc);
            ctx->launches++;
            e = cudaGetLastError();
        }
    } else if (e == cudaSuccess && n_vertices > 0) {          // no entries: every vertex is dangling
        if (T == ARROW_F64)
            k_pr_out_sums<double><<<grid(n_vertices), 256, 0, s>>>(nullptr, nullptr, 0, n_vertices, (double *)W->p, (double *)I->p, dc);
        else
            k_pr_out_sums<float><<<grid(n_vertices), 256, 0, s>>>(nullptr, nullptr, 0, n_vertices, (double *)W->p, I->p, dc);
        ctx->launches++;
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(h_cnt, cnt.p, sizeof h_cnt, cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return fail(ctx, e == cudaErrorMemoryAllocation ? ARROW_ERR_NOMEM : ARROW_ERR_CUDA, "out-weight pass failed: %s",
                    cudaGetErrorString(e));
    }
    if (dangling) *dangling = (int64_t)h_cnt[0];
    if (bad_inverses) *bad_inverses = (int64_t)h_cnt[1];
    if (bad_entries) *bad_entries = (int64_t)h_cnt[2];
    return ARROW_OK;
}

int arrow_csr_scale_columns(arrow_ctx *ctx, int csr, int map, int scale_buf, int *csr_out) {
    CHECK_CTX(ctx);
    CHECK_POISON(ctx);
    Csr *c = get_csr(ctx, csr);
    if (!c) return fail(ctx, ARROW_ERR_HANDLE, "bad csr handle %d", csr);
    if (!csr_out) return fail(ctx, ARROW_ERR_ARG, "csr_out is null");
    const IdxMap *m = nullptr;
    if (map != -1 && !(m = get_map(ctx, map))) return fail(ctx, ARROW_ERR_HANDLE, "bad map handle %d", map);
    DenseBuf *S = get_dense(ctx, scale_buf);
    if (!S) return fail(ctx, ARROW_ERR_HANDLE, "bad dense handle scale=%d", scale_buf);
    if (S->dtype != c->dtype || S->k != 1)
        return fail(ctx, ARROW_ERR_ARG, "scale is a %s tile of %d columns, expected %s x 1", dtype_name(S->dtype), S->k, dtype_name(c->dtype));
    if (m ? (m->n < c->n_cols || m->limit > S->rows) : c->n_cols > S->rows)
        return fail(ctx, ARROW_ERR_ARG, "the block's %lld columns%s reach past the %lld scale rows", (long long)c->n_cols,
                    m ? " mapped" : "", (long long)S->rows);
    if (c->nnz > 0 && !c->vals) return fail(ctx, ARROW_ERR_ARG, "the block has no values to scale");
    if (ctx->capturing) return fail(ctx, ARROW_ERR_UNSUPPORTED, "arrow_csr_scale_columns allocates: not during graph capture");
    Csr d = *c;
    d.owns_indptr = d.owns_indices = d.owns_long = false;     // shared with the source block (and its own source)
    d.owns_vals = true;
    d.vals = nullptr;
    d.parent = csr;
    d.children = 0;
    const size_t esz = dtype_size(c->dtype);
    CUDA_TRY(ctx, cudaMalloc(&d.vals, ((size_t)c->nnz + 8) * esz));
    cudaError_t e = cudaSuccess;
    if (c->nnz > 0) {
        const int grid = (int)std::min<long long>((c->nnz + 255) / 256, (long long)ctx->sm_count * 8);
        if (c->dtype == ARROW_F64)
            k_pr_scale<double><<<grid, 256, 0, ctx->stream>>>(c->indices, (const double *)c->vals, m ? m->p : nullptr,
                                                              (const double *)S->p, (double *)d.vals, c->nnz);
        else
            k_pr_scale<float><<<grid, 256, 0, ctx->stream>>>(c->indices, c->vals, m ? m->p : nullptr, S->p, d.vals, c->nnz);
        ctx->launches++;
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) {
        cudaFree(d.vals);
        return fail(ctx, ARROW_ERR_CUDA, "column scaling failed: %s", cudaGetErrorString(e));
    }
    const int h = new_slot(ctx->csrs);       // may grow the table: `c` is not used past this point
    ctx->csrs[h] = d;
    ctx->csrs[csr].children++;
    *csr_out = h;
    return ARROW_OK;
}

int arrow_pagerank_restart(arrow_ctx *ctx, int x_buf, int inv_buf, int s_buf, int scratch_buf, int state_buf, double *col_sums,
                           int64_t *bad_columns, int64_t *first_bad_column) {
    CHECK_CTX(ctx);
    CHECK_POISON(ctx);
    DenseBuf *t[6];
    if (const int rc = pr_tiles(ctx, "arrow_pagerank_restart", true, x_buf, -1, s_buf, inv_buf, scratch_buf, state_buf, t)) return rc;
    const long long n = t[0]->rows, nch = pr_chunks(n);
    const int k = t[0]->k;
    const bool f64 = t[0]->dtype == ARROW_F64;
    double *part = reinterpret_cast<double *>(t[4]->p), *state = reinterpret_cast<double *>(t[5]->p);
    cudaStream_t s = cur_stream(ctx);
    if (k == 0) {
        if (bad_columns) *bad_columns = 0;
        if (first_bad_column) *first_bad_column = -1;
        return ARROW_OK;
    }
    if (nch > 0) {
        if (f64) k_pr_restart_partials<double><<<pr_grid(ctx, nch * k), 256, 0, s>>>((const double *)t[0]->p, n, k, nch, part);
        else k_pr_restart_partials<float><<<pr_grid(ctx, nch * k), 256, 0, s>>>(t[0]->p, n, k, nch, part);
        ctx->launches++;
    }
    k_pr_chunk_sums<<<2 * k, 256, 0, s>>>(part, nch, state + 2 * k);      // rows 2 (sigma) and 3 (bad flags)
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
    std::vector<double> h((size_t)2 * k);
    CUDA_TRY(ctx, cudaMemcpyAsync(h.data(), state + 2 * k, h.size() * 8, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(ctx, cudaStreamSynchronize(s));
    int64_t bad = 0, first = -1;
    for (int c = 0; c < k; ++c) {
        const double sigma = h[c];
        if (h[k + c] != 0.0 || !(sigma > 0.0) || !std::isfinite(sigma)) {
            if (first < 0) first = c;
            ++bad;
        }
    }
    if (col_sums) memcpy(col_sums, h.data(), (size_t)k * 8);
    if (bad_columns) *bad_columns = bad;
    if (first_bad_column) *first_bad_column = first;
    if (bad > 0) return ARROW_OK;
    if (nch > 0) {
        if (f64)
            k_pr_restart_write<double><<<pr_grid(ctx, nch * k), 256, 0, s>>>((const double *)t[0]->p, (const double *)t[3]->p, state,
                                                                        (double *)t[2]->p, n, k, nch, part);
        else
            k_pr_restart_write<float><<<pr_grid(ctx, nch * k), 256, 0, s>>>(t[0]->p, t[3]->p, state, t[2]->p, n, k, nch, part);
        ctx->launches++;
    }
    k_pr_chunk_sums<<<k, 256, 0, s>>>(part, nch, state);                  // row 0: m_0
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
    return ARROW_OK;
}

int arrow_pagerank_update(arrow_ctx *ctx, int y_buf, int p_buf, int s_buf, int inv_buf, int scratch_buf, int state_buf,
                          double alpha, double *residuals) {
    CHECK_CTX(ctx);
    CHECK_POISON(ctx);
    if (!(alpha >= 0.0 && alpha < 1.0)) return fail(ctx, ARROW_ERR_ARG, "alpha = %g lies outside [0, 1)", alpha);
    DenseBuf *t[6];
    if (const int rc = pr_tiles(ctx, "arrow_pagerank_update", false, y_buf, p_buf, s_buf, inv_buf, scratch_buf, state_buf, t))
        return rc;
    const long long n = t[0]->rows, nch = pr_chunks(n);
    const int k = t[0]->k;
    if (k == 0) return ARROW_OK;
    const double beta = 1.0 - alpha;
    double *part = reinterpret_cast<double *>(t[4]->p), *state = reinterpret_cast<double *>(t[5]->p);
    cudaStream_t s = cur_stream(ctx);
    if (nch > 0) {
        if (t[0]->dtype == ARROW_F64)
            k_pr_update<double><<<pr_grid(ctx, nch * k), 256, 0, s>>>((double *)t[0]->p, (const double *)t[1]->p, (const double *)t[2]->p,
                                                                 (const double *)t[3]->p, state, alpha, beta, n, k, nch, part);
        else
            k_pr_update<float><<<pr_grid(ctx, nch * k), 256, 0, s>>>(t[0]->p, t[1]->p, t[2]->p, t[3]->p, state, alpha, beta, n, k, nch, part);
        ctx->launches++;
    }
    k_pr_chunk_sums<<<2 * k, 256, 0, s>>>(part, nch, state);              // rows 0 (m_{t+1}) and 1 (r_{t+1})
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
    if (residuals) CUDA_TRY(ctx, cudaMemcpyAsync(residuals, state + k, (size_t)k * 8, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(ctx, cudaStreamSynchronize(s));
    return ARROW_OK;
}

int arrow_connected_components(arrow_ctx *ctx, int n_parts, const int *csrs, const int *maps, int64_t n_vertices,
                               int labels_buf, int sizes_buf, int64_t *n_components) {
    CHECK_CTX(ctx);
    CHECK_POISON(ctx);
    if (n_parts < 0 || (n_parts > 0 && (!csrs || !maps)) || n_vertices < 0)
        return fail(ctx, ARROW_ERR_ARG, "bad arguments (n_parts=%d, n_vertices=%lld)", n_parts, (long long)n_vertices);
    if (n_vertices > 2147483646LL) return fail(ctx, ARROW_ERR_RANGE, "%lld vertices exceed the int32 device layout", (long long)n_vertices);
    DenseBuf *L = get_dense(ctx, labels_buf), *S = nullptr;
    if (!L) return fail(ctx, ARROW_ERR_HANDLE, "bad dense handle labels=%d", labels_buf);
    if (sizes_buf != -1 && !(S = get_dense(ctx, sizes_buf))) return fail(ctx, ARROW_ERR_HANDLE, "bad dense handle sizes=%d", sizes_buf);
    for (const DenseBuf *t : {L, S}) {
        if (t && (t->dtype != ARROW_I32 || t->rows != n_vertices || t->k != 1))
            return fail(ctx, ARROW_ERR_ARG, "%s is a %s tile of %lld x %d, expected int32 %lld x 1", t == L ? "labels" : "sizes",
                        dtype_name(t->dtype), (long long)t->rows, t->k, (long long)n_vertices);
    }
    if (S && (sizes_buf == labels_buf || S->p == L->p)) return fail(ctx, ARROW_ERR_ARG, "sizes aliases labels");
    std::vector<std::pair<const Csr *, const IdxMap *>> blocks;
    if (const int rc = operator_parts(ctx, n_parts, csrs, maps, n_vertices, blocks)) return rc;
    if (ctx->capturing) return fail(ctx, ARROW_ERR_UNSUPPORTED, "arrow_connected_components synchronises: not during graph capture");
    int *parent = reinterpret_cast<int *>(L->p);
    int *sizes = S ? reinterpret_cast<int *>(S->p) : nullptr;
    cudaStream_t s = cur_stream(ctx);
    DevTmp cnt;
    unsigned long long roots = 0;
    CUDA_TRY(ctx, cudaMalloc(&cnt.p, sizeof roots));
    unsigned long long *d_roots = reinterpret_cast<unsigned long long *>(cnt.p);
    CUDA_TRY(ctx, cudaMemsetAsync(d_roots, 0, sizeof roots, s));
    if (sizes) CUDA_TRY(ctx, cudaMemsetAsync(sizes, 0, (size_t)n_vertices * 4, s));
    if (n_vertices > 0) {
        k_cc_init<<<pr_grid(ctx, n_vertices), 256, 0, s>>>(parent, n_vertices);
        ctx->launches++;
        for (const auto &b : blocks) {
            const Csr *c = b.first;
            if (c->nnz == 0) continue;
            const AdjPart p{c->indptr, c->indices, b.second ? b.second->p : nullptr, (long long)c->nnz, (int)c->n_rows};
            k_cc_hook<<<pr_grid(ctx, (p.nnz + CC_CHUNK - 1) / CC_CHUNK * 32), 256, 0, s>>>(p, parent);
            ctx->launches++;
        }
        k_cc_label<<<pr_grid(ctx, n_vertices), 256, 0, s>>>(parent, n_vertices, sizes, d_roots);
        ctx->launches++;
    }
    CUDA_TRY(ctx, cudaGetLastError());
    CUDA_TRY(ctx, cudaMemcpyAsync(&roots, d_roots, sizeof roots, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(ctx, cudaStreamSynchronize(s));
    if (n_components) *n_components = (int64_t)roots;
    return ARROW_OK;
}

int arrow_gather_rows_multi(arrow_ctx *ctx, int dst_buf, const int *src_bufs, const int64_t *row_bounds, int n_src, int map, int flags) {
    CHECK_CTX(ctx);
    DenseBuf *D = get_dense(ctx, dst_buf);
    IdxMap *m = get_map(ctx, map);
    if (!D) return fail(ctx, ARROW_ERR_HANDLE, "bad dense handle %d", dst_buf);
    if (!m) return fail(ctx, ARROW_ERR_HANDLE, "bad map handle %d", map);
    if (!src_bufs || !row_bounds || n_src < 1 || n_src > MAX_SRC) return fail(ctx, ARROW_ERR_ARG, "need 1..%d sources", MAX_SRC);
    REFUSE_I32(ctx, D, "arrow_gather_rows_multi");
    REFUSE_B1(ctx, D, "arrow_gather_rows_multi");
    if (D->dtype != ARROW_F32) return fail(ctx, ARROW_ERR_UNSUPPORTED, "the multi-source gather is float32 only");
    if (m->n > D->rows) return fail(ctx, ARROW_ERR_ARG, "map has %lld entries, destination has %lld rows", (long long)m->n, (long long)D->rows);
    MultiSrc ms;
    memset(&ms, 0, sizeof ms);
    ms.n = n_src;
    for (int s = 0; s < n_src; ++s) {
        DenseBuf *S = get_dense(ctx, src_bufs[s]);
        if (!S) return fail(ctx, ARROW_ERR_HANDLE, "bad source handle %d", src_bufs[s]);
        if (S->k != D->k) return fail(ctx, ARROW_ERR_ARG, "feature width mismatch in source %d", s);
        REFUSE_I32(ctx, S, "arrow_gather_rows_multi");
        REFUSE_B1(ctx, S, "arrow_gather_rows_multi");
        if (S->dtype != ARROW_F32) return fail(ctx, ARROW_ERR_UNSUPPORTED, "the multi-source gather is float32 only");
        if (row_bounds[s + 1] < row_bounds[s] || row_bounds[s + 1] - row_bounds[s] > S->rows)
            return fail(ctx, ARROW_ERR_ARG, "source %d owns %lld rows but its tile has %lld", s, (long long)(row_bounds[s + 1] - row_bounds[s]), (long long)S->rows);
        if (S->p == D->p) return fail(ctx, ARROW_ERR_ARG, "gather source and destination must not alias");
        ms.p[s] = S->p;
        ms.bound[s] = row_bounds[s];
    }
    ms.bound[n_src] = row_bounds[n_src];
    if (m->limit > row_bounds[n_src]) return fail(ctx, ARROW_ERR_ARG, "map reaches row %lld beyond the last source bound %lld", (long long)m->limit, (long long)row_bounds[n_src]);
    return gather_common(ctx, D, nullptr, ms, true, m, (flags & ARROW_ACCUMULATE) != 0);
}

int arrow_push_rows(arrow_ctx *ctx, const int *dst_bufs, const int64_t *item_bounds, int n_dst, int src_buf, int map) {
    CHECK_CTX(ctx);
    CHECK_POISON(ctx);
    DenseBuf *S = get_dense(ctx, src_buf);
    IdxMap *m = get_map(ctx, map);
    if (!S) return fail(ctx, ARROW_ERR_HANDLE, "bad dense handle %d", src_buf);
    if (!m) return fail(ctx, ARROW_ERR_HANDLE, "bad map handle %d", map);
    REFUSE_I32(ctx, S, "arrow_push_rows");
    REFUSE_B1(ctx, S, "arrow_push_rows");
    if (S->dtype != ARROW_F32) return fail(ctx, ARROW_ERR_UNSUPPORTED, "arrow_push_rows is float32 only");
    if (!dst_bufs || !item_bounds || n_dst < 1 || n_dst > MAX_SRC) return fail(ctx, ARROW_ERR_ARG, "need 1..%d destinations", MAX_SRC);
    if (m->limit > S->rows) return fail(ctx, ARROW_ERR_ARG, "map reaches row %lld, source has %lld rows", (long long)m->limit, (long long)S->rows);
    if (item_bounds[0] != 0 || item_bounds[n_dst] != m->n) return fail(ctx, ARROW_ERR_ARG, "item bounds must span [0, %lld]", (long long)m->n);
    MultiDst md;
    memset(&md, 0, sizeof md);
    md.n = n_dst;
    for (int d = 0; d < n_dst; ++d) {
        const int64_t cnt = item_bounds[d + 1] - item_bounds[d];
        if (cnt < 0) return fail(ctx, ARROW_ERR_ARG, "item bounds must not decrease");
        md.bound[d] = item_bounds[d];
        if (cnt == 0) { md.p[d] = nullptr; continue; }
        DenseBuf *D = get_dense(ctx, dst_bufs[d]);
        if (!D) return fail(ctx, ARROW_ERR_HANDLE, "bad destination handle %d", dst_bufs[d]);
        if (D->k != S->k) return fail(ctx, ARROW_ERR_ARG, "feature width mismatch in destination %d", d);
        REFUSE_I32(ctx, D, "arrow_push_rows");
        REFUSE_B1(ctx, D, "arrow_push_rows");
        if (D->dtype != ARROW_F32) return fail(ctx, ARROW_ERR_UNSUPPORTED, "arrow_push_rows is float32 only");
        if (cnt > D->rows) return fail(ctx, ARROW_ERR_ARG, "destination %d receives %lld rows but its region has %lld", d, (long long)cnt, (long long)D->rows);
        if (D->p == S->p) return fail(ctx, ARROW_ERR_ARG, "push source and destination must not alias");
        md.p[d] = D->p;
    }
    md.bound[n_dst] = item_bounds[n_dst];
    md.max_len = 0;
    if (ctx->push_interleave && n_dst > 1)
        for (int d = 0; d < n_dst; ++d) md.max_len = std::max<long long>(md.max_len, md.bound[d + 1] - md.bound[d]);
    const long long n_items = m->n;
    if (n_items == 0) return ARROW_OK;
    const int k = S->k;
    const bool vec = (k % 4 == 0);
    const int vpr = vec ? k / 4 : k;
    int g = 1;
    while (g < vpr && g < 32) g <<= 1;
    if (g > 8 && vpr <= 32) g = 8;
    const int threads = 256;
    const long long rows_per_cta = (threads / 32) * (32 / g);
    const long long want = ctx->push_ctas > 0 ? ctx->push_ctas : (long long)ctx->sm_count * 2;
    int grid = (int)std::max<long long>(1, std::min<long long>((n_items + rows_per_cta - 1) / rows_per_cta, want));
#define LAUNCH_PU(VT, GG) k_push_rows<VT, GG><<<grid, threads, 0, cur_stream(ctx)>>>(md, reinterpret_cast<const VT *>(S->p), m->p, n_items, vpr)
#define DISPATCH_PU(VT)                                                                                          \
    do {                                                                                                         \
        switch (g) {                                                                                             \
            case 1: LAUNCH_PU(VT, 1); break;                                                                     \
            case 2: LAUNCH_PU(VT, 2); break;                                                                     \
            case 4: LAUNCH_PU(VT, 4); break;                                                                     \
            case 8: LAUNCH_PU(VT, 8); break;                                                                     \
            case 16: LAUNCH_PU(VT, 16); break;                                                                   \
            default: LAUNCH_PU(VT, 32); break;                                                                   \
        }                                                                                                        \
    } while (0)
    if (vec) DISPATCH_PU(float4); else DISPATCH_PU(float);
#undef DISPATCH_PU
#undef LAUNCH_PU
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
    return ARROW_OK;
}

int arrow_reduce_rows(arrow_ctx *ctx, int dst_buf, int out_table, const int *src_bufs, int n_src, int64_t rows) {
    CHECK_CTX(ctx);
    CHECK_POISON(ctx);
    if (!src_bufs || n_src < 1 || n_src > MAX_SRC || rows < 0) return fail(ctx, ARROW_ERR_ARG, "need 1..%d sources", MAX_SRC);
    DenseBuf *D = dst_buf >= 0 ? get_dense(ctx, dst_buf) : nullptr;
    if (dst_buf >= 0 && !D) return fail(ctx, ARROW_ERR_HANDLE, "bad dense handle %d", dst_buf);
    REFUSE_I32(ctx, D, "arrow_reduce_rows");
    REFUSE_B1(ctx, D, "arrow_reduce_rows");
    if (D && D->dtype != ARROW_F32) return fail(ctx, ARROW_ERR_UNSUPPORTED, "arrow_reduce_rows is float32 only");
    PtrTable *OT = nullptr;
    if (out_table >= 0) {
        if (out_table >= (int)ctx->ptrtabs.size() || !ctx->ptrtabs[out_table].live)
            return fail(ctx, ARROW_ERR_HANDLE, "bad pointer table handle %d", out_table);
        OT = &ctx->ptrtabs[out_table];
        if (OT->n < rows) return fail(ctx, ARROW_ERR_ARG, "pointer table has %lld entries, %lld rows are reduced", (long long)OT->n, (long long)rows);
    }
    if (!D && !OT) return fail(ctx, ARROW_ERR_ARG, "no destination");
    if (D && D->rows < rows) return fail(ctx, ARROW_ERR_ARG, "destination has %lld rows, %lld are reduced", (long long)D->rows, (long long)rows);
    MultiSrc ms;
    memset(&ms, 0, sizeof ms);
    ms.n = n_src;
    int k = 0;
    for (int s2 = 0; s2 < n_src; ++s2) {
        DenseBuf *S = get_dense(ctx, src_bufs[s2]);
        if (!S) return fail(ctx, ARROW_ERR_HANDLE, "bad source handle %d", src_bufs[s2]);
        if (s2 == 0) k = S->k;
        if (S->k != k || (D && D->k != k) || (OT && OT->k != k)) return fail(ctx, ARROW_ERR_ARG, "feature width mismatch in source %d", s2);
        REFUSE_I32(ctx, S, "arrow_reduce_rows");
        REFUSE_B1(ctx, S, "arrow_reduce_rows");
        if (S->dtype != ARROW_F32) return fail(ctx, ARROW_ERR_UNSUPPORTED, "arrow_reduce_rows is float32 only");
        if (S->rows < rows) return fail(ctx, ARROW_ERR_ARG, "source %d has %lld rows, %lld are reduced", s2, (long long)S->rows, (long long)rows);
        ms.p[s2] = S->p;
    }
    if (rows == 0) return ARROW_OK;
    const bool vec = (k % 4 == 0);
    const int vpr = vec ? k / 4 : k;
    const long long total = rows * vpr;
    const int grid = (int)std::max<long long>(1, std::min<long long>((total + 255) / 256, (long long)ctx->sm_count * 4));
    float *const *tab = OT ? OT->p : nullptr;
    if (vec) k_reduce_rows<float4><<<grid, 256, 0, cur_stream(ctx)>>>(D ? reinterpret_cast<float4 *>(D->p) : nullptr, tab, ms, rows, vpr);
    else k_reduce_rows<float><<<grid, 256, 0, cur_stream(ctx)>>>(D ? D->p : nullptr, tab, ms, rows, vpr);
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
    return ARROW_OK;
}

// ---- IPC / peer barrier -------------------------------------------------------------------------
// cudaIpcGetMemHandle names the whole underlying allocation; a pointer that was sub-allocated inside a larger
// driver block must be re-based on the importing side.  The base comes from the driver (cuMemGetAddressRange),
// resolved at run time so the library does not link libcuda.
static long long ipc_base_offset(void *ptr) {
    typedef int (*range_fn)(unsigned long long *, size_t *, unsigned long long);
    static range_fn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void *h = dlopen("libcuda.so.1", RTLD_LAZY | RTLD_GLOBAL);
        if (h) fn = (range_fn)dlsym(h, "cuMemGetAddressRange_v2");
    }
    if (!fn) return 0;
    unsigned long long base = 0;
    size_t size = 0;
    if (fn(&base, &size, (unsigned long long)ptr) != 0) return 0;
    return (long long)((unsigned long long)ptr - base);
}

int arrow_ipc_export(arrow_ctx *ctx, int buf, void *handle) {
    CHECK_CTX(ctx);
    DenseBuf *d = get_dense(ctx, buf);
    if (!d || !d->owned) return fail(ctx, ARROW_ERR_HANDLE, "ipc export needs a tile this context allocated (handle %d)", buf);
    if (!handle) return fail(ctx, ARROW_ERR_ARG, "handle is null");
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "ipc handle size");
    cudaIpcMemHandle_t h;
    CUDA_TRY(ctx, cudaIpcGetMemHandle(&h, d->p));
    memset(handle, 0, ARROW_IPC_HANDLE_BYTES);
    memcpy(handle, &h, sizeof h);
    const long long off = ipc_base_offset(d->p);
    memcpy((char *)handle + 64, &off, sizeof off);
    return ARROW_OK;
}

int arrow_ipc_import(arrow_ctx *ctx, const void *handle, int64_t rows, int k, int *buf_out) {
    CHECK_CTX(ctx);
    if (!handle || !buf_out || rows < 0 || k < 1) return fail(ctx, ARROW_ERR_ARG, "bad ipc import arguments");
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, sizeof h);
    long long off = 0;
    memcpy(&off, (const char *)handle + 64, sizeof off);
    void *p = nullptr;
    CUDA_TRY(ctx, cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
    DenseBuf d;
    d.p = (float *)((char *)p + off);
    d.ipc_base = p;
    d.rows = rows;
    d.k = k;
    d.ipc = true;
    d.live = true;
    const int hh = new_slot(ctx->dense);
    ctx->dense[hh] = d;
    *buf_out = hh;
    return ARROW_OK;
}

int arrow_peer_barrier(arrow_ctx *ctx, const int *flag_bufs, int rank, int world) {
    CHECK_CTX(ctx);
    CHECK_POISON(ctx);
    if (!flag_bufs || world < 1 || world > MAX_SRC || rank < 0 || rank >= world) return fail(ctx, ARROW_ERR_ARG, "bad barrier arguments");
    PeerFlags pf;
    memset(&pf, 0, sizeof pf);
    for (int s = 0; s < world; ++s) {
        DenseBuf *d = get_dense(ctx, flag_bufs[s]);
        if (!d || (long long)d->rows * d->k < world) return fail(ctx, ARROW_ERR_HANDLE, "bad flag tile for rank %d", s);
        pf.p[s] = reinterpret_cast<unsigned int *>(d->p);
    }
    const long long timeout_clocks = ctx->barrier_timeout_ms * (long long)ctx->clock_khz;
    k_peer_barrier<<<1, 32, 0, cur_stream(ctx)>>>(pf, rank, world, ctx->barrier_epoch + ctx->cur_lane, ctx->dev_status, timeout_clocks);
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
    return ARROW_OK;
}

// ---- lanes: side streams ordered against the main stream with events ---------------------------------
static int lane_stream(arrow_ctx *ctx, int lane, cudaStream_t *out);

int arrow_set_lane(arrow_ctx *ctx, int lane) {
    CHECK_CTX(ctx);
    cudaStream_t st;
    int rc = lane_stream(ctx, lane, &st);          // creates the stream on first use
    if (rc != ARROW_OK) return rc;
    ctx->cur_lane = lane;
    return ARROW_OK;
}

static int lane_stream(arrow_ctx *ctx, int lane, cudaStream_t *out) {
    if (lane < 0 || lane >= ARROW_N_LANES) return fail(ctx, ARROW_ERR_ARG, "lane %d out of range", lane);
    if (lane == ARROW_LANE_MAIN) { *out = ctx->stream; return ARROW_OK; }
    if (!ctx->lanes[lane]) CUDA_TRY(ctx, cudaStreamCreateWithFlags(&ctx->lanes[lane], cudaStreamNonBlocking));
    *out = ctx->lanes[lane];
    return ARROW_OK;
}

int arrow_dense_h2d_lane(arrow_ctx *ctx, int lane, int buf, int64_t row0, int64_t rows, const void *host) {
    CHECK_CTX(ctx);
    DenseBuf *d = get_dense(ctx, buf);
    if (!d) return fail(ctx, ARROW_ERR_HANDLE, "bad dense handle %d", buf);
    if (!host || row0 < 0 || rows < 0 || row0 + rows > d->rows) return fail(ctx, ARROW_ERR_ARG, "h2d range outside tile");
    cudaStream_t st;
    int rc = lane_stream(ctx, lane, &st);
    if (rc != ARROW_OK) return rc;
    if (rows) CUDA_TRY(ctx, cudaMemcpyAsync(dense_row(d, row0), host, (size_t)rows * row_bytes(d->dtype, d->k), cudaMemcpyHostToDevice, st));
    return ARROW_OK;
}

int arrow_dense_d2h_lane(arrow_ctx *ctx, int lane, int buf, int64_t row0, int64_t rows, void *host) {
    CHECK_CTX(ctx);
    DenseBuf *d = get_dense(ctx, buf);
    if (!d) return fail(ctx, ARROW_ERR_HANDLE, "bad dense handle %d", buf);
    if (!host || row0 < 0 || rows < 0 || row0 + rows > d->rows) return fail(ctx, ARROW_ERR_ARG, "d2h range outside tile");
    cudaStream_t st;
    int rc = lane_stream(ctx, lane, &st);
    if (rc != ARROW_OK) return rc;
    if (rows) CUDA_TRY(ctx, cudaMemcpyAsync(host, dense_row(d, row0), (size_t)rows * row_bytes(d->dtype, d->k), cudaMemcpyDeviceToHost, st));
    return ARROW_OK;
}

int arrow_lane_wait(arrow_ctx *ctx, int waiting_lane, int signalling_lane) {
    CHECK_CTX(ctx);
    cudaStream_t w, sgn;
    int rc = lane_stream(ctx, waiting_lane, &w);
    if (rc != ARROW_OK) return rc;
    rc = lane_stream(ctx, signalling_lane, &sgn);
    if (rc != ARROW_OK) return rc;
    if (w == sgn) return ARROW_OK;
    cudaEvent_t &ev = ctx->lane_events[signalling_lane];
    if (!ev) CUDA_TRY(ctx, cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    CUDA_TRY(ctx, cudaEventRecord(ev, sgn));
    CUDA_TRY(ctx, cudaStreamWaitEvent(w, ev, 0));
    return ARROW_OK;
}

int arrow_event_record(arrow_ctx *ctx, int event, int lane) {
    CHECK_CTX(ctx);
    if (event < 0 || event >= ARROW_MAX_EVENTS) return fail(ctx, ARROW_ERR_ARG, "event %d out of range", event);
    cudaStream_t st;
    int rc = lane_stream(ctx, lane, &st);
    if (rc != ARROW_OK) return rc;
    if (!ctx->user_events[event]) CUDA_TRY(ctx, cudaEventCreateWithFlags(&ctx->user_events[event], cudaEventDisableTiming));
    CUDA_TRY(ctx, cudaEventRecord(ctx->user_events[event], st));
    return ARROW_OK;
}

int arrow_event_wait(arrow_ctx *ctx, int event, int lane) {
    CHECK_CTX(ctx);
    if (event < 0 || event >= ARROW_MAX_EVENTS) return fail(ctx, ARROW_ERR_ARG, "event %d out of range", event);
    if (!ctx->user_events[event]) return ARROW_OK;            // never recorded: nothing to wait for
    cudaStream_t st;
    int rc = lane_stream(ctx, lane, &st);
    if (rc != ARROW_OK) return rc;
    CUDA_TRY(ctx, cudaStreamWaitEvent(st, ctx->user_events[event], 0));
    return ARROW_OK;
}

int arrow_lane_sync(arrow_ctx *ctx, int lane) {
    CHECK_CTX(ctx);
    cudaStream_t st;
    int rc = lane_stream(ctx, lane, &st);
    if (rc != ARROW_OK) return rc;
    CUDA_TRY(ctx, cudaStreamSynchronize(st));
    int flag = 0;
    CUDA_TRY(ctx, cudaMemcpy(&flag, ctx->dev_status, sizeof(int), cudaMemcpyDeviceToHost));
    if (flag != 0) {
        ctx->poisoned = true;
        return fail(ctx, ARROW_ERR_CUDA, "device-side failure flag %d: a peer barrier timed out after %lld ms; the context is "
                    "poisoned (results after the time-out are racy) -- destroy it", flag, ctx->barrier_timeout_ms);
    }
    return ARROW_OK;
}

// ---- CUDA graphs: one host call per step ---------------------------------------------------------------
// Everything between begin and end is recorded instead of executed: launches on the main lane and on every lane that
// joined through arrow_lane_wait / arrow_event_wait (fork) and was joined back before the end.  Device-side state
// (tile tickets, barrier epochs) lives in device memory, so the recorded step can be replayed any number of times.
int arrow_graph_begin(arrow_ctx *ctx) {
    CHECK_CTX(ctx);
    CHECK_POISON(ctx);
    if (ctx->capturing) return fail(ctx, ARROW_ERR_ARG, "a capture is already in progress");
    CUDA_TRY(ctx, cudaStreamBeginCapture(ctx->stream, cudaStreamCaptureModeThreadLocal));
    ctx->capturing = true;
    ctx->capture_launches0 = ctx->launches;
    ctx->cur_lane = 0;
    return ARROW_OK;
}

int arrow_graph_end(arrow_ctx *ctx, int *graph_out) {
    CHECK_CTX(ctx);
    if (!ctx->capturing) return fail(ctx, ARROW_ERR_ARG, "no capture in progress");
    ctx->capturing = false;
    const int64_t recorded = ctx->launches - ctx->capture_launches0;
    ctx->launches = ctx->capture_launches0;                  // recorded, not executed
    cudaGraph_t g = nullptr;
    cudaError_t e = cudaStreamEndCapture(ctx->stream, &g);
    if (e != cudaSuccess || !g) {
        cudaGetLastError();
        return fail(ctx, ARROW_ERR_CUDA, "cudaStreamEndCapture: %s (was every side lane joined back into the main lane?)", cudaGetErrorString(e));
    }
    cudaGraphExec_t ex = nullptr;
    e = cudaGraphInstantiate(&ex, g, 0);
    cudaGraphDestroy(g);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return fail(ctx, ARROW_ERR_CUDA, "cudaGraphInstantiate: %s", cudaGetErrorString(e));
    }
    if (!graph_out) { cudaGraphExecDestroy(ex); return fail(ctx, ARROW_ERR_ARG, "graph_out is null"); }
    int h = -1;
    for (size_t i = 0; i < ctx->graphs.size(); ++i)
        if (!ctx->graphs[i]) { h = (int)i; break; }
    if (h < 0) { ctx->graphs.push_back(nullptr); ctx->graph_kernels.push_back(0); h = (int)ctx->graphs.size() - 1; }
    ctx->graphs[h] = ex;
    ctx->graph_kernels[h] = recorded;
    *graph_out = h;
    return ARROW_OK;
}

int arrow_graph_launch(arrow_ctx *ctx, int graph) {
    CHECK_CTX(ctx);
    CHECK_POISON(ctx);
    if (graph < 0 || graph >= (int)ctx->graphs.size() || !ctx->graphs[graph]) return fail(ctx, ARROW_ERR_HANDLE, "bad graph handle %d", graph);
    if (ctx->capturing) return fail(ctx, ARROW_ERR_ARG, "cannot launch a graph while capturing");
    CUDA_TRY(ctx, cudaGraphLaunch(ctx->graphs[graph], ctx->stream));
    ctx->launches += ctx->graph_kernels[graph];
    return ARROW_OK;
}

int arrow_graph_free(arrow_ctx *ctx, int graph) {
    CHECK_CTX(ctx);
    if (graph < 0 || graph >= (int)ctx->graphs.size() || !ctx->graphs[graph]) return fail(ctx, ARROW_ERR_HANDLE, "bad graph handle %d", graph);
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    cudaGraphExecDestroy(ctx->graphs[graph]);
    ctx->graphs[graph] = nullptr;
    return ARROW_OK;
}

// ---- host memory next to the GPU --------------------------------------------------------------------------
// On a two-socket HGX box GPUs 0-3 hang off socket 0 and 4-7 off socket 1: staging buffers that live on the other
// socket cross the inter-socket link on every copy.  These calls
// pin the calling thread to the CPUs of the GPU's NUMA node and place the pinned buffer there.
static int numa_node_of_device(int device) {
    char bus[32] = {0};
    if (cudaDeviceGetPCIBusId(bus, sizeof bus, device) != cudaSuccess) { cudaGetLastError(); return -1; }
    for (char *c = bus; *c; ++c) *c = (char)tolower(*c);
    char path[128];
    snprintf(path, sizeof path, "/sys/bus/pci/devices/%s/numa_node", bus);
    FILE *f = fopen(path, "r");
    if (!f) return -1;
    int node = -1;
    if (fscanf(f, "%d", &node) != 1) node = -1;
    fclose(f);
    return node;
}

int arrow_bind_thread_to_device_numa(int device, int *node_out, int *n_cpus_out) {
    if (device < 0) {                                    // undo: every CPU, default memory policy
        cpu_set_t all;
        CPU_ZERO(&all);
        for (int c = 0; c < CPU_SETSIZE; ++c) CPU_SET(c, &all);
        sched_setaffinity(0, sizeof all, &all);
        syscall(SYS_set_mempolicy, 0 /* MPOL_DEFAULT */, nullptr, 0);
        if (node_out) *node_out = -1;
        if (n_cpus_out) *n_cpus_out = 0;
        return ARROW_OK;
    }
    int node = numa_node_of_device(device);
    if (node_out) *node_out = node;
    if (n_cpus_out) *n_cpus_out = 0;
    if (node < 0) return ARROW_OK;                       // single-node machine or unknown topology: nothing to do
    char path[128];
    snprintf(path, sizeof path, "/sys/devices/system/node/node%d/cpulist", node);
    FILE *f = fopen(path, "r");
    if (!f) return ARROW_OK;
    char buf[4096] = {0};
    const size_t got = fread(buf, 1, sizeof buf - 1, f);
    fclose(f);
    buf[got] = 0;
    cpu_set_t set;
    CPU_ZERO(&set);
    int n = 0;
    for (char *tok = strtok(buf, ",\n"); tok; tok = strtok(nullptr, ",\n")) {
        int a = 0, b = 0;
        if (sscanf(tok, "%d-%d", &a, &b) == 2) { for (int c = a; c <= b && c < CPU_SETSIZE; ++c) { CPU_SET(c, &set); ++n; } }
        else if (sscanf(tok, "%d", &a) == 1 && a < CPU_SETSIZE) { CPU_SET(a, &set); ++n; }
    }
    if (n > 0 && sched_setaffinity(0, sizeof set, &set) == 0) {
        if (n_cpus_out) *n_cpus_out = n;
        unsigned long mask[16] = {0};
        if (node < (int)(sizeof mask * 8)) {
            mask[node / (8 * sizeof(unsigned long))] |= 1UL << (node % (8 * sizeof(unsigned long)));
            syscall(SYS_set_mempolicy, 1 /* MPOL_PREFERRED */, mask, sizeof mask * 8);
        }
    }
    return ARROW_OK;
}

int arrow_host_alloc_numa(size_t bytes, int device, void **ptr) {
    if (!ptr) return ARROW_ERR_ARG;
    *ptr = nullptr;
    const size_t page = 2u << 20;
    const size_t len = ((std::max<size_t>(bytes, 16) + page - 1) / page) * page;
    void *p = mmap(nullptr, len, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
    if (p == MAP_FAILED) return fail(nullptr, ARROW_ERR_NOMEM, "mmap(%zu) failed", len);
    madvise(p, len, MADV_HUGEPAGE);
    const int node = numa_node_of_device(device);
    if (node >= 0) {
        unsigned long mask[16] = {0};
        if (node < (int)(sizeof mask * 8)) {
            mask[node / (8 * sizeof(unsigned long))] |= 1UL << (node % (8 * sizeof(unsigned long)));
            syscall(SYS_mbind, p, len, 2 /* MPOL_BIND */, mask, sizeof mask * 8, 0);      // best effort
        }
    }
    memset(p, 0, len);                                   // first touch: pages materialise on the bound node
    cudaError_t e = cudaHostRegister(p, len, cudaHostRegisterPortable);
    if (e != cudaSuccess) {
        cudaGetLastError();
        munmap(p, len);
        return fail(nullptr, ARROW_ERR_NOMEM, "cudaHostRegister(%zu): %s", len, cudaGetErrorString(e));
    }
    {
        std::lock_guard<std::mutex> lk(g_numa_mu);
        g_numa_allocs[p] = len;
    }
    *ptr = p;
    return ARROW_OK;
}

// ---- timing -------------------------------------------------------------------------------------
int arrow_timer_start(arrow_ctx *ctx, int slot) {
    CHECK_CTX(ctx);
    if (slot < 0 || slot >= ARROW_MAX_TIMERS) return fail(ctx, ARROW_ERR_ARG, "timer slot %d", slot);
    Timer &t = ctx->timers[slot];
    if (!t.a) CUDA_TRY(ctx, cudaEventCreate(&t.a));
    if (!t.b) CUDA_TRY(ctx, cudaEventCreate(&t.b));
    CUDA_TRY(ctx, cudaEventRecord(t.a, ctx->stream));
    return ARROW_OK;
}

int arrow_timer_stop(arrow_ctx *ctx, int slot) {
    CHECK_CTX(ctx);
    if (slot < 0 || slot >= ARROW_MAX_TIMERS || !ctx->timers[slot].b) return fail(ctx, ARROW_ERR_ARG, "timer slot %d not started", slot);
    CUDA_TRY(ctx, cudaEventRecord(ctx->timers[slot].b, ctx->stream));
    return ARROW_OK;
}

int arrow_timer_elapsed_ms(arrow_ctx *ctx, int slot, float *ms) {
    CHECK_CTX(ctx);
    if (slot < 0 || slot >= ARROW_MAX_TIMERS || !ctx->timers[slot].b || !ms) return fail(ctx, ARROW_ERR_ARG, "timer slot %d not started", slot);
    CUDA_TRY(ctx, cudaEventSynchronize(ctx->timers[slot].b));
    CUDA_TRY(ctx, cudaEventElapsedTime(ms, ctx->timers[slot].a, ctx->timers[slot].b));
    return ARROW_OK;
}

int arrow_launch_count(arrow_ctx *ctx, int64_t *count) {
    if (!ctx || !count) return ARROW_ERR_ARG;
    *count = ctx->launches;
    return ARROW_OK;
}

// Lazy module loading (the CUDA default) loads a kernel at its first launch, and loading synchronises the context.  A
// kernel that spin-waits -- arrow_peer_barrier on one lane -- while another lane (or, with rank threads, another
// rank) launches a kernel for the first time therefore deadlocks until the barrier times out.  This runs every kernel
// the step of a given feature width can launch once, on tiny operands, before any barrier is in flight.
int arrow_preload_kernels(arrow_ctx *ctx, int k) {
    CHECK_CTX(ctx);
    if (k < 1) return fail(ctx, ARROW_ERR_ARG, "k must be positive");
    const int64_t n = 700;
    std::vector<int32_t> ip(n + 1), ix;
    std::vector<float> val;
    for (int64_t r = 0; r < n; ++r) {
        ip[r] = (int32_t)ix.size();
        const int len = (r == 3) ? 600 : 3;                       // one long row: the segmented kernels load too
        for (int j = 0; j < len; ++j) { ix.push_back((int32_t)((r * 7 + j) % n)); val.push_back(1.0f); }
        std::sort(ix.begin() + ip[r], ix.end());
        ix.erase(std::unique(ix.begin() + ip[r], ix.end()), ix.end());
        val.resize(ix.size());
    }
    ip[n] = (int32_t)ix.size();
    int csr = -1, x = -1, x2 = -1, c = -1, c2 = -1, map = -1, tab = -1, rc = ARROW_OK;
    std::vector<int64_t> ident(n);
    for (int64_t i = 0; i < n; ++i) ident[i] = i;
    std::vector<int32_t> which(n, 0);
    const int saved_kernel = ctx->tile_kernel, saved_lane = ctx->cur_lane;
    ctx->cur_lane = 0;
#define PRE(expr) do { if (rc == ARROW_OK) rc = (expr); } while (0)
    PRE(arrow_csr_upload(ctx, n, n, (int64_t)ix.size(), ip.data(), 4, ix.data(), 4, val.data(), &csr));
    PRE(arrow_dense_alloc(ctx, n, k, &x));
    PRE(arrow_dense_alloc(ctx, n, k, &x2));
    PRE(arrow_dense_alloc(ctx, n, k, &c));
    PRE(arrow_dense_alloc(ctx, n, k, &c2));
    PRE(arrow_map_upload(ctx, ident.data(), n, n, &map));
    if (rc == ARROW_OK) { const int tiles[1] = {c2}; rc = arrow_ptrtable_upload(ctx, tiles, 1, which.data(), ident.data(), n, &tab); }
    for (int tk = 0; tk < 2 && rc == ARROW_OK; ++tk) {
        ctx->tile_kernel = tk;
        for (int rpg = 1; rpg <= 2; ++rpg) {
            const int variant = ARROW_VARIANT_TILES | (rpg << 8);
            PRE(arrow_spmm(ctx, csr, x, c, -1, 0, variant));
            PRE(arrow_spmm(ctx, csr, x, c, -1, ARROW_ACCUMULATE, variant));
            PRE(arrow_spmm(ctx, csr, x, c, map, 0, variant));
            PRE(arrow_spmm(ctx, csr, x, c, map, ARROW_ACCUMULATE, variant));
            PRE(arrow_spmm_add(ctx, csr, x, c, c2, map, variant));
            PRE(arrow_spmm_ex(ctx, csr, x, x2, n / 2, c, -1, -1, -1, variant));
            PRE(arrow_spmm_ex(ctx, csr, x, x2, n / 2, -1, tab, -1, -1, variant));
            PRE(arrow_spmm_ex(ctx, csr, x, -1, 0, -1, tab, c, map, variant));
        }
    }
    ctx->tile_kernel = saved_kernel;
    PRE(arrow_gather_rows(ctx, c, x, map, 0));
    PRE(arrow_gather_rows(ctx, c, x, map, ARROW_ACCUMULATE));
    if (rc == ARROW_OK) {
        const int srcs[1] = {x};
        const int64_t bounds[2] = {0, n};
        PRE(arrow_gather_rows_multi(ctx, c, srcs, bounds, 1, map, 0));
        PRE(arrow_gather_rows_multi(ctx, c, srcs, bounds, 1, map, ARROW_ACCUMULATE));
        const int dsts[1] = {c};
        PRE(arrow_push_rows(ctx, dsts, bounds, 1, x, map));
        PRE(arrow_reduce_rows(ctx, c, -1, srcs, 1, n));
        PRE(arrow_reduce_rows(ctx, -1, tab, srcs, 1, n));
        PRE(arrow_dense_fill(ctx, c, 1.0f));
        // the barrier kernel against this context's own flag word (world of one): loads it, never waits
        const int flags[1] = {c};
        for (int lane = 0; lane < ARROW_N_LANES && rc == ARROW_OK; lane += ARROW_LANE_SIDE) {
            cudaStream_t st;
            rc = lane_stream(ctx, lane, &st);
            ctx->cur_lane = lane;
            if (lane) PRE(arrow_lane_wait(ctx, lane, 0));
            PRE(arrow_dense_fill(ctx, c, 0.0f));
            PRE(arrow_peer_barrier(ctx, flags, 0, 1));
            if (lane) PRE(arrow_lane_wait(ctx, 0, lane));
        }
    }
#undef PRE
    ctx->cur_lane = saved_lane;
    cudaStreamSynchronize(ctx->stream);
    for (int l = 1; l < ARROW_N_LANES; ++l)
        if (ctx->lanes[l]) cudaStreamSynchronize(ctx->lanes[l]);
    if (tab >= 0) arrow_ptrtable_free(ctx, tab);
    if (map >= 0) arrow_map_free(ctx, map);
    for (int h : {x, x2, c, c2}) if (h >= 0) arrow_dense_free(ctx, h);
    if (csr >= 0) arrow_csr_free(ctx, csr);
    // the barrier test bumped the epoch counters of a flag word that no longer exists: start clean
    cudaMemset(ctx->barrier_epoch, 0, ARROW_N_LANES * sizeof(unsigned int));
    return rc;
}

int arrow_l2_flush(arrow_ctx *ctx) {
    CHECK_CTX(ctx);
    const size_t bytes = (size_t)256 << 20;      // 256 MiB > 50 MB of L2
    if (!ctx->flush_buf) {
        CUDA_TRY(ctx, cudaMalloc(&ctx->flush_buf, bytes));
        ctx->flush_bytes = bytes;
    }
    k_fill<float><<<ctx->sm_count * 8, 256, 0, ctx->stream>>>((float *)ctx->flush_buf, 0.f, (long long)(ctx->flush_bytes / 4));
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
    return ARROW_OK;
}

}  // extern "C"
