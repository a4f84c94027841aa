// common.cuh -- context, error handling and small device helpers shared by every kernel file.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/dss_b200.h"

namespace dss {

void set_error(const char *fmt, ...);

#define DSS_CUDA_TRY(expr)                                                                      \
    do {                                                                                        \
        cudaError_t _e = (expr);                                                                \
        if (_e != cudaSuccess) {                                                                \
            dss::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__,    \
                           __LINE__);                                                           \
            return DSS_E_CUDA;                                                                  \
        }                                                                                       \
    } while (0)

#define DSS_REQUIRE(cond, msg)                                                                  \
    do {                                                                                        \
        if (!(cond)) {                                                                          \
            dss::set_error("invalid argument: %s (%s)", msg, #cond);                            \
            return DSS_E_INVALID;                                                               \
        }                                                                                       \
    } while (0)

#define DSS_LAUNCH_CHECK(ctx)                                                                   \
    do {                                                                                        \
        (ctx)->launches++;                                                                      \
        cudaError_t _e = cudaGetLastError();                                                    \
        if (_e != cudaSuccess) {                                                                \
            dss::set_error("kernel launch failed: %s (%s:%d)", cudaGetErrorString(_e),          \
                           __FILE__, __LINE__);                                                 \
            return DSS_E_CUDA;                                                                  \
        }                                                                                       \
    } while (0)

// grow-only scratch slots
enum BufId {
    BUF_SCAN_STATUS = 0,
    BUF_RECORDS,      // packed 32-byte splat records (2 x float4 per splat)
    BUF_TILE_COUNTS,  // per (view, tile) counts, then cursors
    BUF_TILE_OFFSETS, // exclusive offsets (+1)
    BUF_TILE_IDS,     // CSR id lists
    BUF_SELECT,       // radix-select histograms
    BUF_MISC,
    BUF_RS,
    BUF_GRADXY,
    BUF_ZRANGE,
    BUF_STATS,
    BUF_OCC_REC,      // compact tile-ordered {px,py,rx,ry} of the visible splats (occupancy backward)
    BUF_OCC_PLANES,   // zero-padded g-/g+ planes of the alpha gradient
    BUF_OCC_PARTS,    // work items per tile and their exclusive scan
    BUF_OCC_ITEMS,    // tile of every work item
    BUF_OCC_COUNTS,   // per-cell (pixel) counters of the occupancy binning (kept at zero between calls)
    BUF_OCC_IDS,      // packed splat id of every compact record
    BUF_TILE_ORDER,   // launch order of the forward tiles
    BUF_BIN_RECTS,    // packed tile rectangle + depth slice of every splat (count pass -> scatter pass)
    BUF_BIN_BLOCK_OFFSETS,  // fused route: every preprocess block's offset inside each tile-list bin it touched
    BUF_KNN_COUNTS,   // 3-D grid of the K-NN search: points per cell
    BUF_KNN_OFFSETS,  //   exclusive scan of the counts
    BUF_KNN_SORTED,   //   points in cell order {x, y, z, index}
    BUF_CAMERA,       // per-block fp64 partial sums of the camera gradients
    BUF_LIGHT,        // per-block fp64 partial sums of the light gradients
    BUF_REGULARISER,  // denoised normals (P,3) and per-cloud bounding boxes of the surface regularisers
    BUF_IMAGE_LOSS,   // per-block fp64 partial sums of the image loss, and the finish's block counter
    BUF_MESH_SCREEN,  // mesh rasterizer: screen-space vertices {x, y, z, 0} of a chunk of views
    BUF_MESH_OFFSETS, //   per (view, face) pixel-centre counts, then their exclusive 64-bit scan (+ total)
    BUF_MESH_RECTS,   //   per (view, face) pixel-index rectangle {column lo, row lo, width, 0}
    BUF_MESH_BLOCKS,  //   per-tile sums of the 64-bit scan
    BUF_MESH_KEYS,    //   per-pixel closest (depth, face) key
    BUF_COLOUR_FIXED, // deterministic colour backward: per-record 64-bit fixed-point sums and the call's scale
    BUF_CHAMFER,      // chamfer distance: fp64 per-block partials, then both directions' K = 1 rows (dist, index)
    BUF_PMD_STATE,    // point-mesh distance: face bounding box, grid parameters and the reference total
    BUF_PMD_TRIS,     //   the usable faces' vertices, 3 float4 per face
    BUF_PMD_COUNTS,   //   face references per grid cell
    BUF_PMD_OFFSETS,  //   exclusive scan of the counts
    BUF_PMD_REFS,     //   face indices in cell order
    NUM_BUFS
};

}  // namespace dss

namespace dss {
enum Stage {
    ST_PACK = 0, ST_PREPROCESS, ST_BIN_COUNT, ST_SCAN, ST_BIN_SCATTER, ST_RASTER_FWD, ST_VISIBILITY,
    ST_SEARCH_RADIUS, ST_OCC_BWD, ST_COLOUR_BWD, ST_ZBUF_BWD, ST_CHAIN, ST_GRID, ST_OCC_BIN, ST_KNN,
    ST_CAMERA_BWD, ST_LIGHT_BWD, NUM_STAGES
};
struct ProfPending {
    cudaEvent_t a, b;
    int stage;
    int closed;
};
}  // namespace dss

struct dss_ctx {
    int device;
    int sm_count;
    void *buf[dss::NUM_BUFS];
    size_t cap[dss::NUM_BUFS];
    int64_t launches;
    int64_t *h_pinned;  // small pinned host area for read-backs
    // optional per-stage device timing (CUDA events on the launch stream), see dss_profile_*
    int profiling;
    dss::ProfPending *pending;
    int n_pending, cap_pending;
    int open[8], n_open;
    int raster_stats;   // debug: accumulate raster work counters
    int raster_minb5;   // tuning (env DSS_RASTER_MINB=5): 5 resident CTAs/SM (48 registers) instead of 4 (64)
    int sync_forward;   // tuning (env DSS_SYNC_FORWARD=1): always wait for the tile-list size before the scatter
    int64_t tile_total_hint;   // tile-list size last seen in the mapped word: sizes the key buffer of the next call
    int64_t tile_cap_limit;    // testing (dss_debug_limit_tile_capacity): upper bound on the key buffer, 0 = none
    cudaStream_t side;      // second stream: independent backward work (colour scatter) overlaps the occupancy path
    cudaEvent_t ev_fork, ev_join;
    const void *occ_counts_ptr;   // BUF_OCC_COUNTS block known to be all zero (nullptr: unknown)
    size_t occ_counts_elems;
    int ns_override;    // tuning (env DSS_NS): number of depth slices of the forward tile lists, 0 = automatic
    int no_tile_order;  // tuning (env DSS_NO_TILE_ORDER=1): launch the raster tiles in index order
    int bin_no_rects;   // tuning (env DSS_BIN_NORECTS=1): the scatter pass derives the tile rectangles again
    int bin_direct;     // tuning (env DSS_BIN_DIRECT): tile binning with plain global atomics instead of per-block histograms
    double stage_ms[dss::NUM_STAGES];
    int64_t stage_calls[dss::NUM_STAGES];
};

namespace dss {

int ctx_reserve(dss_ctx *ctx, BufId id, size_t bytes, void **out);

// Scoped stage timer: records an event pair around the enclosed launches when profiling is on.
void prof_begin(dss_ctx *ctx, int stage, cudaStream_t st);
void prof_end(dss_ctx *ctx, cudaStream_t st);
struct StageScope {
    dss_ctx *ctx;
    cudaStream_t st;
    StageScope(dss_ctx *c, int stage, cudaStream_t s) : ctx(c), st(s) {
        if (ctx->profiling) prof_begin(ctx, stage, st);
    }
    ~StageScope() {
        if (ctx->profiling) prof_end(ctx, st);
    }
};

template <typename T>
inline int ctx_get(dss_ctx *ctx, BufId id, size_t count, T **out) {
    void *p = nullptr;
    int rc = ctx_reserve(ctx, id, count * sizeof(T), &p);
    *out = reinterpret_cast<T *>(p);
    return rc;
}

// Grid size of a grid-stride launch: one thread per item, at most per_sm blocks per SM, at least one block.
inline unsigned int grid_blocks(int64_t items, int threads, int sm_count, int per_sm) {
    int64_t b = (items + threads - 1) / threads;
    const int64_t cap = (int64_t)sm_count * per_sm;
    if (b > cap) b = cap;
    if (b < 1) b = 1;
    return (unsigned int)b;
}

// ---- device helpers -------------------------------------------------------------------------

// MUFU reciprocal (rcp.approx, denormals flushed to zero): never contracted or rewritten by the compiler.
__device__ __forceinline__ float rcp_approx(float x) {
    float y;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// Pixel index -> NDC centre, the reference's expression (DSS/csrc/rasterization_utils.cuh:8-11).
// No multiply-add pair, so immune to FMA contraction: int->float, add, IEEE divide, add.
__device__ __forceinline__ float pix_to_ndc(int i, int S) { return -1 + (2 * i + 1.0f) / S; }

// Same value without the division when S is a power of two: (2i+1)/S is then exact, so the single
// rounding of the fused multiply-add equals the single rounding of the reference's final add.
__device__ __forceinline__ float pix_to_ndc_fast(int i, int S, float inv_S, bool pow2) {
    return pow2 ? fmaf((float)(2 * i + 1), inv_S, -1.0f) : pix_to_ndc(i, S);
}

// Sign-preserving clamp of a denominator (DSS/csrc/rasterization_utils.cuh:37-43) with zero treated as
// positive like the Python helper (DSS/utils/mathHelper.py:10-14); see DESIGN.md hazard 11.
__device__ __forceinline__ float eps_denom(float d, float eps) {
    const float a = fmaxf(fabsf(d), eps);
    return d < 0.0f ? -a : a;
}

// Order-preserving float <-> int map: integer atomicMin / atomicMax then give float extremes in any order.
__device__ __forceinline__ int f2ord(float f) {
    const int i = __float_as_int(f);
    return i >= 0 ? i : i ^ 0x7fffffff;
}
__device__ __forceinline__ float ord2f(int i) { return __int_as_float(i >= 0 ? i : i ^ 0x7fffffff); }

// sum of acc[k] over the block (blockDim.x a multiple of 32, at most 256) in a fixed order; thread k < K
// returns sum k, the others 0
template <int K>
__device__ __forceinline__ double block_sum(const double (&acc)[K], double (*sPart)[K]) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < K; ++k) {
        double v = acc[k];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0) sPart[warp][k] = v;
    }
    __syncthreads();
    double v = 0.0;
    if (threadIdx.x < K)
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) v += sPart[w][threadIdx.x];
    return v;
}

// Pass 2 of the fixed-order fp64 sums (camera and light gradients, image loss) over partials (N, nl, blocks, SUMS).
// Block (l, m) sums slice l of output row m -- view m (per_view: cameras, per-view lights, image loss; its partials in
// block order), or, for the only row of shared lights, the partials of view 0 in block order, then view 1, ....  Each
// thread adds a fixed, strided subset, block_sum combines them in a fixed order, rows(totals, l, m, k) writes the
// outputs.
template <int SUMS, class Rows>
__global__ void __launch_bounds__(256) grad_finish_kernel(const double *partials, int blocks, int n_views, int per_view,
                                                          const Rows rows) {
    __shared__ double sPart[8][SUMS];
    __shared__ double sTot[SUMS];
    const int l = blockIdx.x, m = blockIdx.y, nl = gridDim.x, k = threadIdx.x;
    const int n0 = per_view ? m : 0;
    const int64_t count = (int64_t)(per_view ? 1 : n_views) * blocks;
    double acc[SUMS];
#pragma unroll
    for (int j = 0; j < SUMS; ++j) acc[j] = 0.0;
    for (int64_t e = threadIdx.x; e < count; e += blockDim.x) {
        const int64_t n = n0 + e / blocks, b = e % blocks;
        const double *p = partials + ((n * nl + l) * blocks + b) * SUMS;
#pragma unroll
        for (int j = 0; j < SUMS; ++j) acc[j] += p[j];
    }
    const double v = block_sum(acc, sPart);
    if (k < SUMS) sTot[k] = v;
    __syncthreads();
    rows(sTot, l, m, k);
}

struct ViewRange {
    int64_t first;
    int64_t count;
};

__device__ __forceinline__ ViewRange view_range(const int64_t *first_idx, const int64_t *num_points, int n,
                                                int64_t P0_shared) {
    ViewRange r;
    if (first_idx == nullptr) {
        r.first = (int64_t)n * P0_shared;
        r.count = P0_shared;
    } else {
        r.first = first_idx[n];
        r.count = num_points[n];
    }
    return r;
}

}  // namespace dss
