// occ_backward.cu -- occupancy ("fast") backward: point <- pixel gather over tile-sorted compact records.
//
// Replaces the fast branch of EllipticalRasterizer.backward (DSS/core/rasterizer.py:845-972) and
// RasterizePointsBackwardCudaFastKernel (DSS/csrc/rasterize_points_backward.cu:30-212).  The reference
// scatters pixel -> point with two float atomics per (pixel, point) pair after building an FRNN grid with
// per-view host loops.  Here (all on the device, no host round trip, no atomics, deterministic):
//
//   occ_planes   alpha gradient -> two zero-padded planes per view in NDC-index orientation: g- = min(g, 0)
//                (acts on the whole search disc) and g+ = max(g, 0) (acts inside the splat's bbox only,
//                rasterize_points_backward.cu:161-168)
//   occ_bin      visible splats -> the pixel cells of 32x32-pixel tiles by centre (count / scan / scatter; the
//                fused forward does the count); the scatter writes COMPACT records {px, py, rx, ry} + ids in
//                tile order, pixel-ordered inside a tile, so everything downstream reads contiguous memory
//   select x4    exact lower median of the visible radii per view (radix select) over the compact records
//                (rasterizer.py:888) -> search radius r_n
//   occ_tile     one CTA per (tile, chunk of its list): the (32 + 2R)^2 windows of both planes and the
//                chunk's records are staged in shared memory by the TMA engine (cp.async.bulk, one row per
//                copy, completion on an mbarrier); lanes own PAIRS of window columns and walk the rows with
//                one reciprocal per pair, the x half of the sum is factored (sum_rows dx*w = dx * sum_rows w).
#include <math_constants.h>

#include "common.cuh"
#include "kernels.cuh"

namespace dss {

constexpr int OCC_ITEM = 128;           // splats per work item (= records staged per TMA copy)
constexpr int OCC_GROUP = 4;            // consecutive items handed to one CTA
constexpr int OCC_SLACK = 64;           // floats of slack behind each staged plane / the column table
constexpr int OCC_RBOX_MAX = 40;        // largest window halo the tile kernel stages (2 x 2 planes <= ~200 KB)

// ---------------------------------------------------------------------------------------------
// planes: (N, 2, Hp, W) floats, plane 0 = min(g, 0) (and NaN), plane 1 = max(g, 0); element (y, x) holds NDC-index pixel
// (yi, xi) = (y - PAD, x - PAD), i.e. image row S-1-yi, col S-1-xi (rasterize_points_backward.cu:100-104);
// zero outside the image so that border windows need no bounds tests.  One block row per plane row: occ_backward
// requires Hp <= 65535 (gridDim.y).
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
occ_planes_kernel(const float *__restrict__ grad, int pix_stride, int pix_offset, int S, int PAD, int W, int Hp,
                  float *__restrict__ planes) {
    const int n = blockIdx.z, y = blockIdx.y;
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= W) return;
    const int yi = y - PAD, xi = x - PAD;
    float g = 0.0f;
    if (yi >= 0 && yi < S && xi >= 0 && xi < S)
        g = __ldg(grad + (((int64_t)n * S + (S - 1 - yi)) * S + (S - 1 - xi)) * pix_stride + pix_offset);
    float *p = planes + (((int64_t)n * 2) * Hp + y) * W + x;
    // a NaN goes to g- (fminf would drop it): the reference adds it to every point whose disc holds the pixel
    p[0] = isnan(g) ? g : fminf(g, 0.0f);
    p[(int64_t)Hp * W] = fmaxf(g, 0.0f);
}

// The id a compact record carries to the tile kernel's store: the packed id, or -1 for a splat behind the camera,
// which gets no gradient (rasterize_points_backward.cu:145) but stays binned, so that the bins match the counts.
__device__ __forceinline__ int32_t occ_store_id(int64_t p, float z) { return z < 0.0f ? -1 : (int32_t)p; }

// ---------------------------------------------------------------------------------------------
// Bin the visible splats by the PIXEL that contains their (clamped) centre (occ_cell, kernels.cuh): one entry per
// splat, so the lists are bounded by P and no host round trip is needed.  A tile's compact list comes out ordered by
// pixel row, then column.  Consecutive splats of a list then sit in the same or the
// next pixel -- the splats a warp of the tile kernel works on together read (nearly) the same shared-memory rows and
// columns, which turns its 4-way bank conflicts into broadcasts.  Two million bins per 8 views do not fit a block
// histogram: plain global atomics (1.5M visible splats over 0.5M occupied cells -- no hot spots).  PASS 0 counts;
// PASS 1 claims its slot by counting the same counter back down to zero, so the counters are clean again for the
// next call, and scatters the compact records.  Slots are int32: occ_backward requires Ptot < INT32_MAX.
// ---------------------------------------------------------------------------------------------
template <int PASS>
__global__ void __launch_bounds__(256)
occ_cellbin_kernel(const float4 *__restrict__ rec, const uint8_t *__restrict__ visible,
                   const int64_t *__restrict__ first_idx, const int64_t *__restrict__ num_points, int64_t P0_shared,
                   int S, int OB, int32_t *__restrict__ counters, const int32_t *__restrict__ offsets,
                   float4 *__restrict__ crec, int32_t *__restrict__ cids) {
    const int n = blockIdx.y;
    const ViewRange vr = view_range(first_idx, num_points, n, P0_shared);
    // four independent points per thread and trip: the visibility bytes, then the records of the visible ones, are
    // requested together (one point at a time, the kernel waits on each dependent load in turn)
    constexpr int U = 4;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i0 < vr.count; i0 += U * stride) {
        bool vis[U];
        float4 A[U];
        float ry[U];
#pragma unroll
        for (int j = 0; j < U; ++j) {
            const int64_t i = i0 + j * stride;
            vis[j] = i < vr.count && visible[vr.first + i] != 0;
        }
#pragma unroll
        for (int j = 0; j < U; ++j) {
            if (vis[j]) {
                const int64_t p = vr.first + i0 + j * stride;
                A[j] = __ldg(&rec[2 * p]);
                if (PASS == 1) ry[j] = __ldg(&rec[2 * p + 1]).x;
            }
        }
#pragma unroll
        for (int j = 0; j < U; ++j) {
            if (!vis[j]) continue;
            const int64_t p = vr.first + i0 + j * stride;
            const int64_t cell = occ_cell(n, OB, centre_pixel(A[j].x, S), centre_pixel(A[j].y, S));
            if (PASS == 0) {
                atomicAdd(&counters[cell], 1);
            } else {
                const int slot = offsets[cell] + atomicSub(&counters[cell], 1) - 1;
                crec[slot] = make_float4(A[j].x, A[j].y, A[j].w, ry[j]);
                cids[slot] = occ_store_id(p, A[j].z);
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// Search radius: radii_s * lower median of the flattened (rx, ry) of the view's visible points
// (rasterizer.py:888, torch.median = element (m-1)/2 of the ascending sort of m = 2 n_vis values).
// Exact 4-pass (8 bits each, MSB first) radix select on the order-preserving uint image of the floats.
// hist layout: (N, 4, 256) uint32.  Each block first re-derives the prefix chosen by the previous
// passes from their (complete) histograms -- 256-bin scans, negligible -- so no host involvement.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned int float_key(float f) {
    const unsigned int b = __float_as_uint(f);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float key_float(unsigned int k) {
    const unsigned int b = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
    return __uint_as_float(b);
}

// Walk histograms of passes [0, upto) and return (prefix, remaining rank).  Executed by one warp.
__device__ void select_resolve(const unsigned int *hist_n, int upto, unsigned int &prefix,
                               unsigned long long &rank, unsigned long long &total) {
    const int lane = threadIdx.x & 31;
    prefix = 0;
    rank = 0;
    total = 0;
    for (int pass = 0; pass < upto; ++pass) {
        const unsigned int *h = hist_n + pass * 256;
        // each lane owns 8 consecutive bins
        unsigned int c[8];
        unsigned long long s = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            c[j] = h[lane * 8 + j];
            s += c[j];
        }
        unsigned long long incl = s;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const unsigned long long t = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d) incl += t;
        }
        const unsigned long long tot = __shfl_sync(0xffffffffu, incl, 31);
        if (pass == 0) {
            total = tot;
            rank = (tot > 0) ? (tot - 1) / 2 : 0;  // lower median
        }
        unsigned long long excl = incl - s;
        // find the bin containing `rank`
        int found = -1;
        unsigned long long found_excl = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            if (found < 0 && rank >= excl && rank < excl + c[j]) {
                found = lane * 8 + j;
                found_excl = excl;
            }
            excl += c[j];
        }
        const unsigned int who = __ballot_sync(0xffffffffu, found >= 0);
        int digit = 0;
        unsigned long long dexcl = 0;
        if (who) {
            const int src = __ffs(who) - 1;
            digit = __shfl_sync(0xffffffffu, found, src);
            dexcl = __shfl_sync(0xffffffffu, found_excl, src);
        }
        prefix = (prefix << 8) | (unsigned int)digit;
        rank -= dexcl;
    }
}

// Record sources of one histogram pass (`pass` travels with the source, so that every instantiation keeps the parameter
// layout of the kernel it replaced).  range(n, ...) gives view n's record indices [beg, end); load(i, rx, ry) reads
// record i's radii and returns false for a record that does not count.
// Packed records (or, rec == null, the (P,2) radii) of the view's slots, filtered by the visibility bytes.
struct SelectPacked {
    using Index = int64_t;
    const float4 *rec;
    const float *radii;
    const uint8_t *visible;
    const int64_t *first_idx, *num_points;
    int64_t P0_shared;
    int pass;
    __device__ __forceinline__ void range(int n, int64_t &beg, int64_t &end) const {
        const ViewRange vr = view_range(first_idx, num_points, n, P0_shared);
        beg = vr.first;
        end = vr.first + vr.count;
    }
    __device__ __forceinline__ bool load(int64_t p, float &rx, float &ry) const {
        if (!visible[p]) return false;
        if (rec) {
            rx = __ldg(&rec[2 * p]).w;
            ry = __ldg(&rec[2 * p + 1]).x;
        } else {
            rx = radii[p * 2];
            ry = radii[p * 2 + 1];
        }
        return true;
    }
};
// The compact records {px, py, rx, ry} of the visible splats, contiguous per view:
// [tile_offsets[n*nc], tile_offsets[(n+1)*nc]) with nc cells per view.  nc and the record indices are int:
// occ_backward requires OB*OB*OCC_CELLS <= INT32_MAX and Ptot < INT32_MAX.
struct SelectCompact {
    using Index = int;
    const float4 *crec;
    const int32_t *tile_offsets;
    int nc;
    int pass;
    __device__ __forceinline__ void range(int n, int &beg, int &end) const {
        beg = __ldg(&tile_offsets[(int64_t)n * nc]);
        end = __ldg(&tile_offsets[(int64_t)(n + 1) * nc]);
    }
    __device__ __forceinline__ bool load(int i, float &rx, float &ry) const {
        const float4 c = __ldg(&crec[i]);
        rx = c.z;
        ry = c.w;
        return true;
    }
};

// One radix-select pass over the radii of view blockIdx.y: the keys that match the prefix chosen by the earlier passes
// are counted by their next 8 bits in shared memory, then added to the view's histogram of this pass.
template <class Src>
__global__ void __launch_bounds__(256) select_hist_kernel(const __grid_constant__ Src src, unsigned int *__restrict__ hist) {
    __shared__ unsigned int s_hist[256];
    __shared__ unsigned int s_prefix;
    const int n = blockIdx.y, pass = src.pass;
    unsigned int *hist_n = hist + (int64_t)n * 4 * 256;
    s_hist[threadIdx.x] = 0;
    if (threadIdx.x < 32) {
        unsigned int prefix;
        unsigned long long rank, total;
        select_resolve(hist_n, pass, prefix, rank, total);
        if (threadIdx.x == 0) s_prefix = prefix;
    }
    __syncthreads();
    const unsigned int prefix = s_prefix;
    const int shift = 24 - 8 * pass;
    typename Src::Index beg, end;
    src.range(n, beg, end);
    for (typename Src::Index i = beg + blockIdx.x * blockDim.x + threadIdx.x; i < end; i += gridDim.x * blockDim.x) {
        float rx, ry;
        if (!src.load(i, rx, ry)) continue;
        const unsigned int kx = float_key(rx), ky = float_key(ry);
        if (pass == 0 || (kx >> (shift + 8)) == prefix) atomicAdd(&s_hist[(kx >> shift) & 255u], 1u);
        if (pass == 0 || (ky >> (shift + 8)) == prefix) atomicAdd(&s_hist[(ky >> shift) & 255u], 1u);
    }
    __syncthreads();
    const unsigned int v = s_hist[threadIdx.x];
    if (v) atomicAdd(&hist_n[pass * 256 + threadIdx.x], v);
}

__global__ void select_final_kernel(const unsigned int *__restrict__ hist, float radii_s, float *__restrict__ rs) {
    const int n = blockIdx.x;
    unsigned int prefix;
    unsigned long long rank, total;
    select_resolve(hist + (int64_t)n * 4 * 256, 4, prefix, rank, total);
    if (threadIdx.x == 0) rs[n] = (total > 0) ? key_float(prefix) * radii_s : 0.0f;
}

int search_radius(dss_ctx *ctx, const float4 *rec, const float *radii, const uint8_t *visible,
                  const int64_t *first_idx, const int64_t *num_points, int N, int64_t P0, float radii_s,
                  float *rs, cudaStream_t st) {
    if (N <= 0) return DSS_OK;
    unsigned int *hist = nullptr;
    int rc = ctx_get(ctx, BUF_SELECT, (size_t)N * 4 * 256, &hist);
    if (rc) return rc;
    StageScope prof(ctx, ST_SEARCH_RADIUS, st);
    DSS_CUDA_TRY(cudaMemsetAsync(hist, 0, (size_t)N * 4 * 256 * sizeof(unsigned int), st));
    if (P0 > 0) {
        dim3 grid(grid_blocks(P0, 256, ctx->sm_count, 4), N);
        for (int pass = 0; pass < 4; ++pass) {
            select_hist_kernel<<<grid, 256, 0, st>>>(SelectPacked{rec, radii, visible, first_idx, num_points, P0, pass}, hist);
            DSS_LAUNCH_CHECK(ctx);
        }
    }
    select_final_kernel<<<N, 32, 0, st>>>(hist, radii_s, rs);
    DSS_LAUNCH_CHECK(ctx);
    return DSS_OK;
}

// ---------------------------------------------------------------------------------------------
// TMA (bulk async copy) + mbarrier helpers: raw PTX, sm_90+ encoding, issued by single threads.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_copy_g2s(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
                 "l"(src), "r"(bytes), "r"(bar)
                 : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    return ok != 0;
}
// bounded wait: a lost transaction traps (surfaces as a launch error) instead of hanging the device
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    unsigned int spins = 0;
    while (!mbar_try_wait(bar, parity)) {
        if (++spins > (1u << 24)) __trap();
    }
}

__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// 1.0f if a <= b else 0.0f (one FSET instruction); NaN -> 0
__device__ __forceinline__ float set_le(float a, float b) {
    float y;
    asm("set.le.f32.f32 %0, %1, %2;" : "=f"(y) : "f"(a), "f"(b));
    return y;
}

// Column-pair arithmetic.  sm_90 has no packed FP32 instructions, so each pair is two scalar ops; the _rn
// intrinsics are never contracted into FMAs, which keeps every rounding step of the row walk explicit.
__device__ __forceinline__ float2 add2_rn(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 mul2_rn(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fma2_rn(float2 a, float2 b, float2 c) {
    return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}

// ---------------------------------------------------------------------------------------------
// Work decomposition of the tile kernel.  A tile's list is cut into `parts` work items of <= OCC_ITEM splats
// (occ_parts -> exclusive scan -> occ_items writes the tile of every item).  Items are handed to the persistent
// CTAs in groups of OCC_GROUP consecutive items, round-robin, so that a CTA usually keeps the staged window for
// a few items and every CTA sees a mix of views (their windows, hence costs, differ).
// ---------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ int occ_hh(float r, int S) {
    // half-width H of the per-splat pixel window: pixel centres cx + 0.5 + k around a point at cx + f, f in [0,1),
    // lie within r (pixels) only for |k| <= floor(r + 1/2); 1e-3 absorbs the rounding of floor() at pixel borders
    return (int)floorf(r * 0.5f * (float)S + 0.5f + 1e-3f);
}
__host__ __device__ __forceinline__ bool occ_fits(float r, int S, int R_box) {
    if (!(r >= 0.0f) || !(r < 4.0f) || R_box <= 0) return false;
    return occ_hh(r, S) + 1 <= R_box;
}

__global__ void __launch_bounds__(256)
occ_parts_kernel(const int32_t *__restrict__ tile_offsets, const float *__restrict__ rs, int nt_view, int64_t nt,
                 int S, int R_box, int32_t *__restrict__ parts) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t > nt) return;
    int p = 0;
    if (t < nt && occ_fits(rs[t / nt_view], S, R_box))
        p = (tile_offsets[(t + 1) * OCC_CELLS] - tile_offsets[t * OCC_CELLS] + OCC_ITEM - 1) / OCC_ITEM;
    parts[t] = p;   // parts[nt] = 0 so that the scan's last entry is the total
}

// Tile numbers (item_tile) and item numbers (part_off) are int32: occ_backward requires its bound on the items,
// max_items = Ptot / OCC_ITEM + nt + 1, below INT32_MAX.
__global__ void __launch_bounds__(256)
occ_items_kernel(const int32_t *__restrict__ part_off, int64_t nt, int32_t *__restrict__ item_tile) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nt) return;
    for (int i = part_off[t]; i < part_off[t + 1]; ++i) item_tile[i] = (int32_t)t;
}

struct OccTileArgs {
    const float4 *crec;          // compact tile-ordered records {px, py, rx, ry}
    const int32_t *cids;         // packed splat id of every compact record (occ_store_id: -1 behind the camera)
    const int32_t *tile_offsets; // (N*OB*OB*OCC_CELLS + 1) cell offsets: list of tile t (ordered by pixel) =
                                 // [tile_offsets[t*OCC_CELLS], tile_offsets[(t+1)*OCC_CELLS])
    const int32_t *part_off;     // (N*OB*OB + 1) exclusive scan of the items per tile; last = number of items
    const int32_t *item_tile;    // tile (n*OB*OB + tile) of every item
    int *group_counter;          // next group of items to hand out (zero at launch)
    const float *rs;             // (N,) search radius
    const float *planes;         // (N, 2, Hp, W)
    float2 *grad_xy;             // (P,) out
    int S, OB, R_box, side, W, Hp;
    int64_t nt;
};

// Everything the consumers need to know about a staged item (written by the producer warp)
struct OccItem {
    int cnt;        // splats in this item; < 0: no more work
    int beg;        // first compact record
    int wbuf;       // which window buffer holds the tile's planes
    int tx, ty;     // tile coordinates
    int hh;         // window half-width of the view
    float r2;       // squared search radius
    int pad;
};

// Row walk for one batch of splats.  A lane owns PPL pairs of adjacent window columns of its splat (pair s = columns
// 2*(s*LPS + gl) + {0,1}); all lanes walk the rows j0..j1 together.  Per pair and row: one LDS.64, d2 of each column
// with one scalar FMA, ONE reciprocal for both (1/(a*b), then *b and *a), the disc test as a 0/1 factor, and per
// column two accumulations:  sw += w,  swy += w*dy  (the x half is factored: sum_rows dx*w = dx * sum_rows w).
// CENTRE rows (those the splat's own bbox can reach) additionally clamp d2 at 1e-10 (the pixel under the point,
// rasterization_utils.cuh:37-43) and add the positive gradients inside the bbox
// (rasterize_points_backward.cu:161-168) as g+ * colmask * rowmask.
template <int LPS, int PPL, bool CENTRE, bool POW2>
__device__ __forceinline__ void occ_rows(int j0, int j1, const float *__restrict__ gm, const float *__restrict__ gp,
                                         const float *__restrict__ yf_tab, const int side, float2 &yf2,
                                         const float2 pix2, const float2 npy2, const float ry, const float r2,
                                         const float2 (&dx2)[PPL], const float2 (&cmask)[PPL], float2 (&sw)[PPL],
                                         float2 (&swy)[PPL]) {
    gm += j0 * side;
    gp += j0 * side;
    for (int j = j0; j < j1; ++j) {
        if (POW2) {
            yf2 = add2_rn(yf2, pix2);          // exact: multiples of 1/S (see occ_tile_kernel)
        } else {
            const float yf = yf_tab[j];
            yf2 = make_float2(yf, yf);
        }
        const float2 dy2 = add2_rn(yf2, npy2);
        // dist2 = dx*dx + dy*dy as the reference's kernel evaluates it (nvcc: FMUL dy*dy, then FFMA dx*dx + that --
        // checked in the SASS of rasterize_points_backward.cu:150): the same rounding, hence the same disc membership
        const float2 dysq2 = mul2_rn(dy2, dy2);
        float2 rowm2 = make_float2(0.f, 0.f);
        if (CENTRE) {
            const float m = set_le(fabsf(dy2.x), ry);
            rowm2 = make_float2(m, m);
        }
#pragma unroll
        for (int s = 0; s < PPL; ++s) {
            float2 g = *reinterpret_cast<const float2 *>(gm + s * 2 * LPS);
            const float2 d2 = fma2_rn(dx2[s], dx2[s], dysq2);                // fma(dx, dx, dy*dy)
            const float2 in = make_float2(set_le(d2.x, r2), set_le(d2.y, r2));   // rasterize_points_backward.cu:156
            float2 dc = d2;
            if (CENTRE) {
                dc.x = fmaxf(d2.x, 1e-10f);
                dc.y = fmaxf(d2.y, 1e-10f);
                const float2 gpv = *reinterpret_cast<const float2 *>(gp + s * 2 * LPS);
                g = fma2_rn(gpv, mul2_rn(cmask[s], rowm2), g);            // g- and g+ never both non-zero
            }
            const float ip = rcp_approx(dc.x * dc.y);
            const float2 inv = make_float2(ip * dc.y, ip * dc.x);                // 1/dc.x, 1/dc.y
            const float2 w = mul2_rn(mul2_rn(g, inv), in);                 // g / max(d2, 1e-10) inside the disc
            sw[s] = add2_rn(sw[s], w);
            swy[s] = fma2_rn(w, dy2, swy[s]);
        }
        gm += side;
        gp += side;
    }
}

// One staged item: `cnt` splats of one tile.  Warp w takes batches w, w + 8, ...; a batch is 32 / LPS splats.
template <int LPS, int PPL, bool POW2, int NCONS>
__device__ __forceinline__ void occ_item(const OccTileArgs &a, const OccItem &it, const float *__restrict__ s_gm,
                                         const float *__restrict__ s_gp, const float *__restrict__ s_xf,
                                         const float *__restrict__ s_yf, const float4 *__restrict__ s_rec, int warp,
                                         int lane) {
    constexpr int GROUPS = 32 / LPS;
    constexpr unsigned FULL = 0xffffffffu;
    const int S = a.S, side = a.side;
    const int grp = lane / LPS, gl = lane - grp * LPS;
    const int Hh = it.hh, Wwin = 2 * Hh + 1;
    const int wx0 = it.tx * OCC_TILE - a.R_box, wy0 = it.ty * OCC_TILE - a.R_box;
    const float half_S = 0.5f * (float)S;
    const float pixf = 2.0f / (float)S;
    const float2 pix2 = make_float2(pixf, pixf);
    const float r2 = it.r2;
    for (int b = warp; b * GROUPS < it.cnt; b += NCONS) {
        const int k = b * GROUPS + grp;
        const bool have = k < it.cnt;
        const float4 rc = s_rec[have ? k : 0];
        const float px = rc.x, py = rc.y, rx = rc.z, ry = rc.w;
        // the id is only needed for the final store: issue the load now so that its latency hides behind the rows
        const int id = (have && gl == 0) ? __ldg(&a.cids[it.beg + k]) : 0;
        // centre pixel (this tile's by construction; the clamp only absorbs points outside the image) and the
        // window origin in staged coordinates, shifted left to an even column (8-byte aligned LDS.64)
        const int cx = min(max(centre_pixel(px, S), it.tx * OCC_TILE), it.tx * OCC_TILE + OCC_TILE - 1);
        const int cy = min(max(centre_pixel(py, S), it.ty * OCC_TILE), it.ty * OCC_TILE + OCC_TILE - 1);
        const int ox = (cx - Hh - wx0) & ~1, oy = cy - Hh - wy0;
        // rows the splat's own bbox can reach (+1 for rounding), at least the 3 rows around the point
        int bh = have ? min(Hh, (int)fminf(ceilf(ry * half_S) + 1.0f, 4096.0f)) : 0;
        bh = max(__reduce_max_sync(FULL, bh), min(Hh, 1));
        const int jc0 = Hh - bh, jc1 = Hh + bh + 1;
        const float2 npy2 = make_float2(-py, -py);
        float2 dx2[PPL], cmask[PPL], sw[PPL], swy[PPL];
        const float *xfp = s_xf + ox + 2 * gl;
#pragma unroll
        for (int s = 0; s < PPL; ++s) {
            const float2 xf = *reinterpret_cast<const float2 *>(xfp + s * 2 * LPS);
            const float dx0 = xf.x - px, dx1 = xf.y - px;
            dx2[s] = make_float2(dx0, dx1);
            cmask[s] = make_float2(set_le(fabsf(dx0), rx), set_le(fabsf(dx1), rx));
            sw[s] = make_float2(0.f, 0.f);
            swy[s] = make_float2(0.f, 0.f);
        }
        const float yfm1 = s_yf[oy] - pixf;                  // row -1 (POW2: exact)
        float2 yf2 = make_float2(yfm1, yfm1);
        const int off = oy * side + ox + 2 * gl;
        occ_rows<LPS, PPL, false, POW2>(0, jc0, s_gm + off, s_gp + off, s_yf + oy, side, yf2, pix2, npy2, ry, r2, dx2, cmask,
                                        sw, swy);
        occ_rows<LPS, PPL, true, POW2>(jc0, jc1, s_gm + off, s_gp + off, s_yf + oy, side, yf2, pix2, npy2, ry, r2, dx2, cmask,
                                       sw, swy);
        occ_rows<LPS, PPL, false, POW2>(jc1, Wwin, s_gm + off, s_gp + off, s_yf + oy, side, yf2, pix2, npy2, ry, r2, dx2, cmask,
                                        sw, swy);
        float gx = 0.f, gy = 0.f;
#pragma unroll
        for (int s = 0; s < PPL; ++s) {
            gx = fmaf(dx2[s].x, sw[s].x, fmaf(dx2[s].y, sw[s].y, gx));     // sum_rows dx*w = dx * sum_rows w
            gy += swy[s].x + swy[s].y;
        }
#pragma unroll
        for (int d = LPS >> 1; d > 0; d >>= 1) {
            gx += __shfl_xor_sync(FULL, gx, d);
            gy += __shfl_xor_sync(FULL, gy, d);
        }
        // rasterize_points_backward.cu:145 -- points outside the renderable area or behind the camera (id < 0) get no
        // gradient
        if (have && gl == 0 && id >= 0 && !(fabsf(py) > 1.0f || fabsf(px) > 1.0f)) a.grad_xy[id] = make_float2(gx, gy);
    }
}

// Persistent, warp-specialised: warp 8 is the PRODUCER -- it decodes the next work item, computes the window's
// pixel-centre tables and drives the TMA engine (cp.async.bulk row copies of both gradient planes into the free
// window buffer when the tile changes, the item's records into the free record buffer), completion signalled on the
// slot's "full" mbarrier; warps 0-7 are CONSUMERS -- they wait on "full", gather, and release the slot through its
// "empty" mbarrier.  Two item slots and two window buffers are in flight, so staging overlaps the arithmetic.
// (This mapping -- 8 consumer warps, up to 96 registers, the LPS/PPL choices of the host code -- was chosen when the
//  column pairs used packed FP32x2 instructions; it has not been re-tuned for the scalar walk on the H100.  Alternatives
//  that were slower then: 10 consumer warps at 80 registers (spills); 12 consumer warps with at most 2 column pairs per
//  lane (4 instead of 8 splats share the per-row instructions); 8 lanes x 2 pairs per splat.)
template <bool POW2, int NCONS>
__global__ void __launch_bounds__((NCONS + 1) * 32, 2)
occ_tile_kernel(const __grid_constant__ OccTileArgs a) {
    constexpr int OCC_THREADS = (NCONS + 1) * 32;
    extern __shared__ __align__(128) unsigned char occ_smem[];
    const int S = a.S, OB = a.OB, side = a.side, R_box = a.R_box;
    const int plane_elems = side * side + OCC_SLACK;
    const int win_elems = 2 * plane_elems + 2 * side + OCC_SLACK;   // g-, g+, column table (+slack), row table
    float *s_win = reinterpret_cast<float *>(occ_smem);              // 2 window buffers
    float4 *s_rec = reinterpret_cast<float4 *>(s_win + 2 * win_elems);               // 2 x OCC_ITEM records
    OccItem *s_item = reinterpret_cast<OccItem *>(s_rec + 2 * OCC_ITEM);              // 2 item descriptors
    unsigned long long *s_bar = reinterpret_cast<unsigned long long *>(s_item + 2);  // full[2], empty[2]
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t bar_full = smem_u32(s_bar), bar_empty = smem_u32(s_bar + 2);

    if (tid == 0) {
        mbar_init(bar_full, 1);
        mbar_init(bar_full + 8, 1);
        mbar_init(bar_empty, NCONS);
        mbar_init(bar_empty + 8, NCONS);
        mbar_fence_init();
    }
    // the slack behind the planes / column table is read (and masked out) by lanes whose column pairs lie beyond
    // the window: keep it finite
    for (int i = tid; i < 2 * 3 * OCC_SLACK; i += OCC_THREADS) {
        const int wb = i / (3 * OCC_SLACK), q = (i / OCC_SLACK) % 3, e = i % OCC_SLACK;
        float *w = s_win + wb * win_elems;
        (q == 0 ? w + side * side : q == 1 ? w + plane_elems + side * side : w + 2 * plane_elems + side)[e] = 0.0f;
    }
    __syncthreads();

    const int n_items = a.part_off[a.nt];
    const int n_groups = (n_items + OCC_GROUP - 1) / OCC_GROUP;

    if (warp == NCONS) {
        // ------------------------------- producer -------------------------------
        // Groups of OCC_GROUP consecutive items are handed out dynamically (one atomic per group): the views differ
        // up to 3x in cost per splat (window area), a static round-robin leaves CTAs idle at the end of the launch.
        int wt_cur = -1;                       // tile held by the current window buffer
        int wcur = 0;
        int slot_use = 0;                      // items staged so far
        int group = -1, k_in = OCC_GROUP;      // current group, next item inside it
        for (;;) {
            const int slot = slot_use & 1;
            if (k_in >= OCC_GROUP) {
                if (lane == 0) group = atomicAdd(a.group_counter, 1);
                group = __shfl_sync(0xffffffffu, group, 0);
                k_in = 0;
            }
            int item = -1;
            if (group < n_groups) {
                item = group * OCC_GROUP + k_in;
                ++k_in;
                if (item >= n_items) {      // tail of the last group
                    k_in = OCC_GROUP;
                    continue;
                }
            }
            // wait until the consumers have released this slot (its previous use)
            if (slot_use >= 2) mbar_wait(bar_empty + 8 * slot, (uint32_t)(((slot_use >> 1) - 1) & 1));
            OccItem *it = s_item + slot;
            if (item < 0) {
                if (lane == 0) {
                    it->cnt = -1;
                    mbar_arrive(bar_full + 8 * slot);
                }
                break;
            }
            const int t = a.item_tile[item];
            const int n = t / (OB * OB), tile = t - n * OB * OB;
            const int ty = tile / OB, tx = tile - ty * OB;
            const int p = item - a.part_off[t], parts = a.part_off[t + 1] - a.part_off[t];
            const int tb = a.tile_offsets[(int64_t)t * OCC_CELLS], count = a.tile_offsets[(int64_t)(t + 1) * OCC_CELLS] - tb;
            const int per = (count + parts - 1) / parts;
            const int beg = tb + p * per;
            const int cnt = max(0, min(count - p * per, per));
            const float r = a.rs[n];
            const bool load_win = wt_cur != t;
            if (load_win) {
                // the other buffer was last used by items <= (this item - 2) of an earlier tile: already released
                if (wt_cur >= 0) wcur ^= 1;
                wt_cur = t;
            }
            float *w = s_win + wcur * win_elems;
            if (load_win) {
                // exact pixel-centre NDC coordinates of the window's columns / rows (the reference's PixToNdc,
                // division included, once per tile instead of once per pair).  Written before the arrive below so
                // that its release (after __syncwarp) publishes them to the consumers together with the descriptor.
                float *xf = w + 2 * plane_elems, *yf = xf + side + OCC_SLACK;
                const int wx0 = tx * OCC_TILE - R_box, wy0 = ty * OCC_TILE - R_box;
                for (int i = lane; i < side + OCC_SLACK; i += 32) {
                    xf[i] = pix_to_ndc(wx0 + i, S);
                    if (i < side) yf[i] = pix_to_ndc(wy0 + i, S);
                }
            }
            __syncwarp();
            if (lane == 0) {
                it->cnt = cnt;
                it->beg = beg;
                it->wbuf = wcur;
                it->tx = tx;
                it->ty = ty;
                it->hh = occ_hh(r, S);
                it->r2 = r * r;
                mbar_arrive_expect_tx(bar_full + 8 * slot, (uint32_t)((load_win ? 2 * side * side * 4 : 0) + cnt * 16));
            }
            __syncwarp();
            if (load_win) {
                // plane padding == R_box, so the window origin is (ty*32, tx*32) in plane coordinates and every row
                // copy is 16-byte aligned on both sides
                const float *src0 = a.planes + (((int64_t)n * 2) * a.Hp + (int64_t)ty * OCC_TILE) * a.W + tx * OCC_TILE;
                for (int row = lane; row < 2 * side; row += 32) {
                    const int pl = row >= side ? 1 : 0, rr = row - pl * side;
                    bulk_copy_g2s(smem_u32(w + pl * plane_elems + rr * side), src0 + ((int64_t)pl * a.Hp + rr) * a.W,
                                  (uint32_t)(side * 4), bar_full + 8 * slot);
                }
            }
            if (lane == 0 && cnt > 0)
                bulk_copy_g2s(smem_u32(s_rec + slot * OCC_ITEM), a.crec + beg, (uint32_t)(cnt * 16), bar_full + 8 * slot);
            ++slot_use;
        }
        return;
    }
    // --------------------------------- consumers ---------------------------------
    for (int use = 0;; ++use) {
        const int slot = use & 1;
        mbar_wait(bar_full + 8 * slot, (uint32_t)((use >> 1) & 1));
        const OccItem it = s_item[slot];
        if (it.cnt < 0) break;
        const float *w = s_win + it.wbuf * win_elems;
        const float *s_gm = w, *s_gp = w + plane_elems, *s_xf = w + 2 * plane_elems, *s_yf = s_xf + side + OCC_SLACK;
        const float4 *rec = s_rec + slot * OCC_ITEM;
        const int need = 2 * it.hh + 2;          // window columns + 1 for the shift to an even column
        if (need <= 8) occ_item<4, 1, POW2, NCONS>(a, it, s_gm, s_gp, s_xf, s_yf, rec, warp, lane);
        else if (need <= 16) occ_item<4, 2, POW2, NCONS>(a, it, s_gm, s_gp, s_xf, s_yf, rec, warp, lane);
        else if (need <= 24) occ_item<4, 3, POW2, NCONS>(a, it, s_gm, s_gp, s_xf, s_yf, rec, warp, lane);
        else if (need <= 32) occ_item<4, 4, POW2, NCONS>(a, it, s_gm, s_gp, s_xf, s_yf, rec, warp, lane);
        else if (need <= 40) occ_item<4, 5, POW2, NCONS>(a, it, s_gm, s_gp, s_xf, s_yf, rec, warp, lane);   // not 48: -17 % pairs
        else if (need <= 48) occ_item<8, 3, POW2, NCONS>(a, it, s_gm, s_gp, s_xf, s_yf, rec, warp, lane);
        else if (need <= 64) occ_item<8, 4, POW2, NCONS>(a, it, s_gm, s_gp, s_xf, s_yf, rec, warp, lane);
        else occ_item<16, 3, POW2, NCONS>(a, it, s_gm, s_gp, s_xf, s_yf, rec, warp, lane);   // need <= 96 (R_box <= 40)
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_empty + 8 * slot);
    }
}


// ---------------------------------------------------------------------------------------------
// Direct gathers from the gradient image in global memory, one warp per point (no staging, no atomics).
// warp_window_gather: the lanes stride over the pixels of the window |x - px| <= ex, |y - py| <= ey (conservative, in
// NDC-index space, clamped to the image); for every pixel with a non-zero gradient g, rule(dx, dy, g, gx, gy) adds that
// pixel's share.  Returns the warp's sums (gx, gy) in every lane.  Each caller keeps its own expression text for d2,
// the test and eps_denom, so their FMA contraction is the caller's own.
// ---------------------------------------------------------------------------------------------
constexpr int OCC_WARPS = 8;

template <class Rule>
__device__ __forceinline__ float2 warp_window_gather(const float *__restrict__ gview, int pix_stride, int S, float inv_S,
                                                     bool pow2, float px, float py, float ex, float ey, Rule rule) {
    constexpr unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    const float half_S = 0.5f * (float)S;
    // pixel i has centre -1 + (2i+1)/S (clamped in float first: saturating conversions of huge extents must not wrap)
    const float top = (float)(S - 1);
    const int xi_lo = (int)fminf(fmaxf(floorf((px - ex + 1.0f) * half_S - 0.5f) - 1.0f, 0.0f), top + 1.0f);
    const int xi_hi = (int)fmaxf(fminf(ceilf((px + ex + 1.0f) * half_S - 0.5f) + 1.0f, top), -1.0f);
    const int yi_lo = (int)fminf(fmaxf(floorf((py - ey + 1.0f) * half_S - 0.5f) - 1.0f, 0.0f), top + 1.0f);
    const int yi_hi = (int)fmaxf(fminf(ceilf((py + ey + 1.0f) * half_S - 0.5f) + 1.0f, top), -1.0f);
    const int W = xi_hi - xi_lo + 1, H = yi_hi - yi_lo + 1;
    float gx = 0.f, gy = 0.f;
    if (W > 0 && H > 0) {
        const int total = W * H;
        int wy = lane / W, wx = lane - wy * W;
        const int step_y = 32 / W, step_x = 32 - step_y * W;
        for (int w = lane; w < total; w += 32) {
            const int xi = xi_lo + wx, yi = yi_lo + wy;
            const float g = __ldg(gview + ((int64_t)(S - 1 - yi) * S + (S - 1 - xi)) * pix_stride);
            if (g != 0.0f) {
                const float xf = pix_to_ndc_fast(xi, S, inv_S, pow2);
                const float yf = pix_to_ndc_fast(yi, S, inv_S, pow2);
                rule(xf - px, yf - py, g, gx, gy);
            }
            wx += step_x;
            wy += step_y;
            if (wx >= W) {
                wx -= W;
                wy += 1;
            }
        }
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        gx += __shfl_xor_sync(FULL, gx, d);
        gy += __shfl_xor_sync(FULL, gy, d);
    }
    return make_float2(gx, gy);
}

// Generic gather for views whose window does not fit the staged box (very large search radius): the disc of radius r
// around every visible splat, the reference's per-pair rule (rasterize_points_backward.cu:141-178); a warp takes the
// visible splats of its 32 slots in turn.
__global__ void __launch_bounds__(OCC_WARPS * 32)
occ_generic_kernel(const float4 *__restrict__ rec, const uint8_t *__restrict__ visible,
                   const float *__restrict__ rs, const float *__restrict__ grad, int pix_stride,
                   int pix_offset, const int64_t *__restrict__ first_idx,
                   const int64_t *__restrict__ num_points, int64_t P0_shared, int S, int R_box,
                   float2 *__restrict__ grad_xy) {
    const int n = blockIdx.y;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const ViewRange vr = view_range(first_idx, num_points, n, P0_shared);
    const float r = rs[n];
    if (occ_fits(r, S, R_box)) return;   // this view is handled by occ_tile_kernel
    const float r2 = r * r;
    const bool pow2 = (S & (S - 1)) == 0;
    const float inv_S = 1.0f / (float)S;
    const float *gview = grad + ((int64_t)n * S * S) * pix_stride + pix_offset;
    constexpr unsigned FULL = 0xffffffffu;

    for (int64_t g0 = ((int64_t)blockIdx.x * OCC_WARPS + warp) * 32; g0 < vr.count;
         g0 += (int64_t)gridDim.x * OCC_WARPS * 32) {
        const int64_t i = g0 + lane;
        const bool in_range = i < vr.count;
        const int64_t p = vr.first + i;
        float4 A = make_float4(0.f, 0.f, -1.f, 0.f);
        float ry = 0.f;
        bool vis = false;
        if (in_range) {
            vis = visible[p] != 0;
            if (vis) {
                A = __ldg(&rec[2 * p]);
                ry = __ldg(&rec[2 * p + 1]).x;
                // rasterize_points_backward.cu:145 -- outside the renderable area
                if (A.z < 0.0f || fabsf(A.y) > 1.0f || fabsf(A.x) > 1.0f) vis = false;
            }
        }
        float out_x = 0.f, out_y = 0.f;
        unsigned todo = __ballot_sync(FULL, vis);
        while (todo) {
            const int src = __ffs(todo) - 1;
            todo &= todo - 1;
            const float px = __shfl_sync(FULL, A.x, src);
            const float py = __shfl_sync(FULL, A.y, src);
            const float rx = __shfl_sync(FULL, A.w, src);
            const float ryb = __shfl_sync(FULL, ry, src);
            const float2 g2 = warp_window_gather(gview, pix_stride, S, inv_S, pow2, px, py, r, r,
                                                 [&](float dx, float dy, float g, float &gx, float &gy) {
                const float d2 = dx * dx + dy * dy;
                const bool outside = (fabsf(dx) > rx) || (fabsf(dy) > ryb);
                if (!(d2 > r2) && !(g > 0.0f && outside)) {
                    const float den = eps_denom(d2, 1e-10f);
                    gx += dx / den * g;
                    gy += dy / den * g;
                }
            });
            if (lane == src) {
                out_x = g2.x;
                out_y = g2.y;
            }
        }
        if (in_range) grad_xy[p] = make_float2(out_x, out_y);
    }
}

// ---------------------------------------------------------------------------------------------
// "Slow" occupancy backward (RasterizePointsOccBackwardCudaKernel, DSS/csrc/rasterize_points.cu:673-760; disabled in
// the reference by backward_occ_fast = True, rasterizer.py:816, kept for completeness): EVERY renderable point of the view
// (z >= 0, |x|,|y| <= 1 -- not only the visible ones) gathers over the RECTANGLE |dx| <= rx*s, |dy| <= ry*s instead of
// the disc; positive gradients only count inside the splat's own bbox ((rx*s)/s, (ry*s)/s as the reference writes it).
// One warp per point on warp_window_gather, like occ_generic_kernel.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(OCC_WARPS * 32)
occ_slow_kernel(const float *__restrict__ points, const float *__restrict__ radii, float radii_s,
                const float *__restrict__ grad, int pix_stride, int pix_offset, const int64_t *__restrict__ first_idx,
                const int64_t *__restrict__ num_points, int S, float2 *__restrict__ grad_xy) {
    const int n = blockIdx.y;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const ViewRange vr = view_range(first_idx, num_points, n, 0);
    const bool pow2 = (S & (S - 1)) == 0;
    const float inv_S = 1.0f / (float)S;
    const float *gview = grad + ((int64_t)n * S * S) * pix_stride + pix_offset;
    for (int64_t i = (int64_t)blockIdx.x * OCC_WARPS + warp; i < vr.count; i += (int64_t)gridDim.x * OCC_WARPS) {
        const int64_t p = vr.first + i;
        const float px = points[p * 3], py = points[p * 3 + 1], pz = points[p * 3 + 2];
        float2 g2 = make_float2(0.f, 0.f);
        if (!(pz < 0.0f || fabsf(py) > 1.0f || fabsf(px) > 1.0f)) {            // rasterize_points.cu:719
            const float rxs = radii[p * 2] * radii_s, rys = radii[p * 2 + 1] * radii_s;   // :725-726
            const float rxb = rxs / radii_s, ryb = rys / radii_s;                            // :744
            g2 = warp_window_gather(gview, pix_stride, S, inv_S, pow2, px, py, rxs, rys,
                                    [&](float dx, float dy, float g, float &gx, float &gy) {
                const bool in_rect = !(fabsf(dx) > rxs || fabsf(dy) > rys);                       // :728
                const bool outside_splat = (fabsf(dx) > rxb) || (fabsf(dy) > ryb);               // :744
                if (in_rect && !(g > 0.0f && outside_splat)) {
                    const float den = eps_denom(dx * dx + dy * dy, 1e-10f);                       // :752-753
                    gx += dx / den * g;
                    gy += dy / den * g;
                }
            });
        }
        if (lane == 0) grad_xy[p] = g2;
    }
}

// rs: (N,) search radii -- an INPUT when radii_s < 0 (the _C-level op passes them in), otherwise computed here as
// radii_s * lower median of the visible radii and written to rs.  grad_xy (P,2) is fully written.
int occ_backward(dss_ctx *ctx, const float4 *rec, const uint8_t *visible, float *rs, float radii_s,
                 const float *grad_occ, int pix_stride, int pix_offset, const int64_t *first_idx,
                 const int64_t *num_points, int N, int64_t P0, int S, float *grad_xy, const int32_t *cell_counts,
                 cudaStream_t st) {
    if (N <= 0 || P0 <= 0) return DSS_OK;
    const int OB = occ_tiles(S);
    const int64_t nt = (int64_t)N * OB * OB;
    const int64_t Ptot = (first_idx == nullptr) ? (int64_t)N * P0 : P0;   // packed mode passes P0 = P
    const bool compute_rs = radii_s >= 0.0f;
    // Size of the staged window from the radii seen by the previous call (a hint only: both kernels re-derive
    // "fits" from the current radius on the device, views that do not fit take the generic kernel)
    float *h_rs = reinterpret_cast<float *>(ctx->h_pinned + 8);
    float hint = 0.0f;
    for (int i = 0; i < (N < 96 ? N : 96); ++i) hint = fmaxf(hint, h_rs[i]);
    int R_box = 20;
    if (hint > 0.0f && hint < 4.0f) R_box = (occ_hh(hint * 1.15f, S) + 2 + 3) & ~3;
    if (R_box < 8) R_box = 8;
    if (R_box > OCC_RBOX_MAX) R_box = OCC_RBOX_MAX;
    const int side = OCC_TILE + 2 * R_box;
    const size_t win_elems = (size_t)2 * (side * side + OCC_SLACK) + 2 * side + OCC_SLACK;
    const size_t smem = 2 * win_elems * sizeof(float) + 2 * (size_t)OCC_ITEM * sizeof(float4) + 2 * sizeof(OccItem) +
                        4 * sizeof(unsigned long long);
    // The limits of the staged path, each stated at the kernel that has it (occ_cellbin_kernel, SelectCompact,
    // occ_items_kernel, occ_planes_kernel).  Cells are indexed in int64 everywhere (occ_cell, every offset read), so
    // their total needs no limit of its own.
    const int64_t max_items = Ptot / OCC_ITEM + nt + 1;   // >= nt + 1
    const bool tiles_ok = max_items < (int64_t)INT32_MAX && Ptot < (int64_t)INT32_MAX &&
                          (int64_t)OB * OB * OCC_CELLS <= (int64_t)INT32_MAX && OB * OCC_TILE + 2 * R_box <= 65535;
    if (!tiles_ok) R_box = 0;
    int rc;
    DSS_CUDA_TRY(cudaMemsetAsync(grad_xy, 0, (size_t)Ptot * 2 * sizeof(float), st));
    if (R_box > 0) {
        int32_t *counts = nullptr, *offsets = nullptr, *cids = nullptr;
        float4 *crec = nullptr;
        float *planes = nullptr;
        const int PAD = R_box, W = OB * OCC_TILE + 2 * PAD, Hp = W;
        const int64_t nc = nt * OCC_CELLS;
        if ((rc = ctx_get(ctx, BUF_OCC_COUNTS, (size_t)(nc + 1), &counts))) return rc;
        if ((rc = ctx_get(ctx, BUF_TILE_OFFSETS, (size_t)(nc + 1), &offsets))) return rc;
        if ((rc = ctx_get(ctx, BUF_OCC_IDS, (size_t)(Ptot > 0 ? Ptot : 1), &cids))) return rc;
        if ((rc = ctx_get(ctx, BUF_OCC_REC, (size_t)(Ptot > 0 ? Ptot : 1), &crec))) return rc;
        if ((rc = ctx_get(ctx, BUF_OCC_PLANES, (size_t)N * 2 * Hp * W, &planes))) return rc;
        {
            StageScope prof(ctx, ST_OCC_BIN, st);
            // the counters live in their own buffer and are left at zero by every successful call
            const bool clean = ctx->occ_counts_ptr == counts && ctx->occ_counts_elems >= (size_t)(nc + 1);
            ctx->occ_counts_ptr = nullptr;   // restored below; an error in between forces the memset next time
            if (!clean) DSS_CUDA_TRY(cudaMemsetAsync(counts, 0, ctx->cap[BUF_OCC_COUNTS], st));
            dim3 bgrid(grid_blocks(P0, 256 * 4, ctx->sm_count, 8), N);
            if (cell_counts) {
                // the forward's blend epilogue has counted already (one count per visible splat, same cells): take a
                // copy -- pass 1 counts the working copy back down to zero, the caller's tensor stays intact
                DSS_CUDA_TRY(cudaMemcpyAsync(counts, cell_counts, (size_t)nc * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
            } else {
                occ_cellbin_kernel<0><<<bgrid, 256, 0, st>>>(rec, visible, first_idx, num_points, P0, S, OB, counts, nullptr,
                                                             nullptr, nullptr);
                DSS_LAUNCH_CHECK(ctx);
            }
            if ((rc = exclusive_scan_i32(ctx, counts, offsets, nc + 1, st))) return rc;
            occ_cellbin_kernel<1><<<bgrid, 256, 0, st>>>(rec, visible, first_idx, num_points, P0, S, OB, counts, offsets,
                                                         crec, cids);
            DSS_LAUNCH_CHECK(ctx);
            ctx->occ_counts_ptr = counts;
            ctx->occ_counts_elems = ctx->cap[BUF_OCC_COUNTS] / sizeof(int32_t);
        }
        if (compute_rs) {
            unsigned int *hist = nullptr;
            if ((rc = ctx_get(ctx, BUF_SELECT, (size_t)N * 4 * 256, &hist))) return rc;
            StageScope prof(ctx, ST_SEARCH_RADIUS, st);
            DSS_CUDA_TRY(cudaMemsetAsync(hist, 0, (size_t)N * 4 * 256 * sizeof(unsigned int), st));
            dim3 grid(grid_blocks(P0 / 4 + 1, 256, ctx->sm_count, 1), N);
            for (int pass = 0; pass < 4; ++pass) {
                select_hist_kernel<<<grid, 256, 0, st>>>(SelectCompact{crec, offsets, OB * OB * OCC_CELLS, pass}, hist);
                DSS_LAUNCH_CHECK(ctx);
            }
            select_final_kernel<<<N, 32, 0, st>>>(hist, radii_s, rs);
            DSS_LAUNCH_CHECK(ctx);
        }
        StageScope prof(ctx, ST_OCC_BWD, st);
        {
            dim3 pgrid((unsigned)((W + 255) / 256), (unsigned)Hp, (unsigned)N);
            occ_planes_kernel<<<pgrid, 256, 0, st>>>(grad_occ, pix_stride, pix_offset, S, PAD, W, Hp, planes);
            DSS_LAUNCH_CHECK(ctx);
        }
        // work items: parts per tile -> scan -> tile of every item
        int32_t *parts = nullptr, *item_tile = nullptr;
        if ((rc = ctx_get(ctx, BUF_OCC_PARTS, (size_t)(2 * (nt + 1) + 4), &parts))) return rc;
        if ((rc = ctx_get(ctx, BUF_OCC_ITEMS, (size_t)max_items, &item_tile))) return rc;
        int32_t *part_off = parts + (nt + 1);
        occ_parts_kernel<<<(unsigned)((nt + 1 + 255) / 256), 256, 0, st>>>(offsets, rs, OB * OB, nt, S, R_box, parts);
        DSS_LAUNCH_CHECK(ctx);
        if ((rc = exclusive_scan_i32(ctx, parts, part_off, nt + 1, st))) return rc;
        occ_items_kernel<<<(unsigned)((nt + 255) / 256), 256, 0, st>>>(part_off, nt, item_tile);
        DSS_LAUNCH_CHECK(ctx);
        OccTileArgs a;
        a.crec = crec;
        a.cids = cids;
        a.tile_offsets = offsets;
        a.part_off = part_off;
        a.item_tile = item_tile;
        a.group_counter = parts + 2 * (nt + 1);
        DSS_CUDA_TRY(cudaMemsetAsync(a.group_counter, 0, sizeof(int), st));
        a.rs = rs;
        a.planes = planes;
        a.grad_xy = reinterpret_cast<float2 *>(grad_xy);
        a.S = S;
        a.OB = OB;
        a.R_box = R_box;
        a.side = side;
        a.W = W;
        a.Hp = Hp;
        a.nt = nt;
        const bool pow2 = (S & (S - 1)) == 0;
        // persistent: as many CTAs as fit (2 per SM at the usual window sizes), items round-robin in groups
        int per_sm = (int)((size_t)220 * 1024 / (smem + 1024));
        if (per_sm > 2) per_sm = 2;
        if (per_sm < 1) per_sm = 1;
        int64_t want = (max_items + OCC_GROUP - 1) / OCC_GROUP;
        unsigned tgrid = (unsigned)(want < (int64_t)ctx->sm_count * per_sm ? want : (int64_t)ctx->sm_count * per_sm);
        if (tgrid < 1) tgrid = 1;
        auto launch = [&](auto kern, int threads) -> int {
            DSS_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            kern<<<tgrid, threads, smem, st>>>(a);
            return DSS_OK;
        };
        // 8 consumer warps + 1 producer warp per CTA
        rc = pow2 ? launch(occ_tile_kernel<true, 8>, 9 * 32) : launch(occ_tile_kernel<false, 8>, 9 * 32);
        if (rc) return rc;
        DSS_LAUNCH_CHECK(ctx);
    } else if (compute_rs) {
        if ((rc = search_radius(ctx, rec, nullptr, visible, first_idx, num_points, N, P0, radii_s, rs, st))) return rc;
    }
    {
        // views whose window does not fit (very large search radius) take the direct global-memory gather
        StageScope prof(ctx, ST_OCC_BWD, st);
        dim3 grid(grid_blocks(P0, OCC_WARPS * 32, ctx->sm_count, 4), N);   // grid-stride; usually every block returns at once
        occ_generic_kernel<<<grid, OCC_WARPS * 32, 0, st>>>(rec, visible, rs, grad_occ, pix_stride, pix_offset, first_idx,
                                                            num_points, P0, S, R_box,
                                                            reinterpret_cast<float2 *>(grad_xy));
        DSS_LAUNCH_CHECK(ctx);
    }
    // refresh the hint for the next call (asynchronous; may be read stale, it is only a hint)
    return publish_words(ctx, rs, h_rs, N < 96 ? N : 96, st);
}

}  // namespace dss

extern "C" {

int dss_search_radius(dss_ctx *ctx, const float *radii, const uint8_t *visible, const int64_t *first_idx,
                      const int64_t *num_points, int N, int64_t P, float radii_s, float *rs, void *stream) {
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    DSS_REQUIRE(N >= 0 && P >= 0, "negative size");
    if (N == 0) return DSS_OK;
    DSS_REQUIRE(rs && first_idx && num_points && (P == 0 || (radii && visible)), "null pointer");
    return dss::search_radius(ctx, nullptr, radii, visible, first_idx, num_points, N, P, radii_s, rs,
                              (cudaStream_t)stream);
}

int dss_occ_backward_slow(dss_ctx *ctx, const float *points, const float *radii, const float *grad_occ, int pix_stride,
                          int pix_offset, const int64_t *first_idx, const int64_t *num_points, int N, int64_t P,
                          int image_size, float radii_s, float *grad_xy, void *stream) {
    using namespace dss;
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    DSS_REQUIRE(N >= 0 && P >= 0 && image_size > 0, "bad size");
    DSS_REQUIRE(pix_stride >= 1 && pix_offset >= 0 && pix_offset < pix_stride, "bad pixel stride/offset");
    DSS_REQUIRE(radii_s > 0.0f, "radii_s must be positive");
    if (N == 0 || P == 0) return DSS_OK;
    DSS_REQUIRE(points && radii && grad_occ && first_idx && num_points && grad_xy, "null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    DSS_CUDA_TRY(cudaMemsetAsync(grad_xy, 0, (size_t)P * 2 * sizeof(float), st));   // rows outside every view range
    StageScope prof(ctx, ST_OCC_BWD, st);
    dim3 grid(grid_blocks(P, OCC_WARPS, ctx->sm_count, 16), N);
    occ_slow_kernel<<<grid, OCC_WARPS * 32, 0, st>>>(points, radii, radii_s, grad_occ, pix_stride, pix_offset, first_idx,
                                                     num_points, image_size, reinterpret_cast<float2 *>(grad_xy));
    DSS_LAUNCH_CHECK(ctx);
    return DSS_OK;
}

int dss_occ_backward(dss_ctx *ctx, const float *points, const float *radii, const uint8_t *visible,
                     const float *rs, const float *grad_occ, int pix_stride, int pix_offset,
                     const int64_t *first_idx, const int64_t *num_points, int N, int64_t P, int image_size,
                     float *grad_xy, void *stream) {
    using namespace dss;
    cudaStream_t st = (cudaStream_t)stream;
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    DSS_REQUIRE(N >= 0 && P >= 0 && image_size > 0, "bad size");
    DSS_REQUIRE(pix_stride >= 1 && pix_offset >= 0 && pix_offset < pix_stride, "bad pixel stride/offset");
    if (N == 0 || P == 0) return DSS_OK;
    DSS_REQUIRE(points && radii && visible && rs && grad_occ && first_idx && num_points && grad_xy, "null pointer");
    float4 *rec = nullptr;
    int rc;
    if ((rc = ctx_get(ctx, BUF_RECORDS, (size_t)(2 * P), &rec))) return rc;
    if ((rc = pack_records(ctx, points, radii, nullptr, P, rec, st))) return rc;
    return occ_backward(ctx, rec, visible, const_cast<float *>(rs), -1.0f, grad_occ, pix_stride, pix_offset, first_idx,
                        num_points, N, P, image_size, grad_xy, nullptr, st);
}

}  // extern "C"
