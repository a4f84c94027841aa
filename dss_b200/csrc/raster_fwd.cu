// raster_fwd.cu -- per-tile forward rasterization (+ optional fused blend).
//
// Replaces RasterizePointsFineCudaKernel (DSS/csrc/rasterize_points.cu:506-597), whose every pixel
// loops over all M = max(1e4, P) slots of its bin and keeps a 150-entry queue in local memory, and --
// when blending -- the weights/compositor/concat sequence of DSS/core/renderer.py:53-78.
//
// One 256-thread CTA per 16x16 pixel tile.  The tile's splat list (CSR ids) is streamed through shared
// memory in chunks of 256 records.  Each warp owns an 8x4 pixel patch and runs a two-level test:
//   level 1 (lane-parallel, 32 splats at a time): bbox-vs-patch overlap and a depth cull against the
//            warp's current K-th nearest depth -> ballot;
//   level 2 (per surviving splat, broadcast from shared memory): the reference's exact per-pixel test
//            (CheckPixelInsidePoint, rasterize_points.cu:87-97) and a sorted insert into K registers.
// Selection is by (z, id) lexicographic order, so the result does not depend on list order (the
// reference's own CPU path pops a max-heap of (z, idx, q) tuples: rasterize_points_cpu.cpp:87-121).
#include <math_constants.h>

#include "common.cuh"
#include "kernels.cuh"

namespace dss {

constexpr int RASTER_THREADS = RASTER_TILE * RASTER_TILE;  // 256
constexpr int RASTER_CHUNK = RASTER_THREADS;

__device__ __forceinline__ bool frag_less(float za, int ia, float zb, int ib) {
    return (za < zb) || (za == zb && ia < ib);
}

// The output of pixel (xi, yi) of view n, shared by both raster kernels, which must agree to the bit.  fz / fq / fid: the
// pixel's nearest fragments in (z, id) order; emit[k]: fragment k is output (k < K and the depth merge has not stopped the
// list before it); any: the pixel has a fragment at all; centre(k): the NDC centre (x, y) of emitted fragment k's splat,
// asked for only when the epilogue counts cells.  Writes idx / zbuf / qvalue (-1 past the emitted fragments), the
// occupancy and, when blending, the image, the weights, the visibility bytes and the cell counts.
template <int KMAX, bool BLEND, class Centre>
__device__ __forceinline__ void pixel_epilogue(const RasterArgs &a, int n, int xi, int yi, const float (&fz)[KMAX],
                                               const float (&fq)[KMAX], const int (&fid)[KMAX], const bool (&emit)[KMAX],
                                               bool any, Centre centre) {
    const int S = a.S, K = a.K;
    // image row S-1-yi, col S-1-xi: rasterize_points.cu:577-580
    const int64_t pix = ((int64_t)n * S + (S - 1 - yi)) * S + (S - 1 - xi);
#pragma unroll
    for (int k = 0; k < KMAX; ++k) {
        if (k < K) {
            a.idx[pix * K + k] = emit[k] ? fid[k] : -1;
            if (a.zbuf) a.zbuf[pix * K + k] = emit[k] ? fz[k] : -1.0f;
            if (a.qvalue) a.qvalue[pix * K + k] = emit[k] ? fq[k] : -1.0f;
        }
    }
    const float occ = any ? 1.0f : 0.0f;
    if (a.occ) a.occ[pix] = occ;
    if (BLEND) {
        // renderer.py:53 w = exp(-0.5 q) * scaler ; norm_weighted_sum [ext]: sum w f / max(sum w, 1e-4)
        float w[KMAX];
        float wsum = 0.f, r = 0.f, g = 0.f, b = 0.f;
#pragma unroll
        for (int k = 0; k < KMAX; ++k) {
            w[k] = 0.f;
            if (emit[k]) {
                const int id = fid[k];
                w[k] = expf(-0.5f * fq[k]) * __ldg(&a.scaler[id]);
                const float *c = a.colours + ((int64_t)id - (int64_t)n * a.colour_P0) * 3;
                r += w[k] * __ldg(c + 0);
                g += w[k] * __ldg(c + 1);
                b += w[k] * __ldg(c + 2);
                wsum += w[k];
                if (a.cell_counts) {
                    // visibility byte + (first setter only) one count in the backward binning's cell of the splat's
                    // centre pixel: the backward's counting pass over all P splats disappears
                    unsigned int *word = reinterpret_cast<unsigned int *>(a.visible) + (id >> 2);
                    const unsigned int bit = 1u << ((id & 3) * 8);
                    if (!(*reinterpret_cast<volatile unsigned int *>(word) & bit) && !(atomicOr(word, bit) & bit)) {
                        const float2 p = centre(k);
                        atomicAdd(&a.cell_counts[occ_cell(n, occ_tiles(S), centre_pixel(p.x, S), centre_pixel(p.y, S))], 1);
                    }
                } else if (a.visible) {
                    a.visible[id] = 1;
                }
            }
        }
        const float inv = 1.0f / fmaxf(wsum, 1e-4f);
        reinterpret_cast<float4 *>(a.image)[pix] = make_float4(r * inv, g * inv, b * inv, occ);
        if (a.weights) {
#pragma unroll
            for (int k = 0; k < KMAX; ++k)
                if (k < K) a.weights[pix * K + k] = w[k] * inv;
        }
    }
}

template <int KMAX, bool PER_POINT_CUTOFF, bool BLEND>
__global__ void __launch_bounds__(RASTER_THREADS)
raster_fwd_kernel(const __grid_constant__ RasterArgs a) {
    __shared__ float4 sA[RASTER_CHUNK];
    __shared__ float4 sB[RASTER_CHUNK];
    __shared__ int sId[RASTER_CHUNK];
    __shared__ float sCut[PER_POINT_CUTOFF ? RASTER_CHUNK : 1];

    const int S = a.S, B = a.B, K = a.K;
    const int n = blockIdx.y;
    const int tile = blockIdx.x;
    const int ty = tile / B, tx = tile - ty * B;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    constexpr unsigned FULL = 0xffffffffu;

    // NDC-index-space pixel of this thread
    const int ix0 = tx * RASTER_TILE + (warp & 1) * 8;
    const int iy0 = ty * RASTER_TILE + (warp >> 1) * 4;
    const int xi = ix0 + (lane & 7);
    const int yi = iy0 + (lane >> 3);
    const bool valid = (xi < S) && (yi < S);
    const float xf = pix_to_ndc(xi, S);
    const float yf = pix_to_ndc(yi, S);
    // warp patch extents, widened by half a pixel (same slack as the reference's bins)
    const float half_pix = 1.0f / S;
    const bool patch_live = (ix0 < S) && (iy0 < S);
    const float pat_x0 = pix_to_ndc(ix0, S) - half_pix;
    const float pat_x1 = pix_to_ndc(min(ix0 + 7, S - 1), S) + half_pix;
    const float pat_y0 = pix_to_ndc(iy0, S) - half_pix;
    const float pat_y1 = pix_to_ndc(min(iy0 + 3, S - 1), S) + half_pix;

    float fz[KMAX], fq[KMAX];
    int fid[KMAX];
#pragma unroll
    for (int k = 0; k < KMAX; ++k) {
        fz[k] = CUDART_INF_F;
        fq[k] = -1.0f;
        fid[k] = INT32_MAX;
    }
    float thresh = CUDART_INF_F;  // warp-wide max of the KMAX-th nearest depth

    const int64_t tbase = ((int64_t)n * B * B + tile) * a.NS;
    const int beg = min(a.tile_offsets[tbase], a.ids_capacity), end = min(a.tile_offsets[tbase + a.NS], a.ids_capacity);

    for (int base = beg; base < end; base += RASTER_CHUNK) {
        const int cnt = min(RASTER_CHUNK, end - base);
        if (tid < cnt) {
            const int id = a.tile_ids[base + tid];
            sA[tid] = __ldg(&a.rec[2 * (int64_t)id]);
            sB[tid] = __ldg(&a.rec[2 * (int64_t)id + 1]);
            sId[tid] = id;
            if (PER_POINT_CUTOFF) sCut[tid] = __ldg(&a.cutoff[id]);
        }
        __syncthreads();
        if (patch_live) {
            for (int j0 = 0; j0 < cnt; j0 += 32) {
                const int j = j0 + lane;
                bool pass = false;
                if (j < cnt) {
                    const float4 A = sA[j];
                    const float ry = sB[j].x;
                    pass = (A.z >= 0.0f) && (A.x - A.w <= pat_x1) && (pat_x0 <= A.x + A.w) &&
                           (A.y - ry <= pat_y1) && (pat_y0 <= A.y + ry) && (A.z <= thresh);
                }
                unsigned mask = __ballot_sync(FULL, pass);
                bool inserted = false;
                while (mask) {
                    const int jj = j0 + __ffs(mask) - 1;
                    mask &= mask - 1;
                    const float4 A = sA[jj];
                    const float4 Bv = sB[jj];
                    const float dx = xf - A.x;
                    const float dy = yf - A.y;
                    // rasterize_points.cu:92-97 -- same expression tree for q as the reference
                    const float qv = Bv.y * dx * dx + Bv.z * dx * dy + Bv.w * dy * dy;
                    const float cut = PER_POINT_CUTOFF ? sCut[jj] : a.cutoff_uniform;
                    const bool ok = valid && !(fabsf(dx) > A.w || fabsf(dy) > Bv.x) && !(qv > cut);
                    if (ok) {
                        const int id = sId[jj];
                        const float z = A.z + 0.0f;  // canonicalise -0
                        if (frag_less(z, id, fz[KMAX - 1], fid[KMAX - 1])) {
                            inserted = true;
#pragma unroll
                            for (int i = KMAX - 1; i >= 0; --i) {
                                if (frag_less(z, id, fz[i], fid[i])) {
                                    const bool shift = (i > 0) && frag_less(z, id, fz[i > 0 ? i - 1 : 0],
                                                                             fid[i > 0 ? i - 1 : 0]);
                                    fz[i] = shift ? fz[i > 0 ? i - 1 : 0] : z;
                                    fq[i] = shift ? fq[i > 0 ? i - 1 : 0] : qv;
                                    fid[i] = shift ? fid[i > 0 ? i - 1 : 0] : id;
                                }
                            }
                        }
                    }
                }
                if (__any_sync(FULL, inserted)) {
                    const float kz = valid ? fz[KMAX - 1] : -CUDART_INF_F;
                    thresh = __int_as_float(__reduce_max_sync(FULL, __float_as_int(kz)));
                }
            }
        }
        __syncthreads();
    }

    if (!valid) return;
    const bool any = fid[0] != INT32_MAX;
    const float z0 = fz[0];
    bool emit[KMAX];
    bool open = any;
#pragma unroll
    for (int k = 0; k < KMAX; ++k) {
        // rasterize_points.cu:586-595: stop at the first fragment farther than the merge threshold
        open = open && (k < K) && (fid[k] != INT32_MAX) && !(fz[k] - z0 > a.depth_merge);
        emit[k] = open;
    }
    pixel_epilogue<KMAX, BLEND>(a, n, xi, yi, fz, fq, fid, emit, any, [&](int k) {
        return __ldg(reinterpret_cast<const float2 *>(&a.rec[2 * (int64_t)fid[k]]));
    });
}

// ---------------------------------------------------------------------------------------------
// Splat-parallel ("scatter") rasterization: shared-memory K-lists (used by raster_sliced_kernel below).
//
// The pixel-parallel kernel above tests every splat that overlaps a warp's 8x4 patch in all 32 lanes,
// although a ~5 px splat covers only ~1/5 of them.  Here the roles are swapped: the per-pixel K-nearest
// lists of a 16x16 tile live in SHARED memory as sorted 64-bit keys (z bits << 32 | id), every THREAD
// takes its own splat of the tile list and walks only the pixels of that splat's bounding box inside
// the tile:  key >= pixel's current K-th key -> skip (one LDS.64 + compare);  otherwise the reference's
// exact test (rasterize_points.cu:87-97) and a lock-free sorted insert: a chain of atomicMin on the K
// slots, each step keeping the smaller key and carrying the larger one to the next slot.  The slots end
// up holding the K smallest keys in ascending (z, id) order whatever the interleaving, so the result is
// deterministic and identical to the pixel-parallel kernel.  q is recomputed for the K winners in the
// epilogue from the same record with the same expression, hence bit-identical to the accept test.
// ---------------------------------------------------------------------------------------------
constexpr unsigned long long KEY_EMPTY = ~0ull;

__device__ __forceinline__ unsigned long long make_key(float z, int id) {
    return ((unsigned long long)__float_as_uint(z) << 32) | (unsigned int)id;
}

// The fragments of the tile's pixel `tid`: keys from the K-lists in shared memory, records gathered up to the depth merge's
// stop, q recomputed for them with the accept test's expression text.  Then the common epilogue.
template <int KMAX, bool BLEND>
__device__ __forceinline__ void sliced_epilogue(const RasterArgs &a, const unsigned long long *s_keys, bool tile_has_entries,
                                                int n, int tx0, int ty0, bool pow2, float inv_S) {
    const int S = a.S, K = a.K;
    const int tid = threadIdx.x;
    // one thread per pixel
    const int xi = tx0 + (tid & (RASTER_TILE - 1));
    const int yi = ty0 + (tid >> 4);
    if (xi >= S || yi >= S) return;
    const float xf = pix_to_ndc_fast(xi, S, inv_S, pow2);
    const float yf = pix_to_ndc_fast(yi, S, inv_S, pow2);
    float fz[KMAX], fq[KMAX], fcx[KMAX], fcy[KMAX];
    int fid[KMAX];
    bool emit[KMAX];
    bool open = tile_has_entries;
    float z0 = 0.f;
#pragma unroll
    for (int k = 0; k < KMAX; ++k) {
        fz[k] = -1.0f;
        fq[k] = -1.0f;
        fcx[k] = fcy[k] = 0.0f;
        fid[k] = -1;
        emit[k] = false;
        if (open && k < K) {
            const unsigned long long key = s_keys[(tid * KMAX) + k];
            if (key == KEY_EMPTY) {
                open = false;
            } else {
                const float z = __uint_as_float((unsigned int)(key >> 32));
                if (k == 0) z0 = z;
                if (z - z0 > a.depth_merge) {   // rasterize_points.cu:586-595
                    open = false;
                } else {
                    const int id = (int)(unsigned int)(key & 0xffffffffull);
                    const float4 A = __ldg(&a.rec[2 * (int64_t)id]);
                    const float4 Bv = __ldg(&a.rec[2 * (int64_t)id + 1]);
                    const float dx = xf - A.x, dy = yf - A.y;
                    fz[k] = z;
                    fid[k] = id;
                    fcx[k] = A.x;
                    fcy[k] = A.y;
                    fq[k] = Bv.y * dx * dx + Bv.z * dx * dy + Bv.w * dy * dy;
                    emit[k] = true;
                }
            }
        }
    }
    const bool any = tile_has_entries && (s_keys[tid * KMAX] != KEY_EMPTY);
    pixel_epilogue<KMAX, BLEND>(a, n, xi, yi, fz, fq, fid, emit, any, [&](int k) { return make_float2(fcx[k], fcy[k]); });
}

// ---------------------------------------------------------------------------------------------
// Depth-sliced splat-parallel rasterizer (production path for K <= 8).
//
// Shared-memory K-lists as described above, plus the three things that remove most of the
// (splat, pixel) candidate tests on dense clouds:
//   1. the tile's list arrives in NS front-to-back depth slices (binning key = tile x slice); before a slice
//      is touched the kernel compares its lower depth bound with the largest K-th depth of the tile and
//      stops if nothing behind that bound can enter any pixel's list;
//   2. every entry is first tested against the K-th depths of the 4x4-pixel blocks its bbox touches (16
//      values per tile, refreshed after every processing phase) -- one cheap, fully lane-parallel test;
//   3. survivors are compacted into a shared-memory queue and rasterized in full batches, so the expensive
//      per-pixel loops run with (nearly) all lanes busy instead of a small fraction of them.
// ---------------------------------------------------------------------------------------------

// Exact range of pixel indices i in [lo_clip, hi_clip] with |pix_to_ndc(i) - c| <= r, i.e. the pixels that
// pass the reference's bbox test (rasterize_points.cu:92) for one axis: arithmetic estimate, then the
// estimate is corrected by evaluating the very same fp32 test on the neighbouring pixels.
__device__ __forceinline__ void pixel_range(float c, float r, int lo_clip, int hi_clip, int S, float inv_S, bool pow2,
                                            float half_S, int &lo, int &hi) {
    if (!(fabsf(c) < 4.0f) || !(r < 2.0f)) {   // far-away centre / huge splat: estimates lose accuracy, test every pixel
        lo = lo_clip;
        hi = hi_clip;
        return;
    }
    lo = (int)fminf(fmaxf(ceilf((c - r + 1.0f) * half_S - 0.5f), -1.0f), (float)S);
    hi = (int)fmaxf(fminf(floorf((c + r + 1.0f) * half_S - 0.5f), (float)S), -2.0f);
    if (lo > 0 && !(fabsf(pix_to_ndc_fast(lo - 1, S, inv_S, pow2) - c) > r)) --lo;
    else if (lo <= hi && lo < S && (fabsf(pix_to_ndc_fast(max(lo, 0), S, inv_S, pow2) - c) > r)) ++lo;
    if (hi < S - 1 && !(fabsf(pix_to_ndc_fast(hi + 1, S, inv_S, pow2) - c) > r)) ++hi;
    else if (hi >= lo && hi >= 0 && (fabsf(pix_to_ndc_fast(min(hi, S - 1), S, inv_S, pow2) - c) > r)) --hi;
    lo = max(lo, lo_clip);
    hi = min(hi, hi_clip);
}

// explicit shared-space accesses with 32-bit addresses: inside the hot pixel loop the compiler otherwise rebuilds the
// generic->shared window base (S2R CgaCtaId + LEA ...) for every access, a third of the loop's instructions
// (the mov through an opaque asm keeps the value in a register instead of being rematerialised in the loop)
__device__ __forceinline__ uint32_t sh_addr(const void *p) {
    uint32_t a = (uint32_t)__cvta_generic_to_shared(p), r;
    asm volatile("mov.u32 %0, %1;" : "=r"(r) : "r"(a));
    return r;
}
__device__ __forceinline__ unsigned long long lds_u64_volatile(uint32_t addr) {
    unsigned long long v;
    asm volatile("ld.volatile.shared.u64 %0, [%1];" : "=l"(v) : "r"(addr) : "memory");
    return v;
}
__device__ __forceinline__ float lds_f32(uint32_t addr) {
    float v;
    asm("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ void sts_u64(uint32_t addr, unsigned long long v) {
    asm volatile("st.shared.u64 [%0], %1;" ::"r"(addr), "l"(v) : "memory");
}
__device__ __forceinline__ void sts_u16(uint32_t addr, unsigned short v) {
    asm volatile("st.shared.u16 [%0], %1;" ::"r"(addr), "h"(v) : "memory");
}

#ifndef DSS_RASTER_WPEND
#define DSS_RASTER_WPEND 128
#endif
#ifndef DSS_RASTER_QFILL
#define DSS_RASTER_QFILL 768
#endif
constexpr int RASTER_QCAP = 1024;
constexpr int RASTER_WPEND = DSS_RASTER_WPEND;   // accepted fragments a warp buffers before it inserts them
constexpr int RASTER_QFILL = DSS_RASTER_QFILL;   // survivors queued before a rasterization phase starts (<= QCAP - 256)

// lock-free sorted insert of one key into a pixel's K slots (chain of atomicMin, see above)
template <int KMAX>
__device__ __forceinline__ void klist_insert(unsigned long long *slot, unsigned long long carry) {
    // most buffered fragments are stale by the time they are inserted (the pixel's K-th key has dropped below them
    // since the test): one load settles those
    if (carry >= slot[KMAX - 1]) return;
#pragma unroll
    for (int k = 0; k < KMAX; ++k) {
        if (carry < slot[k]) {
            const unsigned long long old = atomicMin(&slot[k], carry);
            carry = old > carry ? old : carry;
        }
    }
}

// A warp inserts the fragments it has buffered: 32 at a time, all lanes busy.  Other warps may be testing
// pixels concurrently; they read the K-th key, which only ever decreases, so a stale value merely lets a
// superfluous fragment into a buffer -- the insert itself re-checks.
template <int KMAX>
__device__ __forceinline__ void pend_flush(unsigned long long *s_keys, const unsigned long long *wkey,
                                           const unsigned short *wpix, int count, int lane) {
    __syncwarp();
    for (int i = lane; i < count; i += 32) klist_insert<KMAX>(s_keys + (int)wpix[i] * KMAX, wkey[i]);
    __syncwarp();
}

// Launch order of the tiles: longest lists first (a counting sort of the tiles by the power of two of their list
// length, one block).  CTAs are handed out in block-index order, so without this the last wave of a launch is whatever
// tiles happen to come last -- often dense ones, with most SMs already idle.
__global__ void __launch_bounds__(1024)
raster_tile_order_kernel(const int32_t *__restrict__ tile_offsets, int NS, int ntiles, int32_t *__restrict__ order) {
    __shared__ int s_cnt[32], s_base[32];
    if (threadIdx.x < 32) s_cnt[threadIdx.x] = 0;
    __syncthreads();
    for (int t = threadIdx.x; t < ntiles; t += blockDim.x) {
        const int len = tile_offsets[(int64_t)(t + 1) * NS] - tile_offsets[(int64_t)t * NS];
        atomicAdd(&s_cnt[len > 0 ? 31 - __clz(len) + 1 : 0], 1);      // bucket 0: empty, k: 2^(k-1) <= len < 2^k
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int run = 0;
        for (int b = 31; b >= 0; --b) {   // descending work
            s_base[b] = run;
            run += s_cnt[b];
        }
    }
    __syncthreads();
    for (int t = threadIdx.x; t < ntiles; t += blockDim.x) {
        const int len = tile_offsets[(int64_t)(t + 1) * NS] - tile_offsets[(int64_t)t * NS];
        order[atomicAdd(&s_base[len > 0 ? 31 - __clz(len) + 1 : 0], 1)] = t;
    }
}

template <int KMAX, bool PER_POINT_CUTOFF, bool BLEND, bool STATS, int MINB>
__global__ void __launch_bounds__(RASTER_THREADS, MINB)
raster_sliced_kernel(const __grid_constant__ RasterArgs a) {
    __shared__ unsigned long long s_keys[RASTER_THREADS * KMAX];   // [pixel][k]
    __shared__ int s_queue[RASTER_QCAP];
    __shared__ unsigned long long s_pend_key[RASTER_THREADS / 32][RASTER_WPEND];   // per warp: accepted fragments
    __shared__ unsigned short s_pend_pix[RASTER_THREADS / 32][RASTER_WPEND];       //           waiting for insertion
    __shared__ float s_xf[RASTER_TILE], s_yf[RASTER_TILE];   // exact pixel centres of the tile
    __shared__ unsigned int s_blk[16];
    __shared__ unsigned int s_wblk[RASTER_THREADS / 32][4];   // per warp: K-th depth maxima of its four 4x2-pixel groups
    __shared__ int s_qcount;
    __shared__ unsigned int s_tilemax;

    const int S = a.S, B = a.B, NS = a.NS;
    const int gt = a.tile_order ? a.tile_order[blockIdx.x] : (int)blockIdx.x;   // global tile: view * B*B + tile
    const int n = gt / (B * B);
    const int tile = gt - n * B * B;
    const int ty = tile / B, tx = tile - ty * B;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t tb = ((int64_t)n * B * B + tile) * NS;
    // The id buffer is sized from the PREVIOUS call (bin_and_raster never waits for the list size).  A tile whose list
    // does not fit it completely (`overflow`) takes its candidates from the view's records directly: every splat of
    // the view is walked, the entry-level cull's rectangle test drops those that miss the tile -- slow, correct, rare.
    const bool overflow = a.tile_offsets[tb + NS] > a.ids_capacity;
    const ViewRange ovr = view_range(a.first_idx, a.num_points, n, a.P0);
    const int beg = overflow ? 0 : a.tile_offsets[tb];
    const int end = overflow ? (int)min(ovr.count, (int64_t)INT32_MAX) : a.tile_offsets[tb + NS];
    const int ofirst = (int)ovr.first;
    auto list_id = [&](int j) -> int { return overflow ? ofirst + j : a.tile_ids[j]; };
    const int tx0 = tx * RASTER_TILE, ty0 = ty * RASTER_TILE;
    const int tx1 = min(tx0 + RASTER_TILE, S) - 1, ty1 = min(ty0 + RASTER_TILE, S) - 1;
    const bool pow2 = (S & (S - 1)) == 0;
    const float inv_S = 1.0f / (float)S, half_S = 0.5f * (float)S;
    constexpr unsigned FULL = 0xffffffffu;
    // An overflowing tile must see the records its list would have held, no more: the binning's closed bin predicate
    // (binning.cu: bin_range) for this tile, with the same fp32 edges (s_xf / s_yf hold the tile's pixel centres, 16 of
    // them even where the tile is cut by the image edge, like the bin's) and the same ordered comparisons.  The rectangle
    // cull below alone would let a record with a NaN centre or radius through (its clamps turn NaN into tile bounds).
    auto in_tile_bin = [&](const float4 &A, float ry) -> bool {
        return (A.x - A.w <= s_xf[RASTER_TILE - 1] + inv_S) && (s_xf[0] - inv_S <= A.x + A.w) &&
               (A.y - ry <= s_yf[RASTER_TILE - 1] + inv_S) && (s_yf[0] - inv_S <= A.y + ry);
    };

    unsigned int st_scanned = 0, st_surv = 0, st_tests = 0, st_acc = 0, st_skip = 0, st_visit = 0;
    if (beg < end) {
#pragma unroll
        for (int k = 0; k < KMAX; ++k) s_keys[k * RASTER_THREADS + tid] = KEY_EMPTY;
        if (tid < 16) s_blk[tid] = 0xffffffffu;
        if (tid < RASTER_TILE) {
            s_xf[tid] = pix_to_ndc(tx0 + tid, S);
            s_yf[tid] = pix_to_ndc(ty0 + tid, S);
        }
        if (tid == 0) {
            s_qcount = 0;
            s_tilemax = 0xffffffffu;
        }
        __syncthreads();
        const SliceMap sm = make_slice_map(a.zrange, n, NS);
        unsigned long long *wkey = s_pend_key[warp];
        unsigned short *wpix = s_pend_pix[warp];
        const uint32_t sa_kth = sh_addr(s_keys) + (KMAX - 1) * 8, sa_xf = sh_addr(s_xf), sa_yf = sh_addr(s_yf);
        const uint32_t sa_wkey = sh_addr(wkey), sa_wpix = sh_addr(wpix);
        // The tile's list is ordered by depth slice: walk it front to back in chunks of 256 entries.  Every entry at
        // or behind position `base` has z >= slice_bound(slice of base): stop as soon as that cannot enter any list.
        int base = beg, s_cur = 0;
        int nq_acc = 0;   // survivors queued since the last rasterization phase (uniform)
        // software pipeline of the list walk: ids are fetched two chunks ahead, the (gathered) records one chunk ahead,
        // so that the dependent id -> record loads of a chunk are in flight while the previous chunk is rasterized
        int id0 = (beg + tid < end) ? list_id(beg + tid) : -1;
        int id1 = (beg + RASTER_THREADS + tid < end) ? list_id(beg + RASTER_THREADS + tid) : -1;
        float4 pA = make_float4(0.f, 0.f, -1.f, 0.f);
        float pry = 0.f;
        if (id0 >= 0) {
            pA = __ldg(&a.rec[2 * (int64_t)id0]);
            pry = __ldg(&a.rec[2 * (int64_t)id0 + 1]).x;
        }
        while (true) {
            bool more = base < end;
            bool chunk_survive = false;
            if (more && !overflow) {
                while (s_cur + 1 < NS && a.tile_offsets[tb + s_cur + 1] <= base) ++s_cur;
                if (s_cur > 0 && __float_as_uint(slice_bound(sm, s_cur)) > s_tilemax) {
                    more = false;
                    if (STATS && tid == 0) st_skip += NS - s_cur;
                }
            }
            if (more) {
                // ---- phase 1: entry-level cull against the block thresholds, survivors -> queue ----
                const int j = base + tid;
                bool survive = false;
                const int id = id0;
                const float4 A = pA;
                const float ry = pry;
                id0 = id1;
                id1 = (j + 2 * RASTER_THREADS < end) ? list_id(j + 2 * RASTER_THREADS) : -1;
                if (id0 >= 0) {
                    pA = __ldg(&a.rec[2 * (int64_t)id0]);
                    pry = __ldg(&a.rec[2 * (int64_t)id0 + 1]).x;
                }
                if (j < end) {
                    if (STATS) st_scanned++;
                    if (A.z >= 0.0f && (!overflow || in_tile_bin(A, ry))) {
                        const int x0 = max(tx0, (int)fmaxf(ceilf((A.x - A.w + 1.0f) * half_S - 0.5f) - 1.0f, -1.0f));
                        const int x1 = min(tx1, (int)fminf(floorf((A.x + A.w + 1.0f) * half_S - 0.5f) + 1.0f, (float)S));
                        const int y0 = max(ty0, (int)fmaxf(ceilf((A.y - ry + 1.0f) * half_S - 0.5f) - 1.0f, -1.0f));
                        const int y1 = min(ty1, (int)fminf(floorf((A.y + ry + 1.0f) * half_S - 0.5f) + 1.0f, (float)S));
                        if (x0 <= x1 && y0 <= y1) {
                            unsigned int zb = 0;
                            for (int by = (y0 - ty0) >> 2; by <= (y1 - ty0) >> 2; ++by)
                                for (int bx = (x0 - tx0) >> 2; bx <= (x1 - tx0) >> 2; ++bx) zb = max(zb, s_blk[by * 4 + bx]);
                            survive = __float_as_uint(A.z + 0.0f) <= zb;
                        }
                    }
                }
                const unsigned m = __ballot_sync(FULL, survive);
                int wbase = 0;
                if (lane == 0 && m) wbase = atomicAdd(&s_qcount, __popc(m));
                wbase = __shfl_sync(FULL, wbase, 0);
                if (survive) {
                    s_queue[wbase + __popc(m & ((1u << lane) - 1u))] = id;
                    if (STATS) st_surv++;
                }
                chunk_survive = survive;
                base += RASTER_THREADS;
            }
            // one barrier gives every thread the number of survivors appended by this chunk (the queue slots themselves
            // come from s_qcount's atomics, which the next chunk may already be using)
            nq_acc += __syncthreads_count(chunk_survive);
            const int nq = nq_acc;
            if (more && nq <= RASTER_QFILL && base < end) continue;   // keep filling
            if (nq > 0) {
                // ---- phase 2: rasterize the queued survivors, one splat per thread: every lane steps through ITS
                //      splat's pixel rectangle (row-major), the trip count is the largest rectangle of the warp's 32
                //      splats.  Accepted fragments go to the warp's own buffer (no atomics, no election: the fill
                //      level is a warp-uniform register) and are inserted 32 at a time when it runs full ----
                int wcount = 0;
                for (int ib = 0; ib < nq; ib += RASTER_THREADS) {
                    const int i = ib + tid;
                    const bool have = i < nq;
                    const int sid = have ? s_queue[i] : 0;
                    float4 A = make_float4(0.f, 0.f, 0.f, 0.f), Bv = make_float4(0.f, 0.f, 0.f, 0.f);
                    float cut = 0.f;
                    if (have) {
                        A = __ldg(&a.rec[2 * (int64_t)sid]);
                        Bv = __ldg(&a.rec[2 * (int64_t)sid + 1]);
                        cut = (PER_POINT_CUTOFF && a.cutoff) ? __ldg(&a.cutoff[sid]) : a.cutoff_uniform;
                    }
                    const unsigned long long key = make_key(A.z + 0.0f, sid);
                    int x0 = tx0, x1 = tx0 - 1, y0 = ty0, y1 = ty0 - 1;
                    if (have) {
                        pixel_range(A.x, A.w, tx0, tx1, S, inv_S, pow2, half_S, x0, x1);
                        pixel_range(A.y, Bv.x, ty0, ty1, S, inv_S, pow2, half_S, y0, y1);
                    }
                    const int w = max(x1 - x0 + 1, 0), h = max(y1 - y0 + 1, 0);
                    const int c = w * h;
                    const int Cm = __reduce_max_sync(FULL, c);
                    int xl = (c > 0) ? x0 - tx0 : 0, yl = (c > 0) ? y0 - ty0 : 0;
                    const int xl0 = xl, xl1 = (c > 0) ? x1 - tx0 : 0;
                    for (int t = 0; t < Cm; ++t) {
                        const bool active = t < c;
                        const int pixl = yl * RASTER_TILE + xl;
                        const unsigned long long kth = lds_u64_volatile(sa_kth + pixl * (KMAX * 8));
                        const float dx = lds_f32(sa_xf + xl * 4) - A.x;
                        const float dy = lds_f32(sa_yf + yl * 4) - A.y;
                        // rasterize_points.cu:92-97 -- same expression tree for q as the reference
                        const float qv = Bv.y * dx * dx + Bv.z * dx * dy + Bv.w * dy * dy;
                        const bool ok = active && (key < kth) && !(fabsf(dx) > A.w) && !(fabsf(dy) > Bv.x) && !(qv > cut);
                        if (STATS) st_tests += active ? 1u : 0u;
                        const unsigned pm = __ballot_sync(FULL, ok);
                        if (pm) {
                            if (wcount + 32 > RASTER_WPEND) {
                                pend_flush<KMAX>(s_keys, wkey, wpix, wcount, lane);
                                wcount = 0;
                            }
                            if (ok) {
                                if (STATS) st_acc++;
                                const int pi = wcount + __popc(pm & ((1u << lane) - 1u));
                                sts_u64(sa_wkey + pi * 8, key);
                                sts_u16(sa_wpix + pi * 2, (unsigned short)pixl);
                            }
                            wcount += __popc(pm);
                        }
                        // next pixel of this lane's rectangle; lanes that are done stay on their last pixel
                        if (t + 1 < c) {
                            if (++xl > xl1) {
                                xl = xl0;
                                ++yl;
                            }
                        }
                    }
                }
                pend_flush<KMAX>(s_keys, wkey, wpix, wcount, lane);
                __syncthreads();
                // ---- phase 3: refresh the block / tile thresholds (K-th depth, pixels outside the image never block).
                //      A warp covers two pixel rows: the 8 lanes of a 4-pixel x 2-row group reduce among themselves,
                //      the two warps of a block row are combined after one barrier (no atomics, nothing to zero) ----
                {
                    const int pxl = tid & (RASTER_TILE - 1), pyl = tid >> 4;
                    const bool in_img = (tx0 + pxl < S) && (ty0 + pyl < S);
                    const unsigned int kz = in_img ? (unsigned int)(s_keys[tid * KMAX + KMAX - 1] >> 32) : 0u;
                    const unsigned int gmask = 0x000f000fu << (4 * ((lane & 15) >> 2));
                    const unsigned int gmax = __reduce_max_sync(gmask, kz);
                    if ((lane & 19) == 0) s_wblk[warp][lane >> 2] = gmax;   // lanes 0, 4, 8, 12
                    if (tid == 0) s_qcount = 0;
                }
                __syncthreads();
                if (tid < 16) s_blk[tid] = max(s_wblk[2 * (tid >> 2)][tid & 3], s_wblk[2 * (tid >> 2) + 1][tid & 3]);
                if (tid == 32) {
                    unsigned int mx = 0;
#pragma unroll
                    for (int i = 0; i < RASTER_THREADS / 32; ++i)
#pragma unroll
                        for (int c = 0; c < 4; ++c) mx = max(mx, s_wblk[i][c]);
                    s_tilemax = mx;
                }
                __syncthreads();
                nq_acc = 0;
                if (STATS && tid == 0) st_visit++;
            }
            if (!more || base >= end) break;
        }
    }
    if (STATS && a.stats) {
        atomicAdd(&a.stats[0], (unsigned long long)st_scanned);
        atomicAdd(&a.stats[1], (unsigned long long)st_surv);
        atomicAdd(&a.stats[2], (unsigned long long)st_tests);
        atomicAdd(&a.stats[3], (unsigned long long)st_acc);
        if (tid == 0) {
            atomicAdd(&a.stats[4], (unsigned long long)st_skip);
            atomicAdd(&a.stats[5], (unsigned long long)st_visit);
            if (overflow) atomicAdd(&a.stats[6], 1ull);
        }
    }
    sliced_epilogue<KMAX, BLEND>(a, s_keys, beg < end, n, tx0, ty0, pow2, inv_S);
}


template <int KMAX>
static int launch_scatter(dss_ctx *ctx, const RasterArgs &a_in, cudaStream_t st) {
    RasterArgs a = a_in;
    const int ntiles = a.B * a.B * a.N;
    dim3 grid((unsigned)ntiles);
    StageScope prof(ctx, ST_RASTER_FWD, st);
    a.tile_order = nullptr;
    if (!ctx->no_tile_order && ntiles > 4 * ctx->sm_count) {
        int32_t *order = nullptr;
        int rc = ctx_get(ctx, BUF_TILE_ORDER, (size_t)ntiles, &order);
        if (rc) return rc;
        raster_tile_order_kernel<<<1, 1024, 0, st>>>(a.tile_offsets, a.NS, ntiles, order);
        DSS_LAUNCH_CHECK(ctx);
        a.tile_order = order;
    }
    const bool blend = a.image != nullptr;
    if (a.stats) {   // debug counters on: one generic instantiation is enough
        if (blend) raster_sliced_kernel<KMAX, true, true, true, 4><<<grid, RASTER_THREADS, 0, st>>>(a);
        else raster_sliced_kernel<KMAX, true, false, true, 4><<<grid, RASTER_THREADS, 0, st>>>(a);
    } else if (blend) {
        if (a.cutoff)
            raster_sliced_kernel<KMAX, true, true, false, 4><<<grid, RASTER_THREADS, 0, st>>>(a);
        else if (ctx->raster_minb5)
            raster_sliced_kernel<KMAX, false, true, false, 5><<<grid, RASTER_THREADS, 0, st>>>(a);
        else
            raster_sliced_kernel<KMAX, false, true, false, 4><<<grid, RASTER_THREADS, 0, st>>>(a);
    } else {
        if (a.cutoff)
            raster_sliced_kernel<KMAX, true, false, false, 4><<<grid, RASTER_THREADS, 0, st>>>(a);
        else
            raster_sliced_kernel<KMAX, false, false, false, 4><<<grid, RASTER_THREADS, 0, st>>>(a);
    }
    DSS_LAUNCH_CHECK(ctx);
    return DSS_OK;
}

template <int KMAX>
static int launch_raster(dss_ctx *ctx, const RasterArgs &a, cudaStream_t st) {
    dim3 grid((unsigned)(a.B * a.B), (unsigned)a.N);
    StageScope prof(ctx, ST_RASTER_FWD, st);
    const bool blend = a.image != nullptr;
    if (blend) {
        if (a.cutoff)
            raster_fwd_kernel<KMAX, true, true><<<grid, RASTER_THREADS, 0, st>>>(a);
        else
            raster_fwd_kernel<KMAX, false, true><<<grid, RASTER_THREADS, 0, st>>>(a);
    } else {
        if (a.cutoff)
            raster_fwd_kernel<KMAX, true, false><<<grid, RASTER_THREADS, 0, st>>>(a);
        else
            raster_fwd_kernel<KMAX, false, false><<<grid, RASTER_THREADS, 0, st>>>(a);
    }
    DSS_LAUNCH_CHECK(ctx);
    return DSS_OK;
}

int raster_forward(dss_ctx *ctx, const RasterArgs &a, cudaStream_t st) {
    if (a.N <= 0 || a.S <= 0) return DSS_OK;
    if (a.K <= 5) return launch_scatter<5>(ctx, a, st);
    if (a.K <= 8) return launch_scatter<8>(ctx, a, st);
    if (a.K <= 16) return launch_raster<16>(ctx, a, st);
    return launch_raster<DSS_MAX_POINTS_PER_PIXEL>(ctx, a, st);
}

int plan_tiles(dss_ctx *ctx, int N, int S, int K, TilePlan *plan) {
    const int B = (S + RASTER_TILE - 1) / RASTER_TILE;
    int NS = K <= 8 ? choose_depth_slices(B) : 1;   // the sliced rasterizer (K <= 8) walks its lists by depth slice
    if (NS > 1 && ctx->ns_override > 0 && ctx->ns_override < NS) NS = ctx->ns_override;
    const int64_t nb = (int64_t)N * B * B * NS;
    if (nb + 1 >= (int64_t)INT32_MAX) {
        set_error("too many tiles (%lld)", (long long)nb);
        return DSS_E_INVALID;
    }
    plan->B = B;
    plan->NS = NS;
    // (the packed rectangle needs B <= 128 tiles per side and <= 16 slices, like the block histograms)
    plan->packed = B <= 128 && NS <= 16 && (int64_t)B * B * NS <= 48 * 1024 && !ctx->bin_direct && !ctx->bin_no_rects;
    return DSS_OK;
}

int bin_and_raster(dss_ctx *ctx, RasterArgs a, const int64_t *first_idx, const int64_t *num_points,
                   int64_t P0, cudaStream_t st, const CountedBins *counted) {
    const int S = a.S;
    const bool scatter_path = a.K <= 8;
    TilePlan plan;
    int rc;
    if ((rc = plan_tiles(ctx, a.N, S, a.K, &plan))) return rc;
    a.B = plan.B;
    a.NS = plan.NS;
    a.first_idx = first_idx;
    a.num_points = num_points;
    a.P0 = P0;
    const int64_t nb = (int64_t)a.N * a.B * a.B * a.NS;
    int32_t *counts = nullptr, *offsets = nullptr;
    int32_t *ids = nullptr;
    float *zrange = const_cast<float *>(a.zrange);   // non-null: the caller's preprocess already produced it
    if ((rc = ctx_get(ctx, BUF_TILE_COUNTS, (size_t)(nb + 1), &counts))) return rc;
    if ((rc = ctx_get(ctx, BUF_TILE_OFFSETS, (size_t)(nb + 1), &offsets))) return rc;
    unsigned int *rects = nullptr;
    if (counted) {
        if ((rc = exclusive_scan_i32(ctx, counts, offsets, nb + 1, st))) return rc;
    } else {
        if (a.NS > 1 && zrange == nullptr) {
            if ((rc = ctx_get(ctx, BUF_ZRANGE, (size_t)(2 * a.N), &zrange))) return rc;
            if ((rc = compute_zrange(ctx, a.rec, first_idx, num_points, a.N, P0, zrange, st))) return rc;
        }
        const int64_t Ptot = (first_idx == nullptr) ? (int64_t)a.N * P0 : P0;
        if (plan.packed && Ptot > 0 && (rc = ctx_get(ctx, BUF_BIN_RECTS, (size_t)Ptot, &rects))) return rc;
        if ((rc = bin_count_and_scan(ctx, a.rec, first_idx, num_points, a.N, P0, S, RASTER_TILE, a.NS, zrange, counts,
                                     offsets, rects, st)))
            return rc;
    }
    a.zrange = zrange;
    a.tile_offsets = offsets;
    a.stats = nullptr;
    if (ctx->raster_stats) {
        unsigned long long *sp = nullptr;
        if ((rc = ctx_get(ctx, BUF_STATS, 8, &sp))) return rc;
        a.stats = sp;
    }
    // Size of the CSR id list.  It is only known on the device (last entry of the scan), and the host never waits for
    // it in steady state: the scan's total is published into mapped pinned memory (no copy engine, no sync) and read
    // by the NEXT call, which grows the buffer if the lists have outgrown it.  Meanwhile scatter and rasterizer run
    // with the buffer they have: the scatter drops entries beyond the capacity, the rasterizer recognises the tiles
    // whose lists are incomplete (offset past the capacity) and takes their candidates from the view's records
    // directly -- slower for those tiles, same result.  Only a context that has never sized the buffer (first call)
    // and the pixel-parallel fallback for K > 8 (which has no such path) wait for the total.
    int64_t cap = (int64_t)(ctx->cap[BUF_TILE_IDS] / sizeof(int32_t));
    volatile int32_t *h_total = reinterpret_cast<volatile int32_t *>(ctx->h_pinned);
    if ((rc = publish_words(ctx, offsets + nb, ctx->h_pinned, 1, st))) return rc;
    const bool must_wait = cap == 0 || !scatter_path || ctx->sync_forward;
    int64_t want = 0;
    if (must_wait) {
        DSS_CUDA_TRY(cudaStreamSynchronize(st));
        want = (int64_t)h_total[0];
    } else {
        want = ctx->tile_total_hint;    // what the previous call published (read below, after its kernels were queued)
    }
    if (want < 0) {
        set_error("tile list size overflowed int32");
        return DSS_E_INVALID;
    }
    if (want > cap) cap = want + want / 4 + 1024;   // headroom so that slowly growing lists never outgrow the buffer
    if (cap > (int64_t)INT32_MAX) cap = INT32_MAX;
    if (cap < 1) cap = 1;
    if ((rc = ctx_get(ctx, BUF_TILE_IDS, (size_t)cap, &ids))) return rc;      // grows when needed, otherwise a no-op
    {
        const size_t have = ctx->cap[BUF_TILE_IDS] / sizeof(int32_t);
        a.ids_capacity = (int)(have > (size_t)INT32_MAX ? (size_t)INT32_MAX : have);
        // testing (dss_debug_limit_tile_capacity): pretend the buffer is smaller, which forces the overflow path
        if (ctx->tile_cap_limit > 0 && a.ids_capacity > ctx->tile_cap_limit) a.ids_capacity = (int)ctx->tile_cap_limit;
    }
    if (!scatter_path && (int64_t)h_total[0] > a.ids_capacity) {
        set_error("internal: tile list buffer too small for the pixel-parallel path");
        return DSS_E_CAPACITY;
    }
    if (counted)
        rc = bin_scatter_counted(ctx, first_idx, num_points, a.N, P0, a.B, a.NS, offsets, counted->block_offsets,
                                 counted->blocks, counted->rects, ids, a.ids_capacity, st);
    else
        rc = bin_scatter(ctx, a.rec, first_idx, num_points, a.N, P0, S, RASTER_TILE, a.NS, zrange, offsets, counts, ids,
                         a.ids_capacity, rects, st);
    if (rc) return rc;
    a.tile_ids = ids;
    if ((rc = raster_forward(ctx, a, st))) return rc;
    // hint for the next call: whatever total the device has published by now (this call's, if the GPU is ahead of
    // the host, otherwise an earlier one) -- it only sizes the buffer, correctness never depends on it
    ctx->tile_total_hint = (int64_t)h_total[0];
    return DSS_OK;
}

}  // namespace dss

extern "C" {

int dss_debug_raster_stats(dss_ctx *ctx, int enable, uint64_t out[8]) {
    using namespace dss;
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    unsigned long long *sp = nullptr;
    int rc = ctx_get(ctx, BUF_STATS, 8, &sp);
    if (rc) return rc;
    DSS_CUDA_TRY(cudaDeviceSynchronize());
    if (out) DSS_CUDA_TRY(cudaMemcpy(out, sp, 8 * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    if (enable) DSS_CUDA_TRY(cudaMemset(sp, 0, 8 * sizeof(unsigned long long)));
    ctx->raster_stats = enable ? 1 : 0;
    return DSS_OK;
}

int64_t dss_debug_tile_total(const dss_ctx *ctx) {
    // the tile-list size the device published last (mapped pinned word, read without synchronising)
    return ctx ? (int64_t)(*reinterpret_cast<volatile int32_t *>(ctx->h_pinned)) : 0;
}

int dss_debug_limit_tile_capacity(dss_ctx *ctx, int64_t max_entries) {
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    DSS_REQUIRE(max_entries >= 0 && max_entries <= (int64_t)INT32_MAX, "bad limit");
    ctx->tile_cap_limit = max_entries;
    return DSS_OK;
}

int dss_debug_bin_no_rects(dss_ctx *ctx, int on) {
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    ctx->bin_no_rects = on ? 1 : 0;
    return DSS_OK;
}

int dss_debug_tile_lists(dss_ctx *ctx, int n_views, float *zrange, int64_t n_offsets, int32_t *offsets, int64_t n_ids,
                         int32_t *ids, void *stream) {
    using namespace dss;
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    DSS_REQUIRE(n_views >= 0 && n_offsets >= 0 && n_ids >= 0, "negative size");
    const struct {
        BufId id;
        void *dst;
        size_t bytes;
    } copies[3] = {{BUF_ZRANGE, zrange, (size_t)n_views * 2 * sizeof(float)},
                   {BUF_TILE_OFFSETS, offsets, (size_t)n_offsets * sizeof(int32_t)},
                   {BUF_TILE_IDS, ids, (size_t)n_ids * sizeof(int32_t)}};
    for (const auto &c : copies) {
        if (!c.dst || c.bytes == 0) continue;
        DSS_REQUIRE(c.bytes <= ctx->cap[c.id], "more entries than the scratch holds");
        DSS_CUDA_TRY(cudaMemcpyAsync(c.dst, ctx->buf[c.id], c.bytes, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
    }
    return DSS_OK;
}

int dss_splat_points(dss_ctx *ctx, const float *points, const float *ellipse_params, const float *cutoff_thres,
                     const float *radii, const int64_t *first_idx, const int64_t *num_points, int N, int64_t P,
                     float depth_merging_thres, int image_size, int points_per_pixel, int bin_size, int32_t *idx,
                     float *zbuf, float *qvalue, float *occupancy, void *stream) {
    using namespace dss;
    (void)bin_size;
    cudaStream_t st = (cudaStream_t)stream;
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    DSS_REQUIRE(N >= 0 && P >= 0, "negative size");
    DSS_REQUIRE(image_size > 0, "image_size must be positive");
    DSS_REQUIRE(points_per_pixel > 0 && points_per_pixel <= DSS_MAX_POINTS_PER_PIXEL,
                "points_per_pixel must be in [1, 64]");
    DSS_REQUIRE(P < (int64_t)INT32_MAX, "more than 2^31-1 packed points");
    if (N == 0) return DSS_OK;
    DSS_REQUIRE(idx && occupancy && first_idx && num_points, "null pointer");
    DSS_REQUIRE(P == 0 || (points && ellipse_params && cutoff_thres && radii), "null input array");
    float4 *rec = nullptr;
    int rc;
    if ((rc = ctx_get(ctx, BUF_RECORDS, (size_t)(2 * (P > 0 ? P : 1)), &rec))) return rc;
    if ((rc = pack_records(ctx, points, radii, ellipse_params, P, rec, st))) return rc;
    RasterArgs a;
    memset(&a, 0, sizeof(a));
    a.rec = rec;
    a.cutoff = cutoff_thres;
    a.cutoff_uniform = 0.f;
    a.N = N;
    a.S = image_size;
    a.K = points_per_pixel;
    a.depth_merge = depth_merging_thres;
    a.idx = idx;
    a.zbuf = zbuf;
    a.qvalue = qvalue;
    a.occ = occupancy;
    return bin_and_raster(ctx, a, first_idx, num_points, P, st);
}

}  // extern "C"
