// binning.cu -- splat records, screen-tile binning (count -> scan -> scatter), 2-D grid binning.
//
// Replaces RasterizePointsCoarseCuda (DSS/csrc/rasterize_points.cu:293-500): instead of a dense
// (N,B,B,M) int32 tensor filled by 64 CTAs that brute-force all B^2 bins per point, every splat
// computes its bin rectangle in O(1), counts go through an on-device exclusive scan and ids are
// scattered into exact-size CSR lists.
#include "binning.cuh"
#include "common.cuh"
#include "kernels.cuh"

namespace dss {

// ---------------------------------------------------------------------------------------------
// pack: (points (P,3), radii (P,2), ellipse (P,3)) -> 32-byte records
//   rec[2p]   = {px, py, pz, rx}
//   rec[2p+1] = {ry, a, b, c}
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
pack_records_kernel(const float *__restrict__ points, const float *__restrict__ radii,
                    const float *__restrict__ ellipse, int64_t P, float4 *__restrict__ rec) {
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= P) return;
    float a = 0.f, b = 0.f, c = 0.f;
    if (ellipse) {
        a = ellipse[p * 3 + 0];
        b = ellipse[p * 3 + 1];
        c = ellipse[p * 3 + 2];
    }
    rec[2 * p] = make_float4(points[p * 3 + 0], points[p * 3 + 1], points[p * 3 + 2], radii[p * 2 + 0]);
    rec[2 * p + 1] = make_float4(radii[p * 2 + 1], a, b, c);
}

int pack_records(dss_ctx *ctx, const float *points, const float *radii, const float *ellipse, int64_t P,
                 float4 *rec, cudaStream_t st) {
    if (P == 0) return DSS_OK;
    StageScope prof(ctx, ST_PACK, st);
    pack_records_kernel<<<(unsigned)((P + 255) / 256), 256, 0, st>>>(points, radii, ellipse, P, rec);
    DSS_LAUNCH_CHECK(ctx);
    return DSS_OK;
}

// ---------------------------------------------------------------------------------------------
// Depth slices.  Tile lists are ordered front to back in NS coarse slices of the view's depth range so
// that the rasterizer can stop as soon as every pixel of a tile already holds K nearer fragments.
// zrange[n] = {zmin, zmax} over the renderable (z >= 0) splats of view n.  Slice s covers
// [slice_bound(s), slice_bound(s+1)); depth_slice() guarantees slice_bound(slice) <= z.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
zrange_kernel(const float4 *__restrict__ rec, const int64_t *__restrict__ first_idx,
              const int64_t *__restrict__ num_points, int64_t P0_shared, int32_t *__restrict__ zrange) {
    const int n = blockIdx.y;
    const ViewRange vr = view_range(first_idx, num_points, n, P0_shared);
    int zmin = 0x7f7fffff, zmax = 0;   // float bits; non-negative floats order like ints
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < vr.count;
         i += (int64_t)gridDim.x * blockDim.x) {
        const float z = __ldg(&rec[2 * (vr.first + i)]).z;
        if (z >= 0.0f && z < 3.0e38f) {
            const int b = __float_as_int(z + 0.0f);
            zmin = min(zmin, b);
            zmax = max(zmax, b);
        }
    }
    zmin = __reduce_min_sync(0xffffffffu, zmin);
    zmax = __reduce_max_sync(0xffffffffu, zmax);
    if ((threadIdx.x & 31) == 0) {
        atomicMin(&zrange[2 * n], zmin);
        atomicMax(&zrange[2 * n + 1], zmax);
    }
}

__global__ void zrange_init_kernel(int32_t *zrange, int N) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < N) {
        zrange[2 * i] = 0x7f7fffff;
        zrange[2 * i + 1] = 0;
    }
}

int init_zrange(dss_ctx *ctx, float *zrange, int N, cudaStream_t st) {
    zrange_init_kernel<<<(N + 127) / 128, 128, 0, st>>>(reinterpret_cast<int32_t *>(zrange), N);
    DSS_LAUNCH_CHECK(ctx);
    return DSS_OK;
}

int compute_zrange(dss_ctx *ctx, const float4 *rec, const int64_t *first_idx, const int64_t *num_points, int N,
                   int64_t P0, float *zrange, cudaStream_t st) {
    StageScope prof(ctx, ST_BIN_COUNT, st);
    zrange_init_kernel<<<(N + 127) / 128, 128, 0, st>>>(reinterpret_cast<int32_t *>(zrange), N);
    DSS_LAUNCH_CHECK(ctx);
    if (P0 > 0) {
        int64_t b = (P0 + 2047) / 2048;
        if (b > ctx->sm_count * 4) b = ctx->sm_count * 4;
        dim3 grid((unsigned)b, N);
        zrange_kernel<<<grid, 256, 0, st>>>(rec, first_idx, num_points, P0, reinterpret_cast<int32_t *>(zrange));
        DSS_LAUNCH_CHECK(ctx);
    }
    return DSS_OK;
}

// ---------------------------------------------------------------------------------------------
// count / scatter with block-level aggregation.  A block owns a contiguous chunk of BIN_ITEMS*256
// splats of one view, keeps the per-tile histogram of that chunk in shared memory and touches global
// memory with ONE atomic per (block, non-empty tile) instead of one per (splat, tile): the per-tile
// counters are a few hundred hot addresses and L2 serialises same-address atomics.
// Fallback (plain global atomics) when the histogram of B*B tiles does not fit in shared memory.
// ---------------------------------------------------------------------------------------------
constexpr int BIN_THREADS = 256;
constexpr int BIN_ITEMS = 16;   // splats per thread (32 measured slower: fewer, longer blocks)
constexpr int BIN_CHUNK = BIN_THREADS * BIN_ITEMS;
constexpr int BIN_MAX_SMEM_TILES = 48 * 1024;   // 192 KB of histogram at most

template <bool SMEM, bool POW2>
__global__ void __launch_bounds__(BIN_THREADS)
bin_count_kernel(const float4 *__restrict__ rec, const int64_t *__restrict__ first_idx,
                 const int64_t *__restrict__ num_points, int64_t P0_shared, int S, int bin, int B, int NS,
                 const float *__restrict__ zrange, int32_t *__restrict__ counts, unsigned int *__restrict__ rects) {
    extern __shared__ int32_t s_hist[];
    const int n = blockIdx.y;
    const int nt = B * B * NS;
    const SliceMap sm = make_slice_map(zrange, n, NS);
    const ViewRange vr = view_range(first_idx, num_points, n, P0_shared);
    const int64_t chunk0 = (int64_t)blockIdx.x * BIN_CHUNK;
    if (chunk0 >= vr.count) return;
    int32_t *cnt = counts + (int64_t)n * nt;
    if (SMEM) {
        for (int t = threadIdx.x; t < nt; t += BIN_THREADS) s_hist[t] = 0;
        __syncthreads();
    }
#pragma unroll 2
    for (int j = 0; j < BIN_ITEMS; ++j) {
        const int64_t i = chunk0 + j * BIN_THREADS + threadIdx.x;
        if (i >= vr.count) break;
        const int64_t p = vr.first + i;
        const float4 A = __ldg(&rec[2 * p]);
        const float ry = __ldg(&rec[2 * p + 1]).x;
        const BinRect r = splat_bin_rect<POW2>(A, ry, bin, S, B);
        const int sl = r.empty ? 0 : depth_slice(sm, A.z);
        // the scatter pass reuses the rectangle instead of deriving it again (and never touches the records)
        if (rects) rects[p] = pack_rect(r, sl);
        if (r.empty) continue;
        for (int by = r.y0; by <= r.y1; ++by)
            for (int bx = r.x0; bx <= r.x1; ++bx) {
                const int key = (by * B + bx) * NS + sl;
                atomicAdd(SMEM ? &s_hist[key] : &cnt[key], 1);
            }
    }
    if (SMEM) {
        __syncthreads();
        for (int t = threadIdx.x; t < nt; t += BIN_THREADS) {
            const int v = s_hist[t];
            if (v) atomicAdd(&cnt[t], v);
        }
    }
}

// cursors: copy of offsets (N*B*B), advanced atomically; ids: CSR payload.
template <bool SMEM, bool POW2>
__global__ void __launch_bounds__(BIN_THREADS)
bin_scatter_kernel(const float4 *__restrict__ rec, const int64_t *__restrict__ first_idx,
                   const int64_t *__restrict__ num_points, int64_t P0_shared, int S, int bin, int B, int NS,
                   const float *__restrict__ zrange, int32_t *__restrict__ cursors, int32_t *__restrict__ ids,
                   int ids_capacity, const unsigned int *__restrict__ rects) {
    extern __shared__ int32_t s_hist[];
    const int n = blockIdx.y;
    const int nt = B * B * NS;
    const SliceMap sm = make_slice_map(zrange, n, NS);
    const ViewRange vr = view_range(first_idx, num_points, n, P0_shared);
    const int64_t chunk0 = (int64_t)blockIdx.x * BIN_CHUNK;
    if (chunk0 >= vr.count) return;
    int32_t *cur = cursors + (int64_t)n * nt;
    if (SMEM) {
        for (int t = threadIdx.x; t < nt; t += BIN_THREADS) s_hist[t] = 0;
        __syncthreads();
    }
    unsigned int rect[SMEM ? BIN_ITEMS : 1];
#pragma unroll
    for (int j = 0; j < BIN_ITEMS; ++j) {
        if (SMEM) rect[j] = BIN_PACK_EMPTY;
        const int64_t i = chunk0 + j * BIN_THREADS + threadIdx.x;
        if (i < vr.count) {
            const int64_t p = vr.first + i;
            if (SMEM && rects) {
                // rectangle + slice packed by the count pass: no record load, no edge arithmetic
                const unsigned int pr = __ldg(&rects[p]);
                rect[j] = pr;
                if (pr != BIN_PACK_EMPTY) {
                    const int x0 = pr & 127, x1 = (pr >> 7) & 127, y0 = (pr >> 14) & 127, y1 = (pr >> 21) & 127, sl = pr >> 28;
                    for (int by = y0; by <= y1; ++by)
                        for (int bx = x0; bx <= x1; ++bx) atomicAdd(&s_hist[(by * B + bx) * NS + sl], 1);
                }
                continue;
            }
            const float4 A = __ldg(&rec[2 * p]);
            const float ry = __ldg(&rec[2 * p + 1]).x;
            const BinRect r = splat_bin_rect<POW2>(A, ry, bin, S, B);
            if (!r.empty) {
                const int sl = depth_slice(sm, A.z);
                if (SMEM) rect[j] = pack_rect(r, sl);
                for (int by = r.y0; by <= r.y1; ++by)
                    for (int bx = r.x0; bx <= r.x1; ++bx) {
                        const int key = (by * B + bx) * NS + sl;
                        if (SMEM) {
                            atomicAdd(&s_hist[key], 1);
                        } else {
                            const int slot = atomicAdd(&cur[key], 1);
                            if (slot < ids_capacity) ids[slot] = (int32_t)p;
                        }
                    }
            }
        }
    }
    if (!SMEM) return;
    __syncthreads();
    // reserve a contiguous range per non-empty tile; s_hist becomes the block's write cursor
    for (int t = threadIdx.x; t < nt; t += BIN_THREADS) {
        const int v = s_hist[t];
        if (v) s_hist[t] = atomicAdd(&cur[t], v);
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < BIN_ITEMS; ++j) {
        const unsigned int pr = rect[j];
        if (pr == BIN_PACK_EMPTY) continue;
        const int x0 = pr & 127, x1 = (pr >> 7) & 127, y0 = (pr >> 14) & 127, y1 = (pr >> 21) & 127, sl = pr >> 28;
        const int32_t p = (int32_t)(vr.first + chunk0 + j * BIN_THREADS + threadIdx.x);
        for (int by = y0; by <= y1; ++by)
            for (int bx = x0; bx <= x1; ++bx) {
                const int slot = atomicAdd(&s_hist[(by * B + bx) * NS + sl], 1);
                if (slot < ids_capacity) ids[slot] = p;
            }
    }
}

template <typename Kern>
static int prepare_smem(Kern kern, size_t bytes) {
    if (bytes > 48 * 1024)
        DSS_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    return DSS_OK;
}

// Number of depth slices of the forward tile lists.  On the 1M-point / 512^2 workload (bench.py) the rasterizer was
// as fast with 8 slices as with 16 (early termination is decided per chunk of the list anyway) and the
// binning histograms are half as large; more tiles -> fewer slices so that the per-block histogram (B*B*NS ints)
// stays within 32 KB of shared memory.
int choose_depth_slices(int B) {
    int ns = 8;
    while (ns > 1 && (int64_t)B * B * ns > 8 * 1024) ns >>= 1;
    return ns;
}

// count + scan.  counts / offsets have N*B*B*NS + 1 entries (the last count stays 0).
int bin_count_and_scan(dss_ctx *ctx, const float4 *rec, const int64_t *first_idx, const int64_t *num_points,
                       int N, int64_t P0, int S, int bin, int NS, const float *zrange, int32_t *counts,
                       int32_t *offsets, unsigned int *rects, cudaStream_t st) {
    const int B = 1 + (S - 1) / bin;
    const int64_t nb = (int64_t)N * B * B * NS;
    DSS_CUDA_TRY(cudaMemsetAsync(counts, 0, (size_t)(nb + 1) * sizeof(int32_t), st));
    if (P0 > 0) {
        dim3 grid((unsigned)((P0 + BIN_CHUNK - 1) / BIN_CHUNK), N);
        const bool pow2 = (S & (S - 1)) == 0;
        StageScope prof(ctx, ST_BIN_COUNT, st);
        if ((int64_t)B * B * NS <= BIN_MAX_SMEM_TILES && B <= BIN_PACK_MAX_B && NS <= 16 && !ctx->bin_direct) {
            const size_t smem = (size_t)B * B * NS * sizeof(int32_t);
            int rc = pow2 ? prepare_smem(bin_count_kernel<true, true>, smem) : prepare_smem(bin_count_kernel<true, false>, smem);
            if (rc) return rc;
            if (pow2)
                bin_count_kernel<true, true><<<grid, BIN_THREADS, smem, st>>>(rec, first_idx, num_points, P0, S, bin, B, NS, zrange, counts, rects);
            else
                bin_count_kernel<true, false><<<grid, BIN_THREADS, smem, st>>>(rec, first_idx, num_points, P0, S, bin, B, NS, zrange, counts, rects);
        } else if (pow2) {
            bin_count_kernel<false, true><<<grid, BIN_THREADS, 0, st>>>(rec, first_idx, num_points, P0, S, bin, B, NS, zrange, counts, nullptr);
        } else {
            bin_count_kernel<false, false><<<grid, BIN_THREADS, 0, st>>>(rec, first_idx, num_points, P0, S, bin, B, NS, zrange, counts, nullptr);
        }
        DSS_LAUNCH_CHECK(ctx);
    }
    return exclusive_scan_i32(ctx, counts, offsets, nb + 1, st);
}

int bin_scatter(dss_ctx *ctx, const float4 *rec, const int64_t *first_idx, const int64_t *num_points, int N,
                int64_t P0, int S, int bin, int NS, const float *zrange, const int32_t *offsets, int32_t *cursors,
                int32_t *ids, int64_t ids_capacity, const unsigned int *rects, cudaStream_t st) {
    const int B = 1 + (S - 1) / bin;
    const int64_t nb = (int64_t)N * B * B * NS;
    const int cap = (int)(ids_capacity > (int64_t)INT32_MAX ? (int64_t)INT32_MAX : ids_capacity);
    DSS_CUDA_TRY(cudaMemcpyAsync(cursors, offsets, (size_t)nb * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
    if (P0 > 0) {
        dim3 grid((unsigned)((P0 + BIN_CHUNK - 1) / BIN_CHUNK), N);
        const bool pow2 = (S & (S - 1)) == 0;
        StageScope prof(ctx, ST_BIN_SCATTER, st);
        if ((int64_t)B * B * NS <= BIN_MAX_SMEM_TILES && B <= BIN_PACK_MAX_B && NS <= 16 && !ctx->bin_direct) {
            const size_t smem = (size_t)B * B * NS * sizeof(int32_t);
            int rc = pow2 ? prepare_smem(bin_scatter_kernel<true, true>, smem) : prepare_smem(bin_scatter_kernel<true, false>, smem);
            if (rc) return rc;
            if (pow2)
                bin_scatter_kernel<true, true><<<grid, BIN_THREADS, smem, st>>>(rec, first_idx, num_points, P0, S, bin, B, NS, zrange, cursors, ids, cap, rects);
            else
                bin_scatter_kernel<true, false><<<grid, BIN_THREADS, smem, st>>>(rec, first_idx, num_points, P0, S, bin, B, NS, zrange, cursors, ids, cap, rects);
        } else if (pow2) {
            bin_scatter_kernel<false, true><<<grid, BIN_THREADS, 0, st>>>(rec, first_idx, num_points, P0, S, bin, B, NS, zrange, cursors, ids, cap, nullptr);
        } else {
            bin_scatter_kernel<false, false><<<grid, BIN_THREADS, 0, st>>>(rec, first_idx, num_points, P0, S, bin, B, NS, zrange, cursors, ids, cap, nullptr);
        }
        DSS_LAUNCH_CHECK(ctx);
    }
    return DSS_OK;
}

// ---------------------------------------------------------------------------------------------
// Scatter of lists that the fused preprocess counted (render.cu, preprocess_splats<..., BIN>): each preprocess block
// stored the packed rectangle of its splats and, per non-empty bin, the value its flush atomic returned -- the block's
// offset inside the bin.  This kernel runs on the same grid with the same grid-stride loop, so block b of view n sees
// exactly the splats block b counted: its cursors are the scanned bin offsets plus its own offsets, and the slots are
// claimed with shared-memory atomics only.  block_offsets: (N, gridDim.x, B*B*NS), entries of empty bins unset (never
// read back, the block has no splat in them).
// ---------------------------------------------------------------------------------------------
constexpr int SCATTER_BATCH = 8;   // rectangle words per thread whose loads are issued together

__global__ void __launch_bounds__(PREPROCESS_THREADS)
bin_scatter_counted_kernel(const int64_t *__restrict__ first_idx, const int64_t *__restrict__ num_points,
                           int64_t P0_shared, int B, int NS, const int32_t *__restrict__ offsets,
                           const int32_t *__restrict__ block_offsets, const unsigned int *__restrict__ rects,
                           int32_t *__restrict__ ids, int ids_capacity) {
    extern __shared__ int32_t s_cur[];
    const int n = blockIdx.y;
    const int nt = B * B * NS;
    const ViewRange vr = view_range(first_idx, num_points, n, P0_shared);
    const int32_t *off = offsets + (int64_t)n * nt;
    const int32_t *own = block_offsets + ((int64_t)n * gridDim.x + blockIdx.x) * nt;
    // (unsigned: the unset entries of empty bins may hold anything)
#pragma unroll 8
    for (int t = threadIdx.x; t < nt; t += PREPROCESS_THREADS) s_cur[t] = (int32_t)((unsigned int)off[t] + (unsigned int)own[t]);
    __syncthreads();
    const int64_t stride = (int64_t)gridDim.x * PREPROCESS_THREADS;
    for (int64_t i0 = (int64_t)blockIdx.x * PREPROCESS_THREADS + threadIdx.x; i0 < vr.count; i0 += SCATTER_BATCH * stride) {
        unsigned int pr[SCATTER_BATCH];
#pragma unroll
        for (int j = 0; j < SCATTER_BATCH; ++j) {
            const int64_t i = i0 + j * stride;
            pr[j] = i < vr.count ? __ldg(&rects[vr.first + i]) : BIN_PACK_EMPTY;
        }
#pragma unroll
        for (int j = 0; j < SCATTER_BATCH; ++j) {
            if (pr[j] == BIN_PACK_EMPTY) continue;
            const int x0 = pr[j] & 127, x1 = (pr[j] >> 7) & 127, y0 = (pr[j] >> 14) & 127, y1 = (pr[j] >> 21) & 127,
                      sl = pr[j] >> 28;
            const int32_t p = (int32_t)(vr.first + i0 + j * stride);
            for (int by = y0; by <= y1; ++by)
                for (int bx = x0; bx <= x1; ++bx) {
                    const int slot = atomicAdd(&s_cur[(by * B + bx) * NS + sl], 1);
                    if (slot < ids_capacity) ids[slot] = p;
                }
        }
    }
}

int bin_scatter_counted(dss_ctx *ctx, const int64_t *first_idx, const int64_t *num_points, int N, int64_t P0, int B,
                        int NS, const int32_t *offsets, const int32_t *block_offsets, unsigned int blocks,
                        const unsigned int *rects, int32_t *ids, int64_t ids_capacity, cudaStream_t st) {
    if (P0 == 0) return DSS_OK;
    const int cap = (int)(ids_capacity > (int64_t)INT32_MAX ? (int64_t)INT32_MAX : ids_capacity);
    const size_t smem = (size_t)B * B * NS * sizeof(int32_t);
    int rc = prepare_smem(bin_scatter_counted_kernel, smem);
    if (rc) return rc;
    StageScope prof(ctx, ST_BIN_SCATTER, st);
    bin_scatter_counted_kernel<<<dim3(blocks, N), PREPROCESS_THREADS, smem, st>>>(first_idx, num_points, P0, B, NS, offsets,
                                                                           block_offsets, rects, ids, cap);
    DSS_LAUNCH_CHECK(ctx);
    return DSS_OK;
}

// ---------------------------------------------------------------------------------------------
// 2-D uniform grid insert / counting sort (FRNN replacements; grid.cu:62-99, counting_sort.cu:5-36).
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
grid_insert_2d_kernel(const float *__restrict__ points, const int64_t *__restrict__ lengths,
                      const float *__restrict__ params, int32_t *grid_cnt, int32_t *__restrict__ grid_cell,
                      int32_t *__restrict__ grid_idx, int Pmax, int G) {
    const int n = blockIdx.y;
    const int64_t len = lengths[n];
    const float min_x = params[n * 6 + 0], min_y = params[n * 6 + 1], delta = params[n * 6 + 2];
    const int res_x = (int)params[n * 6 + 3], res_y = (int)params[n * 6 + 4];
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < len;
         p += (int64_t)gridDim.x * blockDim.x) {
        const float2 xy = reinterpret_cast<const float2 *>(points)[(int64_t)n * Pmax + p];
        int gx = (int)((xy.x - min_x) * delta);
        int gy = (int)((xy.y - min_y) * delta);
        gx = max(min(gx, res_x - 1), 0);
        gy = max(min(gy, res_y - 1), 0);
        const int gs = gx * res_y + gy;
        grid_cell[(int64_t)n * Pmax + p] = gs;
        grid_idx[(int64_t)n * Pmax + p] = atomicAdd(&grid_cnt[(int64_t)n * G + gs], 1);
    }
}

__global__ void __launch_bounds__(256)
grid_counting_sort_2d_kernel(const float *__restrict__ points, const int64_t *__restrict__ lengths,
                             const int32_t *__restrict__ grid_cell, const int32_t *__restrict__ grid_idx,
                             const int32_t *__restrict__ grid_off, float *__restrict__ sorted_points,
                             int32_t *__restrict__ sorted_idx, int Pmax, int G) {
    const int n = blockIdx.y;
    const int64_t len = lengths[n];
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < len;
         p += (int64_t)gridDim.x * blockDim.x) {
        const int cell = grid_cell[(int64_t)n * Pmax + p];
        const int64_t s = (int64_t)grid_off[(int64_t)n * G + cell] + grid_idx[(int64_t)n * Pmax + p];
        if (s < 0 || s >= len) continue;  // corrupt offsets: never write out of the view's rows
        reinterpret_cast<float2 *>(sorted_points)[(int64_t)n * Pmax + s] =
            reinterpret_cast<const float2 *>(points)[(int64_t)n * Pmax + p];
        sorted_idx[(int64_t)n * Pmax + s] = (int32_t)p;
    }
}

}  // namespace dss

extern "C" {

int dss_grid_insert_points_2d(dss_ctx *ctx, const float *points, const int64_t *lengths, const float *params,
                              int32_t *grid_cnt, int32_t *grid_cell, int32_t *grid_idx, int N, int Pmax,
                              int G, void *stream) {
    DSS_REQUIRE(ctx && points && lengths && params && grid_cnt && grid_cell && grid_idx, "null pointer");
    DSS_REQUIRE(N >= 0 && Pmax >= 0 && G >= 0, "negative size");
    if (N == 0 || Pmax == 0) return DSS_OK;
    dim3 grid(dss::grid_blocks(Pmax, 256, ctx->sm_count, 8), N);
    dss::grid_insert_2d_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(points, lengths, params, grid_cnt,
                                                                       grid_cell, grid_idx, Pmax, G);
    DSS_LAUNCH_CHECK(ctx);
    return DSS_OK;
}

int dss_grid_counting_sort_2d(dss_ctx *ctx, const float *points, const int64_t *lengths,
                              const int32_t *grid_cell, const int32_t *grid_idx, const int32_t *grid_off,
                              float *sorted_points, int32_t *sorted_idx, int N, int Pmax, int G, void *stream) {
    DSS_REQUIRE(ctx && points && lengths && grid_cell && grid_idx && grid_off && sorted_points && sorted_idx,
                "null pointer");
    DSS_REQUIRE(N >= 0 && Pmax >= 0 && G >= 0, "negative size");
    if (N == 0 || Pmax == 0) return DSS_OK;
    dim3 grid(dss::grid_blocks(Pmax, 256, ctx->sm_count, 8), N);
    dss::grid_counting_sort_2d_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(
        points, lengths, grid_cell, grid_idx, grid_off, sorted_points, sorted_idx, Pmax, G);
    DSS_LAUNCH_CHECK(ctx);
    return DSS_OK;
}

int dss_rasterize_coarse(dss_ctx *ctx, const float *points, const float *radii, const int64_t *first_idx,
                         const int64_t *num_points, int N, int64_t P, int image_size, int bin_size,
                         int32_t *bin_offsets, int32_t *bin_ids, int64_t bin_ids_capacity,
                         int64_t *total_required_host, void *stream) {
    using namespace dss;
    cudaStream_t st = (cudaStream_t)stream;
    DSS_REQUIRE(ctx && points && radii && first_idx && num_points && bin_offsets, "null pointer");
    DSS_REQUIRE(N > 0 && P >= 0 && image_size > 0 && bin_size > 0, "bad size");
    const int S = image_size, B = 1 + (S - 1) / bin_size;
    const int64_t nb = (int64_t)N * B * B;
    DSS_REQUIRE(nb + 1 < (int64_t)INT32_MAX, "too many bins");
    float4 *rec = nullptr;
    int32_t *counts = nullptr;
    int rc;
    if ((rc = ctx_get(ctx, BUF_RECORDS, (size_t)(2 * (P > 0 ? P : 1)), &rec))) return rc;
    if ((rc = ctx_get(ctx, BUF_TILE_COUNTS, (size_t)(nb + 1), &counts))) return rc;
    if ((rc = pack_records(ctx, points, radii, nullptr, P, rec, st))) return rc;
    if ((rc = bin_count_and_scan(ctx, rec, first_idx, num_points, N, P, S, bin_size, 1, nullptr, counts, bin_offsets, nullptr, st)))
        return rc;
    if ((rc = publish_words(ctx, bin_offsets + nb, ctx->h_pinned, 1, st))) return rc;
    DSS_CUDA_TRY(cudaStreamSynchronize(st));
    const int64_t total = (int64_t)(*reinterpret_cast<int32_t *>(ctx->h_pinned));
    if (total_required_host) *total_required_host = total;
    if (total > bin_ids_capacity || (total > 0 && bin_ids == nullptr)) {
        set_error("bin_ids capacity %lld < required %lld", (long long)bin_ids_capacity, (long long)total);
        return DSS_E_CAPACITY;
    }
    if (total == 0) return DSS_OK;
    return bin_scatter(ctx, rec, first_idx, num_points, N, P, S, bin_size, 1, nullptr, bin_offsets, counts, bin_ids,
                       bin_ids_capacity, nullptr, st);
}

}  // extern "C"
