// knn.cu -- K nearest neighbours within a radius on a 3-D uniform grid (SURVEY.md section 8(f), row 1).
//
// Replaces frnn.frnn_grid_points(points1, points2, lengths1, lengths2, K, r) (external/FRNN/frnn/frnn.py:15-175;
// kernels external/FRNN/frnn/csrc/grid/grid.cu:62-99 insert, counting_sort.cu:5-36, grid.cu:285-373 search), which DSS
// calls with K = 7, r = 0.2 on the world-space cloud in every forward to size the splats (DSS/core/rasterizer.py:
// 313-326, 369-388).  Semantics = the reference's own ground truth FRNNBruteForceCPU (external/FRNN/frnn/csrc/
// bruteforce/bruteforce_cpu.cpp:8-64): per query the K points of the same cloud with the smallest (d2, index), d2 < r^2,
// ascending; missing neighbours are reported as dist -1 / idx -1.
//
// FRNN fixes the cell size at r / 2 and scans the 5^3 cells around the query -- with r = 0.2 on a unit-sized cloud that
// is a large share of ALL points per query (72 ms per 1M random points in the reference's own table,
// tests/output/frnn_individual.csv:26).  Here the cell size follows the point density (a few points per occupied cell),
// and every query grows its search cube ring by ring until the K-th best distance is proven final
// (d_K < ring * cell) or the radius is exhausted -- the same result, ~100 candidates per query instead of ~10^4.
// Everything (bounding box, grid parameters, counting sort) is computed on the device; no host round trip.
#include <math_constants.h>

#include <cfloat>

#include "common.cuh"
#include "kernels.cuh"

namespace dss {

constexpr int KNN_GMAX = 1 << 21;        // grid cells per cloud at most (counts + offsets: 2 x 8 MB per cloud)
constexpr int KNN_MAX_K = 32;

struct KnnGrid {          // per cloud, lives on the device
    float gmin[3];
    float cell, inv_cell;
    int res[3];
};

__global__ void knn_bbox_init_kernel(int *bbox, int N) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < N * 6) bbox[i] = (i % 6 < 3) ? INT32_MAX : INT32_MIN;
}

__global__ void __launch_bounds__(256)
knn_bbox_kernel(const float *__restrict__ pts, const int64_t *__restrict__ first, const int64_t *__restrict__ num,
                int *__restrict__ bbox) {
    const int n = blockIdx.y;
    const int64_t f = first[n], c = num[n];
    int lo[3] = {INT32_MAX, INT32_MAX, INT32_MAX}, hi[3] = {INT32_MIN, INT32_MIN, INT32_MIN};
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < c; i += (int64_t)gridDim.x * blockDim.x) {
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const float v = pts[(f + i) * 3 + k];
            if (isfinite(v)) {                      // NaN and +-inf coordinates do not shape the grid
                lo[k] = min(lo[k], f2ord(v));
                hi[k] = max(hi[k], f2ord(v));
            }
        }
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        lo[k] = __reduce_min_sync(0xffffffffu, lo[k]);
        hi[k] = __reduce_max_sync(0xffffffffu, hi[k]);
    }
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            atomicMin(&bbox[n * 6 + k], lo[k]);
            atomicMax(&bbox[n * 6 + 3 + k], hi[k]);
        }
    }
}

// Cell size from the density: clouds on this path are surfaces, so aim at ~3 points per occupied cell of a surface
// with the bounding box's face area; never more than KNN_GMAX cells; never finer than 1/1024 of the largest extent.
//
// The grid holds for every input, 1 <= res[k] and res[0] res[1] res[2] <= KNN_GMAX, so no cell index leaves the cloud's
// counters.  The bounding box holds finite coordinates only, so each extent is finite once an overflowing difference
// (+-3e38 in one cloud) is clamped to FLT_MAX; `cell` is finite and positive (an overflowing density cell is clamped to
// FLT_MAX, a zero one replaced by 1).  Then e/cell is in [0, inf] and r = floor(e/cell) + 1 in [1, inf]; the growth test
// compares integers below 2^24 exactly (a product of such r that rounds is larger than 2^21 before and after rounding),
// so a loop exit means the grid fits.  If 64 steps of x1.26 do not suffice (far outliers, a radius far below the
// extent), cell >= emax / 126 gives e/cell <= 126 (1 + 3u) < 127 on every axis: res <= 127 and 127^3 < 2^21.
__global__ void knn_params_kernel(const int *__restrict__ bbox, const int64_t *__restrict__ num, float radius, int N,
                                  KnnGrid *__restrict__ grids) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    KnnGrid g;
    float e[3];
    for (int k = 0; k < 3; ++k) {
        const float lo = ord2f(bbox[n * 6 + k]), hi = ord2f(bbox[n * 6 + 3 + k]);
        g.gmin[k] = (num[n] > 0 && hi >= lo) ? lo : 0.0f;
        e[k] = (num[n] > 0 && hi >= lo) ? fminf(fmaxf(hi - lo, 0.0f), FLT_MAX) : 0.0f;
    }
    const float emax = fmaxf(e[0], fmaxf(e[1], e[2]));
    const float P = (float)(num[n] > 0 ? num[n] : 1);
    const float area = 2.0f * (e[0] * e[1] + e[1] * e[2] + e[0] * e[2]);
    float cell = sqrtf(3.0f * area / P);
    cell = fmaxf(cell, emax * (1.0f / 1024.0f));
    if (radius > 0.0f) cell = fminf(cell, radius);
    cell = fminf(cell, FLT_MAX);
    if (!(cell > 0.0f)) cell = 1.0f;                               // degenerate cloud (single point / all equal)
    bool fits = false;
    for (int it = 0; it < 64 && !fits; ++it) {                     // grow until the grid fits
        const float r0 = floorf(e[0] / cell) + 1.0f, r1 = floorf(e[1] / cell) + 1.0f, r2 = floorf(e[2] / cell) + 1.0f;
        fits = r0 * r1 * r2 <= (float)KNN_GMAX;
        if (!fits) cell *= 1.26f;
    }
    if (!fits) cell = fmaxf(cell, emax * (1.0f / 126.0f));
    g.cell = cell;
    g.inv_cell = 1.0f / cell;
    for (int k = 0; k < 3; ++k) g.res[k] = (int)(floorf(e[k] / cell) + 1.0f);
    grids[n] = g;
}

__device__ __forceinline__ int knn_axis_cell(float v, float gmin, float inv_cell, int res) {
    const float t = (v - gmin) * inv_cell;
    int c = (t >= 0.0f) ? ((t < (float)res) ? (int)t : res - 1) : 0;     // NaN -> 0
    return c;
}

template <int PASS>   // 0: count, 1: scatter (claims slots by counting the same counters back down to zero)
__global__ void __launch_bounds__(256)
knn_bin_kernel(const float *__restrict__ pts, const int64_t *__restrict__ first, const int64_t *__restrict__ num,
               const KnnGrid *__restrict__ grids, int32_t *__restrict__ counts, const int32_t *__restrict__ offsets,
               float4 *__restrict__ sorted) {
    const int n = blockIdx.y;
    const int64_t f = first[n], c = num[n];
    const KnnGrid g = grids[n];
    int32_t *cnt = counts + (int64_t)n * KNN_GMAX;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < c; i += (int64_t)gridDim.x * blockDim.x) {
        const float x = pts[(f + i) * 3], y = pts[(f + i) * 3 + 1], z = pts[(f + i) * 3 + 2];
        const int cell = (knn_axis_cell(x, g.gmin[0], g.inv_cell, g.res[0]) * g.res[1] +
                          knn_axis_cell(y, g.gmin[1], g.inv_cell, g.res[1])) * g.res[2] +
                         knn_axis_cell(z, g.gmin[2], g.inv_cell, g.res[2]);
        if (PASS == 0) {
            atomicAdd(&cnt[cell], 1);
        } else {
            const int slot = offsets[(int64_t)n * KNN_GMAX + cell] + atomicSub(&cnt[cell], 1) - 1;
            sorted[slot] = make_float4(x, y, z, __int_as_float((int)i));
        }
    }
}

// sorted insert of (d2, id) into the K best, ascending by (d2, id)
template <int KMAX>
__device__ __forceinline__ void knn_insert(float (&bd)[KMAX], int (&bi)[KMAX], int K, float d, int id) {
    if (!(d < bd[K - 1] || (d == bd[K - 1] && id < bi[K - 1]))) return;
#pragma unroll
    for (int k = KMAX - 1; k >= 0; --k) {
        if (k < K) {
            const bool here = d < bd[k] || (d == bd[k] && id < bi[k]);
            const bool prev = (k > 0) && (d < bd[k > 0 ? k - 1 : 0] || (d == bd[k > 0 ? k - 1 : 0] && id < bi[k > 0 ? k - 1 : 0]));
            if (here) {
                bd[k] = prev ? bd[k > 0 ? k - 1 : 0] : d;
                bi[k] = prev ? bi[k > 0 ? k - 1 : 0] : id;
            }
        }
    }
}

// One thread per query.  self_mode: the queries are the data points themselves, visited in grid order so that
// neighbouring threads read the same cells.
//
// The ring bound.  After ring R every cell within R of the query's cell (cx, cy, cz) has been visited, so an unseen
// point lies R + 1 or more cells away along some axis.  The computed coordinate t = fl(fl(v - gmin) * inv_cell) differs
// from (v - gmin) * inv_cell by at most err = 2.0001 u t (two roundings, u = 2^-24); clamping into a border cell only
// moves t outward, and only t < res + 1 decides a cell, so err <= 2.0001 u (maxres + 1).  The unseen point is
// therefore at least (R - 2 err) / inv_cell away along that axis, and 1 / inv_cell >= cell (1 - u).  Its computed
// squared distance (one difference, one square, two sums of non-negative terms) is at least (1 - 5u) times the exact
// one, and reach2 = fl(fl(fl(R - slack) * cell)^2) at most (1 + 5u) (R - slack)^2 cell^2.  Hence bd[K-1] < reach2
// proves that no unseen point can enter the list once R - slack <= (R - 2 err)(1 - 6.1u), i.e. for
// slack >= 2 err + 6.1 u R; with R <= maxres, slack = 16 u (maxres + 2) covers it.  That is ~1e-3 cells at the
// density floor's res <= 1025, and ~2 cells at the res = 2^21 the radius clamp allows along one axis, where t itself
// is only known to ~0.25 cells.
template <int KMAX>
__global__ void __launch_bounds__(128)
knn_search_kernel(const float *__restrict__ queries, const int64_t *__restrict__ qfirst, const int64_t *__restrict__ qnum,
                  const KnnGrid *__restrict__ grids, const int32_t *__restrict__ offsets,
                  const float4 *__restrict__ sorted, int self_mode, int K, float radius, float *__restrict__ out_d,
                  int32_t *__restrict__ out_i) {
    const int n = blockIdx.y;
    const int64_t qf = qfirst[n], qc = qnum[n];
    const KnnGrid g = grids[n];
    const int32_t *off = offsets + (int64_t)n * KNN_GMAX;
    // the scan runs over all clouds, so cloud n's first slot in `sorted` is the sum of the earlier clouds' sizes, whatever
    // gaps the caller's first_idx leaves between them
    const int64_t dbase = off[0];
    const float r2 = radius > 0.0f ? radius * radius : CUDART_INF_F;
    const int maxres = max(g.res[0], max(g.res[1], g.res[2]));
    const float slack = (float)(maxres + 2) * 0x1p-20f;             // 16 u (maxres + 2), see above
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < qc; t += (int64_t)gridDim.x * blockDim.x) {
        float qx, qy, qz;
        int64_t row;
        if (self_mode) {
            const float4 s = sorted[dbase + t];
            qx = s.x, qy = s.y, qz = s.z;
            row = qf + __float_as_int(s.w);
        } else {
            qx = queries[(qf + t) * 3], qy = queries[(qf + t) * 3 + 1], qz = queries[(qf + t) * 3 + 2];
            row = qf + t;
        }
        float bd[KMAX];
        int bi[KMAX];
#pragma unroll
        for (int k = 0; k < KMAX; ++k) {
            bd[k] = CUDART_INF_F;
            bi[k] = INT32_MAX;
        }
        const int cx = knn_axis_cell(qx, g.gmin[0], g.inv_cell, g.res[0]);
        const int cy = knn_axis_cell(qy, g.gmin[1], g.inv_cell, g.res[1]);
        const int cz = knn_axis_cell(qz, g.gmin[2], g.inv_cell, g.res[2]);
        // a non-finite query is at distance inf or NaN from every point, so it has no neighbour: skip the search
        // (which no bound would cut short)
        const bool finite = isfinite(qx) && isfinite(qy) && isfinite(qz);
        // distance from the query to the faces of its own cell along the grid: queries outside the box (general mode)
        // are clamped into a border cell, the ring bound below then starts from their distance to that cell's far side
        for (int ring = 0; finite && ring <= maxres; ++ring) {
            const int x0 = max(cx - ring, 0), x1 = min(cx + ring, g.res[0] - 1);
            const int y0 = max(cy - ring, 0), y1 = min(cy + ring, g.res[1] - 1);
            for (int x = x0; x <= x1; ++x)
                for (int y = y0; y <= y1; ++y) {
                    const bool shell_xy = (abs(x - cx) == ring) || (abs(y - cy) == ring);
                    // cells along z are contiguous in memory: one run for a full column, two single cells otherwise
                    int zruns[2][2];
                    int nruns = 0;
                    if (shell_xy) {
                        zruns[0][0] = max(cz - ring, 0);
                        zruns[0][1] = min(cz + ring, g.res[2] - 1);
                        nruns = 1;
                    } else {
                        if (cz - ring >= 0) zruns[nruns][0] = zruns[nruns][1] = cz - ring, ++nruns;
                        if (cz + ring < g.res[2] && ring > 0) zruns[nruns][0] = zruns[nruns][1] = cz + ring, ++nruns;
                    }
                    for (int rr = 0; rr < nruns; ++rr) {
                        const int c0 = (x * g.res[1] + y) * g.res[2] + zruns[rr][0];
                        const int c1 = (x * g.res[1] + y) * g.res[2] + zruns[rr][1];
                        const int b = off[c0], e = off[c1 + 1];
                        for (int j = b; j < e; ++j) {
                            const float4 s = __ldg(&sorted[j]);
                            // bruteforce_cpu.cpp:41-45: dist = sum over d of diff*diff, in this order
                            const float dx = qx - s.x, dy = qy - s.y, dz = qz - s.z;
                            const float d = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
                            if (d < r2) knn_insert<KMAX>(bd, bi, K, d, __float_as_int(s.w));
                        }
                    }
                }
            // every point not yet seen lies outside the cube of (2 ring + 1)^3 cells around the query's cell, i.e. at
            // least ring cells away (minus rounding slack): stop when that cannot beat the K-th best or the radius
            const float reach = fmaxf((float)ring - slack, 0.0f) * g.cell;
            const float reach2 = reach * reach;
            if (reach2 >= r2 || bd[K - 1] < reach2) break;
            if (x0 == 0 && y0 == 0 && x1 == g.res[0] - 1 && y1 == g.res[1] - 1 && cz - ring <= 0 && cz + ring >= g.res[2] - 1)
                break;                                                   // the whole grid has been visited
        }
#pragma unroll
        for (int k = 0; k < KMAX; ++k)
            if (k < K) {
                const bool ok = bi[k] != INT32_MAX;
                out_d[row * K + k] = ok ? bd[k] : -1.0f;
                if (out_i) out_i[row * K + k] = ok ? bi[k] : -1;
            }
    }
}

}  // namespace dss

extern "C" {

int dss_knn_points(dss_ctx *ctx, const float *queries, const int64_t *query_first_idx, const int64_t *query_num,
                   const float *points, const int64_t *first_idx, const int64_t *num_points, int N, int64_t Pq,
                   int64_t P, int K, float radius, float *sq_dists, int32_t *idxs, void *stream) {
    using namespace dss;
    cudaStream_t st = (cudaStream_t)stream;
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    DSS_REQUIRE(N >= 0 && P >= 0 && Pq >= 0, "negative size");
    DSS_REQUIRE(K >= 1 && K <= KNN_MAX_K, "K must be in [1, 32]");
    DSS_REQUIRE(P < (int64_t)INT32_MAX && Pq < (int64_t)INT32_MAX, "more than 2^31-1 points");
    if (N == 0 || Pq == 0) return DSS_OK;
    DSS_REQUIRE(points && first_idx && num_points && sq_dists, "null pointer");
    const bool self_mode = (queries == nullptr || queries == points) && (query_first_idx == nullptr || query_first_idx == first_idx);
    if (self_mode) {
        queries = points;
        query_first_idx = first_idx;
        query_num = num_points;
    }
    DSS_REQUIRE(query_first_idx && query_num, "query offsets missing");
    DSS_REQUIRE((int64_t)N * KNN_GMAX + 1 < (int64_t)INT32_MAX, "too many clouds for one call (N * 2^21 cells)");
    int *bbox = nullptr;
    KnnGrid *grids = nullptr;
    int32_t *counts = nullptr, *offsets = nullptr;
    float4 *sorted = nullptr;
    int rc;
    const int64_t ncell = (int64_t)N * KNN_GMAX + 1;
    if ((rc = ctx_get(ctx, BUF_MISC, (size_t)(N * 6 + N * (sizeof(KnnGrid) / 4 + 1) + 64), &bbox))) return rc;
    grids = reinterpret_cast<KnnGrid *>(bbox + ((N * 6 + 15) & ~15));
    if ((rc = ctx_get(ctx, BUF_KNN_COUNTS, (size_t)ncell, &counts))) return rc;
    if ((rc = ctx_get(ctx, BUF_KNN_OFFSETS, (size_t)ncell, &offsets))) return rc;
    if ((rc = ctx_get(ctx, BUF_KNN_SORTED, (size_t)(P > 0 ? P : 1), &sorted))) return rc;
    StageScope prof(ctx, ST_KNN, st);
    knn_bbox_init_kernel<<<(N * 6 + 127) / 128, 128, 0, st>>>(bbox, N);
    DSS_LAUNCH_CHECK(ctx);
    const unsigned nb = (unsigned)((P + 256 * 8 - 1) / (256 * 8) > 0 ? (P + 256 * 8 - 1) / (256 * 8) : 1);
    {
        dim3 grid(nb < 1184u ? nb : 1184u, N);
        knn_bbox_kernel<<<grid, 256, 0, st>>>(points, first_idx, num_points, bbox);
        DSS_LAUNCH_CHECK(ctx);
    }
    knn_params_kernel<<<(N + 63) / 64, 64, 0, st>>>(bbox, num_points, radius, N, grids);
    DSS_LAUNCH_CHECK(ctx);
    DSS_CUDA_TRY(cudaMemsetAsync(counts, 0, (size_t)ncell * sizeof(int32_t), st));
    {
        dim3 grid(nb < 4736u ? nb : 4736u, N);
        knn_bin_kernel<0><<<grid, 256, 0, st>>>(points, first_idx, num_points, grids, counts, nullptr, nullptr);
        DSS_LAUNCH_CHECK(ctx);
        if ((rc = exclusive_scan_i32(ctx, counts, offsets, ncell, st))) return rc;
        knn_bin_kernel<1><<<grid, 256, 0, st>>>(points, first_idx, num_points, grids, counts, offsets, sorted);
        DSS_LAUNCH_CHECK(ctx);
    }
    {
        const unsigned qb = (unsigned)((Pq + 127) / 128 > 0 ? (Pq + 127) / 128 : 1);
        dim3 grid(qb < 65535u ? qb : 65535u, N);
        // offsets index `sorted` globally (the scan runs over all clouds), so cloud n's first slot is offsets[n*GMAX]
        if (K <= 8)
            knn_search_kernel<8><<<grid, 128, 0, st>>>(queries, query_first_idx, query_num, grids, offsets, sorted,
                                                       self_mode ? 1 : 0, K, radius, sq_dists, idxs);
        else if (K <= 16)
            knn_search_kernel<16><<<grid, 128, 0, st>>>(queries, query_first_idx, query_num, grids, offsets, sorted,
                                                        self_mode ? 1 : 0, K, radius, sq_dists, idxs);
        else
            knn_search_kernel<32><<<grid, 128, 0, st>>>(queries, query_first_idx, query_num, grids, offsets, sorted,
                                                        self_mode ? 1 : 0, K, radius, sq_dists, idxs);
        DSS_LAUNCH_CHECK(ctx);
    }
    return DSS_OK;
}

}  // extern "C"
