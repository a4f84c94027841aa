// rimls.cu -- move point clouds onto the RIMLS surface of their samples, and smooth their normals first
// (project_to_latent_surface, denoise_normals, DSS/core/cloud.py:442-553).  The rules are in include/dss_b200.h and
// DESIGN.md.
//
// Both kernels run one warp per row: lane j holds neighbour j of the row (k <= 31, so lane 31 and the lanes past k hold
// nothing), in float64.  A neighbour is the row's dss_knn_points entry at K = k + 1 less its own index (knn_own_entry),
// kept when its squared distance is at most r_n^2; a dropped or -1 entry contributes zero to every sum.  Every sum over
// the neighbours is the xor butterfly 16, 8, 4, 2, 1 of __shfl_xor_sync, so every lane holds the same bits, every
// decision is uniform over the warp, and every call gives the same bits (tests/project_oracle.py restates the tree).
// The samples q_j, n_j are the input's and never change, so the rows are independent: one launch, no scratch, no
// atomics, no host synchronisation.
#include <math_constants.h>

#include "common.cuh"
#include "kernels.cuh"

namespace dss {

constexpr int RIMLS_THREADS = 128;               // four rows per block
constexpr int RIMLS_ROWS = RIMLS_THREADS / 32;
constexpr int RIMLS_MAX_K = 31;                  // the K-NN runs at k + 1 <= 32
constexpr double RIMLS_ALPHA_TOL = 1e-4;         // the inner loop stops when no weight changed by this much
constexpr double RIMLS_MOVE_TOL = 5e-4;          // a row stays active while it moved farther than this
constexpr double NORMALIZE_EPS = 1e-12;          // F.normalize

struct RimlsArgs {
    const float *points;        // (P,3)
    const float *normals;       // (P,3)
    const int64_t *first;       // (N,)
    const int64_t *num;         // (N,)
    const int32_t *knn_idx;     // (P, k + 1), local to the cloud
    int k;
    const double *radius;       // (N,) r_n
    double sigma;               // denoise: sharpness_sigma
    int max_proj_iters, max_est_iters;
    float *out;                 // (P,3): denoised normals or projected points
    int32_t *iterations;        // (P,) projection only
};

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ double warp_min(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmin(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ D3 warp_sum3(D3 v) { return d3(warp_sum(v.x), warp_sum(v.y), warp_sum(v.z)); }

__device__ __forceinline__ D3 load_d3(const float *p, int64_t row) {
    return d3((double)p[row * 3], (double)p[row * 3 + 1], (double)p[row * 3 + 2]);
}

// F.normalize in float64: v / max(|v|, 1e-12), so a zero vector stays zero
__device__ __forceinline__ D3 normalize_d3(D3 v) {
    const double l = fmax(sqrt(ddot(v, v)), NORMALIZE_EPS);
    return d3(v.x / l, v.y / l, v.z / l);
}

__device__ __forceinline__ void store_f3(float *p, int64_t row, D3 v) {
    p[row * 3] = (float)v.x, p[row * 3 + 1] = (float)v.y, p[row * 3 + 2] = (float)v.z;
}

// This lane's neighbour of local row i at p (cloud rows from f, radius^2 r2): its position, unit normal and squared
// distance; ok is false for the lanes past k, a -1 entry and an entry beyond the radius.
struct Neighbour {
    D3 q, n;
    double d2;
    bool ok;
};
__device__ __forceinline__ Neighbour rimls_neighbour(const RimlsArgs &a, int64_t f, int64_t i, D3 p, double r2) {
    Neighbour b;
    b.q = b.n = d3(0.0, 0.0, 0.0);
    b.d2 = 0.0;
    b.ok = false;
    const int lane = threadIdx.x & 31;
    if (lane < a.k) {
        const int32_t *nb = a.knn_idx + (f + i) * (a.k + 1);
        const int32_t j = nb[knn_other(lane, knn_own_entry(nb, a.k, (int32_t)i))];
        if (j >= 0) {
            b.q = load_d3(a.points, f + j);
            b.d2 = ddot(dsub(p, b.q), dsub(p, b.q));
            b.ok = b.d2 <= r2;
            if (b.ok) b.n = normalize_d3(load_d3(a.normals, f + j));
        }
    }
    if (!b.ok) b.q = b.n = d3(0.0, 0.0, 0.0), b.d2 = 0.0;
    return b;
}

// the rows of cloud blockIdx.y, one per warp
#define RIMLS_ROWS_OF_CLOUD(a, i_)                                                                               \
    const int n_ = blockIdx.y;                                                                                   \
    const int64_t f_ = (a).first[n_], c_ = (a).num[n_];                                                          \
    const double r2_ = (a).radius[n_] * (a).radius[n_];                                                          \
    for (int64_t i_ = (int64_t)blockIdx.x * RIMLS_ROWS + (threadIdx.x >> 5); i_ < c_;                            \
         i_ += (int64_t)gridDim.x * RIMLS_ROWS)

// denoise_normals: normalize(sum w_j n_j / eps_denom(sum w_j)), w_j = exp(-((1 - n_i.n_j) / sigma)^2)
// exp(-d2_j c / 2), zero where d2_j > 16 / (c / 2); a row whose weights are all zero keeps normalize(n_i)
__global__ void __launch_bounds__(RIMLS_THREADS, 4) denoise_normals_kernel(const __grid_constant__ RimlsArgs a) {
    RIMLS_ROWS_OF_CLOUD(a, i) {
        const int64_t row = f_ + i;
        const D3 p = load_d3(a.points, row), ni = normalize_d3(load_d3(a.normals, row));
        const Neighbour b = rimls_neighbour(a, f_, i, p, r2_);
        const double inv = (double)c_ / 2.0, cut = 16.0 / inv;
        double w = 0.0;
        if (b.ok && !(b.d2 > cut)) {
            const double t = (1.0 - ddot(ni, b.n)) / a.sigma;
            w = exp(-b.d2 * inv) * exp(-(t * t));
        }
        const double sw = warp_sum(w);
        const D3 sn = warp_sum3(d3(b.n.x * w, b.n.y * w, b.n.z * w));
        D3 out = ni;
        if (sw != 0.0) {
            const double e = eps_denom_f64(sw);
            out = normalize_d3(d3(sn.x / e, sn.y / e, sn.z / e));
        }
        if ((threadIdx.x & 31) == 0) store_f3(a.out, row, out);
    }
}

// project_to_latent_surface with the samples fixed at the input (DESIGN.md §3)
__global__ void __launch_bounds__(RIMLS_THREADS) project_surface_kernel(const __grid_constant__ RimlsArgs a) {
    RIMLS_ROWS_OF_CLOUD(a, i) {
        const int64_t row = f_ + i;
        const D3 p = load_d3(a.points, row);
        const Neighbour b = rimls_neighbour(a, f_, i, p, r2_);
        // the nearest neighbour at a positive distance fixes the spatial scale; without one the row stays
        const double d2min = warp_min(b.ok && b.d2 > 0.0 ? b.d2 : CUDART_INF);
        D3 x = p;
        int moved = 0;
        if (d2min < CUDART_INF) {
            const double inv = 1.0 / (16.0 * d2min);
            for (int t = 0; t < a.max_proj_iters; ++t) {
                const D3 dx = dsub(x, b.q);
                const double fx = b.ok ? ddot(dx, b.n) : 0.0;
                double alpha = 1.0, f = 0.0;
                D3 g = d3(0.0, 0.0, 0.0);
                for (int s = 0; s < a.max_est_iters; ++s) {
                    if (s > 0) {
                        const D3 dn = dsub(b.n, g);
                        const double u = sqrt(ddot(dn, dn)) / 0.5, v = fx - f;
                        const double next = exp(-(u * u)) * exp(-(v * v * inv / 4.0));
                        if (warp_max(b.ok ? fabs(next - alpha) : 0.0) < RIMLS_ALPHA_TOL) break;
                        alpha = next;
                    }
                    double w = 0.0, gs = 0.0;
                    if (b.ok) {
                        const double phi = exp(-ddot(dx, dx) * inv);
                        w = phi * alpha;
                        gs = (inv * phi) * w;
                    }
                    const D3 gw = d3(2.0 * dx.x * gs, 2.0 * dx.y * gs, 2.0 * dx.z * gs);
                    const double sw = warp_sum(w), sf = warp_sum(fx * w);
                    const D3 sgw = warp_sum3(gw), sgf = warp_sum3(d3(gw.x * fx, gw.y * fx, gw.z * fx));
                    const D3 sn = warp_sum3(d3(w * b.n.x, w * b.n.y, w * b.n.z));
                    const double e = eps_denom_f64(sw);
                    f = sf / e;
                    g = d3(__dadd_rn(__dsub_rn(sgf.x, __dmul_rn(f, sgw.x)), sn.x) / e,
                           __dadd_rn(__dsub_rn(sgf.y, __dmul_rn(f, sgw.y)), sn.y) / e,
                           __dadd_rn(__dsub_rn(sgf.z, __dmul_rn(f, sgw.z)), sn.z) / e);
                }
                const D3 mv = d3(f * g.x, f * g.y, f * g.z);
                x = dsub(x, mv);
                moved += (mv.x != 0.0 || mv.y != 0.0 || mv.z != 0.0);
                if (!(sqrt(ddot(mv, mv)) > RIMLS_MOVE_TOL)) break;
            }
        }
        if ((threadIdx.x & 31) == 0) {
            store_f3(a.out, row, x);
            a.iterations[row] = moved;
        }
    }
}

int rimls_launch(dss_ctx *ctx, const RimlsArgs &a, int N, int64_t P, bool project, void *stream) {
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    DSS_REQUIRE(P >= 0 && P < (int64_t)INT32_MAX, "P out of range");
    DSS_REQUIRE(N >= 1 && N <= 65535, "N out of range");
    DSS_REQUIRE(a.k >= 3 && a.k <= RIMLS_MAX_K, "k must lie in [3, 31]");
    if (P == 0) return DSS_OK;
    DSS_REQUIRE(a.points && a.normals && a.first && a.num && a.knn_idx && a.radius && a.out, "null pointer");
    const dim3 grid(grid_blocks(P, RIMLS_ROWS, ctx->sm_count, 16), N);
    cudaStream_t st = (cudaStream_t)stream;
    if (project)
        project_surface_kernel<<<grid, RIMLS_THREADS, 0, st>>>(a);
    else
        denoise_normals_kernel<<<grid, RIMLS_THREADS, 0, st>>>(a);
    DSS_LAUNCH_CHECK(ctx);
    return DSS_OK;
}

}  // namespace dss

extern "C" {

int dss_denoise_normals(dss_ctx *ctx, const float *points, const float *normals, const int64_t *first_idx,
                        const int64_t *num_points, int N, int64_t P, const int32_t *knn_idx, int k,
                        const double *radius, double sharpness_sigma, float *out_normals, void *stream) {
    using namespace dss;
    RimlsArgs a = {};
    a.points = points, a.normals = normals, a.first = first_idx, a.num = num_points, a.knn_idx = knn_idx, a.k = k;
    a.radius = radius, a.sigma = sharpness_sigma, a.out = out_normals;
    return rimls_launch(ctx, a, N, P, false, stream);
}

int dss_project_to_surface(dss_ctx *ctx, const float *points, const float *normals, const int64_t *first_idx,
                           const int64_t *num_points, int N, int64_t P, const int32_t *knn_idx, int k,
                           const double *radius, int max_proj_iters, int max_est_iters, float *out_points,
                           int32_t *iterations, void *stream) {
    using namespace dss;
    DSS_REQUIRE(max_proj_iters >= 0 && max_est_iters >= 0, "negative iteration count");
    DSS_REQUIRE(iterations != nullptr, "null pointer");
    RimlsArgs a = {};
    a.points = points, a.normals = normals, a.first = first_idx, a.num = num_points, a.knn_idx = knn_idx, a.k = k;
    a.radius = radius, a.max_proj_iters = max_proj_iters, a.max_est_iters = max_est_iters, a.out = out_points;
    a.iterations = iterations;
    return rimls_launch(ctx, a, N, P, true, stream);
}

}  // extern "C"
