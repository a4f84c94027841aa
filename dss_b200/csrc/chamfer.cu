// chamfer.cu -- chamfer point and normal distances of two batches of clouds, forward only.
//
// The sums behind pytorch3d's chamfer_distance(x, y, x_lengths, y_lengths, x_normals, y_normals) [ext, pytorch3d 0.4.0],
// which the reference's trainer uses as its model-selection metric under no_grad (DSS/training/trainer.py:144-171).
// Nearest neighbours come from dss_knn_points with K = 1 (the (squared distance, index) order), one search per
// direction.  Then one thread per query row of both directions forms its two terms and every block writes its fp64
// sums to a partials array, which grad_finish_kernel adds in a fixed order: the result is the same bits on every run.
#include <math_constants.h>

#include "common.cuh"

namespace dss {

constexpr int CH_THREADS = 256;

struct ChamferDir {
    const float *normals, *other_normals;
    const int64_t *first, *num, *other_first;
    const float *nn_d;        // (rows,) float32 squared distance to the nearest row of the other cloud, -1: none
    const int32_t *nn_i;      // (rows,) its index local to the other cloud, -1: none
    int64_t other_rows;       // 0: the other batch has no rows at all, so no search ran and nothing has a neighbour
};

// torch's cosine_similarity(a, b, eps): each vector over max(|a|, eps), then the dot product
__device__ __forceinline__ double cosine_eps(const float *a, const float *b) {
    const double a0 = a[0], a1 = a[1], a2 = a[2], b0 = b[0], b1 = b[1], b2 = b[2];
    const double na = fmax(sqrt(a0 * a0 + a1 * a1 + a2 * a2), 1e-6), nb = fmax(sqrt(b0 * b0 + b1 * b1 + b2 * b2), 1e-6);
    return (a0 / na) * (b0 / nb) + (a1 / na) * (b1 / nb) + (a2 / na) * (b2 / nb);
}

// grid (blocks, N, 2): blockIdx.z is the direction (0: x -> y, 1: y -> x); partials (N, 2, blocks, 2) {sum d, sum c}
__global__ void __launch_bounds__(CH_THREADS) chamfer_terms_kernel(ChamferDir dx, ChamferDir dy, double *partials) {
    __shared__ double sPart[CH_THREADS / 32][2];
    // field by field: selecting a whole parameter struct would copy it to the stack
    const bool z = blockIdx.z != 0;
    ChamferDir d;
    d.normals = z ? dy.normals : dx.normals, d.other_normals = z ? dy.other_normals : dx.other_normals;
    d.first = z ? dy.first : dx.first, d.num = z ? dy.num : dx.num, d.other_first = z ? dy.other_first : dx.other_first;
    d.nn_d = z ? dy.nn_d : dx.nn_d, d.nn_i = z ? dy.nn_i : dx.nn_i, d.other_rows = z ? dy.other_rows : dx.other_rows;
    const int n = blockIdx.y;
    const int64_t f = d.first[n], c = d.num[n];
    const int64_t of = d.other_rows > 0 ? d.other_first[n] : 0;
    double acc[2] = {0.0, 0.0};
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < c; t += (int64_t)gridDim.x * blockDim.x) {
        const int64_t row = f + t;
        const int i = d.other_rows > 0 ? d.nn_i[row] : -1;
        if (i < 0) {
            acc[0] += CUDART_NAN;
            if (d.normals) acc[1] += CUDART_NAN;
            continue;
        }
        acc[0] += (double)d.nn_d[row];
        if (d.normals) acc[1] += 1.0 - fabs(cosine_eps(d.normals + row * 3, d.other_normals + (of + i) * 3));
    }
    const double v = block_sum(acc, sPart);
    if (threadIdx.x < 2) partials[(((int64_t)n * 2 + blockIdx.z) * gridDim.x + blockIdx.x) * 2 + threadIdx.x] = v;
}

// grad_finish_kernel's rows: slice l is the direction, row m the cloud, k the term
struct ChamferRows {
    double *sums;
    __device__ __forceinline__ void operator()(const double *tot, int l, int m, int k) const {
        if (k < 2) sums[m * 4 + k * 2 + l] = tot[k];
    }
};

}  // namespace dss

extern "C" {

int dss_chamfer(dss_ctx *ctx, const float *x, const float *x_normals, const int64_t *x_first, const int64_t *x_num,
                int64_t Px, const float *y, const float *y_normals, const int64_t *y_first, const int64_t *y_num,
                int64_t Py, int N, double *sums, void *stream) {
    using namespace dss;
    cudaStream_t st = (cudaStream_t)stream;
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    DSS_REQUIRE(N >= 0 && N <= 65535, "N out of range");
    DSS_REQUIRE(Px >= 0 && Py >= 0 && Px < (int64_t)INT32_MAX && Py < (int64_t)INT32_MAX, "row count out of range");
    DSS_REQUIRE((x_normals == nullptr) == (y_normals == nullptr), "give normals for both clouds or for neither");
    if (N == 0) return DSS_OK;
    DSS_REQUIRE(sums && x_first && x_num && y_first && y_num, "null pointer");
    DSS_REQUIRE((Px == 0 || x) && (Py == 0 || y), "null points");
    const int64_t Pmax = Px > Py ? Px : Py;
    const unsigned blocks = grid_blocks((Pmax + N - 1) / N, CH_THREADS, ctx->sm_count, 4);
    const size_t npart = (size_t)N * 2 * blocks * 2;
    // one slot: partials (doubles), a copy of the offsets (N int64), then x's rows {dist f32, index i32}, then y's
    double *partials = nullptr;
    int rc;
    if ((rc = ctx_get(ctx, BUF_CHAMFER, npart + (size_t)N + (size_t)(Px + Py), &partials))) return rc;
    int64_t *first_copy = reinterpret_cast<int64_t *>(partials + npart);
    float *xd = reinterpret_cast<float *>(first_copy + N);
    int32_t *xi = reinterpret_cast<int32_t *>(xd + Px);
    float *yd = reinterpret_cast<float *>(xi + Px);
    int32_t *yi = reinterpret_cast<int32_t *>(yd + Py);
    // x and y the same rows: dss_knn_points would take its self mode (each row's own index first, not the smallest index
    // among exact duplicates); the queries get a copy of the offsets, so that both searches run in the general mode
    const int64_t *qx_first = x_first, *qy_first = y_first;
    if (x == y && x_first == y_first) {
        DSS_CUDA_TRY(cudaMemcpyAsync(first_copy, x_first, (size_t)N * sizeof(int64_t), cudaMemcpyDeviceToDevice, st));
        qx_first = qy_first = first_copy;
    }
    if (Px > 0 && Py > 0) {
        if ((rc = dss_knn_points(ctx, x, qx_first, x_num, y, y_first, y_num, N, Px, Py, 1, -1.0f, xd, xi, stream)))
            return rc;
        if ((rc = dss_knn_points(ctx, y, qy_first, y_num, x, x_first, x_num, N, Py, Px, 1, -1.0f, yd, yi, stream)))
            return rc;
    }
    ChamferDir dx, dy;
    dx.normals = x_normals, dx.other_normals = y_normals, dx.first = x_first, dx.num = x_num, dx.other_first = y_first;
    dx.nn_d = xd, dx.nn_i = xi, dx.other_rows = Px > 0 ? Py : 0;
    dy.normals = y_normals, dy.other_normals = x_normals, dy.first = y_first, dy.num = y_num, dy.other_first = x_first;
    dy.nn_d = yd, dy.nn_i = yi, dy.other_rows = Py > 0 ? Px : 0;
    chamfer_terms_kernel<<<dim3(blocks, N, 2), CH_THREADS, 0, st>>>(dx, dy, partials);
    DSS_LAUNCH_CHECK(ctx);
    grad_finish_kernel<2><<<dim3(2, N), 256, 0, st>>>(partials, (int)blocks, N, 1, ChamferRows{sums});
    DSS_LAUNCH_CHECK(ctx);
    return DSS_OK;
}

}  // extern "C"
