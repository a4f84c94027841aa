// local_frames.cu -- per-point principal frames of the anisotropic reconstruction kernel (Vrk_invariant = false,
// Vrk_isotropic = false: DSS/core/rasterizer.py:256-291 over DSS/utils/mathHelper.py:34-91).
//
// The reference takes, per point, its 8 nearest neighbours (the point itself included), the 8x3 matrix D of their
// offsets from the neighbourhood mean and D's SVD (a cuSolver batched Jacobi SVD); curvature = S^2 / 8 are then the
// eigenvalues of the population covariance C = D^T D / 8 and V's columns its eigenvectors.  It keeps the two largest
// pairs: Vr = F diag(lambda) F^T, Sk = F^T with F = [f1 f2].  Here that is one thread per row: gather the neighbours
// (the rows dss_knn_points wrote for K = 8, r = -1), form C in float64, diagonalise it by a fixed number of cyclic
// Jacobi sweeps in float64 (sym3_eigen.cuh, shared with normals.cu) and round once to float32 at the output.  Every row takes the same instruction path up to
// the rotation guards, so the result does not depend on how fast a solver converges, and the launch needs no scratch,
// no atomics and no host synchronisation (capturable in a CUDA graph).
//
// Degenerate rows: where the two smallest eigenvalues agree to 2^-40 of the largest (collinear neighbours, duplicate
// points) the reference's f1 is whatever its SVD returned.  Here it is fixed: f1 = normalize(f2 x e_k), e_k the axis
// of the smallest |f2_k| (the first such axis); where all three agree (a cluster of duplicates, lambda = 0),
// f2 = e_x first, so that f1 = e_z.  Rows with a missing neighbour (-1: a non-finite point, a cloud of fewer than 8
// points) get an all-NaN record, which the preprocess turns into a non-finite splat that every later stage drops.
#include <math_constants.h>

#include "common.cuh"
#include "sym3_eigen.cuh"

namespace dss {

constexpr int LF_K = 8;            // neighbourhood size (rasterizer.py:272-273)

struct LocalFrameArgs {
    const float *points;       // (P,3)
    const int64_t *first_idx;  // (N,) or nullptr: one cloud of P rows
    const int64_t *num_points; // (N,) or nullptr
    const int32_t *knn_idx;    // (P,8) local to the cloud, ascending distance, -1 missing
    float *frames;             // (P,8) {f1.xyz, l1, f2.xyz, l2}
    int64_t P;
};

__global__ void __launch_bounds__(256) local_frames_kernel(const __grid_constant__ LocalFrameArgs a) {
    const ViewRange cr = view_range(a.first_idx, a.num_points, blockIdx.y, a.P);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < cr.count; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t row = cr.first + i;
        const int32_t *nb = a.knn_idx + row * LF_K;
        float4 *out = reinterpret_cast<float4 *>(a.frames + row * 8);
        double q[LF_K][3];
        bool ok = true;
#pragma unroll
        for (int k = 0; k < LF_K; ++k) {
            const int32_t j = nb[k];
            ok = ok && j >= 0;
            const int64_t src = cr.first + (j >= 0 ? j : 0);
#pragma unroll
            for (int e = 0; e < 3; ++e) q[k][e] = (double)a.points[src * 3 + e];
        }
        if (!ok) {
            out[0] = out[1] = make_float4(CUDART_NAN_F, CUDART_NAN_F, CUDART_NAN_F, CUDART_NAN_F);
            continue;
        }
        // neighbourhood mean and population covariance C = sum d d^T / 8 (mathHelper.py:77-85)
        double m[3];
#pragma unroll
        for (int e = 0; e < 3; ++e) {
            double s = 0.0;
#pragma unroll
            for (int k = 0; k < LF_K; ++k) s += q[k][e];
            m[e] = s * (1.0 / LF_K);
        }
        double A[3][3] = {{0.0, 0.0, 0.0}, {0.0, 0.0, 0.0}, {0.0, 0.0, 0.0}};
#pragma unroll
        for (int k = 0; k < LF_K; ++k) {
            const double d0 = q[k][0] - m[0], d1 = q[k][1] - m[1], d2 = q[k][2] - m[2];
            A[0][0] = fma(d0, d0, A[0][0]);
            A[0][1] = fma(d0, d1, A[0][1]);
            A[0][2] = fma(d0, d2, A[0][2]);
            A[1][1] = fma(d1, d1, A[1][1]);
            A[1][2] = fma(d1, d2, A[1][2]);
            A[2][2] = fma(d2, d2, A[2][2]);
        }
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = r; c < 3; ++c) A[r][c] *= 1.0 / LF_K;
        double l0, l1, l2, f0[3], f1[3], f2[3];
        sym3_eigen(A, l0, l1, l2, f0, f1, f2);
        sym3_fix_degenerate(l0, l1, l2, f1, f2);
        out[0] = make_float4((float)f1[0], (float)f1[1], (float)f1[2], (float)l1);
        out[1] = make_float4((float)f2[0], (float)f2[1], (float)f2[2], (float)l2);
    }
}

}  // namespace dss

extern "C" {

int dss_local_frames(dss_ctx *ctx, const float *points, const int64_t *first_idx, const int64_t *num_points, int N,
                     int64_t P, const int32_t *knn_idx, float *frames, void *stream) {
    using namespace dss;
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    DSS_REQUIRE(P >= 0 && P < (int64_t)INT32_MAX, "P out of range");
    DSS_REQUIRE((first_idx == nullptr) == (num_points == nullptr), "first_idx and num_points go together");
    DSS_REQUIRE(first_idx ? (N >= 1 && N <= 65535) : N == 1, "N out of range (one cloud without first_idx)");
    if (P == 0) return DSS_OK;
    DSS_REQUIRE(points && knn_idx && frames, "null pointer");
    DSS_REQUIRE((reinterpret_cast<uintptr_t>(frames) & 15) == 0, "frames must be 16-byte aligned");
    LocalFrameArgs a;
    a.points = points, a.first_idx = first_idx, a.num_points = num_points, a.knn_idx = knn_idx, a.frames = frames;
    a.P = P;
    StageScope prof(ctx, ST_KNN, (cudaStream_t)stream);
    local_frames_kernel<<<dim3(grid_blocks(P, 256, ctx->sm_count, 8), N), 256, 0, (cudaStream_t)stream>>>(a);
    DSS_LAUNCH_CHECK(ctx);
    return DSS_OK;
}

}  // extern "C"
