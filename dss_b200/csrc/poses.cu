// poses.cu -- per-view camera pose corrections: the map from V corrections xi_v = (w, t) in R^6 (a rotation vector and
// a translation, applied in the camera frame) to the refined world-to-view and full projection matrices of a batch of
// views, and its backward.  Row-vector convention, as everywhere in the library:
//
//   E(xi) = [[R(w), 0], [t, 1]],   R(w) = I + s [w]x + c [w]x^2,   s = sin(th) / th,   c = (1 - cos(th)) / th^2
//   view  = view0 E = view0 + view0 D,              D = E - I = [[A, 0], [t, 0]],   A = s [w]x + c [w]x^2
//   proj  = view E K = proj0 + view0 D K,           K = view0^-1 proj0  (view0^-1 the rigid inverse)
//
// R(w) is scipy's Rotation.from_rotvec(w).as_matrix().  The delta form is what makes xi = 0 give view0 and proj0 bit
// for bit: D is formed directly (never as E - I), so it is exactly zero there and the outputs are the inputs' bits.
// Every output element is computed in float64 and rounded once to float32.  s, c and the derivatives' s1 = s' / th,
// c1 = c' / th switch to their Taylor series below th = 0.1 (truncation error under 1e-17 relative there; the closed
// forms lose at most three digits of float64 to cancellation above it), so both branches agree to float64 rounding.
//
// The backward is linear in (d view, d proj), so each pose row first sums the d view / d proj of its batch entries in
// batch order, in float64, and applies the chain rule once.  One thread per pose row: no atomics, no scratch, and the
// same bits on every run; rows of views outside the batch are written as +0.
#include "common.cuh"

namespace dss {

constexpr int POSE_THREADS = 128;
constexpr double POSE_SERIES_BELOW = 0.1;

struct PoseCoeffs {
    double s, c, s1, c1;   // sin(th)/th, (1-cos(th))/th^2 and their th-derivatives over th
};

__device__ __forceinline__ PoseCoeffs pose_coeffs(double th2) {
    PoseCoeffs k;
    if (th2 < POSE_SERIES_BELOW * POSE_SERIES_BELOW) {
        const double x = th2;
        k.s = 1.0 + x * (-1.0 / 6 + x * (1.0 / 120 + x * (-1.0 / 5040 + x * (1.0 / 362880 + x * (-1.0 / 39916800)))));
        k.c = 0.5 + x * (-1.0 / 24 + x * (1.0 / 720 + x * (-1.0 / 40320 + x * (1.0 / 3628800 + x * (-1.0 / 479001600)))));
        k.s1 = -1.0 / 3 + x * (1.0 / 30 + x * (-1.0 / 840 + x * (1.0 / 45360 + x * (-1.0 / 3991680))));
        k.c1 = -1.0 / 12 + x * (1.0 / 180 + x * (-1.0 / 6720 + x * (1.0 / 453600 + x * (-1.0 / 47900160))));
    } else {
        const double th = sqrt(th2), sn = sin(th), cs = cos(th), h = sin(0.5 * th);
        const double omc = 2.0 * h * h;   // 1 - cos(th) without cancellation
        k.s = sn / th;
        k.c = omc / th2;
        k.s1 = (th * cs - sn) / (th2 * th);
        k.c1 = (th * sn - 2.0 * omc) / (th2 * th2);
    }
    return k;
}

// D = E - I of pose p (6 floats), as the (4,3) block of its non-zero columns
__device__ __forceinline__ void pose_delta(const float *p, double D[4][3]) {
    const double w[3] = {p[0], p[1], p[2]};
    const double th2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2];
    const PoseCoeffs k = pose_coeffs(th2);
    // [w]x = [[0, -w2, w1], [w2, 0, -w0], [-w1, w0, 0]];  [w]x^2 = w w^T - th^2 I
    const double W[3][3] = {{0.0, -w[2], w[1]}, {w[2], 0.0, -w[0]}, {-w[1], w[0], 0.0}};
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) D[i][j] = k.s * W[i][j] + k.c * (w[i] * w[j] - (i == j ? th2 : 0.0));
    D[3][0] = p[3], D[3][1] = p[4], D[3][2] = p[5];
}

// K = view0^-1 proj0 with the rigid inverse [[R^T, 0], [-t R^T, 1]] of view0 = [[R, 0], [t, 1]]
__device__ __forceinline__ void pose_intrinsics(const float *v0, const float *p0, double K[4][4]) {
    double inv[4][4];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
#pragma unroll
        for (int j = 0; j < 3; ++j) inv[i][j] = v0[j * 4 + i];
        inv[i][3] = 0.0;
    }
#pragma unroll
    for (int j = 0; j < 3; ++j)
        inv[3][j] = -((double)v0[12] * v0[j * 4 + 0] + (double)v0[13] * v0[j * 4 + 1] + (double)v0[14] * v0[j * 4 + 2]);
    inv[3][3] = 1.0;
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            double a = 0.0;
#pragma unroll
            for (int l = 0; l < 4; ++l) a += inv[i][l] * p0[l * 4 + j];
            K[i][j] = a;
        }
}

// x + d rounded once; an exact zero d keeps x's bits (its sign of zero included): the xi = 0 identity
__device__ __forceinline__ float pose_add(float x, double d) { return d == 0.0 ? x : (float)((double)x + d); }

__global__ void __launch_bounds__(POSE_THREADS) pose_forward_kernel(const float *poses, const int64_t *idx, int V, int B,
                                                                    const float *view0, const float *proj0, float *view,
                                                                    float *proj) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const int64_t v = idx[b];
    float *vo = view + (int64_t)b * 16, *po = proj + (int64_t)b * 16;
    if (v < 0 || v >= V) {   // the host checks the indices; a bad one gives NaN cameras rather than a wild read
        for (int e = 0; e < 16; ++e) vo[e] = po[e] = __int_as_float(0x7fffffff);
        return;
    }
    const float *v0 = view0 + v * 16, *p0 = proj0 + v * 16;
    double D[4][3], K[4][4], M[4][3];
    pose_delta(poses + v * 6, D);
    pose_intrinsics(v0, p0, K);
    // M = view0 D: the non-zero columns of the view's delta
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            double a = 0.0;
#pragma unroll
            for (int l = 0; l < 4; ++l) a += (double)v0[i * 4 + l] * D[l][j];
            M[i][j] = a;
        }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            vo[i * 4 + j] = j < 3 ? pose_add(v0[i * 4 + j], M[i][j]) : v0[i * 4 + j];
            double a = 0.0;
#pragma unroll
            for (int l = 0; l < 3; ++l) a += M[i][l] * K[l][j];
            po[i * 4 + j] = pose_add(p0[i * 4 + j], a);
        }
    }
}

__global__ void __launch_bounds__(POSE_THREADS) pose_backward_kernel(const float *poses, const int64_t *idx, int V,
                                                                     int B, const float *view0, const float *proj0,
                                                                     const float *grad_view, const float *grad_proj,
                                                                     float *grad_poses) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V) return;
    // the row's d view and d proj, summed over its batch entries in batch order
    double Gv[4][4] = {}, Gp[4][4] = {};
    int n = 0;
    for (int b = 0; b < B; ++b) {
        if (idx[b] != v) continue;
        ++n;
#pragma unroll
        for (int e = 0; e < 16; ++e) {
            if (grad_view) Gv[e / 4][e % 4] += grad_view[(int64_t)b * 16 + e];
            if (grad_proj) Gp[e / 4][e % 4] += grad_proj[(int64_t)b * 16 + e];
        }
    }
    float *out = grad_poses + (int64_t)v * 6;
    if (n == 0) {
        for (int k = 0; k < 6; ++k) out[k] = 0.f;
        return;
    }
    const float *v0 = view0 + (int64_t)v * 16, *p0 = proj0 + (int64_t)v * 16;
    double K[4][4];
    pose_intrinsics(v0, p0, K);
    // d L / d D = view0^T (Gv + Gp K^T), of which only the first three columns matter (D's last column is zero)
    double Q[4][3], G[4][3];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            double a = Gv[i][j];
#pragma unroll
            for (int l = 0; l < 4; ++l) a += Gp[i][l] * K[j][l];
            Q[i][j] = a;
        }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            double a = 0.0;
#pragma unroll
            for (int l = 0; l < 4; ++l) a += (double)v0[l * 4 + i] * Q[l][j];
            G[i][j] = a;
        }
    // A = s W + c (w w^T - th^2 I), W = [w]x:
    // d L / d w = w (s1 <G,W> + c1 (w^T G w - th^2 tr G)) + s g + c (G w + G^T w - 2 tr(G) w),  g_k = <G, [e_k]x>
    const float *p = poses + (int64_t)v * 6;
    const double w[3] = {p[0], p[1], p[2]};
    const double th2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2];
    const PoseCoeffs k = pose_coeffs(th2);
    const double g[3] = {G[2][1] - G[1][2], G[0][2] - G[2][0], G[1][0] - G[0][1]};
    const double tr = G[0][0] + G[1][1] + G[2][2];
    double Gw[3], GTw[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        Gw[i] = G[i][0] * w[0] + G[i][1] * w[1] + G[i][2] * w[2];
        GTw[i] = G[0][i] * w[0] + G[1][i] * w[1] + G[2][i] * w[2];
    }
    const double wGw = w[0] * Gw[0] + w[1] * Gw[1] + w[2] * Gw[2];
    const double radial = k.s1 * (w[0] * g[0] + w[1] * g[1] + w[2] * g[2]) + k.c1 * (wGw - th2 * tr);
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        out[i] = (float)(w[i] * radial + k.s * g[i] + k.c * (Gw[i] + GTw[i] - 2.0 * tr * w[i]));
        out[3 + i] = (float)G[3][i];
    }
}

}  // namespace dss

extern "C" {

int dss_pose_forward(dss_ctx *ctx, const float *poses, const int64_t *idx, int V, int B, const float *view0,
                     const float *proj0, float *view, float *proj, void *stream) {
    using namespace dss;
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    DSS_REQUIRE(V >= 1 && B >= 0, "size out of range");
    if (B == 0) return DSS_OK;
    DSS_REQUIRE(poses && idx && view0 && proj0 && view && proj, "null pointer");
    pose_forward_kernel<<<(B + POSE_THREADS - 1) / POSE_THREADS, POSE_THREADS, 0, (cudaStream_t)stream>>>(
        poses, idx, V, B, view0, proj0, view, proj);
    DSS_LAUNCH_CHECK(ctx);
    return DSS_OK;
}

int dss_pose_backward(dss_ctx *ctx, const float *poses, const int64_t *idx, int V, int B, const float *view0,
                      const float *proj0, const float *grad_view, const float *grad_proj, float *grad_poses,
                      void *stream) {
    using namespace dss;
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    DSS_REQUIRE(V >= 1 && B >= 0, "size out of range");
    DSS_REQUIRE(poses && view0 && proj0 && grad_poses && (B == 0 || idx), "null pointer");
    pose_backward_kernel<<<(V + POSE_THREADS - 1) / POSE_THREADS, POSE_THREADS, 0, (cudaStream_t)stream>>>(
        poses, idx, V, B, view0, proj0, grad_view, grad_proj, grad_poses);
    DSS_LAUNCH_CHECK(ctx);
    return DSS_OK;
}

}  // extern "C"
