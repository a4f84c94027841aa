// regularisers.cu -- the projection and repulsion regularisers of the training step, fused (SURVEY.md section 8(f)2).
//
// Replaces the torch bodies of dss_b200/training/losses.py: ProjectionLoss / RepulsionLoss (DSS/training/losses.py:
// 282-497), which the trainer rebuilds every iteration with knn_k = 12 (trainer.py:134-137, 321-326).  In the reference
// the weights (phi, normal_w, visibility_w, spatial_w, density_w), the neighbour positions and the denoised normals are
// all computed under no_grad or detached (losses.py:337-374, 432-470), so row i's loss depends differentiably on p_i
// only and its gradient is a closed form of what the forward already has: the forward saves it per row, and the
// backward is one contraction with the incoming gradient.  Nothing is scattered to neighbours, so there are no atomics
// on floats and the bits do not change from run to run.
//
// Input: one K-NN row per packed row as dss_knn_points writes it ((P,K) squared distances, indices local to the cloud,
// the query in column 0, -1 padded), or the same without column 0 (self_col = 0).  Column j of the row WITHOUT the
// query is "neighbour j" below, j = 0 .. K-2.  The torch body's corners are kept formula by formula:
//   - a missing neighbour (index < 0) is pytorch3d's padding: distance 0, index 0;
//   - knn_gather(..., lengths) zeroes neighbour j >= length in the denoise, the visibility and the sdf / projection
//     normals; get_normal_w gathers without lengths and does not zero it;
//   - the neighbour POSITIONS are the ones the torch body keeps with its tree: either given per column (knn_pos, a
//     caller's knn, used as they are), or read at the neighbour's index from the positions the rows were built on
//     (nbr_points, which may be older than `points` when the rows are reused), zeroed from column length of the given
//     row on (knn_gather on the given layout, or knn_points' positions, zero where the index is missing);
//   - torch's clamp keeps NaN, so h = 0 (K-1 neighbours at distance 0) gives a NaN row that reaches the neighbours
//     through the denoised normal, as in the torch body.
// Pass 1 (denoise, + the per-cloud bounding box for the repulsion): n^_i = sum phi_j n_j / eps_denom(sum phi_j), or
// n_i itself for reliable rows.  Pass 2 (loss): the loss and the gradient coefficients of row i.
#include "common.cuh"

namespace dss {

constexpr int REG_THREADS = 256;

struct RegArgs {
    const float *points, *normals;       // (P,3) packed
    const int64_t *first, *num;          // (N,)
    const float *knn_d;                  // (P, K - 1 + self_col)
    const int32_t *knn_i;                // same shape, local to the cloud
    const float *knn_pos;                // (P, K - 1 + self_col, 3) neighbour positions per column, or NULL
    const float *nbr_points;             // (P,3) positions the neighbours are read from when knn_pos is NULL
    int K;                               // knn_k: neighbours per row, the query included
    int self_col;                        // 1: column 0 of every row is the query (dropped, losses.py:305)
    const uint8_t *reliable;             // (P,) or NULL: these rows keep their own normal (losses.py:207-214)
    const uint8_t *visible;              // (P,) or NULL: visibility weight 1 / 0.1 of a neighbour (losses.py:335-337)
    float inv_sigma2;                    // 1 / sharpness_sigma^2
    float filter_scale;
    float *nhat;                         // (P,3) denoised normals (scratch)
    int *bbox;                           // (N,6) ordered-int min xyz, max xyz (scratch)
    float *loss;                         // (P,) projection, (P,3) repulsion
    float *coef;                         // (P,3) d loss_i / d p_i, or (P,9) row-major M with d L / d p_i = M g_i
};

// torch's clamp(min=lo) keeps NaN; fmaxf would not
__device__ __forceinline__ float clamp_min_keep_nan(float x, float lo) { return x < lo ? lo : x; }

// eps_denom (DSS/utils/mathHelper.py:10-14, eps 1e-17, zero counts as positive) with NaN kept like torch
__device__ __forceinline__ float reg_eps_denom(float d) {
    const float a = clamp_min_keep_nan(fabsf(d), 1e-17f);
    return d < 0.0f ? -a : a;
}

// F.normalize(x, eps=1e-12): x / clamp_min(|x|, eps)
__device__ __forceinline__ void normalize3(const float *x, float *y) {
    const float den = clamp_min_keep_nan(sqrtf(x[0] * x[0] + x[1] * x[1] + x[2] * x[2]), 1e-12f);
    y[0] = x[0] / den, y[1] = x[1] / den, y[2] = x[2] / den;
}

// neighbour j (query column dropped) of packed row `row` of a cloud of L points
__device__ __forceinline__ void reg_neighbour(const RegArgs &a, int64_t row, int j, int64_t L, float &d, int64_t &id) {
    const int64_t o = row * (a.K - 1 + a.self_col) + j + a.self_col;
    const int k = a.knn_i[o];
    d = k >= 0 ? a.knn_d[o] : 0.0f;
    id = (k >= 0 && k < L) ? k : 0;              // an index outside the cloud is never read
}

// h = 4 * mean squared neighbour distance (losses.py:258-277)
__device__ __forceinline__ float reg_h(const RegArgs &a, int64_t row, int64_t L) {
    float s = 0.0f;
    for (int j = 0; j < a.K - 1; ++j) {
        float d;
        int64_t id;
        reg_neighbour(a, row, j, L, d, id);
        s += d;
    }
    return s / (float)(a.K - 1) * 4.0f;
}

// phi = clamp(1 - d / h, 0)^4, squared twice as the torch body does
__device__ __forceinline__ float reg_phi(float d, float h) {
    float w = clamp_min_keep_nan(1.0f - d / h, 0.0f);
    w = w * w;
    return w * w;
}

__global__ void reg_bbox_init_kernel(int *bbox, int N) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < N * 6) bbox[i] = (i % 6 < 3) ? INT32_MAX : INT32_MIN;
}

// grid (blocks, N): cloud n's rows, grid-stride.  BBOX: also the cloud's min / max coordinates, NaN included (torch's
// min / max propagate it), through integer atomics on the ordered map, so the order of the rows does not matter.
template <bool BBOX>
__global__ void __launch_bounds__(REG_THREADS) reg_denoise_kernel(RegArgs a) {
    const int n = blockIdx.y;
    const int64_t f = a.first[n], L = a.num[n];
    int lo[3] = {INT32_MAX, INT32_MAX, INT32_MAX}, hi[3] = {INT32_MIN, INT32_MIN, INT32_MIN};
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < L; t += (int64_t)gridDim.x * blockDim.x) {
        const int64_t row = f + t;
        float out[3];
        if (a.reliable != nullptr && a.reliable[row]) {
#pragma unroll
            for (int c = 0; c < 3; ++c) out[c] = a.normals[row * 3 + c];
        } else {
            const float h = reg_h(a, row, L);
            float sw = 0.0f, s[3] = {0.0f, 0.0f, 0.0f};
            for (int j = 0; j < a.K - 1; ++j) {
                float d;
                int64_t id;
                reg_neighbour(a, row, j, L, d, id);
                const float phi = reg_phi(d, h);
                sw += phi;
                const bool zero = j >= L;                      // knn_gather(normals, idx, lengths)
#pragma unroll
                for (int c = 0; c < 3; ++c) s[c] += (zero ? 0.0f : a.normals[(f + id) * 3 + c]) * phi;
            }
            const float e = reg_eps_denom(sw);
#pragma unroll
            for (int c = 0; c < 3; ++c) out[c] = s[c] / e;
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) a.nhat[row * 3 + c] = out[c];
        if (BBOX) {
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const int v = f2ord(a.points[row * 3 + c]);
                lo[c] = min(lo[c], v);
                hi[c] = max(hi[c], v);
            }
        }
    }
    if (BBOX) {
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            lo[c] = __reduce_min_sync(0xffffffffu, lo[c]);
            hi[c] = __reduce_max_sync(0xffffffffu, hi[c]);
        }
        if ((threadIdx.x & 31) == 0) {
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                atomicMin(&a.bbox[n * 6 + c], lo[c]);
                atomicMax(&a.bbox[n * 6 + 3 + c], hi[c]);
            }
        }
    }
}

// KIND 0: projection (losses.py:326-395), KIND 1: repulsion (losses.py:420-487)
template <int KIND>
__global__ void __launch_bounds__(REG_THREADS) reg_loss_kernel(RegArgs a) {
    const int n = blockIdx.y;
    const int64_t f = a.first[n], L = a.num[n];
    float inv_spatial = 0.0f;                    // P / diag^2 (losses.py:248-256)
    if (KIND == 1 && L > 0) {
        float diag2 = 0.0f;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float e = ord2f(a.bbox[n * 6 + 3 + c]) - ord2f(a.bbox[n * 6 + c]);
            diag2 += e * e;
        }
        inv_spatial = (float)L / diag2;
    }
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < L; t += (int64_t)gridDim.x * blockDim.x) {
        const int64_t row = f + t;
        const float p[3] = {a.points[row * 3], a.points[row * 3 + 1], a.points[row * 3 + 2]};
        float ni[3];
        {
            const float m[3] = {a.nhat[row * 3], a.nhat[row * 3 + 1], a.nhat[row * 3 + 2]};
            normalize3(m, ni);
        }
        const float h = reg_h(a, row, L);
        float sw = 0.0f;
        float acc[3] = {0.0f, 0.0f, 0.0f};       // projection: sum w sdf n^; repulsion: sum w proj
        float sws = 0.0f;                         // projection: sum w sdf^2; repulsion: sum spatial_w
        float A[6] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f};   // repulsion: sum w n^ n^T (xx xy xz yy yz zz)
        for (int j = 0; j < a.K - 1; ++j) {
            float d;
            int64_t id;
            reg_neighbour(a, row, j, L, d, id);
            const int64_t q = f + id;
            const float m[3] = {a.nhat[q * 3], a.nhat[q * 3 + 1], a.nhat[q * 3 + 2]};
            float mu[3];
            normalize3(m, mu);
            const float dx = mu[0] - ni[0], dy = mu[1] - ni[1], dz = mu[2] - ni[2];
            const float nw = expf(-(dx * dx + dy * dy + dz * dz) * a.inv_sigma2);       // losses.py:224-246
            const bool zero = j >= L;                                                  // knn_gather(..., lengths)
            const float nz[3] = {zero ? 0.0f : m[0], zero ? 0.0f : m[1], zero ? 0.0f : m[2]};
            const bool pzero = j >= L - a.self_col;                                    // neighbour position zeroed
            const float *qp = a.knn_pos != nullptr ? a.knn_pos + (row * (a.K - 1 + a.self_col) + j + a.self_col) * 3
                                                   : a.nbr_points + q * 3;
            float u[3];                                                                // q_j - p_i
#pragma unroll
            for (int c = 0; c < 3; ++c) u[c] = ((pzero && a.knn_pos == nullptr) ? 0.0f : qp[c]) - p[c];
            const float phi = reg_phi(d, h);
            if (KIND == 0) {
                const float vw = a.visible == nullptr ? 1.0f : ((!zero && a.visible[q]) ? 1.0f : 0.1f);
                const float w = phi * nw * vw;
                const float sdf = u[0] * nz[0] + u[1] * nz[1] + u[2] * nz[2];
                sw += w;
                sws += w * sdf * sdf;
#pragma unroll
                for (int c = 0; c < 3; ++c) acc[c] += w * sdf * nz[c];
            } else {
                const float sp = expf(-(u[0] * u[0] + u[1] * u[1] + u[2] * u[2]) * inv_spatial * a.filter_scale);
                const float w = sp * nw;
                // proj = diff - (diff . n^) n^ with diff = p_i - q_j = -u
                const float dn = -u[0] * nz[0] - u[1] * nz[1] - u[2] * nz[2];
                sw += w;
                sws += sp;
#pragma unroll
                for (int c = 0; c < 3; ++c) acc[c] += (-u[c] - dn * nz[c]) * w;
                A[0] += w * nz[0] * nz[0], A[1] += w * nz[0] * nz[1], A[2] += w * nz[0] * nz[2];
                A[3] += w * nz[1] * nz[1], A[4] += w * nz[1] * nz[2], A[5] += w * nz[2] * nz[2];
            }
        }
        const float e = reg_eps_denom(sw);
        if (KIND == 0) {
            a.loss[row] = sws / e;
#pragma unroll
            for (int c = 0; c < 3; ++c) a.coef[row * 3 + c] = -2.0f * acc[c] / e;
        } else {
            // repel = sum w proj / eps_denom(sum w) * density;  d repel / d p_i = density / e (sum w I - sum w n^ n^T)
            const float density = sws + 1.0f;
            float s[3];
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const float r = acc[c] / e * density;
                const float l = expf(-fabsf(r));
                a.loss[row * 3 + c] = l;
                s[c] = r > 0.0f ? -l : (r < 0.0f ? l : r * 0.0f);    // -sign(r) exp(-|r|), sign(0) = 0, NaN kept
            }
            const float k = density / e;
            const float J[9] = {k * (sw - A[0]), -k * A[1], -k * A[2],
                                -k * A[1], k * (sw - A[3]), -k * A[4],
                                -k * A[2], -k * A[4], k * (sw - A[5])};
#pragma unroll
            for (int r = 0; r < 3; ++r)
#pragma unroll
                for (int c = 0; c < 3; ++c) a.coef[row * 9 + r * 3 + c] = J[r * 3 + c] * s[c];
        }
    }
}

}  // namespace dss

extern "C" {

int dss_surface_regulariser(dss_ctx *ctx, int kind, const float *points, const float *normals, const int64_t *first_idx,
                            const int64_t *num_points, int N, int64_t P, const float *knn_dists, const int32_t *knn_idx,
                            int K, int self_col, const float *knn_pos, const float *neighbour_points,
                            const uint8_t *reliable, const uint8_t *visible, float sharpness_sigma,
                            float filter_scale, float *loss, float *grad_coef, void *stream) {
    using namespace dss;
    cudaStream_t st = (cudaStream_t)stream;
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    DSS_REQUIRE(kind == 0 || kind == 1, "kind must be 0 (projection) or 1 (repulsion)");
    DSS_REQUIRE(N >= 0 && N <= 65535 && P >= 0, "size out of range");
    DSS_REQUIRE(K >= 2 && K <= 32, "K must be in [2, 32]");
    DSS_REQUIRE(self_col == 0 || self_col == 1, "self_col must be 0 or 1");
    DSS_REQUIRE(P < (int64_t)INT32_MAX, "more than 2^31-1 points");
    if (N == 0 || P == 0) return DSS_OK;
    DSS_REQUIRE(points && normals && first_idx && num_points && knn_dists && knn_idx && loss && grad_coef, "null pointer");
    float *nhat = nullptr;
    int rc;
    const size_t nh = ((size_t)P * 3 + 63) & ~size_t(63);
    if ((rc = ctx_get(ctx, BUF_REGULARISER, nh + (size_t)N * 6, &nhat))) return rc;
    RegArgs a;
    a.points = points, a.normals = normals, a.first = first_idx, a.num = num_points;
    a.knn_d = knn_dists, a.knn_i = knn_idx, a.K = K, a.self_col = self_col;
    a.knn_pos = knn_pos, a.nbr_points = neighbour_points != nullptr ? neighbour_points : points;
    a.reliable = reliable, a.visible = kind == 0 ? visible : nullptr;
    a.inv_sigma2 = (float)(1.0 / ((double)sharpness_sigma * (double)sharpness_sigma));
    a.filter_scale = filter_scale;
    a.nhat = nhat, a.bbox = reinterpret_cast<int *>(nhat + nh), a.loss = loss, a.coef = grad_coef;
    const dim3 grid(grid_blocks(P, REG_THREADS, ctx->sm_count, 8), N);
    if (kind == 1) {
        reg_bbox_init_kernel<<<(N * 6 + 127) / 128, 128, 0, st>>>(a.bbox, N);
        DSS_LAUNCH_CHECK(ctx);
        reg_denoise_kernel<true><<<grid, REG_THREADS, 0, st>>>(a);
        DSS_LAUNCH_CHECK(ctx);
        reg_loss_kernel<1><<<grid, REG_THREADS, 0, st>>>(a);
    } else {
        reg_denoise_kernel<false><<<grid, REG_THREADS, 0, st>>>(a);
        DSS_LAUNCH_CHECK(ctx);
        reg_loss_kernel<0><<<grid, REG_THREADS, 0, st>>>(a);
    }
    DSS_LAUNCH_CHECK(ctx);
    return DSS_OK;
}

}  // extern "C"
