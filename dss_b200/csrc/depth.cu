// depth.cu -- dense depth of the splat blend and the depth loss of the training step.
//
// Depth map: D[n,y,x] = sum_k w_k z_k over the pixel's K-list in k order (fmaf, one rounding per slot), w_k the
// normalised blend weights the colour uses (after depth merging), z_k the view depth of the record; D = 0 where the
// list is empty.  One launch after the raster, from the forward's idx, weights and records.
// Its backward holds the weights constant, as the reference holds the blend weights' q-dependence (it drops
// qvalue_grad, rasterizer.py:788-813): d L / d z_s = sum g_D w_k over the pixels whose list holds record s.  Those terms
// are summed in 64-bit fixed point with the scale rule of the deterministic colour backward (backward.cu), so the sum
// is the same bits in any order; the result is added to the z gradient the chain kernel reads.
//
// Depth loss: loss = lambda sum_valid |D - D_gt| / M, valid = mask != 0 (NaN counts as set) & alpha != 0 & D_gt finite
// & znear < D_gt < zfar, M = |valid|, 0 when M = 0.  Forward, pass 1: grid (blocks, N), every block writes two fp64 sums
// (M, sum |D - D_gt|) of its pixels; pass 2 (grad_finish_kernel): one block adds all of them in a fixed order and
// writes the total row and the scalar.  Backward: one pass, sign(D - D_gt) lambda g / M on valid pixels, 0 elsewhere.
// View-sharded: dss_depth_loss_partial writes the rank's total row only; the caller sums it over the ranks and
// dss_depth_loss_finish writes the scalar.  Bit-reproducible; no host synchronisation.
#include "common.cuh"
#include "kernels.cuh"

namespace dss {

__global__ void __launch_bounds__(256)
depth_forward_kernel(const int32_t *__restrict__ idx, const float *__restrict__ weights, const float4 *__restrict__ rec,
                     int64_t num_pixels, int K, float *__restrict__ depth) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < num_pixels;
         i += (int64_t)gridDim.x * blockDim.x) {
        float d = 0.0f;
        for (int k = 0; k < K; ++k) {
            const int p = idx[i * K + k];
            if (p < 0) break;
            d = fmaf(weights[i * K + k], rec[2 * (int64_t)p].z, d);
        }
        depth[i] = d;
    }
}

int depth_forward(dss_ctx *ctx, const dss_render_args *g, const float4 *rec, cudaStream_t st) {
    DSS_REQUIRE(g->idx && g->weights, "the depth map needs idx and weights");
    const int64_t npix = (int64_t)g->n_views * g->image_size * g->image_size;
    if (npix == 0) return DSS_OK;
    StageScope prof(ctx, ST_DEPTH_FWD, st);
    depth_forward_kernel<<<grid_blocks(npix, 256, ctx->sm_count, 16), 256, 0, st>>>(g->idx, g->weights, rec, npix,
                                                                                     g->points_per_pixel, g->depth);
    DSS_LAUNCH_CHECK(ctx);
    return DSS_OK;
}

__global__ void __launch_bounds__(256)
depth_gmax_kernel(const float *__restrict__ grad_depth, int64_t num_pixels, int *__restrict__ gmax) {
    int m = 0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < num_pixels;
         i += (int64_t)gridDim.x * blockDim.x)
        m = max(m, finite_abs_bits(__ldg(&grad_depth[i])));
    m = __reduce_max_sync(0xffffffffu, m);
    if ((threadIdx.x & 31) == 0 && m > 0) atomicMax(gmax, m);
}

__global__ void __launch_bounds__(256)
depth_fixed_kernel(const int32_t *__restrict__ idx, const float *__restrict__ weights,
                   const float *__restrict__ grad_depth, int64_t num_pixels, int K, int64_t pixels_per_view,
                   const int *__restrict__ gmax, unsigned long long *__restrict__ acc, float *__restrict__ gz) {
    const int e = colour_fixed_exp(gmax, pixels_per_view);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < num_pixels;
         i += (int64_t)gridDim.x * blockDim.x) {
        if (idx[i * K] < 0) continue;
        const float gd = __ldg(&grad_depth[i]);
        if (gd == 0.0f) continue;
        for (int k = 0; k < K; ++k) {
            const int p = idx[i * K + k];
            if (p < 0) break;
            const float v = gd * weights[i * K + k];
            // a non-finite term goes to the float output: its NaN or infinity does not depend on the order
            if (isfinite(v)) atomicAdd(&acc[p], (unsigned long long)__float2ll_rn(ldexpf(v, e)));
            else atomicAdd(&gz[p], v);
        }
    }
}

__global__ void __launch_bounds__(256)
depth_fixed_finish_kernel(const unsigned long long *__restrict__ acc, int64_t P, int64_t pixels_per_view,
                          const int *__restrict__ gmax, float *__restrict__ gz) {
    const int e = colour_fixed_exp(gmax, pixels_per_view);
    for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < P; j += (int64_t)gridDim.x * blockDim.x)
        if (isfinite(gz[j])) gz[j] += (float)ldexp((double)(long long)acc[j], -e);
}

int depth_backward(dss_ctx *ctx, const dss_render_args *g, float *gz, cudaStream_t st) {
    const int K = g->points_per_pixel;
    const int64_t ppv = (int64_t)g->image_size * g->image_size, npix = (int64_t)g->n_views * ppv, P = g->P;
    if (npix == 0 || P == 0) return DSS_OK;
    unsigned long long *acc = nullptr;      // (P,) sums, then the int bits of G
    int rc;
    if ((rc = ctx_get(ctx, BUF_DEPTH_FIXED, (size_t)P + 1, &acc))) return rc;
    int *gmax = reinterpret_cast<int *>(acc + P);
    DSS_CUDA_TRY(cudaMemsetAsync(acc, 0, ((size_t)P + 1) * sizeof(unsigned long long), st));
    StageScope prof(ctx, ST_DEPTH_BWD, st);
    const unsigned blocks = grid_blocks(npix, 256, ctx->sm_count, 16);
    depth_gmax_kernel<<<blocks, 256, 0, st>>>(g->grad_depth, npix, gmax);
    DSS_LAUNCH_CHECK(ctx);
    depth_fixed_kernel<<<blocks, 256, 0, st>>>(g->idx, g->weights, g->grad_depth, npix, K, ppv, gmax, acc, gz);
    DSS_LAUNCH_CHECK(ctx);
    depth_fixed_finish_kernel<<<grid_blocks(P, 256, ctx->sm_count, 8), 256, 0, st>>>(acc, P, ppv, gmax, gz);
    DSS_LAUNCH_CHECK(ctx);
    return DSS_OK;
}

// ---------------------------------------------------------------------------------------------
// depth loss
// ---------------------------------------------------------------------------------------------
constexpr int DL_THREADS = 256;
constexpr int DL_SUMS = 2;   // M, sum |D - D_gt| over the valid pixels

struct DepthLossArgs {
    const float *depth;          // (N, H*W)
    const float4 *pred;          // (N, H*W) rgba: the alpha channel gates the pixel
    const float *gt;             // (N, H*W)
    const void *mask;            // (N, H*W) float32, or bytes (bool / uint8)
    int mask_bytes;
    int64_t HW;
    float znear, zfar;
};

__device__ __forceinline__ bool dl_valid(const DepthLossArgs &a, int64_t i, float gt) {
    const float m = a.mask_bytes ? (float)static_cast<const uint8_t *>(a.mask)[i] : static_cast<const float *>(a.mask)[i];
    return m != 0.0f && a.pred[i].w != 0.0f && isfinite(gt) && gt > a.znear && gt < a.zfar;
}

__global__ void __launch_bounds__(DL_THREADS) depth_loss_partials_kernel(const __grid_constant__ DepthLossArgs a,
                                                                          double *partials) {
    __shared__ double sPart[DL_THREADS / 32][DL_SUMS];
    const int n = blockIdx.y;
    double acc[DL_SUMS] = {0.0, 0.0};
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < a.HW; p += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = n * a.HW + p;
        const float gt = a.gt[i];
        if (dl_valid(a, i, gt)) {
            acc[0] += 1.0;
            acc[1] += fabs((double)a.depth[i] - (double)gt);
        }
    }
    const double v = block_sum(acc, sPart);
    if (threadIdx.x < DL_SUMS) partials[((int64_t)n * gridDim.x + blockIdx.x) * DL_SUMS + threadIdx.x] = v;
}

__device__ __forceinline__ float dl_scalar(double M, double sum_abs, double lambda) {
    return M > 0.0 ? (float)(lambda * (sum_abs / M)) : 0.0f;
}

// grad_finish_kernel's output: the total row (M, sum |D - D_gt|) and, unless a rank's share of a view-sharded loss
// (loss == nullptr), the scalar
struct DepthLossRow {
    double *totals;
    float *loss;
    double lambda;
    __device__ __forceinline__ void operator()(const double *tot, int, int, int k) const {
        if (k < DL_SUMS) totals[k] = tot[k];
        if (k == 0 && loss) *loss = dl_scalar(tot[0], tot[1], lambda);
    }
};

__global__ void depth_loss_finish_kernel(const double *row, double lambda, float *loss) {
    *loss = dl_scalar(row[0], row[1], lambda);
}

__global__ void __launch_bounds__(DL_THREADS) depth_loss_backward_kernel(const __grid_constant__ DepthLossArgs a,
                                                                          const double *totals, const float *g_loss,
                                                                          double lambda, float *grad) {
    const int n = blockIdx.y;
    const double M = totals[0];
    const float w = M > 0.0 ? (float)(lambda * (double)*g_loss / M) : 0.0f;
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < a.HW; p += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = n * a.HW + p;
        const float gt = a.gt[i], d = a.depth[i];
        // torch's sign (as abs' backward takes it): -1, 0 or 1, and 0 for NaN
        const float s = d > gt ? 1.0f : (d < gt ? -1.0f : 0.0f);
        grad[i] = dl_valid(a, i, gt) ? s * w : 0.0f;
    }
}

// blocks per view: one wave over all views at per_sm resident blocks per SM, and no more blocks than the pixels need
static unsigned int dl_blocks(const dss_ctx *ctx, int N, int64_t HW, int per_sm) {
    const int64_t want = ((int64_t)ctx->sm_count * per_sm + N - 1) / N, need = (HW + DL_THREADS - 1) / DL_THREADS;
    return (unsigned int)(want < need ? want : need);
}

static int dl_args(DepthLossArgs &a, const float *depth, const float *pred, const float *gt, const void *mask,
                   int mask_kind, int N, int H, int W, float znear, float zfar) {
    DSS_REQUIRE(N >= 1 && N <= 65535 && H >= 1 && W >= 1, "size out of range");
    DSS_REQUIRE((int64_t)H * W <= (int64_t)INT32_MAX, "more than 2^31-1 pixels per view");
    DSS_REQUIRE(mask_kind == 0 || mask_kind == 1, "mask_kind must be 0 (float32) or 1 (bytes)");
    DSS_REQUIRE(depth && pred && gt && mask, "null pointer");
    DSS_REQUIRE((reinterpret_cast<uintptr_t>(pred) & 15) == 0, "pred must be 16-byte aligned");
    a.depth = depth;
    a.pred = reinterpret_cast<const float4 *>(pred);
    a.gt = gt;
    a.mask = mask;
    a.mask_bytes = mask_kind;
    a.HW = (int64_t)H * W;
    a.znear = znear;
    a.zfar = zfar;
    return DSS_OK;
}

static int dl_forward(dss_ctx *ctx, const float *depth, const float *pred, const float *gt, const void *mask,
                      int mask_kind, int N, int H, int W, float znear, float zfar, double lambda, double *totals,
                      float *loss, void *stream) {
    cudaStream_t st = (cudaStream_t)stream;
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    DepthLossArgs a;
    int rc = dl_args(a, depth, pred, gt, mask, mask_kind, N, H, W, znear, zfar);
    if (rc) return rc;
    DSS_REQUIRE(totals != nullptr, "null pointer");
    const unsigned int blocks = dl_blocks(ctx, N, a.HW, 4);
    double *partials = nullptr;
    if ((rc = ctx_get(ctx, BUF_DEPTH_LOSS, (size_t)N * blocks * DL_SUMS, &partials))) return rc;
    depth_loss_partials_kernel<<<dim3(blocks, N), DL_THREADS, 0, st>>>(a, partials);
    DSS_LAUNCH_CHECK(ctx);
    grad_finish_kernel<DL_SUMS><<<dim3(1, 1), 256, 0, st>>>(partials, (int)blocks, N, 0,
                                                            DepthLossRow{totals, loss, lambda});
    DSS_LAUNCH_CHECK(ctx);
    return DSS_OK;
}

}  // namespace dss

extern "C" {

int dss_depth_loss_forward(dss_ctx *ctx, const float *depth, const float *pred, const float *gt, const void *mask,
                           int mask_kind, int N, int H, int W, float znear, float zfar, double lambda, double *totals,
                           float *loss, void *stream) {
    DSS_REQUIRE(loss != nullptr, "null pointer");
    return dss::dl_forward(ctx, depth, pred, gt, mask, mask_kind, N, H, W, znear, zfar, lambda, totals, loss, stream);
}

int dss_depth_loss_partial(dss_ctx *ctx, const float *depth, const float *pred, const float *gt, const void *mask,
                           int mask_kind, int N, int H, int W, float znear, float zfar, double *totals, void *stream) {
    return dss::dl_forward(ctx, depth, pred, gt, mask, mask_kind, N, H, W, znear, zfar, 0.0, totals, nullptr, stream);
}

int dss_depth_loss_finish(dss_ctx *ctx, const double *total_row, double lambda, float *loss, void *stream) {
    using namespace dss;
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    DSS_REQUIRE(total_row && loss, "null pointer");
    depth_loss_finish_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(total_row, lambda, loss);
    DSS_LAUNCH_CHECK(ctx);
    return DSS_OK;
}

int dss_depth_loss_backward(dss_ctx *ctx, const float *depth, const float *pred, const float *gt, const void *mask,
                            int mask_kind, int N, int H, int W, float znear, float zfar, double lambda,
                            const double *totals, const float *grad_loss, float *grad_depth, void *stream) {
    using namespace dss;
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    DepthLossArgs a;
    int rc = dl_args(a, depth, pred, gt, mask, mask_kind, N, H, W, znear, zfar);
    if (rc) return rc;
    DSS_REQUIRE(totals && grad_loss && grad_depth, "null pointer");
    depth_loss_backward_kernel<<<dim3(dl_blocks(ctx, N, a.HW, 8), N), DL_THREADS, 0, (cudaStream_t)stream>>>(
        a, totals, grad_loss, lambda, grad_depth);
    DSS_LAUNCH_CHECK(ctx);
    return DSS_OK;
}

}  // extern "C"
