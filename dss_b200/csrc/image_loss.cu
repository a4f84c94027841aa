// image_loss.cu -- the image loss of the training step, fused: Trainer.calc_dr_loss (DSS/training/trainer.py:332-376)
// with L1Loss(reduction='mean') and IouLoss(reduction='mean', channel_dim=None) (trainer.py:138-140, losses.py:130-137,
// 498-513), on the renderer's RGBA:
//
//   mask_pred = m.bool() & alpha.bool()                                   m: the ground-truth mask, NaN counts as true
//   loss_rgb  = l_rgb * sum_{mask_pred} sum_c |gt - pred| / M             M = |mask_pred|; 0 when M == 0
//   loss_sil  = l_sil * (sum |m - alpha| / (N H W) + 0.01 * mean_n (1 - I_n / eps_denom(U_n)))
//               I_n = sum m alpha, U_n = sum (m + alpha - m alpha) over view n
//
// A term whose lambda is not > 0 is absent, as in the reference: 0, no gradient, no NaN from its inputs (without the
// RGB term the GT RGB is not read).
// Forward, pass 1: grid (blocks, N), every block writes the five fp64 sums of its pixels of view n (M, sum |d rgb|,
// sum |m - alpha|, I, U) to the partials.  Pass 2 (grad_finish_kernel): block n adds view n's partials in block order and
// writes the view's totals; the last block to finish (an integer counter; no float atomics) adds the N totals in a
// fixed order and writes the loss scalars.  Backward: one pass, the coefficients of view n from the totals and the
// upstream gradients of the three scalars, read from device memory.  Bit-reproducible; no host synchronisation.
// View-sharded (each rank holds some of the views): dss_image_loss_partial runs both forward passes but, instead of the
// scalars, puts the rank's view count into the fifth slot of the total row; the caller sums that row over the ranks
// and image_loss_finish_kernel writes the scalars from it.  The backward reads M and the view count from the (summed)
// total row and I_n, U_n from the rank's own view rows.
#include "common.cuh"

namespace dss {

constexpr int IL_THREADS = 256;
constexpr int IL_SUMS = 5;   // M, sum |d rgb| over mask_pred, sum |m - alpha|, I, U

struct ImageLossArgs {
    const float4 *pred;          // (N, H*W) rgba
    const float *gt;             // rgb at gt[n*gs[0] + y*gs[1] + x*gs[2] + c*gs[3]]
    int64_t gs[4];
    const void *mask;            // (N, H*W) float32, or bytes (bool / uint8)
    int mask_bytes;
    int W;
    int64_t HW;
    int use_rgb, use_sil;
};

__device__ __forceinline__ float il_mask(const ImageLossArgs &a, int64_t i) {
    return a.mask_bytes ? (float)static_cast<const uint8_t *>(a.mask)[i] : static_cast<const float *>(a.mask)[i];
}

// the rgb of view n's pixel p = y * W + x
__device__ __forceinline__ float3 il_gt(const ImageLossArgs &a, int n, int64_t p) {
    const unsigned int y = (unsigned int)p / (unsigned int)a.W, x = (unsigned int)p - y * (unsigned int)a.W;
    const float *g = a.gt + n * a.gs[0] + (int64_t)y * a.gs[1] + (int64_t)x * a.gs[2];
    return make_float3(g[0], g[a.gs[3]], g[2 * a.gs[3]]);
}

// torch's sign (as abs' backward takes it): -1, 0 or 1, and 0 for NaN
__device__ __forceinline__ float il_sign(float d) { return d > 0.0f ? 1.0f : (d < 0.0f ? -1.0f : 0.0f); }

__global__ void __launch_bounds__(IL_THREADS) image_loss_partials_kernel(const __grid_constant__ ImageLossArgs a,
                                                                          double *partials, unsigned int *done) {
    __shared__ double sPart[IL_THREADS / 32][IL_SUMS];
    const int n = blockIdx.y;
    if (blockIdx.x == 0 && n == 0 && threadIdx.x == 0) *done = 0;   // the finish's counter, read after this kernel
    double acc[IL_SUMS] = {0.0, 0.0, 0.0, 0.0, 0.0};
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < a.HW; p += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = n * a.HW + p;
        const float4 q = a.pred[i];
        const float m = il_mask(a, i);
        if (m != 0.0f && q.w != 0.0f) {
            acc[0] += 1.0;
            if (a.use_rgb) {
                const float3 g = il_gt(a, n, p);
                acc[1] += fabs((double)g.x - q.x) + fabs((double)g.y - q.y) + fabs((double)g.z - q.z);
            }
        }
        const double md = m, al = q.w;
        acc[2] += fabs(md - al);
        acc[3] += md * al;
        acc[4] += md + al - md * al;
    }
    const double v = block_sum(acc, sPart);
    if (threadIdx.x < IL_SUMS) partials[((int64_t)n * gridDim.x + blockIdx.x) * IL_SUMS + threadIdx.x] = v;
}

// the three loss scalars from the total row's sums over Nv views of HW pixels each
__device__ __forceinline__ void il_scalars(double M, double abs_rgb, double abs_sil, double iou, double Nv,
                                           double npix, double lambda_rgb, double lambda_sil, int use_rgb, int use_sil,
                                           float *loss, float *loss_rgb, float *loss_sil) {
    const double rgb = (use_rgb && M > 0.0) ? lambda_rgb * (abs_rgb / M) : 0.0;
    const double sil = use_sil ? lambda_sil * (0.01 * (iou / Nv) + abs_sil / npix) : 0.0;
    *loss_rgb = (float)rgb;
    *loss_sil = (float)sil;
    *loss = (float)(rgb + sil);
}

// grad_finish_kernel's output rows: view m's totals, then, in the last block, the total row and either the loss scalars
// or (loss == nullptr: one rank's share of a view-sharded loss) the view count in the row's fifth slot
struct ImageLossRows {
    double *totals;              // (N + 1, IL_SUMS): the views', then (M, sum |d rgb|, sum |m - alpha|, sum_n iou_n, 0 or N)
    unsigned int *done;
    float *loss, *loss_rgb, *loss_sil;
    double lambda_rgb, lambda_sil, npix;
    int use_rgb, use_sil;
    __device__ __forceinline__ void operator()(const double *tot, int, int m, int k) const {
        __shared__ double sPart[IL_THREADS / 32][4];
        __shared__ double sAll[4];
        const int N = gridDim.y;
        if (k < IL_SUMS) totals[(int64_t)m * IL_SUMS + k] = tot[k];
        if (!finish_last_block(done, N)) return;
        // every view's totals are written: add them in view order
        double acc[4] = {0.0, 0.0, 0.0, 0.0};
        for (int v = k; v < N; v += blockDim.x) {
            const double *t = totals + (int64_t)v * IL_SUMS;
            acc[0] += __ldcg(t);
            acc[1] += __ldcg(t + 1);
            acc[2] += __ldcg(t + 2);
            acc[3] += 1.0 - __ldcg(t + 3) / eps_denom_f64(__ldcg(t + 4));
        }
        const double s = block_sum(acc, sPart);
        if (k < 4) sAll[k] = s;
        __syncthreads();
        if (k != 0) return;
        double *row = totals + (int64_t)N * IL_SUMS;
        row[0] = sAll[0], row[1] = sAll[1], row[2] = sAll[2], row[3] = sAll[3], row[4] = loss ? 0.0 : (double)N;
        if (loss)
            il_scalars(sAll[0], sAll[1], sAll[2], sAll[3], N, npix, lambda_rgb, lambda_sil, use_rgb, use_sil, loss,
                       loss_rgb, loss_sil);
    }
};

// the scalars of a view-sharded loss from its total row summed over the ranks (the fifth slot: the view count)
__global__ void image_loss_finish_kernel(const double *row, double HW, double lambda_rgb, double lambda_sil,
                                         int use_rgb, int use_sil, float *loss, float *loss_rgb, float *loss_sil) {
    const double Nv = row[4];
    il_scalars(row[0], row[1], row[2], row[3], Nv, Nv * HW, lambda_rgb, lambda_sil, use_rgb, use_sil, loss, loss_rgb,
               loss_sil);
}

struct ImageLossGradArgs {
    const double *totals;                          // as ImageLossRows writes them, the total row maybe summed over ranks
    const float *g_loss, *g_rgb, *g_sil;           // upstream gradients of the three scalars (device)
    double lambda_rgb, lambda_sil;
    float4 *grad;                                  // (N, H*W) d L / d rgba
};

__global__ void __launch_bounds__(IL_THREADS) image_loss_backward_kernel(const __grid_constant__ ImageLossArgs a,
                                                                          const __grid_constant__ ImageLossGradArgs b) {
    const int n = blockIdx.y, N = gridDim.y;
    const double gl = *b.g_loss;
    // the view count of the loss: this call's N, or, for a view-sharded loss, the total row's fifth slot
    const double Nt = b.totals[(int64_t)N * IL_SUMS + 4], Nv = Nt > 0.0 ? Nt : (double)N, npix = Nv * (double)a.HW;
    // rgb: sign(pred - gt) w_rgb inside mask_pred; alpha: sign(alpha - m) w_l1 - m A + (1 - m) B, where
    // d(1 - I/E)/d alpha = -(m E - I (1 - m) dE/dU) / E^2 gives A = w_iou / E and B = w_iou I dE/dU / E^2
    float w_rgb = 0.0f;
    double w_l1 = 0.0, A = 0.0, B = 0.0;
    if (a.use_rgb) {
        const double M = b.totals[(int64_t)N * IL_SUMS];
        w_rgb = M > 0.0 ? (float)(b.lambda_rgb * (gl + (double)*b.g_rgb) / M) : 0.0f;
    }
    if (a.use_sil) {
        const double ws = b.lambda_sil * (gl + (double)*b.g_sil), w_iou = 0.01 * ws / Nv;
        const double I = b.totals[(int64_t)n * IL_SUMS + 3], U = b.totals[(int64_t)n * IL_SUMS + 4];
        const double E = eps_denom_f64(U);   // dE / dU is 1 where the clamp passes the gradient (|U| >= eps), else 0
        w_l1 = ws / npix;
        A = w_iou / E;
        B = fabs(U) >= EPS_DENOM ? w_iou * I / (E * E) : 0.0;
    }
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < a.HW; p += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = n * a.HW + p;
        const float4 q = a.pred[i];
        const float m = il_mask(a, i);
        float4 o = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        if (a.use_rgb && m != 0.0f && q.w != 0.0f) {
            const float3 g = il_gt(a, n, p);
            o.x = il_sign(q.x - g.x) * w_rgb;
            o.y = il_sign(q.y - g.y) * w_rgb;
            o.z = il_sign(q.z - g.z) * w_rgb;
        }
        if (a.use_sil) {
            const double md = m;
            o.w = (float)((double)il_sign(q.w - m) * w_l1 - md * A + (1.0 - md) * B);
        }
        b.grad[i] = o;
    }
}

// blocks per view: one wave over all views at per_sm resident blocks per SM (partials 48 registers: 4, backward 30: 8),
// and no more blocks than the pixels need
static unsigned int il_blocks(const dss_ctx *ctx, int N, int64_t HW, int per_sm) {
    const int64_t want = ((int64_t)ctx->sm_count * per_sm + N - 1) / N, need = (HW + IL_THREADS - 1) / IL_THREADS;
    return (unsigned int)(want < need ? want : need);
}

static int il_args(ImageLossArgs &a, const float *pred, const float *gt, const int64_t *gt_strides, const void *mask,
                   int mask_kind, int N, int H, int W, double lambda_rgb, double lambda_sil) {
    DSS_REQUIRE(N >= 1 && N <= 65535 && H >= 1 && W >= 1, "size out of range");
    DSS_REQUIRE((int64_t)H * W <= (int64_t)INT32_MAX, "more than 2^31-1 pixels per view");
    DSS_REQUIRE(mask_kind == 0 || mask_kind == 1, "mask_kind must be 0 (float32) or 1 (bytes)");
    DSS_REQUIRE(pred && gt && gt_strides && mask, "null pointer");
    DSS_REQUIRE((reinterpret_cast<uintptr_t>(pred) & 15) == 0, "pred must be 16-byte aligned");
    a.pred = reinterpret_cast<const float4 *>(pred);
    a.gt = gt;
    for (int d = 0; d < 4; ++d) a.gs[d] = gt_strides[d];
    a.mask = mask;
    a.mask_bytes = mask_kind;
    a.W = W;
    a.HW = (int64_t)H * W;
    a.use_rgb = lambda_rgb > 0.0;
    a.use_sil = lambda_sil > 0.0;
    return DSS_OK;
}

// both forward passes; loss == nullptr: a rank's share of a view-sharded loss (no scalars, the view count in the row)
static int il_forward(dss_ctx *ctx, const float *pred, const float *gt, const int64_t *gt_strides, const void *mask,
                      int mask_kind, int N, int H, int W, double lambda_rgb, double lambda_sil, double *totals,
                      float *loss, float *loss_rgb, float *loss_sil, void *stream) {
    cudaStream_t st = (cudaStream_t)stream;
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    ImageLossArgs a;
    int rc = il_args(a, pred, gt, gt_strides, mask, mask_kind, N, H, W, lambda_rgb, lambda_sil);
    if (rc) return rc;
    DSS_REQUIRE(totals != nullptr, "null pointer");
    const unsigned int blocks = il_blocks(ctx, N, a.HW, 4);
    const size_t np = (size_t)N * blocks * IL_SUMS;
    double *partials = nullptr;
    if ((rc = ctx_get(ctx, BUF_IMAGE_LOSS, np + 1, &partials))) return rc;
    unsigned int *done = reinterpret_cast<unsigned int *>(partials + np);
    image_loss_partials_kernel<<<dim3(blocks, N), IL_THREADS, 0, st>>>(a, partials, done);
    DSS_LAUNCH_CHECK(ctx);
    ImageLossRows rows;
    rows.totals = totals, rows.done = done, rows.loss = loss, rows.loss_rgb = loss_rgb, rows.loss_sil = loss_sil;
    rows.lambda_rgb = lambda_rgb, rows.lambda_sil = lambda_sil, rows.npix = (double)N * (double)a.HW;
    rows.use_rgb = a.use_rgb, rows.use_sil = a.use_sil;
    grad_finish_kernel<IL_SUMS><<<dim3(1, N), 256, 0, st>>>(partials, (int)blocks, N, 1, rows);
    DSS_LAUNCH_CHECK(ctx);
    return DSS_OK;
}

}  // namespace dss

extern "C" {

int dss_image_loss_forward(dss_ctx *ctx, const float *pred, const float *gt, const int64_t *gt_strides,
                           const void *mask, int mask_kind, int N, int H, int W, double lambda_rgb, double lambda_sil,
                           double *totals, float *loss, float *loss_rgb, float *loss_sil, void *stream) {
    using namespace dss;
    DSS_REQUIRE(loss && loss_rgb && loss_sil, "null pointer");
    return il_forward(ctx, pred, gt, gt_strides, mask, mask_kind, N, H, W, lambda_rgb, lambda_sil, totals, loss,
                      loss_rgb, loss_sil, stream);
}

int dss_image_loss_partial(dss_ctx *ctx, const float *pred, const float *gt, const int64_t *gt_strides,
                           const void *mask, int mask_kind, int N, int H, int W, double lambda_rgb, double lambda_sil,
                           double *totals, void *stream) {
    return dss::il_forward(ctx, pred, gt, gt_strides, mask, mask_kind, N, H, W, lambda_rgb, lambda_sil, totals,
                           nullptr, nullptr, nullptr, stream);
}

int dss_image_loss_finish(dss_ctx *ctx, const double *total_row, int H, int W, double lambda_rgb, double lambda_sil,
                          float *loss, float *loss_rgb, float *loss_sil, void *stream) {
    using namespace dss;
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    DSS_REQUIRE(H >= 1 && W >= 1 && (int64_t)H * W <= (int64_t)INT32_MAX, "size out of range");
    DSS_REQUIRE(total_row && loss && loss_rgb && loss_sil, "null pointer");
    image_loss_finish_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(total_row, (double)H * (double)W, lambda_rgb,
                                                                lambda_sil, lambda_rgb > 0.0, lambda_sil > 0.0, loss,
                                                                loss_rgb, loss_sil);
    DSS_LAUNCH_CHECK(ctx);
    return DSS_OK;
}

int dss_image_loss_backward(dss_ctx *ctx, const float *pred, const float *gt, const int64_t *gt_strides,
                            const void *mask, int mask_kind, int N, int H, int W, double lambda_rgb, double lambda_sil,
                            const double *totals, const float *grad_loss, const float *grad_loss_rgb,
                            const float *grad_loss_sil, float *grad_pred, void *stream) {
    using namespace dss;
    cudaStream_t st = (cudaStream_t)stream;
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    ImageLossArgs a;
    int rc = il_args(a, pred, gt, gt_strides, mask, mask_kind, N, H, W, lambda_rgb, lambda_sil);
    if (rc) return rc;
    DSS_REQUIRE(totals && grad_loss && grad_loss_rgb && grad_loss_sil && grad_pred, "null pointer");
    DSS_REQUIRE((reinterpret_cast<uintptr_t>(grad_pred) & 15) == 0, "grad_pred must be 16-byte aligned");
    ImageLossGradArgs b;
    b.totals = totals, b.g_loss = grad_loss, b.g_rgb = grad_loss_rgb, b.g_sil = grad_loss_sil;
    b.lambda_rgb = lambda_rgb, b.lambda_sil = lambda_sil;
    b.grad = reinterpret_cast<float4 *>(grad_pred);
    image_loss_backward_kernel<<<dim3(il_blocks(ctx, N, a.HW, 8), N), IL_THREADS, 0, st>>>(a, b);
    DSS_LAUNCH_CHECK(ctx);
    return DSS_OK;
}

}  // extern "C"
