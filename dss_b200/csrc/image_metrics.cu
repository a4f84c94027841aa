// image_metrics.cu -- the image-space validation metrics of the reference's Trainer.eval_step
// (DSS/training/trainer.py:173-212) for renders of s x s pixels against ground truth of H x W pixels:
//
//   g^, m^   = the ground-truth RGB and mask resized to s x s as F.interpolate(mode='bilinear', align_corners=False)
//   iou_n    = 1 - I_n / eps_denom(U_n)      I_n = sum m^ alpha, U_n = sum (m^ + alpha - m^ alpha)   (IouLoss)
//   psnr_n   = E_n / s^2                     E_n = sum_pixels sum_c (g^_c - p_c)^2      (L2Loss(channel_dim=1), a mean
//                                                                                     squared error despite its name)
//
// on the raw render (no clamping, as eval_step reads it).  The resize is torch's upsample_bilinear2d without antialias,
// in float32: src = max((dst + 0.5) H / s - 0.5, 0), i0 = (int)src, i1 = i0 + (i0 < H - 1), weights src - i0 and
// 1 - (src - i0), combined in ATen's order, so that s == H returns every input value unchanged.
// Pass 1: grid (blocks, V), every block writes the three fp64 sums (I, U, E) of its pixels of view n to the partials.
// Pass 2 (grad_finish_kernel): block n adds view n's partials in block order and writes the view's row; the last block
// to finish (an integer counter; no float atomics) adds the rows' iou_n and psnr_n in view order and writes the means.
// Bit-reproducible; no host synchronisation.
#include "common.cuh"

namespace dss {

constexpr int IM_THREADS = 256;
constexpr int IM_SUMS = 3;   // I, U, E

struct ImageMetricsArgs {
    const float4 *pred;          // (V, s*s) rgba
    const float *gt;             // rgb at gt[n*gs[0] + y*gs[1] + x*gs[2] + c*gs[3]]
    int64_t gs[4];
    const void *mask;            // (V, H*W) float32, or bytes (bool / uint8)
    int mask_bytes;
    int H, W, s;
    float scale_y, scale_x;      // H / s, W / s as torch's area_pixel_compute_scale forms them
};

__device__ __forceinline__ float im_mask(const ImageMetricsArgs &a, int64_t i) {
    return a.mask_bytes ? (float)static_cast<const uint8_t *>(a.mask)[i] : static_cast<const float *>(a.mask)[i];
}

// area_pixel_compute_source_index (align_corners = false, not cubic) and the two taps of upsample_bilinear2d
struct Taps {
    int i0, i1;
    float l0, l1;
};
__device__ __forceinline__ Taps im_taps(float scale, int dst, int size) {
    float src = scale * ((float)dst + 0.5f) - 0.5f;
    src = src < 0.0f ? 0.0f : src;
    Taps t;
    t.i0 = (int)src;
    t.i1 = t.i0 + (t.i0 < size - 1 ? 1 : 0);
    t.l1 = src - (float)t.i0;
    t.l0 = 1.0f - t.l1;
    return t;
}

__device__ __forceinline__ float im_lerp(const Taps &ty, const Taps &tx, float a, float b, float c, float d) {
    return ty.l0 * (tx.l0 * a + tx.l1 * b) + ty.l1 * (tx.l0 * c + tx.l1 * d);
}

__global__ void __launch_bounds__(IM_THREADS) image_metrics_partials_kernel(const __grid_constant__ ImageMetricsArgs a,
                                                                            double *partials, unsigned int *done) {
    __shared__ double sPart[IM_THREADS / 32][IM_SUMS];
    const int n = blockIdx.y;
    if (blockIdx.x == 0 && n == 0 && threadIdx.x == 0) *done = 0;   // the finish's counter, read after this kernel
    const int64_t ss = (int64_t)a.s * a.s, HW = (int64_t)a.H * a.W;
    const float *gv = a.gt + n * a.gs[0];
    const int64_t mv = n * HW;
    double acc[IM_SUMS] = {0.0, 0.0, 0.0};
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < ss; p += (int64_t)gridDim.x * blockDim.x) {
        const int y = (int)((unsigned int)p / (unsigned int)a.s), x = (int)p - y * a.s;
        const float4 q = a.pred[n * ss + p];
        const Taps ty = im_taps(a.scale_y, y, a.H), tx = im_taps(a.scale_x, x, a.W);
        const int64_t r0 = (int64_t)ty.i0 * a.W, r1 = (int64_t)ty.i1 * a.W;
        const float m = im_lerp(ty, tx, im_mask(a, mv + r0 + tx.i0), im_mask(a, mv + r0 + tx.i1),
                                im_mask(a, mv + r1 + tx.i0), im_mask(a, mv + r1 + tx.i1));
        const float *g00 = gv + (int64_t)ty.i0 * a.gs[1] + (int64_t)tx.i0 * a.gs[2];
        const float *g01 = gv + (int64_t)ty.i0 * a.gs[1] + (int64_t)tx.i1 * a.gs[2];
        const float *g10 = gv + (int64_t)ty.i1 * a.gs[1] + (int64_t)tx.i0 * a.gs[2];
        const float *g11 = gv + (int64_t)ty.i1 * a.gs[1] + (int64_t)tx.i1 * a.gs[2];
        const float pc[3] = {q.x, q.y, q.z};
        double e = 0.0;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const int64_t o = c * a.gs[3];
            const double d = (double)im_lerp(ty, tx, g00[o], g01[o], g10[o], g11[o]) - (double)pc[c];
            e += d * d;
        }
        const double md = m, al = q.w;
        acc[0] += md * al;
        acc[1] += md + al - md * al;
        acc[2] += e;
    }
    const double v = block_sum(acc, sPart);
    if (threadIdx.x < IM_SUMS) partials[((int64_t)n * gridDim.x + blockIdx.x) * IM_SUMS + threadIdx.x] = v;
}

// grad_finish_kernel's output rows: view m's (I, U, E, iou_m, psnr_m), then, in the last block, the two means
struct ImageMetricsRows {
    double *per_view;            // (V, 5)
    double *means;               // (2,): mean_n iou_n, mean_n psnr_n
    unsigned int *done;
    double npix;                 // s^2
    __device__ __forceinline__ void operator()(const double *tot, int, int m, int k) const {
        __shared__ double sPart[IM_THREADS / 32][2];
        const int V = gridDim.y;
        if (k == 0) {
            double *row = per_view + (int64_t)m * 5;
            row[0] = tot[0], row[1] = tot[1], row[2] = tot[2];
            row[3] = 1.0 - tot[0] / eps_denom_f64(tot[1]);
            row[4] = tot[2] / npix;
        }
        if (!finish_last_block(done, V)) return;
        // every view's row is written: add them in view order
        double acc[2] = {0.0, 0.0};
        for (int v = k; v < V; v += blockDim.x) {
            acc[0] += __ldcg(per_view + (int64_t)v * 5 + 3);
            acc[1] += __ldcg(per_view + (int64_t)v * 5 + 4);
        }
        const double s = block_sum(acc, sPart);
        if (k < 2) means[k] = s / (double)V;
    }
};

}  // namespace dss

extern "C" {

int dss_image_metrics(dss_ctx *ctx, const float *pred, int s, const float *gt, const int64_t *gt_strides,
                      const void *mask, int mask_kind, int V, int H, int W, double *per_view, double *means,
                      void *stream) {
    using namespace dss;
    cudaStream_t st = (cudaStream_t)stream;
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    DSS_REQUIRE(V >= 1 && V <= 65535 && s >= 1 && H >= 1 && W >= 1, "size out of range");
    DSS_REQUIRE((int64_t)s * s <= (int64_t)INT32_MAX && (int64_t)H * W <= (int64_t)INT32_MAX,
                "more than 2^31-1 pixels per view");
    DSS_REQUIRE(mask_kind == 0 || mask_kind == 1, "mask_kind must be 0 (float32) or 1 (bytes)");
    DSS_REQUIRE(pred && gt && gt_strides && mask && per_view && means, "null pointer");
    DSS_REQUIRE((reinterpret_cast<uintptr_t>(pred) & 15) == 0, "pred must be 16-byte aligned");
    ImageMetricsArgs a;
    a.pred = reinterpret_cast<const float4 *>(pred);
    a.gt = gt;
    for (int d = 0; d < 4; ++d) a.gs[d] = gt_strides[d];
    a.mask = mask;
    a.mask_bytes = mask_kind;
    a.H = H, a.W = W, a.s = s;
    a.scale_y = (float)H / (float)s;
    a.scale_x = (float)W / (float)s;
    // one wave over all views at 4 resident blocks per SM, and no more blocks than the pixels need
    const int64_t ss = (int64_t)s * s;
    const int64_t want = ((int64_t)ctx->sm_count * 4 + V - 1) / V, need = (ss + IM_THREADS - 1) / IM_THREADS;
    const unsigned int blocks = (unsigned int)(want < need ? want : need);
    const size_t np = (size_t)V * blocks * IM_SUMS;
    double *partials = nullptr;
    int rc;
    if ((rc = ctx_get(ctx, BUF_IMAGE_METRICS, np + 1, &partials))) return rc;
    unsigned int *done = reinterpret_cast<unsigned int *>(partials + np);
    image_metrics_partials_kernel<<<dim3(blocks, V), IM_THREADS, 0, st>>>(a, partials, done);
    DSS_LAUNCH_CHECK(ctx);
    ImageMetricsRows rows;
    rows.per_view = per_view, rows.means = means, rows.done = done, rows.npix = (double)ss;
    grad_finish_kernel<IM_SUMS><<<dim3(1, V), 256, 0, st>>>(partials, (int)blocks, V, 1, rows);
    DSS_LAUNCH_CHECK(ctx);
    return DSS_OK;
}

}  // extern "C"
