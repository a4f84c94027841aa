// backward.cu -- visibility, z-buffer and colour scatters (the occupancy gather lives in occ_backward.cu).
#include <math_constants.h>

#include "common.cuh"
#include "kernels.cuh"

namespace dss {

// ---------------------------------------------------------------------------------------------
// visibility (rasterizer.py:854-860): any slot of a pixel whose first slot is occupied.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
visibility_kernel(const int32_t *__restrict__ idx, int64_t num_pixels, int K, int64_t P,
                  uint8_t *__restrict__ visible) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < num_pixels;
         i += (int64_t)gridDim.x * blockDim.x) {
        const int32_t *row = idx + i * K;
        if (row[0] < 0) continue;
        for (int k = 0; k < K; ++k) {
            const int p = row[k];
            if (p >= 0 && p < P) visible[p] = 1;
        }
    }
}

int visibility_from_idx(dss_ctx *ctx, const int32_t *idx, int64_t num_pixels, int K, int64_t P,
                        uint8_t *visible, cudaStream_t st) {
    DSS_CUDA_TRY(cudaMemsetAsync(visible, 0, (size_t)(P > 0 ? P : 0), st));
    if (num_pixels == 0 || P == 0) return DSS_OK;
    StageScope prof(ctx, ST_VISIBILITY, st);
    visibility_kernel<<<grid_blocks(num_pixels, 256, ctx->sm_count, 16), 256, 0, st>>>(idx, num_pixels, K, P, visible);
    DSS_LAUNCH_CHECK(ctx);
    return DSS_OK;
}

// ---------------------------------------------------------------------------------------------
// z-buffer backward (rasterize_points.cu:823-846).  z_grad element stride in floats (1 for (P,),
// 3 to write the z column of a (P,3) gradient).
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
zbuf_backward_kernel(const int32_t *__restrict__ idx, const float *__restrict__ grad_zbuf, int64_t num_pixels,
                     int K, float *z_grad, int z_stride) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < num_pixels;
         i += (int64_t)gridDim.x * blockDim.x) {
        for (int k = 0; k < K; ++k) {
            const float g = grad_zbuf[i * K + k];
            if (g == 0.0f) continue;
            const int p = idx[i * K + k];
            if (p < 0) break;
            atomicAdd(z_grad + (int64_t)p * z_stride, g);
        }
    }
}

int zbuf_backward(dss_ctx *ctx, const int32_t *idx, const float *grad_zbuf, int64_t num_pixels, int K,
                  float *z_grad, int z_stride, cudaStream_t st) {
    if (num_pixels == 0) return DSS_OK;
    StageScope prof(ctx, ST_ZBUF_BWD, st);
    zbuf_backward_kernel<<<grid_blocks(num_pixels, 256, ctx->sm_count, 16), 256, 0, st>>>(idx, grad_zbuf, num_pixels,
                                                                                      K, z_grad, z_stride);
    DSS_LAUNCH_CHECK(ctx);
    return DSS_OK;
}

// ---------------------------------------------------------------------------------------------
// Colour backward: dL/dcolour[idx_k] += g_rgb * w_k / max(sum w, 1e-4)  (norm_weighted_sum backward [ext]);
// `weights` already holds the normalised weights written by the forward pass.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
colour_backward_kernel(const int32_t *__restrict__ idx, const float *__restrict__ weights,
                       const float4 *__restrict__ grad_image, int64_t num_pixels, int K,
                       float *grad_colours, int64_t colour_P0, int64_t pixels_per_view) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < num_pixels;
         i += (int64_t)gridDim.x * blockDim.x) {
        if (idx[i * K] < 0) continue;
        const float4 g = __ldg(&grad_image[i]);
        if (g.x == 0.0f && g.y == 0.0f && g.z == 0.0f) continue;
        for (int k = 0; k < K; ++k) {
            const int p = idx[i * K + k];
            if (p < 0) break;
            const float w = weights[i * K + k];
            float *dst = grad_colours + ((int64_t)p - (colour_P0 > 0 ? (i / pixels_per_view) * colour_P0 : 0)) * 3;
            atomicAdd(dst + 0, g.x * w);
            atomicAdd(dst + 1, g.y * w);
            atomicAdd(dst + 2, g.z * w);
        }
    }
}

// Deterministic colour backward of per-record colours (the shading's d L / d shaded scratch, one row per (view, point)
// record): the same products g * w_k, summed in 64-bit fixed point, where integer atomics give the same bits in any
// order.  One scale 2^e per call: G is the largest finite |g| of the image gradient's rgb (one pass over the pixels),
// and a record gathers at most one term per pixel of its view, each |g * w_k| <= G (w_k <= 1), so with
// e = 62 - exponent(G * pixels_per_view) every sum stays below 2^62 in magnitude.  Each term is rounded to the nearest
// integer once: the error of a record is at most (its terms / 2) * G * pixels_per_view * 2^-62, about 2^-45 G per term at
// 512^2.  The finish writes sum * 2^-e.  A non-finite term is added to the float output with float atomics instead:
// its NaN or infinity does not depend on the order, and the finish leaves such entries as they are.
__global__ void __launch_bounds__(256)
colour_gmax_kernel(const float4 *__restrict__ grad_image, int64_t num_pixels, int *__restrict__ gmax) {
    int m = 0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < num_pixels;
         i += (int64_t)gridDim.x * blockDim.x) {
        const float4 g = __ldg(&grad_image[i]);
        m = max(m, max(finite_abs_bits(g.x), max(finite_abs_bits(g.y), finite_abs_bits(g.z))));
    }
    m = __reduce_max_sync(0xffffffffu, m);
    if ((threadIdx.x & 31) == 0 && m > 0) atomicMax(gmax, m);
}

__global__ void __launch_bounds__(256)
colour_fixed_kernel(const int32_t *__restrict__ idx, const float *__restrict__ weights,
                    const float4 *__restrict__ grad_image, int64_t num_pixels, int K, int64_t pixels_per_view,
                    const int *__restrict__ gmax, unsigned long long *__restrict__ acc, float *__restrict__ grad_colours) {
    const int e = colour_fixed_exp(gmax, pixels_per_view);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < num_pixels;
         i += (int64_t)gridDim.x * blockDim.x) {
        if (idx[i * K] < 0) continue;
        const float4 g = __ldg(&grad_image[i]);
        if (g.x == 0.0f && g.y == 0.0f && g.z == 0.0f) continue;
        for (int k = 0; k < K; ++k) {
            const int p = idx[i * K + k];
            if (p < 0) break;
            const float w = weights[i * K + k];
            const float v[3] = {g.x * w, g.y * w, g.z * w};
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                if (isfinite(v[c]))
                    atomicAdd(&acc[(int64_t)p * 3 + c], (unsigned long long)__float2ll_rn(ldexpf(v[c], e)));
                else
                    atomicAdd(&grad_colours[(int64_t)p * 3 + c], v[c]);
            }
        }
    }
}

__global__ void __launch_bounds__(256)
colour_fixed_finish_kernel(const unsigned long long *__restrict__ acc, int64_t n, int64_t pixels_per_view,
                           const int *__restrict__ gmax, float *__restrict__ grad_colours) {
    const int e = colour_fixed_exp(gmax, pixels_per_view);
    for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (int64_t)gridDim.x * blockDim.x)
        if (isfinite(grad_colours[j])) grad_colours[j] = (float)ldexp((double)(long long)acc[j], -e);
}

int colour_backward_fixed(dss_ctx *ctx, const int32_t *idx, const float *weights, const float *grad_image,
                          int64_t num_pixels, int K, float *grad_colours, int64_t P, int64_t pixels_per_view,
                          cudaStream_t st) {
    DSS_CUDA_TRY(cudaMemsetAsync(grad_colours, 0, (size_t)P * 3 * sizeof(float), st));
    if (num_pixels == 0 || P == 0) return DSS_OK;
    unsigned long long *acc = nullptr;      // (P,3) sums, then the int bits of G
    int rc;
    if ((rc = ctx_get(ctx, BUF_COLOUR_FIXED, (size_t)P * 3 + 1, &acc))) return rc;
    int *gmax = reinterpret_cast<int *>(acc + P * 3);
    DSS_CUDA_TRY(cudaMemsetAsync(acc, 0, ((size_t)P * 3 + 1) * sizeof(unsigned long long), st));
    StageScope prof(ctx, ST_COLOUR_BWD, st);
    const unsigned blocks = grid_blocks(num_pixels, 256, ctx->sm_count, 16);
    const float4 *g = reinterpret_cast<const float4 *>(grad_image);
    colour_gmax_kernel<<<blocks, 256, 0, st>>>(g, num_pixels, gmax);
    DSS_LAUNCH_CHECK(ctx);
    colour_fixed_kernel<<<blocks, 256, 0, st>>>(idx, weights, g, num_pixels, K, pixels_per_view, gmax, acc,
                                                grad_colours);
    DSS_LAUNCH_CHECK(ctx);
    colour_fixed_finish_kernel<<<grid_blocks(P * 3, 256, ctx->sm_count, 8), 256, 0, st>>>(acc, P * 3, pixels_per_view,
                                                                                         gmax, grad_colours);
    DSS_LAUNCH_CHECK(ctx);
    return DSS_OK;
}

int colour_backward(dss_ctx *ctx, const int32_t *idx, const float *weights, const float *grad_image,
                    int64_t num_pixels, int K, float *grad_colours, int64_t colour_P0, int64_t pixels_per_view,
                    cudaStream_t st) {
    if (num_pixels == 0) return DSS_OK;
    StageScope prof(ctx, ST_COLOUR_BWD, st);
    colour_backward_kernel<<<grid_blocks(num_pixels, 256, ctx->sm_count, 16), 256, 0, st>>>(
        idx, weights, reinterpret_cast<const float4 *>(grad_image), num_pixels, K, grad_colours, colour_P0, pixels_per_view);
    DSS_LAUNCH_CHECK(ctx);
    return DSS_OK;
}

}  // namespace dss

extern "C" {

int dss_visibility_from_idx(dss_ctx *ctx, const int32_t *idx, int64_t num_pixels, int K, int64_t P,
                            uint8_t *visible, void *stream) {
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    DSS_REQUIRE(num_pixels >= 0 && K > 0 && P >= 0, "bad size");
    DSS_REQUIRE((num_pixels == 0 || idx) && (P == 0 || visible), "null pointer");
    return dss::visibility_from_idx(ctx, idx, num_pixels, K, P, visible, (cudaStream_t)stream);
}

int dss_zbuf_backward(dss_ctx *ctx, const int32_t *idx, const float *grad_zbuf, int64_t num_pixels, int K,
                      float *z_grad, void *stream) {
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    DSS_REQUIRE(num_pixels >= 0 && K > 0, "bad size");
    if (num_pixels == 0) return DSS_OK;
    DSS_REQUIRE(idx && grad_zbuf && z_grad, "null pointer");
    return dss::zbuf_backward(ctx, idx, grad_zbuf, num_pixels, K, z_grad, 1, (cudaStream_t)stream);
}

}  // extern "C"
