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
