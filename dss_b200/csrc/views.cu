// views.cu -- the training views resident on the device: gather a batch of views out of one (n_store, H, W, 4) store
// of r, g, b, mask per pixel into the float32 image (B, H, W, 3) and mask (B, H, W) the training step reads.
//
// A byte store holds the 8-bit values the data directory's PNGs hold: rgb = u / 255 (IEEE division, __fdiv_rn, which
// numpy's float32 u / 255.0 also is), mask = (u != 0), the values MVRData.load_all_images / load_all_masks give.  A
// float32 store is copied bit for bit.  One grid row per batch view; when H W % 4 == 0 and every pointer is 16-byte
// aligned, each thread moves four pixels (one 16-byte load from a byte store, four from a float32 one; three float4
// image stores and one float4 mask store), otherwise one.  No atomics, no scratch, no host synchronisation.
#include "common.cuh"

namespace dss {

constexpr int VW_THREADS = 256;

struct Px {
    float r, g, b, m;
};

__device__ __forceinline__ Px vw_pixel(uchar4 u) {
    Px p;
    p.r = __fdiv_rn((float)u.x, 255.0f);
    p.g = __fdiv_rn((float)u.y, 255.0f);
    p.b = __fdiv_rn((float)u.z, 255.0f);
    p.m = u.w != 0 ? 1.0f : 0.0f;
    return p;
}

__device__ __forceinline__ Px vw_pixel(float4 f) {
    Px p;
    p.r = f.x, p.g = f.y, p.b = f.z, p.m = f.w;
    return p;
}

// the four pixels of group g of a view starting at pixel `base`
__device__ __forceinline__ void vw_load4(const uchar4 *store, int64_t base, int64_t g, Px (&p)[4]) {
    const uint4 w = __ldg(reinterpret_cast<const uint4 *>(store + base) + g);
    const unsigned int v[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
    for (int k = 0; k < 4; ++k)
        p[k] = vw_pixel(make_uchar4(v[k] & 0xff, (v[k] >> 8) & 0xff, (v[k] >> 16) & 0xff, v[k] >> 24));
}

__device__ __forceinline__ void vw_load4(const float4 *store, int64_t base, int64_t g, Px (&p)[4]) {
#pragma unroll
    for (int k = 0; k < 4; ++k) p[k] = vw_pixel(__ldg(store + base + 4 * g + k));
}

template <typename T>
__global__ void __launch_bounds__(VW_THREADS) gather_views_vec_kernel(const T *store, const int64_t *idx, int64_t HW,
                                                                      float4 *img, float4 *mask) {
    const int b = blockIdx.y;
    const int64_t src = __ldg(idx + b) * HW, dst4 = (int64_t)b * (HW >> 2);
    for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < (HW >> 2); g += (int64_t)gridDim.x * blockDim.x) {
        Px p[4];
        vw_load4(store, src, g, p);
        float4 *o = img + 3 * (dst4 + g);
        o[0] = make_float4(p[0].r, p[0].g, p[0].b, p[1].r);
        o[1] = make_float4(p[1].g, p[1].b, p[2].r, p[2].g);
        o[2] = make_float4(p[2].b, p[3].r, p[3].g, p[3].b);
        mask[dst4 + g] = make_float4(p[0].m, p[1].m, p[2].m, p[3].m);
    }
}

template <typename T>
__global__ void __launch_bounds__(VW_THREADS) gather_views_kernel(const T *store, const int64_t *idx, int64_t HW,
                                                                  float *img, float *mask) {
    const int b = blockIdx.y;
    const int64_t src = __ldg(idx + b) * HW, dst = (int64_t)b * HW;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += (int64_t)gridDim.x * blockDim.x) {
        const Px p = vw_pixel(__ldg(store + src + i));
        float *o = img + 3 * (dst + i);
        o[0] = p.r, o[1] = p.g, o[2] = p.b;
        mask[dst + i] = p.m;
    }
}

template <typename T>
int gather_views(dss_ctx *ctx, const T *store, int64_t HW, const int64_t *idx, int B, float *img, float *mask,
                 cudaStream_t st) {
    const bool vec = HW % 4 == 0 && ((reinterpret_cast<uintptr_t>(store) | reinterpret_cast<uintptr_t>(img) |
                                      reinterpret_cast<uintptr_t>(mask)) & 15) == 0;
    const int64_t items = vec ? HW / 4 : HW;
    // about 8 resident blocks per SM over the whole batch, and no more blocks per view than its items need
    const int64_t want = ((int64_t)ctx->sm_count * 8 + B - 1) / B, need = (items + VW_THREADS - 1) / VW_THREADS;
    const dim3 grid((unsigned int)(want < need ? want : need), (unsigned int)B);
    if (vec)
        gather_views_vec_kernel<T><<<grid, VW_THREADS, 0, st>>>(store, idx, HW, reinterpret_cast<float4 *>(img),
                                                                reinterpret_cast<float4 *>(mask));
    else
        gather_views_kernel<T><<<grid, VW_THREADS, 0, st>>>(store, idx, HW, img, mask);
    DSS_LAUNCH_CHECK(ctx);
    return DSS_OK;
}

}  // namespace dss

extern "C" {

int dss_gather_views(dss_ctx *ctx, const void *store, int store_f32, int64_t n_store, int H, int W, const int64_t *idx,
                     int B, float *img, float *mask, void *stream) {
    using namespace dss;
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    DSS_REQUIRE(n_store >= 1 && H >= 1 && W >= 1 && B >= 0 && B <= 65535, "size out of range");
    DSS_REQUIRE(store_f32 == 0 || store_f32 == 1, "store_f32 must be 0 (uint8) or 1 (float32)");
    if (B == 0) return DSS_OK;
    DSS_REQUIRE(store && idx && img && mask, "null pointer");
    DSS_REQUIRE((reinterpret_cast<uintptr_t>(store) & (store_f32 ? 15 : 3)) == 0,
                "store must be aligned to its pixel (4 bytes for uint8, 16 for float32)");
    DSS_REQUIRE(((reinterpret_cast<uintptr_t>(img) | reinterpret_cast<uintptr_t>(mask)) & 3) == 0,
                "img and mask must be 4-byte aligned");
    const int64_t HW = (int64_t)H * W;
    cudaStream_t st = (cudaStream_t)stream;
    return store_f32 ? gather_views(ctx, static_cast<const float4 *>(store), HW, idx, B, img, mask, st)
                     : gather_views(ctx, static_cast<const uchar4 *>(store), HW, idx, B, img, mask, st);
}

}  // extern "C"
