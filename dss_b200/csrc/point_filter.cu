// point_filter.cu -- the point filters of the training step for one shared cloud seen by N cameras
// (Model.forward, DSS/models/point_modeling.py:172-173, 188-212):
//
//   visibility[i] = any_n visible[n, i]
//   inmask[i]     = visibility[i] && any_n (grid_sample(mask_n, clamp(-xy[n, i], -1, 1)) != 0)
//
// grid_sample is bilinear with padding_mode='reflection' and align_corners=False (DSS/utils/__init__.py:266-300); its
// coordinate and tap arithmetic is restated below in ATen's order (GridSampler.cuh: unnormalize, reflect, clip, then the
// nw, ne, sw, se taps, each skipped when out of bounds), so a sample is zero exactly when the reference's is.  x, y are
// the NDC positions the forward's preprocess wrote into the records: the filter samples where the render projected.
// A non-finite x or y (a point on the camera plane, a NaN input) is outside the mask and never indexes it.
// One thread per world point ORs over the views in registers: one launch, no atomics, no scratch, deterministic.
// View-sharded (each rank holds some of the views): the visibility gate is the visibility ORed over all ranks, and
// replaces this call's own; inmask ORed over the ranks is then the filter of all views.
#include "common.cuh"

namespace dss {

constexpr int PF_THREADS = 256;

struct PointFilterArgs {
    const float *records;        // (N*P0, 8): x, y at [s*8], [s*8+1] of slot s = n*P0 + i
    const uint8_t *visible;      // (N*P0,)
    const void *mask;            // mask_n(y, x) at mask[n*ms[0] + y*ms[1] + x*ms[2]], float32 or bytes
    int64_t ms[3];
    int mask_bytes;
    int N, H, W;
    int64_t P0;
    const uint8_t *gate;            // (P0,) visibility over all ranks, or nullptr: this call's views decide
    uint8_t *visibility, *inmask;   // (P0,)
};

__device__ __forceinline__ float pf_mask(const PointFilterArgs &a, int n, int y, int x) {
    const int64_t o = n * a.ms[0] + (int64_t)y * a.ms[1] + (int64_t)x * a.ms[2];
    return a.mask_bytes ? (float)static_cast<const uint8_t *>(a.mask)[o] : static_cast<const float *>(a.mask)[o];
}

// grid_sampler_compute_source_index for align_corners=False, reflection padding, a finite coordinate in [-1, 1]
__device__ __forceinline__ float pf_source_index(float coord, int size) {
    coord = ((coord + 1.f) * size - 1) / 2;
    const float lo = -0.5f, span = (float)size;
    const float in = fabsf(coord - lo);
    const float extra = fmodf(in, span);
    const int flips = (int)floorf(in / span);
    coord = (flips % 2 == 0) ? extra + lo : span - extra + lo;
    return fminf((float)(size - 1), fmaxf(coord, 0.f));
}

__device__ __forceinline__ bool pf_in_mask(const PointFilterArgs &a, int n, float x, float y) {
    if (!isfinite(x) || !isfinite(y)) return false;
    // p = -xy (NDC +X left, +Y up), clamped like torch.clamp(-1, 1); grid x indexes W, grid y indexes H
    const float ix = pf_source_index(fminf(fmaxf(-x, -1.f), 1.f), a.W);
    const float iy = pf_source_index(fminf(fmaxf(-y, -1.f), 1.f), a.H);
    const int ix_nw = (int)floorf(ix), iy_nw = (int)floorf(iy);
    const int ix_ne = ix_nw + 1, iy_ne = iy_nw;
    const int ix_sw = ix_nw, iy_sw = iy_nw + 1;
    const int ix_se = ix_nw + 1, iy_se = iy_nw + 1;
    const float nw = (ix_se - ix) * (iy_se - iy);
    const float ne = (ix - ix_sw) * (iy_sw - iy);
    const float sw = (ix_ne - ix) * (iy - iy_ne);
    const float se = (ix - ix_nw) * (iy - iy_nw);
    auto inb = [&](int yy, int xx) { return yy >= 0 && yy < a.H && xx >= 0 && xx < a.W; };
    float acc = 0.f;
    if (inb(iy_nw, ix_nw)) acc += pf_mask(a, n, iy_nw, ix_nw) * nw;
    if (inb(iy_ne, ix_ne)) acc += pf_mask(a, n, iy_ne, ix_ne) * ne;
    if (inb(iy_sw, ix_sw)) acc += pf_mask(a, n, iy_sw, ix_sw) * sw;
    if (inb(iy_se, ix_se)) acc += pf_mask(a, n, iy_se, ix_se) * se;
    return acc != 0.f;
}

__global__ void __launch_bounds__(PF_THREADS) point_filter_kernel(const __grid_constant__ PointFilterArgs a) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.P0; i += (int64_t)gridDim.x * blockDim.x) {
        bool vis = false;
        if (a.gate)
            vis = a.gate[i] != 0;
        else
            for (int n = 0; n < a.N && !vis; ++n) vis = a.visible[n * a.P0 + i] != 0;
        bool in = false;
        // inmask is false wherever visibility is: the masks are only sampled for visible points
        for (int n = 0; vis && n < a.N && !in; ++n) {
            const float2 xy = __ldg(reinterpret_cast<const float2 *>(a.records + (n * a.P0 + i) * 8));
            in = pf_in_mask(a, n, xy.x, xy.y);
        }
        a.visibility[i] = vis;
        a.inmask[i] = in;
    }
}

static int pf_launch(dss_ctx *ctx, const float *records, const uint8_t *visible, int shared_cloud, int N, int64_t P0,
                     const void *mask, int mask_kind, const int64_t *mask_strides, int H, int W, const uint8_t *gate,
                     uint8_t *visibility, uint8_t *inmask, void *stream) {
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    DSS_REQUIRE(shared_cloud == 1, "the point filters take a shared cloud (one cloud seen by N cameras)");
    DSS_REQUIRE(N >= 1 && N <= DSS_MAX_SHARED_VIEWS && P0 >= 0, "size out of range");
    DSS_REQUIRE(H >= 1 && W >= 1, "mask size out of range");
    DSS_REQUIRE(mask_kind == 0 || mask_kind == 1, "mask_kind must be 0 (float32) or 1 (bytes)");
    if (P0 == 0) return DSS_OK;
    DSS_REQUIRE(records && visible && mask && mask_strides && visibility && inmask, "null pointer");
    DSS_REQUIRE((reinterpret_cast<uintptr_t>(records) & 7) == 0, "records must be 8-byte aligned");
    PointFilterArgs a;
    a.records = records, a.visible = visible, a.mask = mask, a.mask_bytes = mask_kind;
    for (int d = 0; d < 3; ++d) a.ms[d] = mask_strides[d];
    a.N = N, a.H = H, a.W = W, a.P0 = P0, a.gate = gate, a.visibility = visibility, a.inmask = inmask;
    point_filter_kernel<<<grid_blocks(P0, PF_THREADS, ctx->sm_count, 8), PF_THREADS, 0, (cudaStream_t)stream>>>(a);
    DSS_LAUNCH_CHECK(ctx);
    return DSS_OK;
}

}  // namespace dss

extern "C" {

int dss_point_filters(dss_ctx *ctx, const float *records, const uint8_t *visible, int shared_cloud, int N, int64_t P0,
                      const void *mask, int mask_kind, const int64_t *mask_strides, int H, int W, uint8_t *visibility,
                      uint8_t *inmask, void *stream) {
    return dss::pf_launch(ctx, records, visible, shared_cloud, N, P0, mask, mask_kind, mask_strides, H, W, nullptr,
                          visibility, inmask, stream);
}

int dss_point_filters_gated(dss_ctx *ctx, const float *records, const uint8_t *visible, int shared_cloud, int N,
                            int64_t P0, const void *mask, int mask_kind, const int64_t *mask_strides, int H, int W,
                            const uint8_t *visibility_gate, uint8_t *visibility, uint8_t *inmask, void *stream) {
    return dss::pf_launch(ctx, records, visible, shared_cloud, N, P0, mask, mask_kind, mask_strides, H, W,
                          visibility_gate, visibility, inmask, stream);
}

}  // extern "C"
