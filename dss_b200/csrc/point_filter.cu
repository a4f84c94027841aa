// point_filter.cu -- the point filters of the training step for one shared cloud seen by N cameras
// (Model.forward, DSS/models/point_modeling.py:172-173, 188-212):
//
//   visibility[i] = any_n visible[n, i]
//   inmask[i]     = visibility[i] && any_n (grid_sample(mask_n, clamp(-xy[n, i], -1, 1)) != 0)
//
// The masks are sampled by mask_sample.cuh (torch's grid_sample, bilinear, reflection padding, align_corners=False).
// x, y are the NDC positions the forward's preprocess wrote into the records: the filter samples where the render
// projected.  A non-finite x or y (a point on the camera plane, a NaN input) is outside the mask and never indexes it.
// One thread per world point ORs over the views in registers: one launch, no atomics, no scratch, deterministic.
// View-sharded (each rank holds some of the views): the visibility gate is the visibility ORed over all ranks, and
// replaces this call's own; inmask ORed over the ranks is then the filter of all views.
#include "mask_sample.cuh"

namespace dss {

constexpr int PF_THREADS = 256;

struct PointFilterArgs {
    const float *records;        // (N*P0, 8): x, y at [s*8], [s*8+1] of slot s = n*P0 + i
    const uint8_t *visible;      // (N*P0,)
    MaskSampler m;
    int N;
    int64_t P0;
    const uint8_t *gate;            // (P0,) visibility over all ranks, or nullptr: this call's views decide
    uint8_t *visibility, *inmask;   // (P0,)
};

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
            in = pf_in_mask(a.m, n, xy.x, xy.y);
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
    PointFilterArgs a;
    int rc = make_mask_sampler(mask, mask_kind, mask_strides, H, W, &a.m);
    if (rc) return rc;
    if (P0 == 0) return DSS_OK;
    DSS_REQUIRE(records && visible && mask && mask_strides && visibility && inmask, "null pointer");
    DSS_REQUIRE((reinterpret_cast<uintptr_t>(records) & 7) == 0, "records must be 8-byte aligned");
    a.records = records, a.visible = visible;
    a.N = N, a.P0 = P0, a.gate = gate, a.visibility = visibility, a.inmask = inmask;
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
