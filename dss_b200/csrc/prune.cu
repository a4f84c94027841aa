// prune.cu -- per-point view coverage of one shared cloud seen by N cameras, the evidence the training loop prunes on:
//
//   seen[i]    += sum_n visible[n, i]                                      (in some pixel's K-list of view n)
//   outside[i] += sum_n [z[n, i] > 0 && |x[n, i]|, |y[n, i]| <= 1 && grid_sample(mask_n, -xy[n, i]) == 0]
//
// The second count is a visual-hull test: a point the preprocess kept in view n (z > 0: inside the depth range, and
// facing the camera under backface culling), projected inside the frame, over background of view n's mask.  It is not
// gated on visibility -- a point hidden behind the surface but over background still counts -- while a point off the
// frame or outside the depth range gives no evidence either way.  A non-finite x or y fails |x|, |y| <= 1.  The mask is
// sampled as the point filters sample it (mask_sample.cuh), at the NDC position the render projected the point to.
// One thread per world point sums over the views in registers and adds once to each counter: no atomics, no scratch,
// deterministic, capturable.
#include "mask_sample.cuh"

namespace dss {

constexpr int PC_THREADS = 256;

struct CoverageArgs {
    const float *records;        // (N*P0, 8): x, y, z at [s*8 .. s*8+2] of slot s = n*P0 + i, 16-byte aligned
    const uint8_t *visible;      // (N*P0,)
    MaskSampler m;
    int N;
    int64_t P0;
    int32_t *seen, *outside;     // (P0,), added to
};

__global__ void __launch_bounds__(PC_THREADS) point_coverage_kernel(const __grid_constant__ CoverageArgs a) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.P0; i += (int64_t)gridDim.x * blockDim.x) {
        int seen = 0, outside = 0;
        for (int n = 0; n < a.N; ++n) {
            const int64_t s = n * a.P0 + i;
            seen += a.visible[s] != 0;
            const float4 r = __ldg(reinterpret_cast<const float4 *>(a.records + s * 8));
            outside += r.z > 0.f && fabsf(r.x) <= 1.f && fabsf(r.y) <= 1.f && !pf_in_mask(a.m, n, r.x, r.y);
        }
        a.seen[i] += seen;
        a.outside[i] += outside;
    }
}

}  // namespace dss

extern "C" {

int dss_point_coverage(dss_ctx *ctx, const float *records, const uint8_t *visible, int shared_cloud, int N, int64_t P0,
                       const void *mask, int mask_kind, const int64_t *mask_strides, int H, int W, int32_t *seen,
                       int32_t *outside, void *stream) {
    using namespace dss;
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    DSS_REQUIRE(shared_cloud == 1, "the view coverage takes a shared cloud (one cloud seen by N cameras)");
    DSS_REQUIRE(N >= 1 && N <= DSS_MAX_SHARED_VIEWS && P0 >= 0, "size out of range");
    CoverageArgs a;
    int rc = make_mask_sampler(mask, mask_kind, mask_strides, H, W, &a.m);
    if (rc) return rc;
    if (P0 == 0) return DSS_OK;
    DSS_REQUIRE(records && visible && mask && mask_strides && seen && outside, "null pointer");
    DSS_REQUIRE((reinterpret_cast<uintptr_t>(records) & 15) == 0, "records must be 16-byte aligned");
    a.records = records, a.visible = visible, a.N = N, a.P0 = P0, a.seen = seen, a.outside = outside;
    point_coverage_kernel<<<grid_blocks(P0, PC_THREADS, ctx->sm_count, 8), PC_THREADS, 0, (cudaStream_t)stream>>>(a);
    DSS_LAUNCH_CHECK(ctx);
    return DSS_OK;
}

}  // extern "C"
