// mask_sample.cuh -- the ground-truth mask sample of the point filters (point_filter.cu) and the view coverage
// (prune.cu): torch's grid_sample(mask_n, clamp(-xy, -1, 1)), bilinear with padding_mode='reflection' and
// align_corners=False (DSS/utils/__init__.py:266-300), its coordinate and tap arithmetic restated in ATen's order
// (GridSampler.cuh: unnormalize, reflect, clip, then the nw, ne, sw, se taps, each skipped when out of bounds), so a
// sample is zero exactly when the reference's is.
#pragma once
#include "common.cuh"

namespace dss {

struct MaskSampler {
    const void *mask;            // mask_n(y, x) at mask[n*ms[0] + y*ms[1] + x*ms[2]], float32 or bytes
    int64_t ms[3];
    int mask_bytes;
    int H, W;
};

__device__ __forceinline__ float pf_mask(const MaskSampler &a, int n, int y, int x) {
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

// whether mask n samples non-zero at the record position (x, y); a non-finite x or y (a point on the camera plane, a
// NaN input) is outside the mask and never indexes it
__device__ __forceinline__ bool pf_in_mask(const MaskSampler &a, int n, float x, float y) {
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

// the MaskSampler of a C-ABI call's mask arguments, checked
static inline int make_mask_sampler(const void *mask, int mask_kind, const int64_t *mask_strides, int H, int W,
                                    MaskSampler *m) {
    DSS_REQUIRE(H >= 1 && W >= 1, "mask size out of range");
    DSS_REQUIRE(mask_kind == 0 || mask_kind == 1, "mask_kind must be 0 (float32) or 1 (bytes)");
    m->mask = mask, m->mask_bytes = mask_kind, m->H = H, m->W = W;
    for (int d = 0; d < 3; ++d) m->ms[d] = mask_strides ? mask_strides[d] : 0;
    return DSS_OK;
}

}  // namespace dss
