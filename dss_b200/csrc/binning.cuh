// binning.cuh -- the tile rectangle and packed bin word of a splat, shared by the binning kernels (binning.cu) and the
// preprocess that counts the forward tile lists itself (render.cu).
#pragma once
#include "common.cuh"

namespace dss {

// ---------------------------------------------------------------------------------------------
// Bin range of an interval [p0, p1] -- the reference's closed fp32 predicate
//     (p0 <= b1(b)) && (b0(b) <= p1),   b0(b) = PixToNdc(b*bin) - 1/S,  b1(b) = PixToNdc((b+1)*bin-1) + 1/S
// (DSS/csrc/rasterize_points.cu:355-383) is monotone in b, so the overlapping bins form a contiguous
// range [lo, hi].  We estimate it arithmetically and fix it up with the exact predicate, which makes
// the membership bit-identical to the reference's brute-force loop at O(1) cost.
// ---------------------------------------------------------------------------------------------
// (pix_to_ndc_fast: for a power-of-two S the division-free form is bit-identical to the reference's expression,
//  see common.cuh -- the edges are evaluated up to eight times per splat and axis, the IEEE division dominated the
//  instruction count of both binning kernels)
struct EdgeCtx {
    int bin, S, B;
    float inv_S, half_pix;
};
__device__ __forceinline__ EdgeCtx make_edge_ctx(int bin, int S, int B) {
    EdgeCtx e;
    e.bin = bin;
    e.S = S;
    e.B = B;
    e.inv_S = 1.0f / (float)S;
    e.half_pix = 1.0f / S;
    return e;
}
template <bool POW2>
__device__ __forceinline__ float bin_lo_edge_eval(int b, const EdgeCtx &e) {
    return pix_to_ndc_fast(b * e.bin, e.S, e.inv_S, POW2) - e.half_pix;
}
template <bool POW2>
__device__ __forceinline__ float bin_hi_edge_eval(int b, const EdgeCtx &e) {
    return pix_to_ndc_fast((b + 1) * e.bin - 1, e.S, e.inv_S, POW2) + e.half_pix;
}
template <bool POW2>
__device__ __forceinline__ float bin_lo_edge(int b, const EdgeCtx &e) { return bin_lo_edge_eval<POW2>(b, e); }
template <bool POW2>
__device__ __forceinline__ float bin_hi_edge(int b, const EdgeCtx &e) { return bin_hi_edge_eval<POW2>(b, e); }
// (tried and dropped: the B edges tabulated once per block in shared memory -- the same float values, 12 loads instead
//  of 12 x (IMAD, I2F, FFMA, FADD) per splat: bin_count did not get faster and bin_scatter got slower; the fix-up loops
//  are latency chains either way and the table reads went through generic loads)

template <bool POW2>
__device__ __forceinline__ void bin_range(float p0, float p1, const EdgeCtx &e, int &lo, int &hi) {
    const int B = e.B;
    const float scale = (float)e.S / (2.0f * (float)e.bin);
    // estimates: the bin that contains the end point (exact unless the point sits within rounding of an edge; NaN/inf are
    // handled by the clamps).  The fix-up loops below correct any start in either direction, so the estimate only sets
    // their trip count: two predicate evaluations per bound from here, three from the "one bin outside" start used before
    // (the edge arithmetic is most of bin_count_kernel's instructions)
    float e0 = floorf((p0 + 1.0f) * scale);
    float e1 = floorf((p1 + 1.0f) * scale);
    lo = (e0 >= 0.0f) ? ((e0 < (float)B) ? (int)e0 : B) : 0;          // NaN -> 0
    hi = (e1 >= 0.0f) ? ((e1 < (float)B) ? (int)e1 : B - 1) : -1;    // NaN -> -1
    if (hi > B - 1) hi = B - 1;
    // lo = smallest b with p0 <= b1(b)
    while (lo > 0 && p0 <= bin_hi_edge<POW2>(lo - 1, e)) --lo;
    while (lo < B && !(p0 <= bin_hi_edge<POW2>(lo, e))) ++lo;
    // hi = largest b with b0(b) <= p1
    while (hi < B - 1 && bin_lo_edge<POW2>(hi + 1, e) <= p1) ++hi;
    while (hi >= 0 && !(bin_lo_edge<POW2>(hi, e) <= p1)) --hi;
}

struct BinRect {
    int x0, x1, y0, y1;
    bool empty;
};

template <bool POW2>
__device__ __forceinline__ BinRect splat_bin_rect(const float4 A, const float ry, int bin, int S, int B) {
    BinRect r;
    r.empty = true;
    r.x0 = r.y0 = 0;
    r.x1 = r.y1 = -1;
    if (A.z < 0) return r;  // behind the camera (rasterize_points.cu:351-352); also NaN-safe below
    const float px0 = A.x - A.w, px1 = A.x + A.w;
    const float py0 = A.y - ry, py1 = A.y + ry;
    const EdgeCtx e = make_edge_ctx(bin, S, B);
    bin_range<POW2>(py0, py1, e, r.y0, r.y1);
    if (r.y0 > r.y1) return r;
    bin_range<POW2>(px0, px1, e, r.x0, r.x1);
    if (r.x0 > r.x1) return r;
    r.empty = false;
    return r;
}

// tile rectangle + depth slice of a splat in one register: 7 bits per coordinate (B <= 128), 4 bits of slice
constexpr int BIN_PACK_MAX_B = 128;
constexpr unsigned int BIN_PACK_EMPTY = 0xffffffffu;
__device__ __forceinline__ unsigned int pack_rect(const BinRect &r, int slice) {
    return r.empty ? BIN_PACK_EMPTY
                   : (unsigned int)r.x0 | ((unsigned int)r.x1 << 7) | ((unsigned int)r.y0 << 14) | ((unsigned int)r.y1 << 21) |
                         ((unsigned int)slice << 28);
}

}  // namespace dss
