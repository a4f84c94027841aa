// kernels.cuh -- host-side entry points shared between the translation units of libdss_b200.
#pragma once
#include "common.cuh"

namespace dss {

constexpr int RASTER_TILE = 16;  // pixels per side of a raster tile (one 256-thread CTA)

// Cells of the occupancy backward's binning: the pixels of 32x32-pixel tiles, a view's tiles row-major (OB = occ_tiles(S)
// per side), 1024 cells per tile, row-major inside the tile.  A splat belongs to the cell of its centre pixel.  The
// forward's blend epilogue counts the visible splats per cell (RasterArgs::cell_counts) and the backward's binning claims
// its slots by counting those counts back down: both must put a splat in the same cell, so both use these functions.
constexpr int OCC_TILE_SHIFT = 5;
constexpr int OCC_TILE = 1 << OCC_TILE_SHIFT;      // pixels per side of a backward tile
constexpr int OCC_CELLS = OCC_TILE * OCC_TILE;     // cells per tile

__host__ __device__ __forceinline__ int occ_tiles(int S) { return (S + OCC_TILE - 1) >> OCC_TILE_SHIFT; }
// counters of the binning (and length of dss_render_args::cell_counts) for N views of S x S pixels
inline int64_t occ_cell_count(int N, int S) { return (int64_t)N * occ_tiles(S) * occ_tiles(S) * OCC_CELLS; }

// centre pixel of NDC coordinate p, clamped to the image
__device__ __forceinline__ int centre_pixel(float p, int S) {
    return min(max((int)floorf((p + 1.0f) * (0.5f * (float)S)), 0), S - 1);
}
// global cell of pixel (cx, cy) of view n (cx, cy >= 0, as centre_pixel returns them)
__device__ __forceinline__ int64_t occ_cell(int n, int OB, int cx, int cy) {
    return (((int64_t)n * OB + (cy >> OCC_TILE_SHIFT)) * OB + (cx >> OCC_TILE_SHIFT)) * OCC_CELLS +
           (cy & (OCC_TILE - 1)) * OCC_TILE + (cx & (OCC_TILE - 1));
}

// Small device -> host read-back WITHOUT the copy engine: a one-block kernel stores the words straight into pinned,
// device-mapped host memory.  A cudaMemcpyAsync would queue behind whatever large D2H copy another stream has in
// flight (copies of one direction are served in order) and, being in stream order, stall every kernel enqueued
// after it, e.g. in bench.py's end-to-end loop while the previous step's image is read back.
int publish_words(dss_ctx *ctx, const void *src_device, void *dst_pinned_host, int n_words, cudaStream_t st);

int exclusive_scan_i32(dss_ctx *ctx, const int32_t *in, int32_t *out, int64_t n, cudaStream_t st);

// 64-bit exclusive scan of v[0, n) in place; the total goes to v[n] (v holds n + 1 entries).  tile_sums: scratch of
// scan_i64_tiles(n) entries.  Three launches, no host synchronisation.
int64_t scan_i64_tiles(int64_t n);
int exclusive_scan_i64(dss_ctx *ctx, int64_t *v, int64_t n, int64_t *tile_sums, cudaStream_t st);

int pack_records(dss_ctx *ctx, const float *points, const float *radii, const float *ellipse, int64_t P,
                 float4 *rec, cudaStream_t st);

int choose_depth_slices(int B);
int init_zrange(dss_ctx *ctx, float *zrange, int N, cudaStream_t st);
int compute_zrange(dss_ctx *ctx, const float4 *rec, const int64_t *first_idx, const int64_t *num_points, int N,
                   int64_t P0, float *zrange, cudaStream_t st);

// rects (optional, one word per packed splat): the count pass stores every splat's tile rectangle + depth slice there and
// the scatter pass, given the same array, reuses them instead of deriving them again from the records
int bin_count_and_scan(dss_ctx *ctx, const float4 *rec, const int64_t *first_idx, const int64_t *num_points,
                       int N, int64_t P0, int S, int bin, int NS, const float *zrange, int32_t *counts,
                       int32_t *offsets, unsigned int *rects, cudaStream_t st);

int bin_scatter(dss_ctx *ctx, const float4 *rec, const int64_t *first_idx, const int64_t *num_points, int N,
                int64_t P0, int S, int bin, int NS, const float *zrange, const int32_t *offsets, int32_t *cursors,
                int32_t *ids, int64_t ids_capacity, const unsigned int *rects, cudaStream_t st);

// Threads per block of the preprocess.  The fused route's scatter (bin_scatter_counted) runs on the preprocess's grid
// and partition of the splats, so both use this.
constexpr int PREPROCESS_THREADS = 256;

// Tile lists that the preprocess counted (dss_render_forward): counts already hold the per-(view, tile, slice) sizes,
// rects the packed rectangle of every splat, block_offsets (N, blocks, B*B*NS) the offset of every preprocess block
// inside each bin it touched.
struct CountedBins {
    const unsigned int *rects;
    const int32_t *block_offsets;
    unsigned int blocks;   // preprocess blocks per view
};
int bin_scatter_counted(dss_ctx *ctx, const int64_t *first_idx, const int64_t *num_points, int N, int64_t P0, int B,
                        int NS, const int32_t *offsets, const int32_t *block_offsets, unsigned int blocks,
                        const unsigned int *rects, int32_t *ids, int64_t ids_capacity, cudaStream_t st);

// Tile grid and depth slices of the forward lists for N views of S x S pixels and K points per pixel; packed: the lists
// can be binned with per-block histograms and the packed rectangle word (B <= 128, <= 16 slices, histogram <= 192 KB, and
// neither DSS_BIN_DIRECT nor DSS_BIN_NORECTS).  Fails when the N*B*B*NS bins do not fit the int32 offsets.
struct TilePlan {
    int B, NS;
    bool packed;
};
int plan_tiles(dss_ctx *ctx, int N, int S, int K, TilePlan *plan);

// Depth slicing shared by the binning and raster kernels (identical arithmetic on both sides).
struct SliceMap {
    float zmin, dz, inv_dz;
    int NS;
};
__device__ __forceinline__ float slice_bound(const SliceMap &m, int s) { return fmaf((float)s, m.dz, m.zmin); }
__device__ __forceinline__ SliceMap make_slice_map(const float *zrange, int n, int NS) {
    SliceMap m;
    m.NS = NS;
    m.zmin = 0.f;
    m.dz = 0.f;
    m.inv_dz = 0.f;
    if (NS > 1 && zrange) {
        const float z0 = zrange[2 * n], z1 = zrange[2 * n + 1];
        if (z1 > z0) {
            m.zmin = z0;
            m.dz = (z1 - z0) / (float)NS;
            m.inv_dz = 1.0f / m.dz;
        }
    }
    return m;
}
// slice index with slice_bound(slice) <= z guaranteed (estimate + exact fix-up)
__device__ __forceinline__ int depth_slice(const SliceMap &m, float z) {
    if (m.NS <= 1 || !(m.dz > 0.f)) return 0;
    int s = (int)((z - m.zmin) * m.inv_dz);
    s = max(0, min(m.NS - 1, s));
    while (s > 0 && z < slice_bound(m, s)) --s;
    while (s < m.NS - 1 && z >= slice_bound(m, s + 1)) ++s;
    return s;
}

struct RasterArgs {
    const float4 *rec;        // 2 per splat
    const float *cutoff;      // per point (P,) or nullptr -> cutoff_uniform
    float cutoff_uniform;
    const int32_t *tile_offsets;  // (N*B*B + 1)
    const int32_t *tile_ids;      // CSR payload: packed splat ids
    const int32_t *tile_order;    // launch order of the tiles (longest lists first) or nullptr: block b = tile b
    int ids_capacity;             // entries tile_ids can hold; a tile whose list does not fit is rasterized from the
                                  // view's records directly (see bin_and_raster)
    const int64_t *first_idx;     // packed layout of the views (nullptr: shared cloud, view n = [n*P0, (n+1)*P0))
    const int64_t *num_points;
    int64_t P0;
    int N, S, K, B;
    int NS;                       // depth slices per tile list
    const float *zrange;          // (N,2) depth range per view (NS > 1)
    float depth_merge;
    // outputs
    int32_t *idx;
    float *zbuf;     // may be null
    float *qvalue;   // may be null
    float *occ;      // may be null (N,S,S)
    // blend (all null when not blending)
    const float *scaler;   // (P,)
    const float *colours;  // (P,3), or (P0,3) shared by every view when colour_P0 > 0
    int64_t colour_P0;     // > 0: colour row of packed splat id in view n is id - n * colour_P0
    float *image;          // (N,S,S,4)
    float *weights;        // (N,S,S,K)
    int32_t *cell_counts;  // optional (occ_cell_count(N, S),), zeroed by the caller: the blend epilogue counts every visible
                           // splat once in its cell (occ_cell; the count pass of the occupancy backward's binning, fused);
                           // needs `visible` 4-byte aligned with capacity rounded up to 4
    uint8_t *visible;      // (P,) must be zeroed by the caller
    unsigned long long *stats; // optional debug counters (dss_debug_raster_stats) or nullptr
};

int raster_forward(dss_ctx *ctx, const RasterArgs &a, cudaStream_t st);

// bin + rasterize, shared by dss_splat_points and dss_render_forward.  Synchronises once.  counted: the preprocess
// already counted the lists (the plan_tiles plan of this call, packed) and a.zrange holds the depth ranges; null: count
// here.
int bin_and_raster(dss_ctx *ctx, RasterArgs a, const int64_t *first_idx, const int64_t *num_points,
                   int64_t P0, cudaStream_t st, const CountedBins *counted = nullptr);

int visibility_from_idx(dss_ctx *ctx, const int32_t *idx, int64_t num_pixels, int K, int64_t P,
                        uint8_t *visible, cudaStream_t st);
int search_radius(dss_ctx *ctx, const float4 *rec, const float *radii, const uint8_t *visible,
                  const int64_t *first_idx, const int64_t *num_points, int N, int64_t P0, float radii_s,
                  float *rs, cudaStream_t st);
// rs is an input when radii_s < 0, otherwise rs[n] = radii_s * lower median of the visible radii is computed here
// cell_counts (optional): per-cell counts of the visible splats produced by the forward (RasterArgs::cell_counts); when
// given and the staged gather runs, the counting pass is replaced by a copy of these counts
int occ_backward(dss_ctx *ctx, const float4 *rec, const uint8_t *visible, float *rs, float radii_s,
                 const float *grad_occ, int pix_stride, int pix_offset, const int64_t *first_idx,
                 const int64_t *num_points, int N, int64_t P0, int S, float *grad_xy, const int32_t *cell_counts,
                 cudaStream_t st);
int zbuf_backward(dss_ctx *ctx, const int32_t *idx, const float *grad_zbuf, int64_t num_pixels, int K,
                  float *z_grad, int z_stride, cudaStream_t st);
// colour_P0 > 0: grad_colours is (P0,3) shared by the views (pixels_per_view = S*S locates a pixel's view)
int colour_backward(dss_ctx *ctx, const int32_t *idx, const float *weights, const float *grad_image,
                    int64_t num_pixels, int K, float *grad_colours, int64_t colour_P0, int64_t pixels_per_view,
                    cudaStream_t st);
// per-record colours (P,3) of views of pixels_per_view pixels, deterministic: 64-bit fixed-point sums (backward.cu);
// zeroes grad_colours first
int colour_backward_fixed(dss_ctx *ctx, const int32_t *idx, const float *weights, const float *grad_image,
                          int64_t num_pixels, int K, float *grad_colours, int64_t P, int64_t pixels_per_view,
                          cudaStream_t st);

// Scale 2^e of a 64-bit fixed-point sum whose terms are at most G in magnitude, at most pixels_per_view of them per
// sum (gmax: the int bits of G): every sum stays below 2^62 in magnitude (see colour_backward_fixed in backward.cu)
__device__ __forceinline__ int colour_fixed_exp(const int *gmax, int64_t pixels_per_view) {
    int x;
    frexp((double)__int_as_float(*gmax) * (double)pixels_per_view, &x);
    return 62 - x;
}

__device__ __forceinline__ int finite_abs_bits(float v) { return isfinite(v) ? __float_as_int(fabsf(v)) : 0; }

// depth.cu: the blend's depth map D = sum_k w_k z_k (N,S,S) from the forward's idx, weights and records ...
int depth_forward(dss_ctx *ctx, const dss_render_args *g, const float4 *rec, cudaStream_t st);
// ... and its record gradient gz[s] += sum g_D w_k over the pixels whose list holds s, the weights held constant,
// summed in 64-bit fixed point (the same bits on every run)
int depth_backward(dss_ctx *ctx, const dss_render_args *g, float *gz, cudaStream_t st);

// The k nearest *other* points of local row i from its dss_knn_points row nb at K = k + 1: the row less entry
// knn_own_entry(nb, k, i), which is i's own index, or the last entry when i is not in the row (more than k duplicates
// of smaller index).  Neighbour s of the k is nb[knn_other(s, own)].  Upsampling and the RIMLS kernels share this rule.
__device__ __forceinline__ int knn_own_entry(const int32_t *nb, int k, int32_t i) {
    for (int s = 0; s <= k; ++s)
        if (nb[s] == i) return s;
    return k;
}
__device__ __forceinline__ int knn_other(int s, int own) { return s < own ? s : s + 1; }

}  // namespace dss
