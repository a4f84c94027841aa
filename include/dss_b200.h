/*
 * dss_b200.h -- C ABI of the H100-native surface-splatting rasterizer (libdss_b200.so).
 *
 * This is the drop-in boundary for ONE hot path of yifita/DSS: the elliptical point rasterizer,
 * forward and backward.  Every entry point is `extern "C"`, takes raw DEVICE pointers (unless a
 * parameter is explicitly marked host), sizes, and a cudaStream_t passed as void*; it enqueues
 * work on that stream and returns an int status (DSS_OK or a negative DSS_E_* code, never a C++
 * exception).  dss_last_error() returns a thread-local description of the last failure.
 *
 * The reference interfaces each entry point replaces are cited as <file>:<line> relative to the
 * yifita/DSS checkout (reference commit 8fd8d86).  Reference-side bindings: INTEGRATION.md.
 *
 * Conventions shared with the reference:
 *   - "packed" arrays hold all N views back to back: view n owns rows
 *     [first_idx[n], first_idx[n] + num_points[n]); first_idx / num_points are int64 DEVICE arrays
 *     exactly as DSS._C receives them (DSS/csrc/rasterize_points.h:461-472);
 *   - points are NDC x,y in [-1,1] (+X left, +Y up) and view-space depth z; points with z < 0 are
 *     never rasterized (DSS/csrc/rasterize_points.cu:87-88);
 *   - output pixel (row r, col c) is the NDC pixel (S-1-r, S-1-c) (rasterize_points.cu:577-580);
 *   - idx / zbuf / qvalue are (N,S,S,K), -1 padded; occupancy (N,S,S) is 0/1 float.
 */
#ifndef DSS_B200_H
#define DSS_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define DSS_API __attribute__((visibility("default")))
#else
#define DSS_API
#endif

#define DSS_OK 0
#define DSS_E_INVALID -1    /* bad argument (null pointer, size out of range, K too large ...) */
#define DSS_E_CUDA -2       /* a CUDA runtime call or kernel launch failed                    */
#define DSS_E_NOMEM -3      /* scratch allocation failed                                      */
#define DSS_E_CAPACITY -4   /* caller-provided output capacity too small (see *_required)     */

#define DSS_MAX_POINTS_PER_PIXEL 64   /* reference allows 150 (rasterization_utils.cuh:18); configs use 5 / 8 */
#define DSS_MAX_SHARED_VIEWS 256      /* views of one shared cloud per render call (checked by forward AND backward) */

typedef struct dss_ctx dss_ctx;   /* owns grow-only device scratch for one device; not thread-safe */

/* ---- library / context ------------------------------------------------------------------- */
DSS_API int dss_version(void);                       /* ABI version, currently 1                        */
DSS_API const char *dss_last_error(void);            /* thread-local message for the last DSS_E_* return */
DSS_API int dss_create(dss_ctx **out);               /* bind to the CURRENT cuda device                  */
DSS_API void dss_destroy(dss_ctx *ctx);
DSS_API size_t dss_scratch_bytes(const dss_ctx *ctx);/* device bytes currently held by the context       */
/* number of kernels the library has launched on this context since creation (bench: gpu_launches) */
DSS_API int64_t dss_launch_count(const dss_ctx *ctx);

/* ---- optional per-stage device timing ------------------------------------------------------
 * When enabled, every stage (preprocess, bin count, scan, scatter, raster, ...) is bracketed by a CUDA
 * event pair on the launch stream.  dss_profile_read synchronises on the recorded events and returns
 * the accumulated milliseconds and number of brackets of one stage since the last reset.  Used by
 * bench.py for the live roofline of the dominant kernel; off by default (zero overhead). */
DSS_API int dss_profile_enable(dss_ctx *ctx, int on);
DSS_API int dss_profile_reset(dss_ctx *ctx);
DSS_API int dss_profile_num_stages(void);
DSS_API const char *dss_profile_stage_name(int stage);
DSS_API int dss_profile_read(dss_ctx *ctx, int stage, double *total_ms, int64_t *brackets);

/* Debug work counters of the depth-sliced rasterizer (off by default; adds global atomics when on):
 * out[0] tile-list entries scanned, [1] survivors of the block-threshold cull, [2] (splat,pixel) tests,
 * [3] accepted fragments queued for insertion, [4] slices skipped by early termination, [5] rasterization passes
 * (queue flushes) executed, [6] tiles rasterized from the records because their list did not fit the id buffer.
 * enable != 0 switches collection on (and zeroes the counters); out may be NULL. Synchronises the device. */
DSS_API int dss_debug_raster_stats(dss_ctx *ctx, int enable, uint64_t out[8]);

/* Total length of the forward's tile lists as the device published it last (mapped pinned word: no synchronisation, may
 * lag one call behind).  Lets a caller that replays a captured CUDA graph notice that the lists have outgrown the buffer
 * the graph was captured with (dss_b200/graph.py). */
DSS_API int64_t dss_debug_tile_total(const dss_ctx *ctx);

/* Testing: cap the forward's tile-list buffer at max_entries (0 = no cap).  Tiles whose list does not fit are then
 * rasterized from the view's records directly -- the path a sudden growth of the lists takes in production, where the
 * buffer is sized from the previous call without the host ever waiting for the device.  Results must not change. */
DSS_API int dss_debug_limit_tile_capacity(dss_ctx *ctx, int64_t max_entries);

/* Testing: on != 0 bins the forward tile lists as DSS_BIN_NORECTS=1 does -- separate count and scatter passes over the
 * records, the depth ranges from the preprocess -- instead of counting them in the preprocess of dss_render_forward.
 * Both must produce the same depth ranges, offsets and lists (as sets). */
DSS_API int dss_debug_bin_no_rects(dss_ctx *ctx, int on);

/* Testing: copies the last forward's binning from the context's scratch, queued on `stream`: the depth ranges of
 * n_views views (2 floats each) into zrange, the first n_offsets tile-list offsets into offsets and the first n_ids list
 * entries into ids (each skipped when its pointer is NULL).  Fails when a count exceeds what the scratch holds. */
DSS_API int dss_debug_tile_lists(dss_ctx *ctx, int n_views, float *zrange, int64_t n_offsets, int32_t *offsets,
                                 int64_t n_ids, int32_t *ids, void *stream);

/* ---- exclusive prefix sum -----------------------------------------------------------------
 * Replaces prefix_sum.prefix_sum_cuda(grid_cnt, num_grids, grid_off)
 * (external/prefix_sum/prefix_sum.h:6-21, prefix_sum.cu:74-87,135-205): exclusive int32 scan of the
 * first n elements of `in` into `out` (in == out allowed).  Single pass, decoupled look-back; no
 * allocation, no device synchronisation. */
DSS_API int dss_exclusive_scan_i32(dss_ctx *ctx, const int32_t *in, int32_t *out, int64_t n, void *stream);

/* ---- 2-D radius binning (uniform grid) ----------------------------------------------------
 * Replace frnn._C.insert_points_cuda / counting_sort_cuda for D = 2
 * (external/FRNN/frnn/csrc/grid/grid.h:43-50, grid.cu:62-99,144-200;
 *  counting_sort.h:4-11, counting_sort.cu:5-36,72-135).
 * points (N,Pmax,2) f32 padded; lengths (N,) i64; params (N,6) f32 = min_x,min_y,1/cell,res_x,res_y,total;
 * grid_cnt (N,G) i32 must be zero on entry; grid_cell, grid_idx (N,Pmax) i32. */
DSS_API int dss_grid_insert_points_2d(dss_ctx *ctx, const float *points, const int64_t *lengths,
                              const float *params, int32_t *grid_cnt, int32_t *grid_cell,
                              int32_t *grid_idx, int N, int Pmax, int G, void *stream);
DSS_API int dss_grid_counting_sort_2d(dss_ctx *ctx, const float *points, const int64_t *lengths,
                              const int32_t *grid_cell, const int32_t *grid_idx,
                              const int32_t *grid_off, float *sorted_points, int32_t *sorted_idx,
                              int N, int Pmax, int G, void *stream);

/* ---- coarse rasterization (screen-tile binning) -------------------------------------------
 * Replaces _C._rasterize_coarse(points, radii, first_idx, num, image_size, bin_size, M)
 * (DSS/csrc/ext.cpp:11; rasterize_points.h:167-203; rasterize_points.cu:293-500).
 * The reference returns a dense (N,B,B,M) int32 tensor (M = max(1e4,P): 8 GB at 1M points); this
 * returns the same bin membership as CSR: bin_offsets (N*B*B + 1) int32 exclusive offsets and
 * bin_ids, the packed point ids of every bin (order inside a bin unspecified, as in the reference).
 * B = 1 + (S-1)/bin_size; bin (by,bx) of view n is entry (n*B + by)*B + bx, in NDC-index space like
 * the reference.  The overlap predicate is the reference's closed fp32 test (rasterize_points.cu:355-383)
 * evaluated with the identical expression sequence, so membership is bit-exact.
 * If the total exceeds bin_ids_capacity nothing is written to bin_ids, *total_required_host receives
 * the needed size and DSS_E_CAPACITY is returned (call again).  Synchronises the stream once (the
 * total is read back to size the id list, like the reference's host-side `at::full`). */
DSS_API int dss_rasterize_coarse(dss_ctx *ctx, const float *points, const float *radii,
                         const int64_t *first_idx, const int64_t *num_points, int N, int64_t P,
                         int image_size, int bin_size, int32_t *bin_offsets, int32_t *bin_ids,
                         int64_t bin_ids_capacity, int64_t *total_required_host, void *stream);

/* ---- forward rasterization ----------------------------------------------------------------
 * Replaces _C.splat_points(points, ellipse_params, cutoff_thres, radii, first_idx, num_points,
 *                          depth_merging_thres, image_size, points_per_pixel, bin_size, max_points_per_bin)
 * (DSS/csrc/ext.cpp:8; rasterize_points.h:461-525 -> RasterizePointsCoarse + RasterizePointsFine,
 *  rasterize_points.cu:293-432,506-597; CheckPixelInsidePoint :64-124).
 * Per pixel: among points of the view with z >= 0, |dx| <= rx, |dy| <= ry and
 * q = a dx^2 + b dx dy + c dy^2 <= cutoff, keep the K with smallest (z, id), ascending; emit while
 * z_k - z_0 <= depth_merging_thres.  `bin_size` is accepted for signature parity and ignored (tiling
 * is internal); max_points_per_bin does not exist here (lists are exact-size CSR).
 * zbuf / qvalue may be NULL (not written).  All outputs are fully written (no pre-fill needed). */
DSS_API int dss_splat_points(dss_ctx *ctx, const float *points, const float *ellipse_params,
                     const float *cutoff_thres, const float *radii, const int64_t *first_idx,
                     const int64_t *num_points, int N, int64_t P, float depth_merging_thres,
                     int image_size, int points_per_pixel, int bin_size, int32_t *idx, float *zbuf,
                     float *qvalue, float *occupancy, void *stream);

/* ---- backward: visibility, search radius, occupancy / z / colour gradients ------------------ */

/* visible[p] = 1 iff p appears in idx at a pixel whose idx[...,0] >= 0
 * (DSS/core/rasterizer.py:854-860; DSS/utils/__init__.py:320-340 -- replaces two torch.unique calls). */
DSS_API int dss_visibility_from_idx(dss_ctx *ctx, const int32_t *idx, int64_t num_pixels, int K, int64_t P,
                            uint8_t *visible, void *stream);

/* rs[n] = radii_s * lower_median(flattened (rx,ry) of the view's visible points); 0 if none
 * (DSS/core/rasterizer.py:888 -- replaces a per-view host loop with .item() syncs).  Exact radix select. */
DSS_API int dss_search_radius(dss_ctx *ctx, const float *radii, const uint8_t *visible,
                      const int64_t *first_idx, const int64_t *num_points, int N, int64_t P,
                      float radii_s, float *rs, void *stream);

/* Occupancy ("fast") backward.  Replaces the whole fast branch of EllipticalRasterizer.backward
 * (DSS/core/rasterizer.py:845-972): visibility compaction, FRNN grid build, per-view prefix sums,
 * counting sort, _C._splat_points_occ_fast_cuda_backward (rasterize_points_backward.cu:30-212,227-322)
 * and the un-sort / scatter, by one gather kernel: for every visible point of view n,
 *   grad_xy[p] = sum over pixels with g != 0, d2 <= rs[n]^2, not (g > 0 and outside bbox)
 *                of (dx,dy) / eps_denom(d2,1e-10) * g .
 * grad_occ is read as grad_occ[(n*S*S + r*S + c) * pix_stride + pix_offset] so that either a dense
 * (N,S,S) map (stride 1, offset 0) or the alpha channel of an (N,S,S,4) image gradient (4, 3) can be
 * passed.  grad_xy: (P,2), fully written (zeros for invisible points).  Deterministic (no atomics). */
DSS_API int dss_occ_backward(dss_ctx *ctx, const float *points, const float *radii, const uint8_t *visible,
                     const float *rs, const float *grad_occ, int pix_stride, int pix_offset,
                     const int64_t *first_idx, const int64_t *num_points, int N, int64_t P,
                     int image_size, float *grad_xy, void *stream);

/* The reference's "slow" occupancy backward, _C._splat_points_occ_backward (DSS/csrc/ext.cpp:10,16;
 * rasterize_points.cu:673-821) -- disabled in the reference by backward_occ_fast = True (rasterizer.py:816), provided
 * for completeness: every renderable point (z >= 0, |x|,|y| <= 1) of view n gathers
 *   grad_xy[p] = sum over pixels with g != 0, |dx| <= rx*s, |dy| <= ry*s, not (g > 0 and outside the splat's bbox)
 *                of (dx,dy) / eps_denom(dx^2 + dy^2, 1e-10) * g .
 * grad_occ addressing as in dss_occ_backward.  grad_xy (P,2) fully written.  Deterministic (gather, no atomics). */
DSS_API int dss_occ_backward_slow(dss_ctx *ctx, const float *points, const float *radii, const float *grad_occ,
                                  int pix_stride, int pix_offset, const int64_t *first_idx, const int64_t *num_points,
                                  int N, int64_t P, int image_size, float radii_s, float *grad_xy, void *stream);

/* z_grad[idx_k] += grad_zbuf_k until the first idx < 0.  Replaces _C._backward_zbuf
 * (DSS/csrc/ext.cpp:17; rasterize_points.h:388-419; rasterize_points.cu:823-885).  z_grad (P,) in-place. */
DSS_API int dss_zbuf_backward(dss_ctx *ctx, const int32_t *idx, const float *grad_zbuf, int64_t num_pixels,
                      int K, float *z_grad, void *stream);

/* ---- splat-size K-NN (SURVEY.md section 8(f) row 1) -------------------------------------------
 * Replaces frnn.frnn_grid_points(points1, points2, lengths1, lengths2, K, r) (external/FRNN/frnn/frnn.py:15-175;
 * grid.cu:62-99,285-373; counting_sort.cu:5-36), called by DSS with K = 7, r = 0.2 on the world-space cloud to size the
 * splats (DSS/core/rasterizer.py:313-326, 369-388).  For every query of cloud n: the K points of cloud n with the
 * smallest (squared distance, index), squared distance < r^2 (r <= 0: no limit), ascending; missing entries are -1.
 * Semantics and tie rule of the reference's ground truth FRNNBruteForceCPU (bruteforce_cpu.cpp:8-64).
 * Packed layout: cloud n owns rows [first_idx[n], first_idx[n] + num_points[n]); the ranges may leave gaps (padded
 * storage passed as packed) but must not overlap, and rows outside every query range are not written.  idxs are local
 * to the cloud.  queries == NULL (or == points): the cloud is searched against itself (the self match, distance 0, is
 * returned first, as in the reference).  A point or query with a NaN or infinite coordinate is at distance inf or NaN
 * from everything, so it is nobody's neighbour and its own row is all -1; it does not shape the grid.
 * sq_dists (Pq,K) f32, idxs (Pq,K) i32 or NULL.  1 <= K <= 32.  No host synchronisation. */
DSS_API int dss_knn_points(dss_ctx *ctx, const float *queries, const int64_t *query_first_idx,
                           const int64_t *query_num, const float *points, const int64_t *first_idx,
                           const int64_t *num_points, int N, int64_t Pq, int64_t P, int K, float radius,
                           float *sq_dists, int32_t *idxs, void *stream);

/* ---- local frames of the anisotropic kernel ------------------------------------------------------------------------
 * Replaces estimate_pointcloud_local_coord_frames(neighborhood_size=8, disambiguate_directions=False) and the frame /
 * curvature selection of _compute_anisotropic_Vrk (DSS/utils/mathHelper.py:34-91, DSS/core/rasterizer.py:256-291).
 * knn_idx (P,8) int32: every row's 8 nearest neighbours as dss_knn_points writes them for K = 8, r = -1 (local to the
 * cloud, the point itself included).  Per row: the population covariance C of the 8 neighbours about their mean,
 * diagonalised in float64 (fixed cyclic Jacobi sweeps), rounded once: frames (P,8) f32, 16-byte aligned,
 * {f1.xyz, l1, f2.xyz, l2} with l0 <= l1 <= l2 the eigenvalues and f2 the eigenvector of the largest.  Where
 * l1 - l0 <= 2^-40 l2, f1 = normalize(f2 x e_k), e_k the axis of the smallest |f2_k|; where l2 - l0 <= 2^-40 l2 too,
 * f2 = e_x.  A row with a -1 neighbour is all NaN.  first_idx / num_points (N,) int64 as for dss_knn_points, or both
 * NULL with N = 1: one cloud of P rows.  Rows outside every range are not written.  One launch, one thread per row; no
 * scratch, no atomics, no host synchronisation. */
DSS_API int dss_local_frames(dss_ctx *ctx, const float *points, const int64_t *first_idx, const int64_t *num_points,
                             int N, int64_t P, const int32_t *knn_idx, float *frames, void *stream);

/* ---- normal estimation and orientation ----------------------------------------------------------------------------
 * PointClouds3D.estimate_normals (DSS/core/cloud.py:210-258) and meshlab's "Compute normals for point sets" with no
 * smoothing and no viewpoint (scripts/poisson_sampling_pca.mlx), for clouds that carry no normals.  knn_idx (P,k)
 * int32, 3 <= k <= 32: every row's k nearest neighbours as dss_knn_points writes them for K = k, r = -1 (local to the
 * cloud, the point itself included); first_idx / num_points (N,) int64 as for dss_knn_points (required; clouds are never
 * connected).  Outputs (P,3) f32 normals, (P,) int32 root and parent, local to the cloud.
 *  - A row with a -1 neighbour (a non-finite point, a cloud of fewer than k finite points) is invalid: NaN normal,
 *    root = parent = -1, and no edge.
 *  - PCA: the population covariance of the k neighbours about their mean in float64, diagonalised as dss_local_frames
 *    does; the normal is the eigenvector f0 of the smallest eigenvalue, rounded once.  Where l1 - l0 <= 2^-40 l2
 *    (collinear neighbours) it is dss_local_frames' f1 = normalize(f2 x e_k), and where all three agree (duplicates)
 *    e_z.  Its canonical sign makes the component of largest |n_k| (the first such axis) positive.
 *  - orient == 0: the canonical normals; root = parent = -1.
 *  - orient != 0: the undirected graph of the edges {i, j}, j != i in i's list; weight w = 1 - |n_i . n_j| in float32,
 *    each product and sum rounded in the order x, y, z; edges ordered by (w, min(i,j), max(i,j)), so the minimum
 *    spanning forest is unique.  Per component the root is the point of largest z (ties: the smallest index), flipped
 *    so that n_z >= 0 (n_z == 0 keeps the canonical sign).  Every other point is flipped exactly when the dot product
 *    of its normal with its parent's oriented normal (same rounding) is negative; zero does not flip.  root: the
 *    component's root; parent: the tree parent, -1 at a root.
 * On the device (DESIGN.md): one PCA thread per row; Boruvka rounds with 64-bit atomicMin keys and pointer jumping,
 * Euler tours ranked by pointer jumping, and ancestor doubling for the signs, each loop of ceil(log2 P) + 1 launches
 * that leave early on a flag written on the device.  Deterministic, no host synchronisation: capturable.  Scratch from
 * the context: 16 bytes per row, and 108 more per row to orient.  P < 2^30. */
DSS_API int dss_estimate_normals(dss_ctx *ctx, const float *points, const int64_t *first_idx,
                                 const int64_t *num_points, int N, int64_t P, const int32_t *knn_idx, int k, int orient,
                                 float *normals, int32_t *root, int32_t *parent, void *stream);

/* ---- outlier ratio -------------------------------------------------------------------------------------------------
 * remove_outliers (DSS/core/cloud.py:363-378).  points, first_idx, num_points, knn_idx and k as for
 * dss_estimate_normals, and the same float64 PCA.  Outputs, per row of every cloud: ratio (P,) f64 = l0 / ((l0 + l1) +
 * l2) with l0 <= l1 <= l2 the covariance's eigenvalues, and keep (P,) uint8 = ratio < tolerance in float64.  A row with
 * a -1 neighbour gets NaN, and so does a row whose neighbours all coincide (0 / 0); NaN is never kept.  Rows outside
 * every range are not written.  One launch, one thread per row; no scratch, no host synchronisation: capturable. */
DSS_API int dss_outlier_ratio(dss_ctx *ctx, const float *points, const int64_t *first_idx, const int64_t *num_points,
                              int N, int64_t P, const int32_t *knn_idx, int k, double tolerance, double *ratio,
                              uint8_t *keep, void *stream);

/* ---- upsampling ----------------------------------------------------------------------------------------------------
 * upsample (DSS/core/cloud.py:555-632), in rounds on preallocated packed buffers.  Cloud n owns rows [first_idx[n],
 * first_idx[n] + sizes[rounds][n]) of points (M,3), and of normals (M,3) and features (M,D) when not NULL; these ranges
 * must tile [0, M).  On entry each cloud holds its sizes[0][n] input rows at the start of its range.  sizes
 * (rounds + 1, N) int64 is the schedule: round r grows cloud n from c = sizes[r][n] to sizes[r + 1][n] = c + m, with
 * m = min(n_n - c, c / 10) (the caller computes it once; a cloud that grows has more than k points).  knn_num
 * (rounds, N) int64 is c where m > 0 and 0 elsewhere.  3 <= k <= 31.  In each round, for every cloud that grows:
 *  - the neighbours q_0 .. q_{k-1} of row i are its dss_knn_points row at K = k + 1, r = -1, less its own index (less
 *    the last entry when its own index is not in the row: more than k duplicates of smaller index);
 *  - in float32, rounded after every operation, without contraction: candidates c_j = (q_j + 2 p_i) / 3 per coordinate;
 *    s_j = min over all k neighbours q_l of sqrt((dx dx + dy dy) + dz dz), d = c_j - q_l; s_i = max_j s_j, attained
 *    first at j*;
 *  - the m rows of largest s_i, ties to the smaller index, are the parents; parent i writes, in increasing order of i,
 *    to the rows that follow the cloud's c current rows: the point c_{j*}, the normal normalize(2 normalize(n_i) +
 *    normalize(n_{j*})) (normalize(v) = v / sqrt((x x + y y) + z z), same rounding), the feature (f_{j*} + 2 f_i) / 3
 *    per channel, and parents (M,2) int32 = (i, j*) in local indices.
 * Rows already written never change; parents of the input rows are left as the caller set them.  On the device
 * (DESIGN.md): per round one K-NN call, one sparsity thread per row (k^2 distances), an 8-pass MSB-first radix select of
 * (bits(s), ~i), flags, an exclusive scan and a write kernel.  Deterministic, no host synchronisation.  Scratch from the
 * context: 8 (k + 1) + 20 bytes per row and 8 KB per cloud.  M < 2^31 - 1. */
DSS_API int dss_upsample_points(dss_ctx *ctx, float *points, float *normals, float *features, int D,
                                const int64_t *first_idx, const int64_t *sizes, const int64_t *knn_num, int N, int64_t M,
                                int rounds, int k, int32_t *parents, void *stream);

/* ---- RIMLS projection and normal denoising -------------------------------------------------------------------------
 * project_to_latent_surface and denoise_normals (DSS/core/cloud.py:442-553).  points, normals (P,3) f32; first_idx,
 * num_points (N,) as for dss_knn_points (gaps allowed); knn_idx (P, k + 1) the dss_knn_points rows at K = k + 1,
 * r = -1; 3 <= k <= 31; radius (N,) f64 the per-cloud r_n.  All arithmetic is float64; each output is rounded once to
 * float32.  For row i of cloud n, with c_n = num_points[n]:
 *  - neighbours: the K-NN row less i's own index (less the last entry when i is not in it), then less the entries
 *    with squared distance d2_j = |p_i - q_j|^2 above r_n^2; dropped and -1 entries contribute nothing;
 *  - unit normals: normalize(v) = v / max(|v|, 1e-12) (F.normalize: zero stays zero);
 *  - every sum over the neighbours is the xor butterfly over 32 lanes (lane j holds neighbour j, the others 0):
 *    the values v_0 .. v_31 become v_l + v_{l+16} for l < 16, then v_l + v_{l+8} for l < 8, ..., down to one;
 *  - eps_denom(s) = sign(s) max(|s|, 1e-17), zero counted as positive.
 * dss_denoise_normals (the caller's r_n = min(4 avg_n k, 0.2)): w_j = exp(-d2_j c_n / 2) exp(-((1 - n_i.n_j) /
 * sigma)^2), zero where d2_j > 16 / (c_n / 2); out = normalize(sum w_j n_j / eps_denom(sum w_j)), or n_i when every
 * w_j is zero.
 * dss_project_to_surface (the caller's r_n = min(16 avg_n k, 0.2)): the samples q_j, n_j are the input's for the
 * whole call.  inv = 1 / (16 d2min), d2min the smallest d2_j > 0; a row without one is written unchanged.  Then, from
 * x = p_i, for t < max_proj_iters while the row is active: fx_j = (x - q_j).n_j; alpha_j = 1, f = 0, g = 0; for
 * s < max_est_iters: when s >= 1, alpha'_j = exp(-(|n_j - g| / 0.5)^2) exp(-(fx_j - f)^2 inv / 4), and if
 * max_j |alpha'_j - alpha_j| < 1e-4 the loop stops keeping f and g, otherwise alpha = alpha'; then phi_j =
 * exp(-|x - q_j|^2 inv), w_j = phi_j alpha_j, gw_j = 2 (x - q_j) (inv phi_j) w_j, f = sum fx_j w_j / eps_denom(sum
 * w_j), g = (sum gw_j fx_j - f sum gw_j + sum w_j n_j) / eps_denom(sum w_j).  x <- x - f g; the row stays active
 * while |f g| > 5e-4.  out_points gets x, iterations (P,) int32 the number of outer iterations with f g != 0.
 * Rows outside every range are not written.  One launch each, one warp per row; no scratch, no host
 * synchronisation: capturable, and the same bits on every call. */
DSS_API int dss_denoise_normals(dss_ctx *ctx, const float *points, const float *normals, const int64_t *first_idx,
                                const int64_t *num_points, int N, int64_t P, const int32_t *knn_idx, int k,
                                const double *radius, double sharpness_sigma, float *out_normals, void *stream);
DSS_API int dss_project_to_surface(dss_ctx *ctx, const float *points, const float *normals, const int64_t *first_idx,
                                   const int64_t *num_points, int N, int64_t P, const int32_t *knn_idx, int k,
                                   const double *radius, int max_proj_iters, int max_est_iters, float *out_points,
                                   int32_t *iterations, void *stream);

/* ---- L0 image smoothing ------------------------------------------------------------------------------------------
 * L0Smooth (DSS/misc/imageFilters.py:133-180; Xu et al. 2011) of N images (N, H, W, C), C in {1, 3}, read at the
 * element strides strides[0..3] (host array, >= 0) as float32 (f64 == 0) or float64 (f64 != 0); out (N, H, W, C)
 * contiguous, same dtype.  2 <= H, W <= DSS_L0_MAX_SIZE, each with no prime factor above 5; lmd finite, >= 0.  Float64
 * throughout, whatever the dtype; a float32 result is rounded once.  Per image, S = I, beta = 0.1, rounds while
 * beta <= 1e5 (20 rounds), beta doubling after each:
 *  - hp, vp: periodic forward differences of S along x and y;
 *  - (hp, vp) = 0 at the pixels where sum_c(hp^2 + vp^2) < lmd / beta, the channels summed in order, each operation
 *    rounded on its own (NaN is kept);
 *  - hv = (hp(x-1, y) - hp(x, y)) + (vp(x, y-1) - vp(x, y)), periodic;
 *  - S = real(ifft2(fft2(I + beta hv) / (1 + beta D))) per channel, D(u, v) = (2 - 2 cos 2 pi u / W) + (2 - 2 cos 2 pi
 *    v / H): the reference's |fft2(dx)|^2 + |fft2(dy)|^2 in closed form.
 * On the device (DESIGN.md): per round a shrink pass, a row FFT whose load forms I + beta hv, a column pass (FFT,
 * spectral division, inverse FFT) and an inverse row FFT whose store takes the real part; the FFTs are mixed-radix
 * (4, 2, 3, 5) Stockham transforms in shared memory.  Deterministic (no atomics), no host synchronisation or
 * allocation: capturable.  Scratch from the context: 32 bytes per value, 1 byte per pixel and 16 (H + W) bytes. */
#define DSS_L0_MAX_SIZE 2048
DSS_API int dss_l0_smooth(dss_ctx *ctx, const void *images, int f64, const int64_t *strides, int N, int H, int W, int C,
                          double lmd, void *out, void *stream);

/* ---- surface regularisers of the training step (SURVEY.md section 8(f) row 2) -----------------------------------
 * Replaces the torch bodies of ProjectionLoss (kind 0) and RepulsionLoss (kind 1) (DSS/training/losses.py:282-497) on
 * packed clouds (points, normals (P,3); first_idx, num_points as for dss_knn_points).  knn_dists (P, K-1+self_col) f32
 * and knn_idx (same shape) i32 hold each row's K-NN as dss_knn_points writes it (local indices, ascending, -1 padded;
 * a missing entry is taken as pytorch3d's padding: distance 0, index 0); self_col = 1: column 0 is the query itself and
 * is dropped, self_col = 0: the rows hold the K-1 neighbours only.  2 <= K <= 32.  The neighbour positions: knn_pos
 * (P, K-1+self_col, 3) f32, one per column, used as given (a caller's pytorch3d `knn`), or, when knn_pos is NULL, read
 * at the neighbour's index from neighbour_points (P,3) f32 -- the positions the rows were built on, which the loss keeps
 * when it reuses its rows after the points moved -- or from `points` when that is NULL too; read by index they are zero
 * from column num_points[n] of the given row on, as knn_gather(..., lengths) gives them.  reliable (P,) bytes or NULL: rows
 * marked keep their own normal in the denoise (visibility & inmask); visible (P,) bytes or NULL (kind 0 only): the
 * neighbour weight 1 / 0.1 (losses.py:335-337).  Outputs:
 *   kind 0: loss (P,) = sum w_j sdf_j^2 / eps_denom(sum w_j), grad_coef (P,3) = d loss_i / d p_i;
 *   kind 1: loss (P,3) = exp(-|r_i|), grad_coef (P,9) = row-major M_i with d L / d p_i = M_i (d L / d loss_i).
 * The neighbours, the weights and the denoised normals are constants, as in the reference: row i's loss depends on p_i
 * only.  Deterministic (no float atomics); no host synchronisation; scratch from the context. */
DSS_API int dss_surface_regulariser(dss_ctx *ctx, int kind, const float *points, const float *normals,
                                    const int64_t *first_idx, const int64_t *num_points, int N, int64_t P,
                                    const float *knn_dists, const int32_t *knn_idx, int K, int self_col,
                                    const float *knn_pos, const float *neighbour_points, const uint8_t *reliable,
                                    const uint8_t *visible, float sharpness_sigma, float filter_scale, float *loss,
                                    float *grad_coef, void *stream);

/* ---- image loss of the training step ----------------------------------------------------------------------------
 * Trainer.calc_dr_loss (DSS/training/trainer.py:332-376) on the renderer's RGBA: with mask_pred = m != 0 && alpha != 0
 * (NaN counts as non-zero, as torch's .bool()),
 *   loss_rgb = lambda_rgb * sum_{mask_pred} sum_c |gt - pred| / M, M = |mask_pred| (0 when M == 0),
 *   loss_sil = lambda_sil * (sum |m - alpha| / (N H W) + 0.01 * mean_n (1 - I_n / eps_denom(U_n))),
 *   I_n = sum_view n m alpha, U_n = sum_view n (m + alpha - m alpha), loss = loss_rgb + loss_sil.
 * A term whose lambda is not > 0 is absent (0, no gradient; without the RGB term gt is not read).  pred (N,H,W,4) f32 contiguous,
 * 16-byte aligned; gt rgb f32 at gt[n*s0 + y*s1 + x*s2 + c*s3] with gt_strides = {s0, s1, s2, s3} (host array, in
 * elements); mask (N,H,W) contiguous, f32 (mask_kind 0) or bytes (mask_kind 1: bool / uint8), its value used in the
 * silhouette terms.  H*W <= 2^31-1, N <= 65535.
 * Forward (2 launches): totals (N+1, 5) f64, caller-owned and kept for the backward -- row n: M_n, sum |d rgb|,
 * sum |m - alpha|, I_n, U_n of view n; row N: the sums of the first three, sum_n (1 - I_n / eps_denom(U_n)), 0 -- and
 * the three f32 scalars loss, loss_rgb, loss_sil, all on the device.
 * Backward (1 launch): grad_pred (N,H,W,4) f32, 16-byte aligned, every element written, from the upstream gradients of
 * the three scalars (device f32 scalars): rgb sign(pred - gt) lambda_rgb (g_loss + g_rgb) / M inside mask_pred, else 0;
 * alpha lambda_sil (g_loss + g_sil) (sign(alpha - m) / (N H W) - 0.01 (m E_n - I_n (1 - m) dE_n) / (N E_n^2)) with
 * E_n = eps_denom(U_n) and dE_n = [|U_n| >= 1e-17]; sign(0) = sign(NaN) = 0, as torch's abs backward.
 * Deterministic: fixed-order fp64 sums, no float atomics; no host synchronisation; partial sums in context scratch.
 * View-sharded loss (each rank holds some of the views, the loss is the one over all of them): dss_image_loss_partial
 * (2 launches) writes the rank's totals as dss_image_loss_forward does, no scalars, and N in row N's fifth slot; the
 * caller sums row N over the ranks (5 doubles) and dss_image_loss_finish (1 launch) writes the three scalars from the
 * summed row: M and N above are then the sums over all ranks (at least one view in all).  dss_image_loss_backward on
 * these totals takes its M and N from the summed row (a non-zero fifth slot replaces its own N) and I_n, U_n from the
 * rank's view rows. */
DSS_API int dss_image_loss_forward(dss_ctx *ctx, const float *pred, const float *gt, const int64_t *gt_strides,
                                   const void *mask, int mask_kind, int N, int H, int W, double lambda_rgb,
                                   double lambda_sil, double *totals, float *loss, float *loss_rgb, float *loss_sil,
                                   void *stream);
DSS_API int dss_image_loss_backward(dss_ctx *ctx, const float *pred, const float *gt, const int64_t *gt_strides,
                                    const void *mask, int mask_kind, int N, int H, int W, double lambda_rgb,
                                    double lambda_sil, const double *totals, const float *grad_loss,
                                    const float *grad_loss_rgb, const float *grad_loss_sil, float *grad_pred,
                                    void *stream);
DSS_API int dss_image_loss_partial(dss_ctx *ctx, const float *pred, const float *gt, const int64_t *gt_strides,
                                   const void *mask, int mask_kind, int N, int H, int W, double lambda_rgb,
                                   double lambda_sil, double *totals, void *stream);
DSS_API int dss_image_loss_finish(dss_ctx *ctx, const double *total_row, int H, int W, double lambda_rgb,
                                  double lambda_sil, float *loss, float *loss_rgb, float *loss_sil, void *stream);

/* ---- depth loss ---------------------------------------------------------------------------------------------------
 * The training step's dense depth term on the blend's depth map (dss_render_args.depth):
 *   loss = lambda sum_valid |depth - gt| / M,  valid = mask != 0 (NaN counts as set) & alpha != 0 & gt finite &
 *          znear < gt < zfar,  M = |valid|;  0 when M = 0
 * depth, gt (N,H,W) f32 contiguous; pred (N,H,W,4) f32 rgba, 16-byte aligned (its alpha gates the pixel); mask
 * (N,H,W) f32 (mask_kind 0) or bytes (1).  Forward (2 launches): totals (2,) f64 (M, sum |depth - gt|), kept for the
 * backward, and the f32 scalar loss.  Backward (1 launch): grad_depth (N,H,W) f32, every element written:
 * sign(depth - gt) lambda g / M on valid pixels, else 0 (sign(0) = sign(NaN) = 0), g the upstream gradient (a device
 * f32 scalar).  Deterministic fixed-order fp64 sums, no host synchronisation.
 * View-sharded: dss_depth_loss_partial (2 launches) writes the rank's totals only; the caller sums them over the ranks
 * (2 doubles) and dss_depth_loss_finish (1 launch) writes the loss from the summed row; the backward then reads M from
 * the summed row. */
DSS_API int dss_depth_loss_forward(dss_ctx *ctx, const float *depth, const float *pred, const float *gt,
                                   const void *mask, int mask_kind, int N, int H, int W, float znear, float zfar,
                                   double lambda, double *totals, float *loss, void *stream);
DSS_API int dss_depth_loss_partial(dss_ctx *ctx, const float *depth, const float *pred, const float *gt,
                                   const void *mask, int mask_kind, int N, int H, int W, float znear, float zfar,
                                   double *totals, void *stream);
DSS_API int dss_depth_loss_finish(dss_ctx *ctx, const double *total_row, double lambda, float *loss, void *stream);
DSS_API int dss_depth_loss_backward(dss_ctx *ctx, const float *depth, const float *pred, const float *gt,
                                    const void *mask, int mask_kind, int N, int H, int W, float znear, float zfar,
                                    double lambda, const double *totals, const float *grad_loss, float *grad_depth,
                                    void *stream);

/* ---- image-space validation metrics -----------------------------------------------------------------------------
 * Trainer.eval_step (DSS/training/trainer.py:173-212) on V renders of s x s pixels: the ground truth of H x W pixels is
 * resized to s x s as torch's F.interpolate(mode='bilinear', align_corners=False) without antialias does it, in float32
 * (src = max((dst + 0.5) H / s - 0.5, 0), i0 = (int)src, i1 = min(i0 + 1, H - 1), weights src - i0 and 1 - (src - i0),
 * the same for x; s == H returns the input values unchanged), giving g^ and m^; then per view n, in fp64,
 *   I_n = sum m^ alpha, U_n = sum (m^ + alpha - m^ alpha), E_n = sum_pixels sum_c (g^_c - p_c)^2,
 *   iou_n = 1 - I_n / eps_denom(U_n) (IouLoss; an empty union gives 1), psnr_n = E_n / s^2 (L2Loss(channel_dim=1)),
 * on the raw render (no clamping).  pred (V,s,s,4) f32 contiguous, 16-byte aligned; gt rgb f32 at
 * gt[n*s0 + y*s1 + x*s2 + c*s3] with gt_strides = {s0, s1, s2, s3} (host array, in elements); mask (V,H,W) contiguous,
 * f32 (mask_kind 0) or bytes (mask_kind 1: bool / uint8), its value used.  s*s, H*W <= 2^31-1, V <= 65535.
 * Outputs (device, f64): per_view (V, 5) rows (I_n, U_n, E_n, iou_n, psnr_n) and means (2,) (mean_n iou_n,
 * mean_n psnr_n).  2 launches; deterministic: fixed-order fp64 sums, no float atomics; no host synchronisation;
 * partial sums in context scratch. */
DSS_API int dss_image_metrics(dss_ctx *ctx, const float *pred, int s, const float *gt, const int64_t *gt_strides,
                              const void *mask, int mask_kind, int V, int H, int W, double *per_view, double *means,
                              void *stream);

/* ---- training views resident on the device ----------------------------------------------------------------------
 * Gathers views idx[0..B) of a store (n_store, H, W, 4) contiguous, r, g, b, mask per pixel, uint8 (store_f32 == 0,
 * 4-byte aligned) or float32 (store_f32 == 1, 16-byte aligned), into img (B, H, W, 3) and mask (B, H, W), float32,
 * contiguous, 4-byte aligned.  uint8: rgb = __fdiv_rn((float)u, 255.f) (what numpy's correctly rounded float32 u / 255.0
 * gives), mask = u != 0 ? 1.f : 0.f; float32: the values' bits unchanged.  idx: B int64 on the device; PRECONDITION:
 * every idx[b] lies in [0, n_store) (not checked: the caller validates the indices before it uploads them).  Repeats
 * are allowed.  0 <= B <= 65535; B == 0 launches nothing.  64-bit offsets throughout.  One launch on the caller's
 * stream, no allocation, no host synchronisation: capturable. */
DSS_API int dss_gather_views(dss_ctx *ctx, const void *store, int store_f32, int64_t n_store, int H, int W,
                             const int64_t *idx, int B, float *img, float *mask, void *stream);

/* ---- point filters of the training step -------------------------------------------------------------------------
 * Model.forward's visibility and inmask filters (DSS/models/point_modeling.py:172-173, 188-212) of one SHARED cloud of
 * P0 points seen by N cameras (shared_cloud must be 1: packed clouds return DSS_E_INVALID), from the forward's records
 * (N*P0, 8) f32, 8-byte aligned, and visible (N*P0,) bytes of dss_render_forward:
 *   visibility[i] = any_n visible[n*P0 + i],
 *   inmask[i]     = visibility[i] && any_n sample_n(clamp(-x, -1, 1), clamp(-y, -1, 1)) != 0,
 * x, y the record's NDC position of (view n, point i) and sample_n torch's grid_sample of mask n (bilinear, reflection
 * padding, align_corners = False), its arithmetic restated in ATen's order.  A non-finite x or y is outside the mask.
 * mask n at mask[n*s0 + y*s1 + x*s2], mask_strides = {s0, s1, s2} (host array, in elements), H x W independent of the
 * render size, f32 (mask_kind 0) or bytes (mask_kind 1: bool / uint8).  Outputs (P0,) bytes, 0 or 1.
 * One launch, one thread per point; deterministic; no scratch, no host synchronisation.
 * dss_point_filters_gated: the same with visibility[i] = visibility_gate[i] != 0 in place of the any over this call's
 * views (NULL: as dss_point_filters).  A view-sharded step passes the visibility ORed over the ranks, so that inmask
 * ORed over the ranks is the filter of all the views. */
DSS_API int dss_point_filters(dss_ctx *ctx, const float *records, const uint8_t *visible, int shared_cloud, int N,
                              int64_t P0, const void *mask, int mask_kind, const int64_t *mask_strides, int H, int W,
                              uint8_t *visibility, uint8_t *inmask, void *stream);
DSS_API int dss_point_filters_gated(dss_ctx *ctx, const float *records, const uint8_t *visible, int shared_cloud,
                                    int N, int64_t P0, const void *mask, int mask_kind, const int64_t *mask_strides,
                                    int H, int W, const uint8_t *visibility_gate, uint8_t *visibility,
                                    uint8_t *inmask, void *stream);

/* ---- per-point view coverage (pruning the cloud) ------------------------------------------------------------------
 * From one dss_render_forward of a SHARED cloud of P0 points seen by N cameras (shared_cloud must be 1: packed clouds
 * return DSS_E_INVALID) -- its records (N*P0, 8) f32, 16-byte aligned, and visible (N*P0,) bytes -- and the N
 * ground-truth masks, passed as dss_point_filters takes them, ADDS to the int32 (P0,) counters:
 *   seen[i]    += sum_n [visible[n*P0 + i] != 0],
 *   outside[i] += sum_n [z > 0 && |x| <= 1 && |y| <= 1 && sample_n(clamp(-x, -1, 1), clamp(-y, -1, 1)) == 0],
 * x, y, z the record of (view n, point i) and sample_n dss_point_filters' mask sample.  z > 0: the preprocess kept the
 * point in view n (its depth range and backface test); a non-finite x or y fails |x|, |y| <= 1.  outside is not gated
 * on visibility: a hidden point over background counts, an off-frame or depth-filtered one does not.
 * One launch, one thread per point; deterministic; no atomics, no scratch, no host synchronisation: capturable. */
DSS_API int dss_point_coverage(dss_ctx *ctx, const float *records, const uint8_t *visible, int shared_cloud, int N,
                               int64_t P0, const void *mask, int mask_kind, const int64_t *mask_strides, int H, int W,
                               int32_t *seen, int32_t *outside, void *stream);

/* ---- fused renderer path (what bench.py times) ----------------------------------------------
 * One call per direction for SurfaceSplattingRenderer.forward / its autograd backward
 * (DSS/core/renderer.py:36-82, DSS/core/rasterizer.py:584-664,749-977).  All pointers device. */
typedef struct dss_render_args {
    /* geometry: `shared_cloud` != 0 -> points/normals are (P0,3), every view renders the same P0 points
     * (the `extend`ed cloud of rasterizer.py:236-240) and first_idx/num_points are ignored;
     * otherwise packed (P,3) with first_idx/num_points as above. */
    const float *points_world;     /* (P0,3) or (P,3)                                            */
    const float *normals_world;    /* same shape, unit length                                    */
    const float *colours;          /* (P,3) per (view,point) features, e.g. shaded rgb; (P0,3) if shared_colours */
    const float *proj;             /* (N,4,4) full projection, row-vector convention [x y z 1] M  */
    const float *view;             /* (N,4,4) world-to-view, same convention                      */
    const float *h;                /* (N,) variance scale per view, or (P,) per splat             */
    const int64_t *first_idx;      /* (N,) or NULL when shared_cloud                              */
    const int64_t *num_points;     /* (N,) or NULL when shared_cloud                              */
    int32_t n_views;
    int32_t shared_cloud;
    int64_t P0;                    /* points per view when shared_cloud, else max points per view */
    int64_t P;                     /* packed total (n_views * P0 when shared_cloud)               */
    int32_t h_per_splat;
    int32_t image_size;            /* S                                                           */
    int32_t points_per_pixel;      /* K                                                           */
    int32_t backface_culling;      /* rasterizer.py:148-181                                       */
    float cutoff_threshold;        /* C   (rasterizer.py:522)                                     */
    float depth_merging_threshold;
    float antialiasing_sigma;
    float znear, zfar;             /* depth filter (rasterizer.py:183-217)                        */
    float radii_backward_scaler;   /* radii_s                                                     */
    float clip_pts_grad;           /* <= 0: no clipping (rasterizer.py:667-673,735-736)           */
    /* forward outputs / backward inputs, all caller-allocated */
    float *records;                /* (P,8) packed splat records {x,y,z,rx, ry,a,b,c}: written by the
                                      forward pass, read by the backward pass; 16-byte aligned.  May
                                      be NULL (scratch is used; backward then rebuilds from ndc/radii) */
    float *ndc;                    /* (P,3) x,y NDC, z view depth; z = -1 for filtered points; may be NULL */
    float *ellipse;                /* (P,3) a,b,c; may be NULL                                     */
    float *radii;                  /* (P,2); may be NULL                                           */
    float *scaler;                 /* (P,)                                                         */
    float *image;                  /* (N,S,S,4) rgb + occupancy                                   */
    int32_t *idx;                  /* (N,S,S,K)                                                    */
    float *weights;                /* (N,S,S,K) normalised blend weights w_k / max(sum w, 1e-4)    */
    float *zbuf;                   /* (N,S,S,K) or NULL                                            */
    float *qvalue;                 /* (N,S,S,K) or NULL                                            */
    uint8_t *visible;              /* (P,)                                                         */
    /* backward */
    const float *grad_image;       /* (N,S,S,4)                                                    */
    const float *grad_zbuf;        /* (N,S,S,K) or NULL                                            */
    float *grad_colours;           /* (P,3), or (P0,3) if shared_colours                           */
    float *grad_ndc;               /* (P,3) gradient w.r.t. ndc (after clipping)                   */
    float *grad_points_world;      /* (P0,3) summed over views when shared_cloud, else (P,3)       */
    float *search_radius;          /* (N,) out                                                     */
    /* != 0 (shared_cloud only): `colours` is (P0,3), one feature row per POINT used by every view (view-independent
     * colour, the common host-side input: the reference only materialises the (N*P0,3) tensor on the device, after
     * shading) and `grad_colours` is (P0,3), summed over the views. */
    int32_t shared_colours;
    /* ---- per-point shading fused into the path (SURVEY.md 8(f)3; DSS/core/texture.py:74-127, lighting.py:10-172) ----
     * shade != 0 (shared or packed clouds): the per-(view,point) colours are COMPUTED instead of read from `colours`:
     *   shaded = albedo * (ambient + sum_l Cd_l relu(n.d_l)) + sum_l Cs_l (relu(v.r_l) [n.d_l > 0])^shininess,
     *   n = normalize(normal), d_l = normalize(direction_l) or normalize(location_l - p), v = normalize(cam - p),
     *   r_l = -d_l + 2 (n.d_l) n          (all normalisations as F.normalize(eps = 1e-6))
     * in the preprocess kernel (forward), and the backward turns the colour gradient into gradients w.r.t. the albedo,
     * the NORMALS and (view direction, point lights) the positions -- what torch autograd does in the reference after
     * ~40 ATen kernels on (N*P0,3) tensors.  Packed clouds (shared_cloud == 0) shade every packed row with the lights
     * and camera centre of the view whose range holds it; albedo and the three gradients below are then (P,3), one row
     * per packed row, and rows that no view range covers are not written (the caller zero-fills them, as for
     * grad_points_world). */
    int32_t shade;
    int32_t n_lights;              /* L, 1 .. DSS_MAX_LIGHTS                                       */
    int32_t light_type;            /* 0: directional (rows of `lights` start with a direction), 1: point (a location) */
    float shininess;               /* specular exponent (texture.py:76: 64)                        */
    /* 0: one set of lights for every view, `lights` (L,9) and `ambient` (3,).  1 (shade only): a set per view, as the
     * reference's data gives every image its own light (texture.py:113-114 gathers the light properties per view):
     * `lights` (N,L,9) and `ambient` (N,3), view n's rows at lights + n*L*9 and ambient + n*3. */
    int32_t lights_per_view;
    const float *albedo;           /* (P0,3) per-point rgb, or (P,3) per packed row                */
    const float *lights;           /* (L,9) {direction | location, diffuse rgb, specular rgb}, or (N,L,9) per view */
    const float *ambient;          /* (3,) ambient colour (summed over the lights' ambient terms), or (N,3) per view */
    const float *cam_centres;      /* (N,3) camera centres in world space                          */
    float *shaded;                 /* (P,3) shaded colours: written by the forward, the blend reads them */
    /* backward (shade): `grad_colours` is then a (P,3) SCRATCH that receives d L / d shaded; outputs: */
    float *grad_albedo;            /* (P0,3) summed over views, or (P,3) per packed row             */
    float *grad_normals_world;     /* (P0,3) summed over views, or (P,3) per packed row             */
    float *grad_points_shading;    /* (P0,3) or (P,3) position gradient through the shading; dss_render_backward adds it
                                      to grad_points_world when it ran the colour half itself (grad_colours != NULL) */
    /* optional (n_views * OB * OB * 1024,) int32, OB = ceil(S / 32): written by the forward (one count per visible splat in
     * the cell -- pixel of a 32x32 tile -- of its centre; `visible` must then be 4-byte aligned with its capacity rounded
     * up to a multiple of 4), read by the backward, whose binning then skips its counting pass over all P splats.  Give
     * the same tensor to both calls or NULL to both. */
    int32_t *cell_counts;
    /* anisotropic splats (Vrk_invariant = Vrk_isotropic = false, rasterizer.py:256-291, 425-439): the (P0,8) (shared
     * cloud) or (P,8) (packed) records {f1.xyz, l1, f2.xyz, l2} of dss_local_frames, indexed like the points.  The
     * splat's world variance is then l1 f1 f1^T + l2 f2 f2^T and |det Mk| = |det([f1 f2]^T J)|, in place of
     * h (I - n n^T); `h` must be NULL.  NULL: the isotropic / invariant kernel with `h`.  The normals still shade and
     * cull. */
    const float *frames;
    /* with `shade`: != 0 sums the colour scatter into d L / d shaded in 64-bit fixed point (the same bits on every run,
     * see dss_colour_backward); 0 adds it with float atomics (faster at large P).  The training step sets it. */
    int32_t deterministic_colours;
    /* dense depth of the blend: (N,S,S) D = sum_k w_k z_k over the pixel's K-list in k order (the normalised weights
     * of `weights`, the records' view depth z), 0 where the list is empty; written by dss_render_forward (one launch
     * after the raster, which needs `weights`) when not NULL. */
    float *depth;
    /* backward: (N,S,S) d L / d depth or NULL.  Adds sum g_D w_k to the view-depth gradient of every record in the
     * pixel's list, the weights held constant, summed in 64-bit fixed point (the same bits on every run); that gradient
     * reaches the positions, `grad_ndc` and so the camera backward, as `grad_zbuf`'s does. */
    const float *grad_depth;
} dss_render_args;
#define DSS_MAX_LIGHTS 8

/* preprocess -> bin -> rasterize + blend.  Never waits for the device in steady state: the tile-list buffer is sized
 * from the total the PREVIOUS call published; tiles whose list has outgrown it are rasterized from the records on the
 * device (see DESIGN.md "Host side").  Only a context's first call synchronises once to size the buffer. */
DSS_API int dss_render_forward(dss_ctx *ctx, const dss_render_args *args, void *stream);
/* visibility/median radius -> occupancy gather -> colour scatter -> z scatter -> clip -> world chain.
 * grad_colours == NULL skips the colour scatter (see dss_colour_backward). */
DSS_API int dss_render_backward(dss_ctx *ctx, const dss_render_args *args, void *stream);
/* The colour half of the backward alone (norm_weighted_sum backward: grad_colours[idx_k] += g_rgb * w_k), on `stream`.
 * With `shade` and `deterministic_colours` the per-record d L / d shaded is summed in 64-bit fixed point (one scale per
 * call, each term rounded once) and is the same bits on every run; otherwise float atomics add the terms in arrival
 * order.
 * Lets a data-parallel caller start the all-reduce of the colour gradients while dss_render_backward (called with
 * grad_colours == NULL on another stream) is still busy with the occupancy path (dss_b200/parallel.py). */
DSS_API int dss_colour_backward(dss_ctx *ctx, const dss_render_args *args, void *stream);
/* Camera gradients, after dss_render_backward has written args->grad_ndc (the clipped NDC gradient of every slot; the
 * reference differentiates the screen positions through pytorch3d's transform, rasterizer.py:614).  With
 * p_h = [p 1], clip = p_h proj[n], w = clip3, (x, y) = clip01 / w, summed over the slots of view n:
 *   grad_proj[n][r][c] = sum p_h[r] (gx / w, gy / w, 0, -(gx x + gy y) / w)[c]      (N,4,4), column 2 zero
 *   grad_view[n][r][c] = c == 2 ? sum p_h[r] gz : 0                                 (N,4,4)
 * grad_cam_centres (N,3) or NULL: with fused shading (shade != 0) the gradient w.r.t. cam_centres through the view
 * direction v = normalize(cam - p); reads the d L / d shaded scratch that the colour backward left in
 * args->grad_colours and the shading inputs.  The splat shapes (ellipse, radii, scaler) are constants, as in the
 * reference.  Deterministic: fixed-order fp64 sums, no atomics. */
DSS_API int dss_camera_backward(dss_ctx *ctx, const dss_render_args *args, float *grad_proj, float *grad_view,
                                float *grad_cam_centres, void *stream);
/* Light gradients of the fused shading (shade != 0), after the colour backward has left d L / d shaded in
 * args->grad_colours (as for grad_cam_centres above).  Outputs have the shape of the inputs: grad_lights (L,9) and
 * grad_ambient (3,), summed over the views, or (N,L,9) and (N,3) with lights_per_view.  Row l holds the gradient w.r.t.
 * light l's direction (directional) or location (point), diffuse rgb and specular rgb; the ambient gradient is that of
 * the summed ambient colour.  `shininess` gets no gradient.  Either output may be NULL.  Deterministic: fixed-order fp64
 * sums, no atomics. */
DSS_API int dss_light_backward(dss_ctx *ctx, const dss_render_args *args, float *grad_lights, float *grad_ambient,
                               void *stream);
/* per-(point,view) preprocess only (rasterizer.py:443-565 fused): writes ndc, ellipse, radii, scaler. */
DSS_API int dss_preprocess(dss_ctx *ctx, const dss_render_args *args, void *stream);

/* ---- opaque triangle meshes (training data from a mesh) -------------------------------------------------------------
 * pytorch3d's rasterize_meshes + HardFlatShader as the reference's scripts/create_mvr_data_from_mesh.py:147-208 calls
 * them (blur_radius 0, perspective_correct off, cull_backfaces off, only the front fragment), for one mesh verts (V,3)
 * f32 / faces (F,3) i32 seen by N cameras proj / view (N,4,4), row-vector convention as in dss_render_args.
 * Per view every vertex gets screen x, y = its NDC (the splat preprocess's expression) and z = its view-space depth;
 * pixel (row, col) has the centre pix_to_ndc of index (S-1-col, S-1-row) as in the point rasterizer.  With
 * E(p, a, b) = (p.x - a.x)(b.y - a.y) - (p.y - a.y)(b.x - a.x), a face is skipped when max(z0, z1, z2) < 0, when
 * |E(v0, v1, v2)| <= 1e-8, or at pixels outside its closed xy bounding box; otherwise, with den = E(v2, v0, v1) + 1e-8,
 *   w0 = E(p, v1, v2) / den,  w1 = E(p, v2, v0) / den,  w2 = E(p, v0, v1) / den,  pz = (w0 z0 + w1 z1) + w2 z2,
 * it covers the pixel when w0 > 0 && w1 > 0 && w2 > 0 && pz >= 0.  The covering face with the smallest pz wins, ties to
 * the smaller face index.  Outputs (caller-allocated, N*S*S each): pix_to_face i32 (face index, -1: none) and zbuf f32
 * (pz, -0 written as +0; -1: none).  rgba (N,S,S,4) f32 or NULL: flat shading, the fused shading's formula (see
 * dss_render_args.shade) with albedo 1 at the face centroid, normal normalize(cross(v1 - v0, v2 - v0)) and view n's
 * lights and camera centre; background (1, 1, 1, 0).  n_lights, light_type, lights_per_view, shininess, lights, ambient
 * and cam_centres as the dss_render_args fields of the same names, read only with rgba.  A face with an index outside
 * [0, V) covers nothing.  Deterministic (a 64-bit integer atomicMin per covered (face, pixel)); no host
 * synchronisation; views are processed in chunks that bound the context's scratch. */
DSS_API int dss_rasterize_mesh(dss_ctx *ctx, const float *verts, int64_t V, const int32_t *faces, int64_t F,
                               const float *proj, const float *view, int N, int image_size, int n_lights,
                               int light_type, int lights_per_view, float shininess, const float *lights,
                               const float *ambient, const float *cam_centres, int32_t *pix_to_face, float *zbuf,
                               float *rgba, void *stream);

/* ---- chamfer distance (evaluation only, no backward) ----------------------------------------------------------------
 * The sums behind pytorch3d's chamfer_distance as Trainer.evaluate_3d calls it (DSS/training/trainer.py:144-171).  x
 * (Px,3) and y (Py,3) f32 hold N clouds each in the dss_knn_points layout (cloud n owns rows [first[n], first[n] +
 * num[n]); gaps allowed, overlaps not); x_normals / y_normals are indexed like the points, both or neither may be NULL.
 * For every query row its nearest row of the other cloud n -- the smallest (squared distance, index), the
 * dss_knn_points rule and its float32 distance -- gives d; with normals, c = 1 - |cos| of the two normals, where
 * cos = sum_k (a_k / max(|a|, 1e-6)) (b_k / max(|b|, 1e-6)) in fp64 (torch's cosine_similarity, eps = 1e-6).  A row
 * without a neighbour (a NaN or infinite coordinate, or an empty other cloud) gives d = c = NaN.
 * Output sums (N,4) f64: {sum_x d, sum_y d, sum_x c, sum_y c} (the normal sums are 0 without normals).  Two K = 1
 * searches (their rows in context scratch), one thread per query row of both directions writing fp64 per-block
 * partials, one fixed-order finish: deterministic, no atomics on floats, no host synchronisation, capturable.  x and y
 * may be the same rows (the tie rule holds there too). */
DSS_API int dss_chamfer(dss_ctx *ctx, const float *x, const float *x_normals, const int64_t *x_first,
                        const int64_t *x_num, int64_t Px, const float *y, const float *y_normals,
                        const int64_t *y_first, const int64_t *y_num, int64_t Py, int N, double *sums, void *stream);

/* ---- point-to-mesh distance (evaluation only, no backward) ---------------------------------------------------------
 * The point-to-surface term of the reference's scripts/evaluatePointClouds.py, exact.  queries (P,3) f32, one mesh
 * verts (V,3) f32 / faces (F,3) i32.  Every face is the closed convex hull of its three vertices, so a zero-area face
 * is a segment or a point.  For every query q:
 *   sq_dist[q]  (P,) f32: the smallest squared Euclidean distance from q to any face, computed in fp64 from the f32
 *               inputs (the closest point of a face by its Voronoi regions, every operation rounded on its own; a face
 *               whose edge vectors have an exactly zero cross product takes the closest of its three edges) and
 *               rounded once to f32;
 *   face_idx[q] (P,) i32: the face attaining it, an exact fp64 tie to the smaller face index;
 *   closest     (P,3) f32 or NULL (not written): the closest point on that face, each coordinate rounded once.
 * A query with a NaN or infinite coordinate gets NaN / -1 (closest NaN).  A face with an index outside [0, V) or a
 * non-finite vertex is ignored: never nearest, and it does not shape the acceleration structure (as in
 * dss_rasterize_mesh).  Without any usable face every query gets NaN / -1.  The result equals a brute force over all
 * faces: a uniform grid over the usable faces' bounding box (built on the device, its cell size from the face density,
 * at most 2^21 cells) only decides which faces a query tests, and each query's search stops once no untested face can
 * be nearer (DESIGN.md).  Deterministic (integer atomics only).  The call synchronises the host ONCE, after counting
 * the grid's face references, to size that list in the context's scratch (so it cannot be captured in a CUDA graph);
 * more than 2^31 - 1 references is DSS_E_CAPACITY.  face_tests (P,) i32 or NULL: for measuring the search, the number
 * of face distances each query evaluated. */
DSS_API int dss_point_mesh_distance(dss_ctx *ctx, const float *queries, int64_t P, const float *verts, int64_t V,
                                    const int32_t *faces, int64_t F, float *sq_dist, int32_t *face_idx, float *closest,
                                    int32_t *face_tests, void *stream);

/* ---- screened Poisson surface reconstruction (forward only) ---------------------------------------------------------
 * The surface of the reference's Generator.generate_mesh (DSS/models/point_modeling.py:256-282, pymeshlab's
 * surface_reconstruction_screened_poisson(depth=8)), restated as Kazhdan & Hoppe's screened Poisson reconstruction on a
 * dense grid with first-order (trilinear) elements.  The discretisation:
 *   - usable sample: finite coordinates and normal, |n| > 0; its unit normal n / |n| (fp64).  Other rows are ignored.
 *   - domain: c = centre of the usable samples' bounding box, L = 1.1 x its longest side, both rounded to float32 as
 *     c_k = (float)(0.5 (lo_k + hi_k)) and L = (float)(1.1 max_k (hi_k - lo_k)) in fp64.  A sample maps to
 *     u = (p - c) / L + 0.5 (fp64, from the float32 c and L), inside [0.045, 0.955]^3.
 *   - grid: R = 2^depth cells per axis, h = 1 / R, nodes u = h (i, j, k) for i, j, k in [0, R], stored x-major:
 *     node (i, j, k) at (i (R+1) + j) (R+1) + k.  phi_n is the trilinear hat of node n.
 *   - A = h^2 x (cells holding at least one usable sample), a = A / N_usable;  V = sum_n V_n phi_n,
 *     V_n = (a / h^3) sum_p phi_n(u_p) n_p.
 *   - chi minimises  integral over [0,1]^3 of |grad chi - V|^2  +  alpha a sum_p chi(u_p)^2,  alpha =
 *     DSS_POISSON_POINT_WEIGHT: (K + alpha a Q) chi = b with K_nm = int grad phi_n . grad phi_m, Q_nm = sum_p phi_n(u_p)
 *     phi_m(u_p), b_n = int grad phi_n . V; natural (Neumann) boundary, every node an unknown.  On the tensor basis
 *     K = K1(x)M1(x)M1 + M1(x)K1(x)M1 + M1(x)M1(x)K1 and b = (D1(x)M1(x)M1) V_x + (M1(x)D1(x)M1) V_y + (M1(x)M1(x)D1) V_z
 *     with the 1-D mass M1, stiffness K1 and D1[n][m] = int phi_n' phi_m.
 *   - iso-value 0: 1^T K = 0 and sum_n b_n = 0, so sum_p chi(u_p) = 0 at the solution.  chi < 0 inside, > 0 outside.
 * Degenerate input (no usable sample, or all of them one point): chi = 1 everywhere (an empty surface), 0 iterations.
 *
 * dss_poisson_solve: points, normals (P,3) f32; depth in [2, DSS_POISSON_MAX_DEPTH].  Writes chi ((R+1)^3 f32, device)
 * and, on the host, center[3] = c, *side = L, *iterations and *residual (|r| / |b| of the depth-d system's CG, both 0
 * when degenerate; either pointer may be NULL).  level_iterations (host, depth + 1 ints) and level_ms (host, 2 (depth +
 * 1) floats: set-up and CG milliseconds of each level) are optional; entries of levels not solved are 0.
 * Solver: cascadic, Jacobi-preconditioned CG in float32 with fp64 dot products, matrix-free (the 27-point stencil of K
 * and the 8 x 8 block of Q of every occupied cell).  Levels min(depth, DSS_POISSON_FIRST_DEPTH) .. depth are solved in
 * turn, each from the trilinear prolongation of the previous level's chi (the first from 0); only the depth-d system
 * defines the result.  Each level stops when |r| / |b| <= DSS_POISSON_TOLERANCE or after DSS_POISSON_MAX_ITERATIONS.
 * Deterministic: every sample-to-grid sum (S_n, the blocks of Q, the occupied-cell count) is an integer (64-bit fixed
 * point, 2^-30) atomic, so the result is the same bits for any order of the samples; dot products are per-block fp64
 * partials added in a fixed order.  Host synchronisations: one after the bounding box, then one every
 * DSS_POISSON_CHECK_EVERY CG iterations of each level (the CG state stays on the device in between).  Workspace (context
 * scratch, kept for later calls): 8 node arrays of the finest level ((R+1)^3 x 4 bytes each: 0.54 GB at depth 9, 67 MB
 * at depth 8), the previous level's solution (1/8 of one), and 544 bytes per cell for min(N_usable, R^3) cells.
 *
 * dss_marching_tetrahedra: the chi = 0 surface of a node grid chi ((R+1)^3 f32, the layout above) placed by center[3]
 * (host) and side: node (i, j, k) lies at c + (h (i, j, k) - 0.5) L.  A node with chi < 0 is inside; chi >= 0 (0 too)
 * and NaN are outside.  Every cube is split into the 6 Kuhn tetrahedra around its corner (0,0,0) - (1,1,1) diagonal, in
 * the order of the axis permutations xyz, xzy, yxz, yzx, zxy, zyx (tetrahedron sigma: corners 0, e_s1, e_s1 + e_s2,
 * (1,1,1)), so neighbouring cubes agree on every face and the mesh is closed without a case table.
 * Vertices: one per crossing edge (a, a + d), d one of the 7 directions d = (dx, dy, dz) != 0 in {0,1}^3 (direction
 * number 4 dx + 2 dy + dz), ordered by (node index of a, direction number).  In float32, each operation rounded once:
 *   t = (0 - chi_a) / (chi_b - chi_a);  g_k = (float)i_k + t where d_k = 1, (float)i_k where d_k = 0;
 *   vertex_k = c_k + (g_k h - 0.5) L   with h = 1 / R (the products and differences in that order, no fused ops).
 * Faces: per tetrahedron with k of its 4 corners inside, none for k = 0 or 4; for k = 1 or 3 one triangle on the 3
 * edges of the lone corner; for k = 2 the quad (i0 o0, i0 o1, i1 o1, i1 o0) of the inside corners i0 < i1 and outside
 * corners o0 < o1 (local order, o0 and o1 swapped when (i0, i1, o0, o1) is an odd permutation of the positively
 * oriented tetrahedron), split along i0 o0 - i1 o1 into (q0, q1, q2), (q0, q2, q3).  Every face's right-hand normal
 * points from inside to outside (along the input normals of a reconstruction).  Faces are ordered by (cube index,
 * tetrahedron, triangle); cube (i, j, k) has index (i R + j) R + k.
 * Count, exclusive scan (dss_exclusive_scan_i32) and write: the call synchronises the host once, after counting, and
 * writes *n_verts / *n_faces (host).  When they exceed max_verts / max_faces nothing is written and DSS_E_CAPACITY is
 * returned (call again with outputs that size); more than 2^31 - 1 of either is DSS_E_CAPACITY as well.  verts (V,3)
 * f32, faces (F,3) i32. */
#define DSS_POISSON_MAX_DEPTH 9
#define DSS_POISSON_FIRST_DEPTH 4      /* the cascade's coarsest level */
#define DSS_POISSON_POINT_WEIGHT 4.0   /* alpha: pymeshlab's default point weight */
#define DSS_POISSON_TOLERANCE 1e-6     /* relative residual |r| / |b| that ends a level's CG */
#define DSS_POISSON_MAX_ITERATIONS 2000
#define DSS_POISSON_CHECK_EVERY 32     /* CG iterations queued between two host reads of the convergence state */
DSS_API int dss_poisson_solve(dss_ctx *ctx, const float *points, const float *normals, int64_t P, int depth,
                              float *chi, float *center, float *side, int *iterations, double *residual,
                              int *level_iterations, float *level_ms, void *stream);
DSS_API int dss_marching_tetrahedra(dss_ctx *ctx, const float *chi, int R, const float *center, float side,
                                    float *verts, int64_t max_verts, int32_t *faces, int64_t max_faces,
                                    int64_t *n_verts, int64_t *n_faces, void *stream);

/* ---- Poisson-disk sampling of a mesh (evaluation ground truth, no backward) ----------------------------------------
 * The samples of the reference's MVRDataset.get_pointclouds(num_points) and scripts/poisson_sampling.mlx (meshlab's
 * Poisson-disk sampling with a Monte Carlo pool of DSS_PD_MONTECARLO_RATE x N samples and an exact-count radius search
 * to 0.5 %), restated as a rule.  Inputs: one mesh verts (V,3) f32 / faces (F,3) i32, a target count N, a seed and
 * the geodesic flag.  Every fp64 operation below is rounded on its own (no contraction).
 *   1. Usable faces: indices in [0, V), finite vertices, area_f = 0.5 sqrt(c . c) > 0 with c = cross(b - a, c - a)
 *      (component k: the two products, then their difference).  A_max = the largest area, W_f = max(1, ceil(area_f
 *      2^32 / A_max)) in [1, 2^32] for a usable face, 0 otherwise; P_f = the exclusive 64-bit prefix of the W_f, W the
 *      total.  A = (double)W A_max 2^-32 is the area the radius search starts from (>= the usable area, within
 *      F A_max 2^-32 of it).  Without a usable face the result is empty.
 *   2. Pool of M = DSS_PD_MONTECARLO_RATE N samples.  The draws of sample i are x_k = splitmix64(seed, 3 i + k + 1) for
 *      k = 0, 1, 2, where splitmix64(s, j) is the j-th output of SplitMix64 seeded with s:
 *        z = s + j 0x9E3779B97F4A7C15;  z = (z ^ z >> 30) 0xBF58476D1CE4E5B9;  z = (z ^ z >> 27) 0x94D049BB133111EB;
 *        x = z ^ z >> 31                                                           (all modulo 2^64).
 *      The face is the f with P_f <= t < P_f + W_f, t = the high 64 bits of the 128-bit product x_0 W (the first
 *      usable face whose inclusive prefix exceeds t).  u = (x_1 >> 11) 2^-53, v = (x_2 >> 11) 2^-53, s = sqrt(u),
 *      w0 = 1 - s, w1 = s (1 - v), w2 = s v, the point ((w0 a + w1 b) + w2 c) per coordinate and its normal c / |c|
 *      (c the face's cross product above), each rounded once to f32.  Pool order is the selection's priority.
 *   3. Selection at radius r (the sequential dart throw): walk the pool in index order and accept a sample unless an
 *      accepted sample conflicts with it.  Samples p0 (the later) and p1 (the earlier) conflict when their distance is
 *      below r.  Euclidean: d2 < r * r with d = p0 - p1 in fp64 from the f32 points and d2 = (dx dx + dy dy) + dz dz.
 *      Geodesic (meshlab's approximate geodesic distance, libm asin, so not bit-reproducible across libraries): 0 when
 *      d2 = 0; otherwise d_e = sqrt(d2), and no conflict unless d_e < r; then v = d / d_e, C0 = v . n0, C1 = v . n1
 *      (the f32 normals), each clamped to [-1, 1], g = (asin C0 - asin C1) / (C0 - C1), or 1 / sqrt(1 - C0 C1) when
 *      |C0 - C1| < 1e-4, g = max(g, 1), and the distance is d_e g.  g equals arc / chord for two points of a circle, is
 *      symmetric and >= 1, so every conflict is also a Euclidean one.
 *   4. The radius: N_tol = floor(N / 200).  Probe r = sqrt(A / (0.7 pi N)) first.  After a probe with n(r) samples:
 *      stop when |n(r) - N| <= N_tol; otherwise r is a lower bound when n(r) > N, an upper one when n(r) < N, and the
 *      next probe is 2 r while no upper bound is known, r / 2 while no lower one is, else (lo + hi) / 2.  After
 *      DSS_PD_MAX_PROBES probes the probe with the smallest |n - N| (the earliest on a tie) is returned.  The radius is
 *      host fp64 arithmetic.
 * Output: the accepted samples of the returned probe in pool order, points and normals (n,3) f32; *n_out = n (host),
 * *radius = its r (host; 0 without a usable face).  When n > max_out nothing is written and DSS_E_CAPACITY is returned
 * (*n_out tells the size; call again).  N <= 0 and M >= 2^31 are DSS_E_INVALID.
 * On the device: a face pass (areas, box, A_max), the weights, the 64-bit scan, one thread per pool sample; then per
 * probe a uniform grid of cell side max(r (1 + 2^-20), extent / DSS_PD_GRID) (27 cells hold every conflict) built by
 * count, dss_exclusive_scan_i32 and fill, and the lexicographically first maximal independent set of the conflict
 * graph in pool order, computed in rounds (DESIGN.md): an undecided sample is rejected when an earlier conflicting
 * sample is accepted and accepted when no earlier conflicting sample is undecided, which is the sequential result.
 * Deterministic.  Host synchronisations: one after the face pass (box, A_max, W), then one every DSS_PD_CHECK_EVERY
 * rounds of every probe, and one to size the output: not capturable.  Scratch from the context: ~80 bytes per pool
 * sample, 16 per face and 8 per grid cell (at most (DSS_PD_GRID + 1)^3 cells). */
#define DSS_PD_MONTECARLO_RATE 20     /* pool samples per requested sample (poisson_sampling.mlx's MontecarloRate) */
#define DSS_PD_MAX_PROBES 64          /* radius probes at most */
#define DSS_PD_CHECK_EVERY 8          /* selection rounds queued between two host reads of the round state */
#define DSS_PD_GRID 256               /* the selection grid's cell side is at least extent / DSS_PD_GRID */
DSS_API int dss_sample_mesh_poisson_disk(dss_ctx *ctx, const float *verts, int64_t V, const int32_t *faces, int64_t F,
                                         int64_t num_samples, int geodesic, uint64_t seed, float *points,
                                         float *normals, int64_t max_out, int64_t *n_out, double *radius,
                                         void *stream);
/* Statistics of the context's last dss_sample_mesh_poisson_disk call, for measuring it (each pointer may be NULL):
 * *probes; per probe (DSS_PD_MAX_PROBES entries, host) its radius, its count and its selection rounds; stage_ms (4
 * floats): the pool build, the radius search, the final selection when the returned probe was not the last one, and
 * the output. */
DSS_API int dss_poisson_disk_stats(dss_ctx *ctx, int *probes, double *radii, int64_t *counts, int *rounds,
                                   float *stage_ms);

/* ---- camera pose corrections ------------------------------------------------------------------------------------
 * V per-view corrections xi_v = (w, t), poses (V,6) f32: a rotation vector w and a translation t applied in the camera
 * frame.  Row-vector convention: E = [[R(w), 0], [t, 1]] with R(w) = I + s [w]x + c [w]x^2 (s = sin th / th, c = (1 -
 * cos th) / th^2, th = |w|: scipy's Rotation.from_rotvec(w).as_matrix()), and for batch entry b of view v = idx[b]
 *   view[b] = view0[v] + view0[v] D,   proj[b] = proj0[v] + view0[v] D K,   D = E - I,   K = view0[v]^-1 proj0[v],
 * view0[v]^-1 the rigid inverse [[R^T, 0], [-t R^T, 1]] (the caller checks that view0's 3x3 blocks are rotations).  D
 * is formed directly, so xi = 0 gives view0 and proj0 bit for bit.  Computed in float64, each output element rounded
 * once.  idx (B,) int64 device, each in [0, V) (the call does not read them on the host; an index out of range gives
 * NaN matrices); view0 / proj0 (V,4,4), view / proj (B,4,4) f32 contiguous.  No scratch, no host synchronisation. */
DSS_API int dss_pose_forward(dss_ctx *ctx, const float *poses, const int64_t *idx, int V, int B, const float *view0,
                             const float *proj0, float *view, float *proj, void *stream);
/* The backward: grad_poses (V,6), every row written, from grad_view / grad_proj (B,4,4) f32 (either may be NULL: zero).
 * Row v sums the batch entries with idx[b] == v in batch order in float64, then applies the chain rule once; rows of
 * views outside the batch are +0.  One thread per row, no atomics: the same bits on every run. */
DSS_API int dss_pose_backward(dss_ctx *ctx, const float *poses, const int64_t *idx, int V, int B, const float *view0,
                              const float *proj0, const float *grad_view, const float *grad_proj, float *grad_poses,
                              void *stream);

#ifdef __cplusplus
}
#endif
#endif /* DSS_B200_H */
