/*
 * dss_oracle.c -- CPU restatement of the DSS surface-splatting hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under dss_b200/ may import, link or call this
 * file; it exists so that tests/, __graft_entry__.smoke() and bench.py's cpu_baseline
 * leg can check the CUDA path against an independent statement of the reference's
 * algorithm.  Paths cited below are relative to /root/reference.
 *
 * Parity status: the reference ships NO golden vectors or known-answer tests for this
 * path (SURVEY.md section 8c), so this restatement is pinned against outputs of the
 * reference's own CPU code compiled here (oracle/_ref, see oracle/build_ref.py) and the
 * fixtures minted from it under tests/golden/ (tests/golden/make_golden.py).
 *
 * Build: gcc -O2 -ffp-contract=off -fopenmp -shared -fPIC (see oracle/build.py).
 * -ffp-contract=off keeps every fp32 expression a sequence of single IEEE roundings,
 * which is what the reference's x86 CPU build does.  The CUDA reference contracts
 * a*dx*dx + b*dx*dy + c*dy*dy into FMAs; `fma_mode` = 1 reproduces that pattern
 * (pinned from SASS, see DESIGN.md "q contraction").
 *
 * All functions are plain C, OpenMP-parallel over pixels / points (deterministic:
 * every output element is produced by exactly one thread in a fixed order).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#ifdef _OPENMP
#include <omp.h>
#endif

#define ORACLE_API __attribute__((visibility("default")))

/* DSS/csrc/rasterization_utils.cuh:8-11 -- pixel index -> NDC centre. */
static inline float pix_to_ndc(int i, int S) { return -1 + (2 * i + 1.0f) / S; }

/* DSS/csrc/rasterization_utils.cuh:37-43 -- sign-preserving clamp of a denominator.
 * NOTE (hazard 11, DESIGN.md): the CUDA helper maps denom==0 to 0 (sign 0), i.e. 0/0 = NaN
 * when a pixel centre coincides exactly with a point.  The Python helper of the same name
 * (DSS/utils/mathHelper.py:10-14) treats 0 as positive.  We follow the Python/intended
 * semantics: 0 -> +eps, so the contribution is 0/eps = 0. */
static inline float eps_denom_f(float d, float eps) {
    float s = (d < 0.0f) ? -1.0f : 1.0f;
    float a = fabsf(d);
    return s * (a > eps ? a : eps);
}
static inline double eps_denom_d(double d, double eps) {
    double s = (d < 0.0) ? -1.0 : 1.0;
    double a = fabs(d);
    return s * (a > eps ? a : eps);
}

/* q = a dx^2 + b dx dy + c dy^2.  DSS/csrc/rasterize_points.cu:94 (CUDA),
 * DSS/csrc/rasterize_points_cpu.cpp:22-25 (CPU).  Left-to-right: ((a*dx)*dx + (b*dx)*dy) + (c*dy)*dy. */
static inline float qvalue_f(float dx, float dy, float a, float b, float c, int fma_mode) {
    if (fma_mode == 1) {
        /* nvcc -fmad=true contraction of the same expression tree, as the sm_90a SASS of the raster kernels has it
         * (CUDA 12.9: FMUL b*dx, FMUL (b*dx)*dy, FFMA dx*(a*dx) + that, FFMA dy*(c*dy) + that):
         * t = fma(a*dx, dx, (b*dx)*dy) ; q = fma(c*dy, dy, t) */
        const float t = fmaf(a * dx, dx, (b * dx) * dy);
        return fmaf(c * dy, dy, t);
    }
    return a * dx * dx + b * dx * dy + c * dy * dy;
}

ORACLE_API int oracle_num_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}

ORACLE_API void oracle_set_num_threads(int n) {
#ifdef _OPENMP
    omp_set_num_threads(n);
#else
    (void)n;
#endif
}

/* ------------------------------------------------------------------------------------------
 * Per-pixel K-nearest queue.  Spec (SURVEY.md A.2): among accepted candidates keep the K
 * smallest by (z, id) lexicographic, emit ascending.  This is exactly what
 * RasterizePointsNaiveCpu does with its max-heap of (z, idx, q) tuples
 * (DSS/csrc/rasterize_points_cpu.cpp:87-121) and what the CUDA queue
 * (DSS/csrc/rasterize_points.cu:99-123 + BubbleSort rasterization_utils.cuh:22-35) produces
 * when candidates are visited in ascending id and no two accepted z are exactly equal.
 * ---------------------------------------------------------------------------------------- */
typedef struct { float z; int32_t id; float q; } frag_t;

static inline int frag_less(const frag_t *a, const frag_t *b) {
    return (a->z < b->z) || (a->z == b->z && a->id < b->id);
}

/* insert into a sorted array of at most K fragments */
static inline void frag_insert(frag_t *buf, int *n, int K, frag_t f) {
    if (*n == K) {
        if (!frag_less(&f, &buf[K - 1])) return;
        (*n)--;
    }
    int i = *n;
    while (i > 0 && frag_less(&f, &buf[i - 1])) { buf[i] = buf[i - 1]; i--; }
    buf[i] = f;
    (*n)++;
}

/* Acceptance test of one (pixel, point) pair.  DSS/csrc/rasterize_points.cu:79-97.
 * bbox_and = 1 reproduces the CPU twin's `&&` (rasterize_points_cpu.cpp:99, hazard 1). */
static inline int accept_pair(const float *points, const float *radii, const float *ellipse,
                              const float *cutoff, int p, float xf, float yf, int fma_mode,
                              int bbox_and, float *q_out) {
    const float px = points[p * 3 + 0], py = points[p * 3 + 1], pz = points[p * 3 + 2];
    if (pz < 0) return 0;
    const float dx = xf - px, dy = yf - py;
    const float rx = radii[p * 2 + 0], ry = radii[p * 2 + 1];
    if (bbox_and) {
        if (fabsf(dx) > rx && fabsf(dy) > ry) return 0;
    } else {
        if (fabsf(dx) > rx || fabsf(dy) > ry) return 0;
    }
    const float q = qvalue_f(dx, dy, ellipse[p * 3 + 0], ellipse[p * 3 + 1], ellipse[p * 3 + 2], fma_mode);
    if (q > cutoff[p]) return 0;
    *q_out = q;
    return 1;
}

static void emit_pixel(const frag_t *buf, int n, int K, float depth_merge, int32_t *idx,
                       float *zbuf, float *qv, float *occ) {
    for (int k = 0; k < K; ++k) { idx[k] = -1; zbuf[k] = -1.0f; qv[k] = -1.0f; }
    *occ = (n > 0) ? 1.0f : 0.0f;   /* rasterize_points.cu:196-200 / 581-585 */
    for (int k = 0; k < n; ++k) {
        if (buf[k].z - buf[0].z > depth_merge) break;   /* rasterize_points.cu:586-595 */
        idx[k] = buf[k].id; zbuf[k] = buf[k].z; qv[k] = buf[k].q;
    }
}

/* Naive forward: every pixel visits every point of its view.
 * DSS/csrc/rasterize_points.cu:131-212 (spec), rasterize_points_cpu.cpp:27-144 (CPU twin).
 * Output pixel (row r, col c) corresponds to NDC indices yi = S-1-r, xi = S-1-c. */
ORACLE_API void oracle_splat_points_naive(
    const float *points, const float *ellipse, const float *cutoff, const float *radii,
    const int64_t *first_idx, const int64_t *num_pts, int N, float depth_merge, int S, int K,
    int fma_mode, int bbox_and, int32_t *idx, float *zbuf, float *qvalue, float *occ) {
    if (K > 64) K = 64;
#pragma omp parallel for schedule(dynamic, 16)
    for (long pix = 0; pix < (long)N * S * S; ++pix) {
        const int n = (int)(pix / ((long)S * S));
        const int rc = (int)(pix % ((long)S * S));
        const int r = rc / S, c = rc % S;
        const float yf = pix_to_ndc(S - 1 - r, S), xf = pix_to_ndc(S - 1 - c, S);
        frag_t buf[64];
        int nb = 0;
        const int64_t p0 = first_idx[n], p1 = first_idx[n] + num_pts[n];
        for (int64_t p = p0; p < p1; ++p) {
            float q;
            if (accept_pair(points, radii, ellipse, cutoff, (int)p, xf, yf, fma_mode, bbox_and, &q)) {
                frag_t f = {points[p * 3 + 2], (int32_t)p, q};
                frag_insert(buf, &nb, K, f);
            }
        }
        emit_pixel(buf, nb, K, depth_merge, idx + pix * K, zbuf + pix * K, qvalue + pix * K, occ + pix);
    }
}

/* ------------------------------------------------------------------------------------------
 * Coarse binning.  DSS/csrc/rasterize_points.cu:293-432 (kernel), :355-390 (the predicate).
 * Bins live in NDC-index space: bin (by,bx) covers NDC
 *   [PixToNdc(b*bin) - 1/S , PixToNdc((b+1)*bin - 1) + 1/S] on each axis, closed, fp32.
 * Output is CSR: bin_offsets (N*B*B + 1) and bin_ids sorted ascending inside each bin
 * (the reference's within-bin order is chunk/atomic dependent, SURVEY.md A.5, so the
 * comparable object is the sorted id set).  Returns total entries; if bin_ids == NULL only
 * counts (bin_offsets filled).
 * ---------------------------------------------------------------------------------------- */
static inline int bin_overlap_1d(float p0, float p1, int b, int bin_size, int S) {
    const float half_pix = 1.0f / S;
    const float b0 = pix_to_ndc(b * bin_size, S) - half_pix;
    const float b1 = pix_to_ndc((b + 1) * bin_size - 1, S) + half_pix;
    return (p0 <= b1) && (b0 <= p1);
}

ORACLE_API long oracle_rasterize_coarse(
    const float *points, const float *radii, const int64_t *first_idx, const int64_t *num_pts,
    int N, int S, int bin_size, int64_t *bin_offsets, int32_t *bin_ids) {
    const int B = 1 + (S - 1) / bin_size;
    const long nb = (long)N * B * B;
    int64_t *cnt = (int64_t *)calloc((size_t)nb + 1, sizeof(int64_t));
    for (int pass = 0; pass < 2; ++pass) {
        if (pass == 1 && bin_ids == NULL) break;
        for (int n = 0; n < N; ++n) {
            for (int64_t p = first_idx[n]; p < first_idx[n] + num_pts[n]; ++p) {
                const float px = points[p * 3 + 0], py = points[p * 3 + 1], pz = points[p * 3 + 2];
                if (pz < 0) continue;
                const float px0 = px - radii[p * 2 + 0], px1 = px + radii[p * 2 + 0];
                const float py0 = py - radii[p * 2 + 1], py1 = py + radii[p * 2 + 1];
                for (int by = 0; by < B; ++by) {
                    if (!bin_overlap_1d(py0, py1, by, bin_size, S)) continue;
                    for (int bx = 0; bx < B; ++bx) {
                        if (!bin_overlap_1d(px0, px1, bx, bin_size, S)) continue;
                        const long b = ((long)n * B + by) * B + bx;
                        if (pass == 0) cnt[b]++;
                        else bin_ids[bin_offsets[b] + cnt[b]++] = (int32_t)p;
                    }
                }
            }
        }
        if (pass == 0) {
            int64_t run = 0;
            for (long b = 0; b < nb; ++b) { bin_offsets[b] = run; run += cnt[b]; cnt[b] = 0; }
            bin_offsets[nb] = run;
        }
    }
    long total = (long)bin_offsets[nb];
    free(cnt);
    return total;
}

/* Binned forward: same per-pixel semantics as the naive path but candidates come from the
 * pixel's bin (ascending id), i.e. what RasterizePointsFineCuda computes
 * (DSS/csrc/rasterize_points.cu:506-597) given the coarse bins.  Used for sizes where the
 * naive oracle is too slow; tests assert it equals oracle_splat_points_naive on small inputs. */
ORACLE_API void oracle_splat_points_binned(
    const float *points, const float *ellipse, const float *cutoff, const float *radii,
    const int64_t *first_idx, const int64_t *num_pts, int N, float depth_merge, int S, int K,
    int bin_size, int fma_mode, int32_t *idx, float *zbuf, float *qvalue, float *occ) {
    const int B = 1 + (S - 1) / bin_size;
    const long nb = (long)N * B * B;
    int64_t *off = (int64_t *)malloc(((size_t)nb + 1) * sizeof(int64_t));
    long total = oracle_rasterize_coarse(points, radii, first_idx, num_pts, N, S, bin_size, off, NULL);
    int32_t *ids = (int32_t *)malloc((size_t)(total > 0 ? total : 1) * sizeof(int32_t));
    oracle_rasterize_coarse(points, radii, first_idx, num_pts, N, S, bin_size, off, ids);
    if (K > 64) K = 64;
#pragma omp parallel for schedule(dynamic, 16)
    for (long pix = 0; pix < (long)N * S * S; ++pix) {
        const int n = (int)(pix / ((long)S * S));
        const int rc = (int)(pix % ((long)S * S));
        const int r = rc / S, c = rc % S;
        const int yi = S - 1 - r, xi = S - 1 - c;
        const float yf = pix_to_ndc(yi, S), xf = pix_to_ndc(xi, S);
        const long b = ((long)n * B + yi / bin_size) * B + xi / bin_size;
        frag_t buf[64];
        int nbuf = 0;
        for (int64_t j = off[b]; j < off[b + 1]; ++j) {
            const int p = ids[j];
            float q;
            if (accept_pair(points, radii, ellipse, cutoff, p, xf, yf, fma_mode, 0, &q)) {
                frag_t f = {points[p * 3 + 2], p, q};
                frag_insert(buf, &nbuf, K, f);
            }
        }
        emit_pixel(buf, nbuf, K, depth_merge, idx + pix * K, zbuf + pix * K, qvalue + pix * K, occ + pix);
    }
    free(off);
    free(ids);
}

/* ------------------------------------------------------------------------------------------
 * Blend.  DSS/core/renderer.py:53-78 + pytorch3d norm_weighted_sum [ext] (SURVEY.md A.3):
 *   w_k = exp(-0.5 q_k) * scaler[idx_k]   (0 where idx_k < 0: rasterizer.py:631-633)
 *   rgb = sum_k w_k colour[idx_k] / max(sum_k w_k, 1e-4);  out = (rgb, occupancy)
 * colours: (P, C) row-major, C channels (3 for rgb).  out: (N,S,S,C+1).
 * ---------------------------------------------------------------------------------------- */
ORACLE_API void oracle_blend_forward(const int32_t *idx, const float *qvalue, const float *occ,
                                     const float *scaler, const float *colours, long npix, int K,
                                     int C, float *out) {
#pragma omp parallel for
    for (long i = 0; i < npix; ++i) {
        double acc[8] = {0}, wsum = 0.0;
        for (int k = 0; k < K; ++k) {
            const int p = idx[i * K + k];
            if (p < 0) continue;
            const float w = expf(-0.5f * qvalue[i * K + k]) * scaler[p];
            wsum += w;
            for (int ch = 0; ch < C; ++ch) acc[ch] += (double)w * colours[(long)p * C + ch];
        }
        const double den = wsum > 1e-4 ? wsum : 1e-4;
        for (int ch = 0; ch < C; ++ch) out[i * (C + 1) + ch] = (float)(acc[ch] / den);
        out[i * (C + 1) + C] = occ[i];
    }
}

/* Colour backward (pytorch3d norm_weighted_sum backward [ext], SURVEY.md A.4):
 *   dL/dcolour[idx_k] += g_rgb * w_k / max(sum w, 1e-4).   grad_w is discarded upstream
 *   (DSS/core/rasterizer.py:788-813).  grad_image is (N,S,S,C+1); accumulates in double. */
ORACLE_API void oracle_blend_backward_colours(const int32_t *idx, const float *qvalue,
                                              const float *scaler, const float *grad_image,
                                              long npix, int K, int C, long P, float *grad_colours) {
    double *acc = (double *)calloc((size_t)P * C, sizeof(double));
    for (long i = 0; i < npix; ++i) {
        double wsum = 0.0;
        float w[64];
        for (int k = 0; k < K; ++k) {
            const int p = idx[i * K + k];
            w[k] = 0.0f;
            if (p < 0) continue;
            w[k] = expf(-0.5f * qvalue[i * K + k]) * scaler[p];
            wsum += w[k];
        }
        const double den = wsum > 1e-4 ? wsum : 1e-4;
        for (int k = 0; k < K; ++k) {
            const int p = idx[i * K + k];
            if (p < 0) continue;
            for (int ch = 0; ch < C; ++ch)
                acc[(long)p * C + ch] += (double)grad_image[i * (C + 1) + ch] * w[k] / den;
        }
    }
    for (long j = 0; j < P * C; ++j) grad_colours[j] = (float)acc[j];
    free(acc);
}

/* ------------------------------------------------------------------------------------------
 * Visibility: a point is visible iff it appears anywhere in idx at a pixel whose idx[...,0] >= 0
 * (DSS/core/rasterizer.py:854-860; DSS/utils/__init__.py:320-340).
 * ---------------------------------------------------------------------------------------- */
ORACLE_API void oracle_visibility(const int32_t *idx, long npix, int K, long P, uint8_t *vis) {
    memset(vis, 0, (size_t)P);
    for (long i = 0; i < npix; ++i) {
        if (idx[i * K] < 0) continue;
        for (int k = 0; k < K; ++k) {
            const int p = idx[i * K + k];
            if (p >= 0) vis[p] = 1;
        }
    }
}

static int cmp_float(const void *a, const void *b) {
    const float x = *(const float *)a, y = *(const float *)b;
    return (x > y) - (x < y);
}

/* Search radius per view: radii_s * lower-median over the flattened (n_vis, 2) radii of the
 * view's visible points (DSS/core/rasterizer.py:888; torch.median = lower median, hazard 10).
 * Views without visible points get 0. */
ORACLE_API void oracle_search_radius(const float *radii, const uint8_t *vis, const int64_t *first_idx,
                                     const int64_t *num_pts, int N, float radii_s, float *rs) {
    for (int n = 0; n < N; ++n) {
        long m = 0;
        float *tmp = (float *)malloc((size_t)(num_pts[n] > 0 ? num_pts[n] : 1) * 2 * sizeof(float));
        for (int64_t p = first_idx[n]; p < first_idx[n] + num_pts[n]; ++p)
            if (vis[p]) { tmp[m++] = radii[p * 2]; tmp[m++] = radii[p * 2 + 1]; }
        if (m == 0) { rs[n] = 0.0f; free(tmp); continue; }
        qsort(tmp, (size_t)m, sizeof(float), cmp_float);
        rs[n] = tmp[(m - 1) / 2] * radii_s;
        free(tmp);
    }
}

/* ------------------------------------------------------------------------------------------
 * Occupancy backward, "fast" semantics.  DSS/csrc/rasterize_points_backward.cu:85-178 with the
 * grid of DSS/core/rasterizer.py:884-950 treated as the pure accelerator it is (SURVEY.md A.4;
 * hazard 9 -- the dropped corner cell -- NOT reproduced: intended semantics).
 * For every visible point p of view n and every pixel with g = grad_occ != 0:
 *   skip p if pz<0 or |px|>1 or |py|>1;  d2 = dx*dx+dy*dy; skip if d2 > r_n^2;
 *   skip if g>0 and (|dx|>rx or |dy|>ry);
 *   grad_x += dx / eps_denom(d2,1e-10) * g  (same for y).
 * fma_mode selects the rounding of d2 in the disc test (and in the fp32 denominator):
 *   0: dx*dx + dy*dy, two products and a sum rounded apart (the x86 build of the reference);
 *   1: fmaf(dx, dx, dy*dy), what nvcc makes of the same expression (SASS of rasterize_points_backward.cu:150:
 *      FMUL dy*dy, FFMA dx*dx + that) and what both of our gathers compute.
 * Pairs within an ulp of r^2 can fall on different sides in the two modes.
 * grad_f32: fp32 accumulation in ascending pixel order (row-major over the output image);
 * grad_f64: double accumulation of the same fp32 terms' exact values (arbiter).
 * abs_f64 (P,2): per point sum |dx/den*g| and sum |dy/den*g| of those terms, in double -- the scale of a rounding
 * bound for any fp32 summation of them; npairs (P,): the number of contributing (point, pixel) pairs.
 * Every output pointer may be NULL; without abs_f64 and npairs the loop does no extra work.
 * Output (P,2), zero for invisible points.
 * ---------------------------------------------------------------------------------------- */
static inline float occ_d2(float dx, float dy, int fma_mode) {
    return fma_mode ? fmaf(dx, dx, dy * dy) : dx * dx + dy * dy;
}

ORACLE_API void oracle_occ_backward_fast(
    const float *points, const float *radii, const uint8_t *vis, const float *rs,
    const float *grad_occ, const int64_t *first_idx, const int64_t *num_pts, int N, int S,
    int fma_mode, float *grad_f32, double *grad_f64, double *abs_f64, int32_t *npairs) {
    const int stats = abs_f64 != NULL || npairs != NULL;
    for (int n = 0; n < N; ++n) {
        const float r = rs[n], r2 = r * r;
        const int64_t p0 = first_idx[n], p1 = first_idx[n] + num_pts[n];
#pragma omp parallel for schedule(dynamic, 64)
        for (int64_t p = p0; p < p1; ++p) {
            float gx = 0.0f, gy = 0.0f;
            double gxd = 0.0, gyd = 0.0, axd = 0.0, ayd = 0.0;
            int32_t pairs = 0;
            const float px = points[p * 3 + 0], py = points[p * 3 + 1], pz = points[p * 3 + 2];
            const float rx = radii[p * 2 + 0], ry = radii[p * 2 + 1];
            if (vis[p] && !(pz < 0 || fabsf(py) > 1.0f || fabsf(px) > 1.0f)) {
                /* conservative pixel window (the d2 test below is the semantics) */
                int c_lo = (int)floorf((1.0f - (px + r)) * 0.5f * S) - 2, c_hi = (int)ceilf((1.0f - (px - r)) * 0.5f * S) + 2;
                int r_lo = (int)floorf((1.0f - (py + r)) * 0.5f * S) - 2, r_hi = (int)ceilf((1.0f - (py - r)) * 0.5f * S) + 2;
                if (c_lo < 0) c_lo = 0;
                if (r_lo < 0) r_lo = 0;
                if (c_hi > S - 1) c_hi = S - 1;
                if (r_hi > S - 1) r_hi = S - 1;
                for (int row = r_lo; row <= r_hi; ++row) {
                    const float yf = pix_to_ndc(S - 1 - row, S);
                    for (int col = c_lo; col <= c_hi; ++col) {
                        const float g = grad_occ[((long)n * S + row) * S + col];
                        if (g == 0.0f) continue;
                        const float xf = pix_to_ndc(S - 1 - col, S);
                        const float dx = xf - px, dy = yf - py;
                        const float d2 = occ_d2(dx, dy, fma_mode);
                        if (d2 > r2) continue;
                        const int outside = (fabsf(dx) > rx) || (fabsf(dy) > ry);
                        if (g > 0.0f && outside) continue;
                        const float den = eps_denom_f(d2, 1e-10f);
                        gx += dx / den * g;
                        gy += dy / den * g;
                        const double dend = eps_denom_d((double)dx * dx + (double)dy * dy, 1e-10);
                        const double tx = (double)dx / dend * g, ty = (double)dy / dend * g;
                        gxd += tx;
                        gyd += ty;
                        if (stats) {
                            axd += fabs(tx);
                            ayd += fabs(ty);
                            ++pairs;
                        }
                    }
                }
            }
            if (grad_f32) { grad_f32[p * 2] = gx; grad_f32[p * 2 + 1] = gy; }
            if (grad_f64) { grad_f64[p * 2] = gxd; grad_f64[p * 2 + 1] = gyd; }
            if (abs_f64) { abs_f64[p * 2] = axd; abs_f64[p * 2 + 1] = ayd; }
            if (npairs) npairs[p] = pairs;
        }
    }
}

/* Brute-force variant with no pixel window at all: every pixel x every visible point.
 * Validates the window logic above on small inputs (same fma_mode and optional outputs). */
ORACLE_API void oracle_occ_backward_fast_bruteforce(
    const float *points, const float *radii, const uint8_t *vis, const float *rs,
    const float *grad_occ, const int64_t *first_idx, const int64_t *num_pts, int N, int S,
    int fma_mode, double *grad_f64, double *abs_f64, int32_t *npairs) {
    for (int n = 0; n < N; ++n) {
        const float r = rs[n], r2 = r * r;
#pragma omp parallel for schedule(dynamic, 64)
        for (int64_t p = first_idx[n]; p < first_idx[n] + num_pts[n]; ++p) {
            double gxd = 0.0, gyd = 0.0, axd = 0.0, ayd = 0.0;
            int32_t pairs = 0;
            const float px = points[p * 3 + 0], py = points[p * 3 + 1], pz = points[p * 3 + 2];
            const float rx = radii[p * 2 + 0], ry = radii[p * 2 + 1];
            if (vis[p] && !(pz < 0 || fabsf(py) > 1.0f || fabsf(px) > 1.0f)) {
                for (int row = 0; row < S; ++row)
                    for (int col = 0; col < S; ++col) {
                        const float g = grad_occ[((long)n * S + row) * S + col];
                        if (g == 0.0f) continue;
                        const float xf = pix_to_ndc(S - 1 - col, S), yf = pix_to_ndc(S - 1 - row, S);
                        const float dx = xf - px, dy = yf - py;
                        const float d2 = occ_d2(dx, dy, fma_mode);
                        if (d2 > r2) continue;
                        if (g > 0.0f && ((fabsf(dx) > rx) || (fabsf(dy) > ry))) continue;
                        const double dend = eps_denom_d((double)dx * dx + (double)dy * dy, 1e-10);
                        const double tx = (double)dx / dend * g, ty = (double)dy / dend * g;
                        gxd += tx;
                        gyd += ty;
                        axd += fabs(tx);
                        ayd += fabs(ty);
                        ++pairs;
                    }
            }
            grad_f64[p * 2] = gxd;
            grad_f64[p * 2 + 1] = gyd;
            if (abs_f64) { abs_f64[p * 2] = axd; abs_f64[p * 2 + 1] = ayd; }
            if (npairs) npairs[p] = pairs;
        }
    }
}

/* Slow occupancy backward, CUDA semantics.  DSS/csrc/rasterize_points.cu:673-760
 * (CPU twin rasterize_points_cpu.cpp:380-477 differs: eps 1e-8, unsigned max, `&&`; hazard 5).
 * cpu_twin = 1 reproduces the CPU twin so it can be checked against oracle/_ref. */
ORACLE_API void oracle_occ_backward_slow(
    const float *points, const float *radii, const float *grad_occ, const int64_t *first_idx,
    const int64_t *num_pts, int N, int S, float radii_s, int cpu_twin, float *grad) {
    for (int n = 0; n < N; ++n) {
#pragma omp parallel for schedule(dynamic, 64)
        for (int64_t p = first_idx[n]; p < first_idx[n] + num_pts[n]; ++p) {
            float gx = 0.0f, gy = 0.0f;
            const float px = points[p * 3 + 0], py = points[p * 3 + 1], pz = points[p * 3 + 2];
            if (!(pz < 0 || fabsf(py) > 1.0f || fabsf(px) > 1.0f)) {
                const float rxs = radii[p * 2 + 0] * radii_s, rys = radii[p * 2 + 1] * radii_s;
                for (int row = 0; row < S; ++row) {
                    const float yf = pix_to_ndc(S - 1 - row, S);
                    for (int col = 0; col < S; ++col) {
                        const float g = grad_occ[((long)n * S + row) * S + col];
                        if (g == 0.0f) continue;
                        const float xf = pix_to_ndc(S - 1 - col, S);
                        const float dx = xf - px, dy = yf - py;
                        const int outside = (fabsf(dx) > rxs / radii_s) || (fabsf(dy) > rys / radii_s);
                        if (g > 0.0f && outside) continue;
                        if (cpu_twin) { if (fabsf(dx) > rxs && fabsf(dy) > rys) continue; }
                        else          { if (fabsf(dx) > rxs || fabsf(dy) > rys) continue; }
                        const float d2 = dx * dx + dy * dy;
                        const float den = cpu_twin ? (d2 > 1e-8f ? d2 : 1e-8f) : eps_denom_f(d2, 1e-10f);
                        gx += dx / den * g;
                        gy += dy / den * g;
                    }
                }
            }
            grad[p * 2] = gx;
            grad[p * 2 + 1] = gy;
        }
    }
}

/* z-buffer backward.  DSS/csrc/rasterize_points.cu:823-846: z_grad[idx_k] += grad_zbuf_k,
 * skipping zero gradients, stopping at the first idx < 0.  In-place on z_grad (P,). */
ORACLE_API void oracle_zbuf_backward(const int32_t *idx, const float *grad_zbuf, long npix, int K,
                                     float *z_grad) {
    for (long i = 0; i < npix; ++i)
        for (int k = 0; k < K; ++k) {
            const float g = grad_zbuf[i * K + k];
            if (g == 0.0f) continue;
            const int p = idx[i * K + k];
            if (p < 0) break;
            z_grad[p] += g;
        }
}

/* Exclusive int32 scan.  external/prefix_sum/prefix_sum.cu:74-87 (API), :135-205 (algorithm);
 * CPU twin external/FRNN/frnn/csrc/grid/prefix_sum_cpu.cpp:5-23. */
ORACLE_API void oracle_exclusive_scan_i32(const int32_t *in, int n, int32_t *out) {
    int32_t run = 0;
    for (int i = 0; i < n; ++i) { const int32_t v = in[i]; out[i] = run; run += v; }
}

/* 2-D uniform-grid insert.  external/FRNN/frnn/csrc/grid/grid.cu:62-99:
 * cell = clamp((int)((p - min) * delta), 0, res-1); linear id = cx*res_y + cy.
 * points (N,Pmax,2); params (N,6) = min_x,min_y,delta,res_x,res_y,total; outputs
 * grid_cnt (N,G) (must be zeroed by caller), grid_cell (N,Pmax).  The slot index the reference
 * takes from atomicAdd is order-dependent; here slots follow ascending point order. */
ORACLE_API void oracle_insert_points_2d(const float *points, const int64_t *lengths, const float *params,
                                        int N, int P, int G, int32_t *grid_cnt, int32_t *grid_cell,
                                        int32_t *grid_idx) {
    for (int n = 0; n < N; ++n)
        for (int64_t p = 0; p < lengths[n]; ++p) {
            const float minx = params[n * 6 + 0], miny = params[n * 6 + 1], delta = params[n * 6 + 2];
            const int resx = (int)params[n * 6 + 3], resy = (int)params[n * 6 + 4];
            int gx = (int)((points[((long)n * P + p) * 2 + 0] - minx) * delta);
            int gy = (int)((points[((long)n * P + p) * 2 + 1] - miny) * delta);
            gx = gx < resx - 1 ? gx : resx - 1; gx = gx > 0 ? gx : 0;
            gy = gy < resy - 1 ? gy : resy - 1; gy = gy > 0 ? gy : 0;
            const int gs = gx * resy + gy;
            grid_cell[(long)n * P + p] = gs;
            grid_idx[(long)n * P + p] = grid_cnt[(long)n * G + gs]++;
        }
}

/* Counting sort scatter.  external/FRNN/frnn/csrc/grid/counting_sort.cu:5-36. */
ORACLE_API void oracle_counting_sort_2d(const float *points, const int64_t *lengths,
                                        const int32_t *grid_cell, const int32_t *grid_idx,
                                        const int32_t *grid_off, int N, int P, int G,
                                        float *sorted_points, int32_t *sorted_idx) {
    for (int n = 0; n < N; ++n)
        for (int64_t p = 0; p < lengths[n]; ++p) {
            const int cell = grid_cell[(long)n * P + p];
            const int s = grid_off[(long)n * G + cell] + grid_idx[(long)n * P + p];
            sorted_points[((long)n * P + s) * 2 + 0] = points[((long)n * P + p) * 2 + 0];
            sorted_points[((long)n * P + s) * 2 + 1] = points[((long)n * P + p) * 2 + 1];
            sorted_idx[(long)n * P + s] = (int32_t)p;
        }
}

/* ------------------------------------------------------------------------------------------
 * Per-(point, view) preprocess in double precision (arbiter for the fp32 CUDA kernel).
 * DSS/core/rasterizer.py:443-565 (SURVEY.md A.1).  Row-vector convention [x y z 1] . M.
 *   M  : (N,4,4) full projection (world -> clip),  V : (N,4,4) world -> view
 *   pts, nrm : (P0,3) one cloud shared by all views (the `extend`ed cloud of rasterizer.py:236-240)
 *   h  : (N,) or (N*P0,) variance scale, h_stride = 0 or 1 (per view / per splat)
 * Outputs, packed (N*P0, .): ndc (x/t, y/t, z_view), ellipse (a,b,c), radii (rx,ry), scaler, and the
 * 3x2 Jacobian J (d ndc_xy / d world) used to chain gradients back to world space.
 * ---------------------------------------------------------------------------------------- */
ORACLE_API void oracle_preprocess_f64(const float *M, const float *V, const float *pts, const float *nrm,
                                      const float *h, int h_per_splat, int N, long P0, float cutoffC,
                                      float sigma, int S, double *ndc, double *ellipse, double *radii,
                                      double *scaler, double *jac) {
    const double PI = 3.14159265358979323846;
    for (int n = 0; n < N; ++n) {
        const float *Mn = M + n * 16, *Vn = V + n * 16;
#pragma omp parallel for
        for (long i = 0; i < P0; ++i) {
            const long s = (long)n * P0 + i;
            const double p[4] = {pts[i * 3], pts[i * 3 + 1], pts[i * 3 + 2], 1.0};
            double x = 0, y = 0, t = 0, zv = 0;
            for (int k = 0; k < 4; ++k) {
                x += p[k] * Mn[k * 4 + 0]; y += p[k] * Mn[k * 4 + 1];
                t += p[k] * Mn[k * 4 + 3]; zv += p[k] * Vn[k * 4 + 2];
            }
            const double t2 = eps_denom_d(t * t, 1e-17);   /* rasterizer.py:482 */
            const double te = eps_denom_d(t, 1e-17);       /* rasterizer.py:484 */
            double J[3][2];
            for (int k = 0; k < 3; ++k) {                  /* Mk = W @ Jk, rasterizer.py:483-494 */
                J[k][0] = Mn[k * 4 + 0] / te - Mn[k * 4 + 3] * x / t2;
                J[k][1] = Mn[k * 4 + 1] / te - Mn[k * 4 + 3] * y / t2;
            }
            const double nx = nrm[i * 3], ny = nrm[i * 3 + 1], nz = nrm[i * 3 + 2];
            /* Pn = I - n n^T = Sk^T Sk (rasterizer.py:337-341; SURVEY.md 7.2 last bullet) */
            const double Pn[3][3] = {{1 - nx * nx, -nx * ny, -nx * nz},
                                     {-ny * nx, 1 - ny * ny, -ny * nz},
                                     {-nz * nx, -nz * ny, 1 - nz * nz}};
            double T[2][2] = {{0, 0}, {0, 0}};
            for (int a = 0; a < 2; ++a)
                for (int b = 0; b < 2; ++b)
                    for (int k = 0; k < 3; ++k)
                        for (int l = 0; l < 3; ++l) T[a][b] += J[k][a] * Pn[k][l] * J[l][b];
            const double hh = h_per_splat ? h[s] : h[n];
            const double pix = 2.0 / S;
            const double G00 = hh * T[0][0] + sigma * pix * pix, G11 = hh * T[1][1] + sigma * pix * pix;
            const double G01 = hh * 0.5 * (T[0][1] + T[1][0]);
            const double detT = T[0][0] * T[1][1] - T[0][1] * T[1][0];
            const double detG = G00 * G11 - G01 * G01;
            const double a = G11 / detG, b = -2.0 * G01 / detG, c = G00 / detG;  /* rasterizer.py:543-551 */
            const double den = eps_denom_d(4 * a * c - b * b, 1e-17);
            double ry2 = fabs(4 * a * cutoffC / den), rx2 = fabs(4 * c * cutoffC / den); /* :509-519 */
            if (ry2 < 1e-17) ry2 = 1e-17;
            if (rx2 < 1e-17) rx2 = 1e-17;
            double sq = fabs(detG * 4 * PI * PI);
            if (sq < 1e-17) sq = 1e-17;
            const double detMk = sqrt(detT > 0 ? detT : 0);    /* |det(Sk J)| = sqrt(det(J^T Pn J)) */
            ndc[s * 3 + 0] = x / t; ndc[s * 3 + 1] = y / t; ndc[s * 3 + 2] = zv;
            ellipse[s * 3 + 0] = a; ellipse[s * 3 + 1] = b; ellipse[s * 3 + 2] = c;
            radii[s * 2 + 0] = sqrt(rx2); radii[s * 2 + 1] = sqrt(ry2);
            scaler[s] = detMk / eps_denom_d(sqrt(sq), 1e-17);   /* rasterizer.py:558-559 */
            if (jac) for (int k = 0; k < 3; ++k) { jac[s * 6 + k * 2] = J[k][0]; jac[s * 6 + k * 2 + 1] = J[k][1]; }
        }
    }
}

/* ---------------------------------------------------------------------------------------------
 * K nearest neighbours within a radius -- restates the reference's own ground truth FRNNBruteForceCPU
 * (external/FRNN/frnn/csrc/bruteforce/bruteforce_cpu.cpp:8-64): per query of cloud n, over the points of the same
 * cloud, dist = sum_d diff*diff accumulated in dimension order (:41-45); a point qualifies iff dist < r*r (:48,51);
 * the K smallest (dist, index) tuples are kept (max-heap of tuples, :38,46-54) and written in ascending order, the
 * rest stays -1 (:22-23,55-61).  Packed layout: cloud n owns rows [first[n], first[n] + num[n]); indices are local to
 * the cloud.  r <= 0: no radius limit (pytorch3d knn_points, rasterizer.py:308-312).
 * ------------------------------------------------------------------------------------------- */
ORACLE_API void oracle_knn_brute(const float *queries, const int64_t *qfirst, const int64_t *qnum, const float *points,
                                 const int64_t *first, const int64_t *num, int N, int K, float r, float *dists,
                                 int32_t *idxs) {
    const float r2 = r > 0 ? r * r : INFINITY;
    for (int n = 0; n < N; ++n) {
#pragma omp parallel for schedule(dynamic, 64)
        for (int64_t a = 0; a < qnum[n]; ++a) {
            const float *q = queries + (qfirst[n] + a) * 3;
            float bd[64];
            int bi[64];
            int cnt = 0;
            for (int64_t b = 0; b < num[n]; ++b) {
                const float *p = points + (first[n] + b) * 3;
                float dist = 0;
                for (int d = 0; d < 3; ++d) {
                    const float diff = q[d] - p[d];
                    dist += diff * diff;
                }
                if (!(dist < r2)) continue;
                if (cnt == K && !(dist < bd[K - 1])) continue;     /* strict: earlier index wins ties (:51) */
                int k = cnt < K ? cnt : K - 1;
                while (k > 0 && (dist < bd[k - 1])) {              /* equal distances keep index order */
                    bd[k] = bd[k - 1];
                    bi[k] = bi[k - 1];
                    --k;
                }
                bd[k] = dist;
                bi[k] = (int)b;
                if (cnt < K) ++cnt;
            }
            float *od = dists + (qfirst[n] + a) * K;
            int32_t *oi = idxs + (qfirst[n] + a) * K;
            for (int k = 0; k < K; ++k) {
                od[k] = k < cnt ? bd[k] : -1.0f;
                oi[k] = k < cnt ? bi[k] : -1;
            }
        }
    }
}
