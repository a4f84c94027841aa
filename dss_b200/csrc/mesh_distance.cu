// mesh_distance.cu -- exact distances from query points to a triangle mesh (dss_point_mesh_distance), forward only.
//
// The point-to-surface ("p2f") term of the reference's evaluation script (scripts/evaluatePointClouds.py), which read
// it from an external CGAL program.  Every face is the closed convex hull of its three vertices; the distance to a face
// is formed in fp64 by tri_closest below, and the result is the face with the smallest (squared distance, index).
//
// The acceleration structure is a uniform grid over the bounding box of the usable faces, built on the device:
//   1. pmd_bbox_kernel   : one thread per face: the box of the usable faces (order-preserving integer atomics) and
//                          their number.
//   2. pmd_params_kernel : one thread: the cell size from the face density (as knn_params_kernel does for points), at
//                          most PMD_GMAX cells.
//   3. pmd_bin_kernel<0> : every usable face counts itself in every cell its bounding box overlaps (plus a margin of
//                          1e-6 cells, so rounding can only add cells), and adds its cell count to a 64-bit total.
//      The host reads that total once (the call's only synchronisation) to size the reference list.
//   4. exclusive_scan_i32 of the counts, pmd_bin_kernel<1> fills the lists (face indices, any order within a cell).
//   5. pmd_query_kernel  : one thread per query walks cubic shells of cells around its clamped cell, skipping a cell
//                          whose box is farther than the best distance so far, and stops once that distance is below
//                          the distance to every cell not yet visited (see the kernel's comment).
// Integer atomics only: the lists' order within a cell varies from run to run, the minimum does not.
#include <math_constants.h>

#include <cfloat>

#include "common.cuh"
#include "kernels.cuh"

namespace dss {

constexpr int PMD_GMAX = 1 << 21;       // grid cells at most (counts + offsets: 2 x 8 MB)
constexpr int PMD_THREADS = 128;
constexpr double PMD_BIN_MARGIN = 1e-6; // in cells: a face's cell range is widened by this much on each side

struct PmdGrid {
    double gmin[3];
    double cell;
    double scale;       // largest |coordinate| of the box, for the search's rounding slack
    int res[3];
    int nfaces;         // usable faces; 0: every query gets NaN / -1
};

struct PmdState {       // device scratch of one call
    int bbox[6];
    int nfaces;
    int pad;
    unsigned long long total;   // cell references of all usable faces
    PmdGrid grid;
};

// closest point of the closed segment [a, b]; a point when a == b
__device__ __forceinline__ D3 seg_closest(D3 p, D3 a, D3 b) {
    const D3 ab = dsub(b, a), ap = dsub(p, a);
    const double l = ddot(ab, ab);
    const double t = l > 0.0 ? fmin(fmax(__ddiv_rn(ddot(ap, ab), l), 0.0), 1.0) : 0.0;
    return daxpy(a, t, ab);
}

// Closest point of the closed triangle (a, b, c) to p: the Voronoi regions of the vertices, the edges and the interior
// (Ericson, Real-Time Collision Detection, 5.1.5).  A face whose edge vectors have an exactly zero cross product (a
// segment or a point), or whose interior denominator is not positive, takes the closest of its three closed edges
// (first of ab, bc, ca on a tie).  Inputs are float32, so an edge vector is exact in fp64 and a nonzero cross product is
// far above the rounding of the region tests.
__device__ D3 tri_closest(D3 p, D3 a, D3 b, D3 c) {
    const D3 ab = dsub(b, a), ac = dsub(c, a), ap = dsub(p, a), bp = dsub(p, b), cp = dsub(p, c);
    const bool flat = ddiff(ab.y, ac.z, ab.z, ac.y) == 0.0 && ddiff(ab.z, ac.x, ab.x, ac.z) == 0.0 &&
                      ddiff(ab.x, ac.y, ab.y, ac.x) == 0.0;
    if (!flat) {
        const double d1 = ddot(ab, ap), d2 = ddot(ac, ap);
        if (d1 <= 0.0 && d2 <= 0.0) return a;
        const double d3v = ddot(ab, bp), d4 = ddot(ac, bp);
        if (d3v >= 0.0 && d4 <= d3v) return b;
        const double vc = ddiff(d1, d4, d3v, d2);
        if (vc <= 0.0 && d1 >= 0.0 && d3v <= 0.0) {
            const double den = __dsub_rn(d1, d3v);
            return daxpy(a, den > 0.0 ? __ddiv_rn(d1, den) : 0.0, ab);
        }
        const double d5 = ddot(ab, cp), d6 = ddot(ac, cp);
        if (d6 >= 0.0 && d5 <= d6) return c;
        const double vb = ddiff(d5, d2, d1, d6);
        if (vb <= 0.0 && d2 >= 0.0 && d6 <= 0.0) {
            const double den = __dsub_rn(d2, d6);
            return daxpy(a, den > 0.0 ? __ddiv_rn(d2, den) : 0.0, ac);
        }
        const double va = ddiff(d3v, d6, d5, d4);
        const double e43 = __dsub_rn(d4, d3v), e56 = __dsub_rn(d5, d6);
        if (va <= 0.0 && e43 >= 0.0 && e56 >= 0.0) {
            const double den = __dadd_rn(e43, e56);
            return daxpy(b, den > 0.0 ? __ddiv_rn(e43, den) : 0.0, dsub(c, b));
        }
        const double denom = __dadd_rn(__dadd_rn(va, vb), vc);
        if (denom > 0.0) return daxpy(daxpy(a, __ddiv_rn(vb, denom), ab), __ddiv_rn(vc, denom), ac);
    }
    const D3 x0 = seg_closest(p, a, b), x1 = seg_closest(p, b, c), x2 = seg_closest(p, c, a);
    const double s0 = ddot(dsub(p, x0), dsub(p, x0)), s1 = ddot(dsub(p, x1), dsub(p, x1));
    const double s2 = ddot(dsub(p, x2), dsub(p, x2));
    D3 x = x0;
    double s = s0;
    if (s1 < s) x = x1, s = s1;
    if (s2 < s) x = x2;
    return x;
}

// the face's three vertices, or false when an index lies outside [0, V) or a coordinate is not finite
__device__ __forceinline__ bool pmd_face(const int32_t *faces, const float *verts, int64_t V, int64_t f, float (&v)[9]) {
    bool ok = true;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int i = faces[f * 3 + k];
        if ((uint64_t)(int64_t)i >= (uint64_t)V) return false;
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            v[k * 3 + j] = verts[(int64_t)i * 3 + j];
            ok = ok && isfinite(v[k * 3 + j]);
        }
    }
    return ok;
}

__global__ void pmd_init_kernel(PmdState *s) {
    if (threadIdx.x < 6) s->bbox[threadIdx.x] = threadIdx.x < 3 ? INT32_MAX : INT32_MIN;
    if (threadIdx.x == 0) s->nfaces = 0, s->total = 0ull;
}

__global__ void __launch_bounds__(256) pmd_bbox_kernel(const float *__restrict__ verts, int64_t V,
                                                       const int32_t *__restrict__ faces, int64_t F,
                                                       float4 *__restrict__ tris, PmdState *s) {
    int lo[3] = {INT32_MAX, INT32_MAX, INT32_MAX}, hi[3] = {INT32_MIN, INT32_MIN, INT32_MIN};
    int usable = 0;
    for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f < F; f += (int64_t)gridDim.x * blockDim.x) {
        float v[9];
        if (!pmd_face(faces, verts, V, f, v)) continue;
        ++usable;
#pragma unroll
        for (int k = 0; k < 9; ++k) {
            lo[k % 3] = min(lo[k % 3], f2ord(v[k]));
            hi[k % 3] = max(hi[k % 3], f2ord(v[k]));
        }
        // the query kernel reads a face's vertices from one 48-byte record instead of gathering them by index
        tris[f * 3 + 0] = make_float4(v[0], v[1], v[2], 0.0f);
        tris[f * 3 + 1] = make_float4(v[3], v[4], v[5], 0.0f);
        tris[f * 3 + 2] = make_float4(v[6], v[7], v[8], 0.0f);
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        lo[k] = __reduce_min_sync(0xffffffffu, lo[k]);
        hi[k] = __reduce_max_sync(0xffffffffu, hi[k]);
    }
    usable = __reduce_add_sync(0xffffffffu, usable);
    if ((threadIdx.x & 31) == 0 && usable > 0) {
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            atomicMin(&s->bbox[k], lo[k]);
            atomicMax(&s->bbox[3 + k], hi[k]);
        }
        atomicAdd(&s->nfaces, usable);
    }
}

// Cell size from the density: aim at a few faces per occupied cell of a surface with the bounding box's face area,
// never finer than 1/1024 of the largest extent, never more than PMD_GMAX cells.  In fp64, where the extents of
// float32 coordinates cannot overflow.
__global__ void pmd_params_kernel(PmdState *s) {
    PmdGrid g;
    g.nfaces = s->nfaces;
    double e[3];
    g.scale = 0.0;
    for (int k = 0; k < 3; ++k) {
        const double lo = g.nfaces > 0 ? (double)ord2f(s->bbox[k]) : 0.0;
        const double hi = g.nfaces > 0 ? (double)ord2f(s->bbox[3 + k]) : 0.0;
        g.gmin[k] = lo;
        e[k] = hi - lo;
        g.scale = fmax(g.scale, fmax(fabs(lo), fabs(hi)));
    }
    const double emax = fmax(e[0], fmax(e[1], e[2]));
    const double area = 2.0 * (e[0] * e[1] + e[1] * e[2] + e[0] * e[2]);
    double cell = sqrt(2.0 * area / (double)(g.nfaces > 0 ? g.nfaces : 1));
    cell = fmax(cell, emax * (1.0 / 1024.0));
    if (!(cell > 0.0)) cell = 1.0;                                  // no faces, or all of them one point
    for (;;) {
        const double r0 = floor(e[0] / cell) + 1.0, r1 = floor(e[1] / cell) + 1.0, r2 = floor(e[2] / cell) + 1.0;
        if (r0 * r1 * r2 <= (double)PMD_GMAX) break;
        cell *= 1.26;
    }
    g.cell = cell;
    for (int k = 0; k < 3; ++k) g.res[k] = (int)(floor(e[k] / cell) + 1.0);
    s->grid = g;
}

// cell index of coordinate v along one axis, shifted by `margin` cells, clamped into [0, res)
__device__ __forceinline__ int pmd_axis_cell(double v, double gmin, double cell, int res, double margin) {
    const double t = floor((v - gmin) / cell + margin);
    return (int)fmin(fmax(t, 0.0), (double)(res - 1));
}

template <int PASS>   // 0: count, 1: fill (claims slots by counting the same counters back down to zero)
__global__ void __launch_bounds__(256) pmd_bin_kernel(const float *__restrict__ verts, int64_t V,
                                                      const int32_t *__restrict__ faces, int64_t F,
                                                      PmdState *s, int32_t *__restrict__ counts,
                                                      const int32_t *__restrict__ offsets, int32_t *__restrict__ refs) {
    const PmdGrid g = s->grid;
    unsigned long long total = 0;
    for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f < F; f += (int64_t)gridDim.x * blockDim.x) {
        float v[9];
        if (!pmd_face(faces, verts, V, f, v)) continue;
        int c0[3], c1[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const float lo = fminf(fminf(v[k], v[3 + k]), v[6 + k]), hi = fmaxf(fmaxf(v[k], v[3 + k]), v[6 + k]);
            c0[k] = pmd_axis_cell(lo, g.gmin[k], g.cell, g.res[k], -PMD_BIN_MARGIN);
            c1[k] = pmd_axis_cell(hi, g.gmin[k], g.cell, g.res[k], PMD_BIN_MARGIN);
        }
        if (PASS == 0) total += (unsigned long long)(c1[0] - c0[0] + 1) * (c1[1] - c0[1] + 1) * (c1[2] - c0[2] + 1);
        for (int x = c0[0]; x <= c1[0]; ++x)
            for (int y = c0[1]; y <= c1[1]; ++y)
                for (int z = c0[2]; z <= c1[2]; ++z) {
                    const int cell = (x * g.res[1] + y) * g.res[2] + z;
                    if (PASS == 0) atomicAdd(&counts[cell], 1);
                    else refs[offsets[cell] + atomicSub(&counts[cell], 1) - 1] = (int32_t)f;
                }
    }
    if (PASS == 0) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) total += __shfl_xor_sync(0xffffffffu, total, o);
        if ((threadIdx.x & 31) == 0 && total) atomicAdd(&s->total, total);
    }
}

// One thread per query.
//
// The stopping rule.  After a shell, the visited cells form the index box [x0, x1] x [y0, y1] x [z0, z1].  A face none
// of whose cells is visited has, on some axis, its whole cell range below x0 or above x1 (say): its bounding box then
// ends before the plane gmin + x0 cell (the binning margin only widens ranges), so every point of it is at least
// p.x - (gmin + x0 cell) away.  A side at the grid's border (x0 == 0, x1 == res - 1) has no face beyond it, because
// face ranges are clamped into the grid.  So the smallest such distance over the sides not at the border, `reach`,
// bounds every face not yet tested, wherever the query lies, inside the box or far outside it.  Rounding: the computed
// side distances and the computed distance of any face are within a few fp64 ulps of the largest coordinate involved
// (`scale`) of the exact ones, far below delta = 2^-40 scale; so best < (reach - delta)^2 proves that no untested face
// can reach the best (distance, index), and the search stops.  The same margin lets a cell be skipped when its box is
// farther than the best distance: a face's closest point lies in one of its cells, and that cell is then not skipped.
__global__ void __launch_bounds__(PMD_THREADS) pmd_query_kernel(const float *__restrict__ queries, int64_t P,
                                                                const PmdState *__restrict__ s,
                                                                const int32_t *__restrict__ offsets,
                                                                const int32_t *__restrict__ refs,
                                                                const float4 *__restrict__ tris,
                                                                float *__restrict__ sq_dist,
                                                                int32_t *__restrict__ face_idx,
                                                                float *__restrict__ closest,
                                                                int32_t *__restrict__ face_tests) {
    const PmdGrid g = s->grid;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < P; t += (int64_t)gridDim.x * blockDim.x) {
        const float qx = queries[t * 3], qy = queries[t * 3 + 1], qz = queries[t * 3 + 2];
        const D3 p = d3(qx, qy, qz);
        double best = CUDART_INF;
        int bi = INT32_MAX;
        int tests = 0;
        if (g.nfaces > 0 && isfinite(qx) && isfinite(qy) && isfinite(qz)) {
            const double pc[3] = {p.x, p.y, p.z};
            const double delta = fmax(g.scale, fmax(fabs(p.x), fmax(fabs(p.y), fabs(p.z)))) * 0x1p-40;
            int c[3];
#pragma unroll
            for (int k = 0; k < 3; ++k) c[k] = pmd_axis_cell(pc[k], g.gmin[k], g.cell, g.res[k], 0.0);
            for (int ring = 0;; ++ring) {
                int lo[3], hi[3];
#pragma unroll
                for (int k = 0; k < 3; ++k) lo[k] = max(c[k] - ring, 0), hi[k] = min(c[k] + ring, g.res[k] - 1);
                for (int x = lo[0]; x <= hi[0]; ++x)
                    for (int y = lo[1]; y <= hi[1]; ++y) {
                        // the shell: a full z column where x or y is on it, else the two z ends
                        const bool shell_xy = abs(x - c[0]) == ring || abs(y - c[1]) == ring;
                        const int zstep = shell_xy || ring == 0 ? 1 : 2 * ring;
                        for (int z = shell_xy ? lo[2] : c[2] - ring; z <= hi[2]; z += zstep) {
                            if (z < 0) continue;
                            const int ci[3] = {x, y, z};
                            double b2 = 0.0;
#pragma unroll
                            for (int k = 0; k < 3; ++k) {
                                const double l = g.gmin[k] + ci[k] * g.cell, h = g.gmin[k] + (ci[k] + 1) * g.cell;
                                const double dk = fmax(fmax(l - pc[k], pc[k] - h), 0.0);
                                b2 += dk * dk;
                            }
                            const double bd = sqrt(b2) - delta;
                            if (bd > 0.0 && bd * bd > best) continue;
                            const int cell = (x * g.res[1] + y) * g.res[2] + z;
                            const int e = offsets[cell + 1];
                            for (int j = offsets[cell]; j < e; ++j) {
                                const int f = __ldg(&refs[j]);
                                const float4 ta = __ldg(&tris[(int64_t)f * 3]), tb = __ldg(&tris[(int64_t)f * 3 + 1]);
                                const float4 tc = __ldg(&tris[(int64_t)f * 3 + 2]);
                                const D3 xq = tri_closest(p, d3(ta.x, ta.y, ta.z), d3(tb.x, tb.y, tb.z),
                                                          d3(tc.x, tc.y, tc.z));
                                const D3 r = dsub(p, xq);
                                const double d = ddot(r, r);
                                ++tests;
                                if (d < best || (d == best && f < bi)) best = d, bi = f;
                            }
                        }
                    }
                double reach = CUDART_INF;
#pragma unroll
                for (int k = 0; k < 3; ++k) {
                    if (lo[k] > 0) reach = fmin(reach, pc[k] - (g.gmin[k] + lo[k] * g.cell));
                    if (hi[k] < g.res[k] - 1) reach = fmin(reach, (g.gmin[k] + (hi[k] + 1) * g.cell) - pc[k]);
                }
                if (reach == CUDART_INF) break;                       // the whole grid has been visited
                const double r = reach - delta;
                if (r > 0.0 && best < r * r) break;
            }
        }
        const bool hit = bi != INT32_MAX;
        sq_dist[t] = hit ? __double2float_rn(best) : CUDART_NAN_F;
        face_idx[t] = hit ? bi : -1;
        if (closest) {
            D3 xq = d3(CUDART_NAN, CUDART_NAN, CUDART_NAN);
            if (hit) {
                const float4 ta = tris[(int64_t)bi * 3], tb = tris[(int64_t)bi * 3 + 1], tc = tris[(int64_t)bi * 3 + 2];
                xq = tri_closest(p, d3(ta.x, ta.y, ta.z), d3(tb.x, tb.y, tb.z), d3(tc.x, tc.y, tc.z));
            }
            closest[t * 3] = __double2float_rn(xq.x);
            closest[t * 3 + 1] = __double2float_rn(xq.y);
            closest[t * 3 + 2] = __double2float_rn(xq.z);
        }
        if (face_tests) face_tests[t] = tests;
    }
}

}  // namespace dss

extern "C" {

int dss_point_mesh_distance(dss_ctx *ctx, const float *queries, int64_t P, const float *verts, int64_t V,
                            const int32_t *faces, int64_t F, float *sq_dist, int32_t *face_idx, float *closest,
                            int32_t *face_tests, void *stream) {
    using namespace dss;
    cudaStream_t st = (cudaStream_t)stream;
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    DSS_REQUIRE(P >= 0 && V >= 0 && F >= 0, "negative size");
    DSS_REQUIRE(P <= (int64_t)INT32_MAX && V <= (int64_t)INT32_MAX && F <= (int64_t)INT32_MAX,
                "P, V and F must be below 2^31");
    if (P == 0) return DSS_OK;
    DSS_REQUIRE(queries && sq_dist && face_idx, "null query or output array");
    DSS_REQUIRE(V == 0 || verts, "verts is null");
    DSS_REQUIRE(F == 0 || faces, "faces is null");
    PmdState *state = nullptr;
    float4 *tris = nullptr;
    int32_t *counts = nullptr, *offsets = nullptr, *refs = nullptr;
    int rc;
    if ((rc = ctx_get(ctx, BUF_PMD_STATE, 1, &state))) return rc;
    pmd_init_kernel<<<1, 32, 0, st>>>(state);
    DSS_LAUNCH_CHECK(ctx);
    const bool build = F > 0 && V > 0;
    const unsigned fb = grid_blocks(F, 256, ctx->sm_count, 8);
    if (build) {
        if ((rc = ctx_get(ctx, BUF_PMD_TRIS, (size_t)F * 3, &tris))) return rc;
        pmd_bbox_kernel<<<fb, 256, 0, st>>>(verts, V, faces, F, tris, state);
        DSS_LAUNCH_CHECK(ctx);
    }
    pmd_params_kernel<<<1, 1, 0, st>>>(state);
    DSS_LAUNCH_CHECK(ctx);
    if (build) {
        const int64_t ncell = (int64_t)PMD_GMAX + 1;
        if ((rc = ctx_get(ctx, BUF_PMD_COUNTS, (size_t)ncell, &counts))) return rc;
        if ((rc = ctx_get(ctx, BUF_PMD_OFFSETS, (size_t)ncell, &offsets))) return rc;
        DSS_CUDA_TRY(cudaMemsetAsync(counts, 0, (size_t)ncell * sizeof(int32_t), st));
        pmd_bin_kernel<0><<<fb, 256, 0, st>>>(verts, V, faces, F, state, counts, nullptr, nullptr);
        DSS_LAUNCH_CHECK(ctx);
        // the call's one host synchronisation: the size of the reference list (h_pinned[32..]: unused elsewhere)
        unsigned long long *h_total = reinterpret_cast<unsigned long long *>(ctx->h_pinned + 32);
        DSS_CUDA_TRY(cudaMemcpyAsync(h_total, &state->total, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
        DSS_CUDA_TRY(cudaStreamSynchronize(st));
        const unsigned long long total = *h_total;
        if (total >= (unsigned long long)INT32_MAX) {
            set_error("dss_point_mesh_distance: %llu face-cell references exceed 2^31 - 1 (faces far larger than the "
                      "mesh's typical face)", total);
            return DSS_E_CAPACITY;
        }
        if ((rc = ctx_get(ctx, BUF_PMD_REFS, (size_t)(total > 0 ? total : 1), &refs))) return rc;
        if ((rc = exclusive_scan_i32(ctx, counts, offsets, ncell, st))) return rc;
        pmd_bin_kernel<1><<<fb, 256, 0, st>>>(verts, V, faces, F, state, counts, offsets, refs);
        DSS_LAUNCH_CHECK(ctx);
    }
    pmd_query_kernel<<<grid_blocks(P, PMD_THREADS, ctx->sm_count, 16), PMD_THREADS, 0, st>>>(
        queries, P, state, offsets, refs, tris, sq_dist, face_idx, closest, face_tests);
    DSS_LAUNCH_CHECK(ctx);
    return DSS_OK;
}

}  // extern "C"
