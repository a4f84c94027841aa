// mesh_sample.cu -- Poisson-disk samples of a triangle mesh (dss_sample_mesh_poisson_disk), forward only.
//
// The ground truth of the reference's evaluation: MVRDataset.get_pointclouds(num_points) and
// scripts/poisson_sampling.mlx run meshlab's Poisson-disk sampling, a dart throw over a Monte Carlo pool with a radius
// searched until the count is within 0.5 % of the request.  The rule is stated in include/dss_b200.h; this file
// computes it:
//   1. pds_face_kernel   : one thread per face: the fp64 area (0 for an unusable face), the box of the usable faces'
//                          vertices (order-preserving integer atomics) and A_max (atomicMax on the bits of a positive
//                          double, which order like the value).
//   2. pds_weight_kernel : the integer weights W_f, then their 64-bit exclusive scan (exclusive_scan_i64).
//      The host reads the box, A_max and W once (the call's first synchronisation).
//   3. pds_pool_kernel   : one thread per pool sample: three SplitMix64 draws, the face by binary search over the scan,
//                          the point and the face normal.
//   4. per probe radius r: pds_count_kernel / exclusive_scan_i32 / pds_fill_kernel sort the pool into a uniform grid
//      of cell side >= r, then rounds of pds_round_kernel + pds_finish_kernel compute the lexicographically first
//      maximal independent set of the conflict graph in pool order (see pds_round_kernel); the host reads the round
//      state every DSS_PD_CHECK_EVERY rounds.
//   5. pds_flags_kernel / exclusive_scan_i32 / pds_write_kernel: the accepted samples of the returned probe in pool
//      order.
// Integer atomics only, and the selection does not depend on the order inside a cell: the result is the same bits on
// every run.
#include <math.h>

#include "common.cuh"
#include "kernels.cuh"

namespace dss {

constexpr int PDS_THREADS = 256;

struct PdsState {
    int bbox[6];                     // usable faces' vertex box, order-preserving ints
    int usable;
    int pad;
    unsigned long long amax_bits;    // the largest area, as the bits of a positive double
    long long pending;               // samples undecided after the last round (the probe is done at 0)
    long long next;                  // samples the running round leaves undecided
    long long accepted;
    long long rounds;
};

struct PdsGrid {
    double lo[3];
    double cell;
    int res[3];
};

// the j-th output of SplitMix64 seeded with s
__device__ __forceinline__ uint64_t splitmix64(uint64_t s, uint64_t j) {
    uint64_t z = s + j * 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

// the face's vertices, or false when an index lies outside [0, V) or a coordinate is not finite
__device__ __forceinline__ bool pds_face(const float *verts, int64_t V, const int32_t *faces, int64_t f, D3 (&p)[3]) {
    bool ok = true;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int i = faces[f * 3 + k];
        if ((uint64_t)(int64_t)i >= (uint64_t)V) return false;
        const float x = verts[(int64_t)i * 3], y = verts[(int64_t)i * 3 + 1], z = verts[(int64_t)i * 3 + 2];
        ok = ok && isfinite(x) && isfinite(y) && isfinite(z);
        p[k] = d3(x, y, z);
    }
    return ok;
}

// cross(b - a, c - a), each component the two products and then their difference
__device__ __forceinline__ D3 pds_cross(const D3 (&p)[3]) {
    const D3 ab = dsub(p[1], p[0]), ac = dsub(p[2], p[0]);
    return d3(ddiff(ab.y, ac.z, ab.z, ac.y), ddiff(ab.z, ac.x, ab.x, ac.z), ddiff(ab.x, ac.y, ab.y, ac.x));
}

__global__ void pds_init_kernel(PdsState *s) {
    if (threadIdx.x < 6) s->bbox[threadIdx.x] = threadIdx.x < 3 ? INT32_MAX : INT32_MIN;
    if (threadIdx.x == 0) s->usable = 0, s->amax_bits = 0ull;
}

// 1. area_f = 0.5 sqrt(c . c), 0 for an unusable face; the usable faces' box, count and largest area
__global__ void __launch_bounds__(PDS_THREADS) pds_face_kernel(const float *__restrict__ verts, int64_t V,
                                                               const int32_t *__restrict__ faces, int64_t F,
                                                               double *__restrict__ area, PdsState *s) {
    int lo[3] = {INT32_MAX, INT32_MAX, INT32_MAX}, hi[3] = {INT32_MIN, INT32_MIN, INT32_MIN};
    int usable = 0;
    unsigned long long amax = 0ull;
    for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f < F; f += (int64_t)gridDim.x * blockDim.x) {
        D3 p[3];
        double a = 0.0;
        if (pds_face(verts, V, faces, f, p)) {
            const D3 c = pds_cross(p);
            a = __dmul_rn(0.5, __dsqrt_rn(ddot(c, c)));
        }
        area[f] = a > 0.0 ? a : 0.0;
        if (!(a > 0.0)) continue;
        ++usable;
        amax = max(amax, (unsigned long long)__double_as_longlong(a));
        const float v[9] = {(float)p[0].x, (float)p[0].y, (float)p[0].z, (float)p[1].x, (float)p[1].y,
                            (float)p[1].z, (float)p[2].x, (float)p[2].y, (float)p[2].z};
#pragma unroll
        for (int k = 0; k < 9; ++k) {
            lo[k % 3] = min(lo[k % 3], f2ord(v[k]));
            hi[k % 3] = max(hi[k % 3], f2ord(v[k]));
        }
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        lo[k] = __reduce_min_sync(0xffffffffu, lo[k]);
        hi[k] = __reduce_max_sync(0xffffffffu, hi[k]);
    }
    usable = __reduce_add_sync(0xffffffffu, usable);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) amax = max(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    if ((threadIdx.x & 31) == 0 && usable > 0) {
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            atomicMin(&s->bbox[k], lo[k]);
            atomicMax(&s->bbox[3 + k], hi[k]);
        }
        atomicAdd(&s->usable, usable);
        atomicMax(&s->amax_bits, amax);
    }
}

// 2. W_f = max(1, ceil(area_f 2^32 / A_max)) for a usable face, else 0
__global__ void __launch_bounds__(PDS_THREADS) pds_weight_kernel(const double *__restrict__ area, int64_t F,
                                                                 const PdsState *__restrict__ s,
                                                                 int64_t *__restrict__ w) {
    const double amax = __longlong_as_double((long long)s->amax_bits);
    for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f < F; f += (int64_t)gridDim.x * blockDim.x) {
        const double a = area[f];
        w[f] = a > 0.0 ? max((int64_t)1, (int64_t)ceil(__ddiv_rn(__dmul_rn(a, 0x1p32), amax))) : 0;
    }
}

// 3. One thread per pool sample (prefix: the exclusive scan of the weights, the total W at prefix[F] > 0)
__global__ void __launch_bounds__(PDS_THREADS) pds_pool_kernel(const float *__restrict__ verts, int64_t V,
                                                               const int32_t *__restrict__ faces,
                                                               const int64_t *__restrict__ prefix, int64_t F,
                                                               int64_t M, uint64_t seed, float4 *__restrict__ pts,
                                                               float4 *__restrict__ nrm) {
    const uint64_t W = (uint64_t)prefix[F];
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < M; i += (int64_t)gridDim.x * blockDim.x) {
        const uint64_t j = 3 * (uint64_t)i + 1;
        const uint64_t x0 = splitmix64(seed, j), x1 = splitmix64(seed, j + 1), x2 = splitmix64(seed, j + 2);
        const int64_t t = (int64_t)__umul64hi(x0, W);
        // the face with prefix[f] <= t < prefix[f + 1] (a face of weight 0 has an empty range)
        int64_t lo = 0, hi = F;
        while (hi - lo > 1) {
            const int64_t mid = (lo + hi) >> 1;
            if (prefix[mid] <= t) lo = mid;
            else hi = mid;
        }
        D3 p[3];
        pds_face(verts, V, faces, lo, p);   // usable: its weight is positive
        const D3 c = pds_cross(p);
        const double len = __dsqrt_rn(ddot(c, c));
        const double u = (double)(x1 >> 11) * 0x1p-53, v = (double)(x2 >> 11) * 0x1p-53;
        const double su = __dsqrt_rn(u);
        const double w0 = __dsub_rn(1.0, su), w1 = __dmul_rn(su, __dsub_rn(1.0, v)), w2 = __dmul_rn(su, v);
        const double px = __dadd_rn(__dadd_rn(__dmul_rn(w0, p[0].x), __dmul_rn(w1, p[1].x)), __dmul_rn(w2, p[2].x));
        const double py = __dadd_rn(__dadd_rn(__dmul_rn(w0, p[0].y), __dmul_rn(w1, p[1].y)), __dmul_rn(w2, p[2].y));
        const double pz = __dadd_rn(__dadd_rn(__dmul_rn(w0, p[0].z), __dmul_rn(w1, p[1].z)), __dmul_rn(w2, p[2].z));
        pts[i] = make_float4(__double2float_rn(px), __double2float_rn(py), __double2float_rn(pz), 0.0f);
        nrm[i] = make_float4(__double2float_rn(__ddiv_rn(c.x, len)), __double2float_rn(__ddiv_rn(c.y, len)),
                             __double2float_rn(__ddiv_rn(c.z, len)), 0.0f);
    }
}

// 4. The selection grid
__device__ __forceinline__ int pds_axis_cell(double x, double lo, double cell, int res) {
    const double t = floor((x - lo) / cell);
    return (int)fmin(fmax(t, 0.0), (double)(res - 1));
}

__global__ void __launch_bounds__(PDS_THREADS) pds_count_kernel(const float4 *__restrict__ pts, int64_t M,
                                                                const PdsGrid g, int32_t *__restrict__ cell,
                                                                int32_t *__restrict__ counts) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < M; i += (int64_t)gridDim.x * blockDim.x) {
        const float4 p = pts[i];
        const int c = (pds_axis_cell(p.x, g.lo[0], g.cell, g.res[0]) * g.res[1] +
                       pds_axis_cell(p.y, g.lo[1], g.cell, g.res[1])) * g.res[2] +
                      pds_axis_cell(p.z, g.lo[2], g.cell, g.res[2]);
        cell[i] = c;
        atomicAdd(&counts[c], 1);
    }
}

// claims slots by counting the counters back down to zero; the order inside a cell varies, the selection does not
// depend on it
__global__ void __launch_bounds__(PDS_THREADS) pds_fill_kernel(const float4 *__restrict__ pts,
                                                               const float4 *__restrict__ nrm, int64_t M,
                                                               const int32_t *__restrict__ cell,
                                                               const int32_t *__restrict__ offsets,
                                                               int32_t *__restrict__ counts, float4 *__restrict__ spts,
                                                               float4 *__restrict__ snrm, int32_t *__restrict__ scell,
                                                               uint8_t *__restrict__ state) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < M; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = cell[i];
        const int slot = offsets[c] + atomicSub(&counts[c], 1) - 1;
        const float4 p = pts[i];
        spts[slot] = make_float4(p.x, p.y, p.z, __int_as_float((int)i));
        if (snrm) snrm[slot] = nrm[i];
        scell[slot] = c;
        state[slot] = 0;
    }
}

__global__ void pds_round_init_kernel(PdsState *s, int64_t M) {
    s->pending = M, s->next = 0, s->accepted = 0, s->rounds = 0;
}

// Whether p0 (the later sample) and p1 (the earlier) lie closer than r: the rule of include/dss_b200.h, step 3.
__device__ __forceinline__ bool pds_conflict(float4 p0, float4 p1, const float4 *snrm, int k0, int k1, double r,
                                             double r2, int geodesic) {
    const D3 d = dsub(d3(p0.x, p0.y, p0.z), d3(p1.x, p1.y, p1.z));
    const double d2 = ddot(d, d);
    if (!geodesic) return d2 < r2;
    if (d2 == 0.0) return true;
    const double de = __dsqrt_rn(d2);
    if (!(de < r)) return false;
    const float4 m0 = snrm[k0], m1 = snrm[k1];
    const D3 v = d3(__ddiv_rn(d.x, de), __ddiv_rn(d.y, de), __ddiv_rn(d.z, de));
    const double c0 = fmin(fmax(ddot(v, d3(m0.x, m0.y, m0.z)), -1.0), 1.0);
    const double c1 = fmin(fmax(ddot(v, d3(m1.x, m1.y, m1.z)), -1.0), 1.0);
    const double dc = __dsub_rn(c0, c1);
    const double g = fabs(dc) < 1e-4 ? __ddiv_rn(1.0, __dsqrt_rn(__dsub_rn(1.0, __dmul_rn(c0, c1))))
                                     : __ddiv_rn(__dsub_rn(asin(c0), asin(c1)), dc);
    return __dmul_rn(de, fmax(g, 1.0)) < r;
}

// One round of the lexicographically first maximal independent set (Blelloch, Fineman & Shun, 2012), priorities the
// pool indices.  An undecided sample j looks at every earlier sample k (smaller pool index) that conflicts with it:
// if one is accepted, j is rejected; if none is undecided, j is accepted; otherwise j waits.  By induction over the pool
// order each decision is the sequential walk's: a sample is accepted only once every earlier conflicting sample has
// been rejected by that walk, and rejected only because one of them was accepted by it.  States only ever move from
// undecided to final, so reading a neighbour's state while another thread of the same round writes it is harmless: a
// stale "undecided" only makes j wait one more round.  The smallest undecided index is decided in every round, so the
// rounds end.
__global__ void __launch_bounds__(PDS_THREADS) pds_round_kernel(const float4 *__restrict__ spts,
                                                                const float4 *__restrict__ snrm,
                                                                const int32_t *__restrict__ scell,
                                                                const int32_t *__restrict__ offsets, int64_t M,
                                                                const PdsGrid g, double r, double r2, int geodesic,
                                                                uint8_t *state, PdsState *s) {
    if (*(volatile long long *)&s->pending == 0) return;   // the probe is decided: the remaining launches do nothing
    long long waiting = 0, accepted = 0;
    for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < M; j += (int64_t)gridDim.x * blockDim.x) {
        if (state[j] != 0) continue;
        const float4 p = spts[j];
        const int idx = __float_as_int(p.w);
        const int c = scell[j];
        const int cz = c % g.res[2], cy = (c / g.res[2]) % g.res[1], cx = c / (g.res[2] * g.res[1]);
        const int z0 = max(cz - 1, 0), z1 = min(cz + 1, g.res[2] - 1);
        bool wait = false, reject = false;
        for (int x = max(cx - 1, 0); x <= min(cx + 1, g.res[0] - 1) && !reject; ++x)
            for (int y = max(cy - 1, 0); y <= min(cy + 1, g.res[1] - 1) && !reject; ++y) {
                const int base = (x * g.res[1] + y) * g.res[2];
                const int e = offsets[base + z1 + 1];   // the z neighbours of one (x, y) are consecutive cells
                for (int k = offsets[base + z0]; k < e; ++k) {
                    const float4 q = spts[k];
                    if (__float_as_int(q.w) >= idx) continue;
                    const uint8_t sk = *(volatile const uint8_t *)&state[k];
                    if (sk == 2) continue;
                    if (!pds_conflict(p, q, snrm, (int)j, k, r, r2, geodesic)) continue;
                    if (sk == 1) {
                        reject = true;
                        break;
                    }
                    wait = true;
                }
            }
        if (reject) state[j] = 2;
        else if (!wait) state[j] = 1, ++accepted;
        else ++waiting;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        waiting += __shfl_xor_sync(0xffffffffu, waiting, o);
        accepted += __shfl_xor_sync(0xffffffffu, accepted, o);
    }
    if ((threadIdx.x & 31) == 0) {
        if (waiting) atomicAdd((unsigned long long *)&s->next, (unsigned long long)waiting);
        if (accepted) atomicAdd((unsigned long long *)&s->accepted, (unsigned long long)accepted);
    }
}

__global__ void pds_finish_kernel(PdsState *s) {
    if (s->pending != 0) s->pending = s->next, s->rounds += 1;
    s->next = 0;
}

// 5. flags[pool index] = accepted
__global__ void __launch_bounds__(PDS_THREADS) pds_flags_kernel(const float4 *__restrict__ spts,
                                                                const uint8_t *__restrict__ state, int64_t M,
                                                                int32_t *__restrict__ flags) {
    for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < M; j += (int64_t)gridDim.x * blockDim.x)
        flags[__float_as_int(spts[j].w)] = state[j] == 1;
}

__global__ void __launch_bounds__(PDS_THREADS) pds_write_kernel(const float4 *__restrict__ pts,
                                                                const float4 *__restrict__ nrm,
                                                                const int32_t *__restrict__ flags,
                                                                const int32_t *__restrict__ pos, int64_t M,
                                                                float *__restrict__ points,
                                                                float *__restrict__ normals) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < M; i += (int64_t)gridDim.x * blockDim.x) {
        if (!flags[i]) continue;
        const int64_t o = pos[i];
        const float4 p = pts[i], n = nrm[i];
        points[o * 3] = p.x, points[o * 3 + 1] = p.y, points[o * 3 + 2] = p.z;
        normals[o * 3] = n.x, normals[o * 3 + 1] = n.y, normals[o * 3 + 2] = n.z;
    }
}

static float ord_to_float(int i) {
    i = i >= 0 ? i : i ^ 0x7fffffff;
    float f;
    memcpy(&f, &i, 4);
    return f;
}

// Scratch and launch sizes of one call
struct PdsRun {
    dss_ctx *ctx;
    cudaStream_t st;
    int64_t M;
    int geodesic;
    double lo[3], ext[3];
    PdsState *state;
    float4 *pts, *nrm, *spts, *snrm;
    int32_t *cell, *scell, *flags, *pos;
    uint8_t *sel;
    unsigned blocks;

    // the sequential selection at radius r: its count and rounds (the accepted set stays in sel / spts)
    int select(double r, int64_t *n, int *rounds) {
        PdsGrid g;
        const double emax = fmax(ext[0], fmax(ext[1], ext[2]));
        g.cell = fmax(r * (1.0 + 0x1p-20), emax / DSS_PD_GRID);
        int64_t ncell = 1;
        for (int k = 0; k < 3; ++k) {
            g.lo[k] = lo[k];
            const double cnt = floor(ext[k] / g.cell) + 1.0;
            g.res[k] = (int)fmin(cnt, (double)(DSS_PD_GRID + 1));
            ncell *= g.res[k];
        }
        int32_t *counts = nullptr;
        int rc;
        if ((rc = ctx_get(ctx, BUF_PDS_GRID, (size_t)(2 * (ncell + 1)), &counts))) return rc;
        int32_t *offsets = counts + ncell + 1;
        DSS_CUDA_TRY(cudaMemsetAsync(counts, 0, (size_t)(ncell + 1) * sizeof(int32_t), st));
        pds_count_kernel<<<blocks, PDS_THREADS, 0, st>>>(pts, M, g, cell, counts);
        DSS_LAUNCH_CHECK(ctx);
        if ((rc = exclusive_scan_i32(ctx, counts, offsets, ncell + 1, st))) return rc;
        pds_fill_kernel<<<blocks, PDS_THREADS, 0, st>>>(pts, nrm, M, cell, offsets, counts, spts, geodesic ? snrm : nullptr,
                                                        scell, sel);
        DSS_LAUNCH_CHECK(ctx);
        pds_round_init_kernel<<<1, 1, 0, st>>>(state, M);
        DSS_LAUNCH_CHECK(ctx);
        const double r2 = r * r;
        PdsState h;
        for (;;) {
            for (int k = 0; k < DSS_PD_CHECK_EVERY; ++k) {
                pds_round_kernel<<<blocks, PDS_THREADS, 0, st>>>(spts, snrm, scell, offsets, M, g, r, r2, geodesic,
                                                                 sel, state);
                DSS_LAUNCH_CHECK(ctx);
                pds_finish_kernel<<<1, 1, 0, st>>>(state);
                DSS_LAUNCH_CHECK(ctx);
            }
            // a host synchronisation every DSS_PD_CHECK_EVERY rounds
            DSS_CUDA_TRY(cudaMemcpyAsync(&h, state, sizeof(PdsState), cudaMemcpyDeviceToHost, st));
            DSS_CUDA_TRY(cudaStreamSynchronize(st));
            if (h.pending == 0) break;
        }
        *n = h.accepted;
        *rounds = (int)h.rounds;
        return DSS_OK;
    }
};

}  // namespace dss

extern "C" {

int dss_sample_mesh_poisson_disk(dss_ctx *ctx, const float *verts, int64_t V, const int32_t *faces, int64_t F,
                                 int64_t num_samples, int geodesic, uint64_t seed, float *points, float *normals,
                                 int64_t max_out, int64_t *n_out, double *radius, void *stream) {
    using namespace dss;
    cudaStream_t st = (cudaStream_t)stream;
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    DSS_REQUIRE(n_out && radius, "null n_out or radius");
    DSS_REQUIRE(num_samples >= 1, "num_samples must be positive");
    DSS_REQUIRE(num_samples <= (int64_t)INT32_MAX / DSS_PD_MONTECARLO_RATE,
                "the pool of DSS_PD_MONTECARLO_RATE x num_samples samples must stay below 2^31");
    DSS_REQUIRE(V >= 0 && V <= (int64_t)INT32_MAX && F >= 0 && F <= (int64_t)INT32_MAX, "V and F must be in [0, 2^31)");
    DSS_REQUIRE(V == 0 || verts, "verts is null");
    DSS_REQUIRE(F == 0 || faces, "faces is null");
    DSS_REQUIRE(max_out >= 0 && (max_out == 0 || (points && normals)), "null output with a capacity");
    *n_out = 0;
    *radius = 0.0;
    ctx->pd_probes = 0;
    for (int k = 0; k < 4; ++k) ctx->pd_ms[k] = 0.0f;
    if (F == 0 || V == 0) return DSS_OK;
    const int64_t N = num_samples, M = DSS_PD_MONTECARLO_RATE * N;

    PdsRun run;
    run.ctx = ctx, run.st = st, run.M = M, run.geodesic = geodesic ? 1 : 0;
    char *buf = nullptr;
    int rc;
    if ((rc = ctx_get(ctx, BUF_PDS_STATE, sizeof(PdsState), &run.state))) return rc;
    const int64_t tiles = scan_i64_tiles(F);
    if ((rc = ctx_get(ctx, BUF_PDS_FACES, (size_t)(F + F + 1 + tiles) * 8, &buf))) return rc;
    double *area = reinterpret_cast<double *>(buf);
    int64_t *prefix = reinterpret_cast<int64_t *>(buf) + F;
    int64_t *tile_sums = prefix + F + 1;
    cudaEvent_t ev[5];
    for (int k = 0; k < 5; ++k) DSS_CUDA_TRY(cudaEventCreate(&ev[k]));
    struct Release {
        cudaEvent_t *e;
        ~Release() {
            for (int k = 0; k < 5; ++k) cudaEventDestroy(e[k]);
        }
    } release{ev};
    DSS_CUDA_TRY(cudaEventRecord(ev[0], st));

    // 1-2. usable faces, their weights and the 64-bit prefix; host synchronisation 1: box, A_max, W
    const unsigned fb = grid_blocks(F, PDS_THREADS, ctx->sm_count, 8);
    pds_init_kernel<<<1, 32, 0, st>>>(run.state);
    DSS_LAUNCH_CHECK(ctx);
    pds_face_kernel<<<fb, PDS_THREADS, 0, st>>>(verts, V, faces, F, area, run.state);
    DSS_LAUNCH_CHECK(ctx);
    pds_weight_kernel<<<fb, PDS_THREADS, 0, st>>>(area, F, run.state, prefix);
    DSS_LAUNCH_CHECK(ctx);
    if ((rc = exclusive_scan_i64(ctx, prefix, F, tile_sums, st))) return rc;
    PdsState hs;
    int64_t W = 0;
    DSS_CUDA_TRY(cudaMemcpyAsync(&hs, run.state, sizeof(PdsState), cudaMemcpyDeviceToHost, st));
    DSS_CUDA_TRY(cudaMemcpyAsync(&W, prefix + F, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    DSS_CUDA_TRY(cudaStreamSynchronize(st));
    if (hs.usable == 0) return DSS_OK;   // no usable face: no sample
    double amax;
    memcpy(&amax, &hs.amax_bits, 8);
    const double A = (double)(uint64_t)W * amax * 0x1p-32;
    for (int k = 0; k < 3; ++k) {
        run.lo[k] = ord_to_float(hs.bbox[k]);
        run.ext[k] = (double)ord_to_float(hs.bbox[3 + k]) - run.lo[k];
    }

    // 3. the pool; every per-sample array in one slot
    if ((rc = ctx_get(ctx, BUF_PDS_POOL, (size_t)M * 2, &run.pts))) return rc;
    run.nrm = run.pts + M;
    const size_t sorted_bytes = (size_t)M * (2 * sizeof(float4) + 4 * sizeof(int32_t) + 1);
    char *sb = nullptr;
    if ((rc = ctx_get(ctx, BUF_PDS_SORTED, sorted_bytes, &sb))) return rc;
    run.spts = reinterpret_cast<float4 *>(sb);
    run.snrm = run.spts + M;
    run.cell = reinterpret_cast<int32_t *>(run.snrm + M);
    run.scell = run.cell + M;
    run.flags = run.scell + M;
    run.pos = run.flags + M;
    run.sel = reinterpret_cast<uint8_t *>(run.pos + M);
    run.blocks = grid_blocks(M, PDS_THREADS, ctx->sm_count, 8);
    pds_pool_kernel<<<run.blocks, PDS_THREADS, 0, st>>>(verts, V, faces, prefix, F, M, seed, run.pts, run.nrm);
    DSS_LAUNCH_CHECK(ctx);
    DSS_CUDA_TRY(cudaEventRecord(ev[1], st));

    // 4. the radius search (host fp64), one selection per probe
    const int64_t tol = N / 200;
    double r = sqrt(A / (0.7 * M_PI * (double)N)), lo = -1.0, hi = -1.0, best_r = r;
    int64_t best_n = 0, best_d = INT64_MAX;
    int probes = 0, best_p = -1;
    while (probes < DSS_PD_MAX_PROBES) {
        int64_t n;
        int rounds;
        if ((rc = run.select(r, &n, &rounds))) return rc;
        ctx->pd_radii[probes] = r, ctx->pd_counts[probes] = n, ctx->pd_rounds[probes] = rounds;
        const int64_t d = n > N ? n - N : N - n;
        if (d < best_d) best_d = d, best_n = n, best_r = r, best_p = probes;
        ++probes;
        ctx->pd_probes = probes;
        if (d <= tol) break;
        if (n > N) lo = r;
        else hi = r;
        r = hi < 0.0 ? 2.0 * r : lo < 0.0 ? 0.5 * r : 0.5 * (lo + hi);
    }
    DSS_CUDA_TRY(cudaEventRecord(ev[2], st));
    if (best_p != probes - 1) {   // the selection state holds the last probe: select the returned one again
        int64_t n;
        int rounds;
        if ((rc = run.select(best_r, &n, &rounds))) return rc;
    }
    DSS_CUDA_TRY(cudaEventRecord(ev[3], st));
    *n_out = best_n;
    *radius = best_r;
    if (best_n > max_out) {
        set_error("dss_sample_mesh_poisson_disk: %lld samples, the outputs hold %lld", (long long)best_n,
                  (long long)max_out);
        return DSS_E_CAPACITY;
    }

    // 5. the accepted samples in pool order
    pds_flags_kernel<<<run.blocks, PDS_THREADS, 0, st>>>(run.spts, run.sel, M, run.flags);
    DSS_LAUNCH_CHECK(ctx);
    if ((rc = exclusive_scan_i32(ctx, run.flags, run.pos, M, st))) return rc;
    pds_write_kernel<<<run.blocks, PDS_THREADS, 0, st>>>(run.pts, run.nrm, run.flags, run.pos, M, points, normals);
    DSS_LAUNCH_CHECK(ctx);
    DSS_CUDA_TRY(cudaEventRecord(ev[4], st));
    DSS_CUDA_TRY(cudaEventSynchronize(ev[4]));   // for the stage times; the selection reads already waited for the rest
    for (int k = 0; k < 4; ++k) DSS_CUDA_TRY(cudaEventElapsedTime(&ctx->pd_ms[k], ev[k], ev[k + 1]));
    return DSS_OK;
}

int dss_poisson_disk_stats(dss_ctx *ctx, int *probes, double *radii, int64_t *counts, int *rounds, float *stage_ms) {
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    if (probes) *probes = ctx->pd_probes;
    for (int k = 0; k < DSS_PD_MAX_PROBES; ++k) {
        const bool on = k < ctx->pd_probes;
        if (radii) radii[k] = on ? ctx->pd_radii[k] : 0.0;
        if (counts) counts[k] = on ? ctx->pd_counts[k] : 0;
        if (rounds) rounds[k] = on ? ctx->pd_rounds[k] : 0;
    }
    if (stage_ms)
        for (int k = 0; k < 4; ++k) stage_ms[k] = ctx->pd_ms[k];
    return DSS_OK;
}

}  // extern "C"
