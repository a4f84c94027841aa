// poisson.cu -- screened Poisson surface reconstruction on a dense grid (dss_poisson_solve) and the chi = 0 surface of
// a node grid by marching tetrahedra (dss_marching_tetrahedra), forward only.
//
// What the reference's Generator.generate_mesh gets from pymeshlab's surface_reconstruction_screened_poisson(depth=8)
// (DSS/models/point_modeling.py:256-282), restated with first-order (trilinear) elements on the full 2^depth grid.  The
// discretisation is the contract of include/dss_b200.h; the system below is that one divided by h, which leaves its
// solution and its relative residual unchanged:
//   (Kn + alpha w h Q) chi = w G S,   w = occupied cells / usable samples,   S_n = sum_p phi_n(u_p) n_p,
// Kn, G the stencils of K / h and of (D1 x M1 x M1, M1 x D1 x M1, M1 x M1 x D1) / h^2 (1-D factors below).
//
// dss_poisson_solve, per level l = first .. depth (first = min(depth, DSS_POISSON_FIRST_DEPTH)):
//   1. psn_mark_kernel / scan / psn_compact_kernel: the occupied cells, numbered in cell order (cellmap, -1: empty).
//   2. psn_splat_kernel: S (3 x 64-bit fixed point per node) and the symmetric 8 x 8 block of Q of every occupied cell
//      (36 x 64-bit fixed point), integer atomics only: the sums do not depend on the order of the samples.
//   3. psn_rhs_kernel (b, |b|^2 partials), psn_cells_kernel (scaled float blocks), psn_diag_kernel (Jacobi).
//   4. the start: the trilinear prolongation of level l-1's chi (zero at the first level), r = b - A chi.
//   5. Jacobi-preconditioned CG, five launches per iteration; dot products are fp64 per-block partials added in a fixed
//      order by one block.  The state lives on the device: once it is done every later launch returns at once, so the
//      host queues DSS_POISSON_CHECK_EVERY iterations between two reads of the state.
// dss_marching_tetrahedra: count (per node the crossing edges of its 7 directions, per cube its triangles), exclusive
// scans, one host synchronisation for the totals, then the vertex and face writes.
#include <cmath>

#include "common.cuh"
#include "kernels.cuh"

namespace dss {

constexpr int PSN_THREADS = 256;
constexpr double PSN_FIX = 1073741824.0;   // 2^30: |phi n_k| <= 1 and |phi_a phi_b| <= 1, P < 2^31 terms fit in 2^61

struct PsnDomain {          // usable samples' bounding box (order-preserving ints) and count
    int lo[3], hi[3];
    int usable;
    int pad;
};

struct PsnCG {              // the CG state of the current level
    double rz, pq, alpha, beta, rr, bb, rel;
    int iter, done;
    int occ, pad;
};

struct PsnEvents {          // per-level timing (level_ms), released on every return
    cudaEvent_t e[3] = {nullptr, nullptr, nullptr};
    ~PsnEvents() {
        for (cudaEvent_t x : e)
            if (x) cudaEventDestroy(x);
    }
};

struct PsnGrid {            // one level
    double c[3], L;         // the domain (centre and side, the float32 values widened)
    int R, N1;              // cells and nodes per axis
    int64_t nodes, cells;
};

// finite coordinates and normal, |n| > 0; the unit normal in fp64
__device__ __forceinline__ bool psn_sample(const float *pts, const float *nrm, int64_t t, double (&p)[3],
                                           double (&n)[3]) {
    bool ok = true;
    double s = 0.0;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float a = pts[t * 3 + k], b = nrm[t * 3 + k];
        ok = ok && isfinite(a) && isfinite(b);
        p[k] = a, n[k] = b;
        s += (double)b * b;
    }
    if (!ok || !(s > 0.0)) return false;
    const double inv = 1.0 / sqrt(s);
#pragma unroll
    for (int k = 0; k < 3; ++k) n[k] *= inv;
    return true;
}

// u = (p - c) / L + 0.5 in fp64; the cell floor(u R) clamped into [0, R) and the offset inside it
__device__ __forceinline__ int64_t psn_locate(const double (&p)[3], const PsnGrid &g, int (&cell)[3], double (&x)[3]) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const double u = __dadd_rn(__ddiv_rn(__dsub_rn(p[k], g.c[k]), g.L), 0.5);
        const double s = u * g.R;
        const int ci = min(max((int)floor(s), 0), g.R - 1);
        cell[k] = ci;
        x[k] = fmin(fmax(s - ci, 0.0), 1.0);
    }
    return ((int64_t)cell[0] * g.R + cell[1]) * g.R + cell[2];
}

__device__ __forceinline__ int psn_pair(int a, int b) { return a * (15 - a) / 2 + b; }   // a <= b: 0 .. 35

// 1-D factors at node i of [0, R], neighbour offset d in {-1, 0, 1}: M1 / h, K1 h, D1
__device__ __forceinline__ float psn_m(int i, int d, int R) {
    if (d == 0) return (i == 0 || i == R) ? (1.0f / 3.0f) : (2.0f / 3.0f);
    return (i + d < 0 || i + d > R) ? 0.0f : (1.0f / 6.0f);
}
__device__ __forceinline__ float psn_k(int i, int d, int R) {
    if (d == 0) return (i == 0 || i == R) ? 1.0f : 2.0f;
    return (i + d < 0 || i + d > R) ? 0.0f : -1.0f;
}
__device__ __forceinline__ double psn_d(int i, int d, int R) {   // integral of phi_i' phi_{i+d}
    if (d == -1) return i > 0 ? 0.5 : 0.0;
    if (d == 1) return i < R ? -0.5 : 0.0;
    return (i > 0 ? 0.5 : 0.0) - (i < R ? 0.5 : 0.0);
}

__device__ __forceinline__ void psn_node(int64_t n, int N1, int &i, int &j, int &k) {
    const int64_t jk = n % ((int64_t)N1 * N1);
    i = (int)(n / ((int64_t)N1 * N1)), j = (int)(jk / N1), k = (int)(jk % N1);
}

// ---- domain -----------------------------------------------------------------------------------------------------

__global__ void psn_domain_init_kernel(PsnDomain *d) {
    if (threadIdx.x < 3) d->lo[threadIdx.x] = INT32_MAX, d->hi[threadIdx.x] = INT32_MIN;
    if (threadIdx.x == 0) d->usable = 0;
}

__global__ void __launch_bounds__(PSN_THREADS) psn_bbox_kernel(const float *__restrict__ pts,
                                                               const float *__restrict__ nrm, int64_t P, PsnDomain *d) {
    int lo[3] = {INT32_MAX, INT32_MAX, INT32_MAX}, hi[3] = {INT32_MIN, INT32_MIN, INT32_MIN};
    int usable = 0;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < P; t += (int64_t)gridDim.x * blockDim.x) {
        double p[3], n[3];
        if (!psn_sample(pts, nrm, t, p, n)) continue;
        ++usable;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            lo[k] = min(lo[k], f2ord(pts[t * 3 + k]));
            hi[k] = max(hi[k], f2ord(pts[t * 3 + k]));
        }
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        lo[k] = __reduce_min_sync(0xffffffffu, lo[k]);
        hi[k] = __reduce_max_sync(0xffffffffu, hi[k]);
    }
    usable = __reduce_add_sync(0xffffffffu, usable);
    if ((threadIdx.x & 31) == 0 && usable > 0) {
#pragma unroll
        for (int k = 0; k < 3; ++k) atomicMin(&d->lo[k], lo[k]), atomicMax(&d->hi[k], hi[k]);
        atomicAdd(&d->usable, usable);
    }
}

__global__ void psn_fill_kernel(float *__restrict__ v, int64_t n, float value) {
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x)
        v[t] = value;
}

// ---- one level's system -----------------------------------------------------------------------------------------

__global__ void __launch_bounds__(PSN_THREADS) psn_mark_kernel(const float *__restrict__ pts,
                                                               const float *__restrict__ nrm, int64_t P, PsnGrid g,
                                                               int32_t *__restrict__ cellmap) {
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < P; t += (int64_t)gridDim.x * blockDim.x) {
        double p[3], n[3], x[3];
        int cell[3];
        if (!psn_sample(pts, nrm, t, p, n)) continue;
        cellmap[psn_locate(p, g, cell, x)] = 1;
    }
}

// cellmap: 1 / 0 -> the cell's rank among the occupied cells / -1
__global__ void __launch_bounds__(PSN_THREADS) psn_compact_kernel(int32_t *__restrict__ cellmap,
                                                                  const int32_t *__restrict__ scan, int64_t cells) {
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < cells; c += (int64_t)gridDim.x * blockDim.x)
        cellmap[c] = cellmap[c] ? scan[c] : -1;
}

__global__ void psn_level_init_kernel(PsnCG *cg, const int32_t *cellmap, const int32_t *scan, int64_t cells) {
    PsnCG s;
    s.rz = s.pq = s.alpha = s.beta = s.rr = s.bb = s.rel = 0.0;
    s.iter = 0, s.done = 0, s.pad = 0;
    s.occ = scan[cells - 1] + (cellmap[cells - 1] >= 0 ? 1 : 0);
    *cg = s;
}

__global__ void __launch_bounds__(PSN_THREADS) psn_splat_kernel(const float *__restrict__ pts,
                                                                const float *__restrict__ nrm, int64_t P, PsnGrid g,
                                                                const int32_t *__restrict__ cellmap,
                                                                unsigned long long *__restrict__ S,
                                                                unsigned long long *__restrict__ qfix) {
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < P; t += (int64_t)gridDim.x * blockDim.x) {
        double p[3], n[3], x[3];
        int cell[3];
        if (!psn_sample(pts, nrm, t, p, n)) continue;
        const int idx = cellmap[psn_locate(p, g, cell, x)];
        double phi[8];
#pragma unroll
        for (int a = 0; a < 8; ++a)
            phi[a] = ((a & 4) ? x[0] : 1.0 - x[0]) * ((a & 2) ? x[1] : 1.0 - x[1]) * ((a & 1) ? x[2] : 1.0 - x[2]);
#pragma unroll
        for (int a = 0; a < 8; ++a) {
            const int64_t node = ((int64_t)(cell[0] + (a >> 2)) * g.N1 + cell[1] + ((a >> 1) & 1)) * g.N1 + cell[2] +
                                 (a & 1);
#pragma unroll
            for (int k = 0; k < 3; ++k)
                atomicAdd(&S[k * g.nodes + node], (unsigned long long)llrint(phi[a] * n[k] * PSN_FIX));
#pragma unroll
            for (int b = a; b < 8; ++b)
                atomicAdd(&qfix[(int64_t)idx * 36 + psn_pair(a, b)], (unsigned long long)llrint(phi[a] * phi[b] * PSN_FIX));
        }
    }
}

// float blocks alpha w h Q of the occupied cells, full 8 x 8 (row a: the cell's corner a)
__global__ void __launch_bounds__(PSN_THREADS) psn_cells_kernel(const unsigned long long *__restrict__ qfix,
                                                                float *__restrict__ qf, const PsnCG *cg, int usable,
                                                                double h) {
    const int occ = cg->occ;
    const double scale = DSS_POISSON_POINT_WEIGHT * ((double)occ / (double)usable) * h / PSN_FIX;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < (int64_t)occ * 64;
         e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t c = e >> 6;
        const int a = (int)(e >> 3) & 7, b = (int)e & 7;
        qf[e] = (float)((double)(long long)qfix[c * 36 + psn_pair(min(a, b), max(a, b))] * scale);
    }
}

// b = w G S into r, and the per-block partials of |b|^2
__global__ void __launch_bounds__(PSN_THREADS) psn_rhs_kernel(const unsigned long long *__restrict__ S, PsnGrid g,
                                                              const PsnCG *cg, int usable, float *__restrict__ r,
                                                              double *__restrict__ partials) {
    __shared__ double sPart[PSN_THREADS / 32][2];
    const double w = (double)cg->occ / (double)usable / PSN_FIX;
    const int64_t s1 = g.N1, s2 = (int64_t)g.N1 * g.N1;
    double acc2[2] = {0.0, 0.0};
    for (int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; n < g.nodes; n += (int64_t)gridDim.x * blockDim.x) {
        int i, j, k;
        psn_node(n, g.N1, i, j, k);
        double acc = 0.0;
        for (int di = -1; di <= 1; ++di) {
            if (i + di < 0 || i + di > g.R) continue;
            const double mi = psn_m(i, di, g.R), dI = psn_d(i, di, g.R);
            for (int dj = -1; dj <= 1; ++dj) {
                if (j + dj < 0 || j + dj > g.R) continue;
                const double mj = psn_m(j, dj, g.R), dJ = psn_d(j, dj, g.R);
                for (int dk = -1; dk <= 1; ++dk) {
                    if (k + dk < 0 || k + dk > g.R) continue;
                    const double mk = psn_m(k, dk, g.R), dK = psn_d(k, dk, g.R);
                    const int64_t m = n + di * s2 + dj * s1 + dk;
                    acc += dI * mj * mk * (double)(long long)S[m] + mi * dJ * mk * (double)(long long)S[g.nodes + m] +
                           mi * mj * dK * (double)(long long)S[2 * g.nodes + m];
                }
            }
        }
        const float b = (float)(acc * w);
        r[n] = b;
        acc2[0] += (double)b * b;
    }
    const double v = block_sum(acc2, sPart);
    if (threadIdx.x < 2) partials[blockIdx.x * 2 + threadIdx.x] = v;
}

// corner a of node n in its adjacent cell q = 0 .. 7 (the cell at node - (bits of q)), or -1 outside the grid
__device__ __forceinline__ int psn_adjacent(int i, int j, int k, int q, int R, int64_t &cell) {
    const int ci = i - ((q >> 2) & 1), cj = j - ((q >> 1) & 1), ck = k - (q & 1);
    if (ci < 0 || cj < 0 || ck < 0 || ci >= R || cj >= R || ck >= R) return -1;
    cell = ((int64_t)ci * R + cj) * R + ck;
    return q;   // the node is corner q of that cell
}

__global__ void __launch_bounds__(PSN_THREADS) psn_diag_kernel(PsnGrid g, const int32_t *__restrict__ cellmap,
                                                               const float *__restrict__ qf, float *__restrict__ inv) {
    for (int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; n < g.nodes; n += (int64_t)gridDim.x * blockDim.x) {
        int i, j, k;
        psn_node(n, g.N1, i, j, k);
        const float mi = psn_m(i, 0, g.R), mj = psn_m(j, 0, g.R), mk = psn_m(k, 0, g.R);
        float d = psn_k(i, 0, g.R) * mj * mk + mi * psn_k(j, 0, g.R) * mk + mi * mj * psn_k(k, 0, g.R);
        for (int q = 0; q < 8; ++q) {
            int64_t c;
            const int a = psn_adjacent(i, j, k, q, g.R, c);
            if (a < 0) continue;
            const int idx = cellmap[c];
            if (idx >= 0) d += qf[(int64_t)idx * 64 + a * 9];
        }
        inv[n] = 1.0f / d;
    }
}

// q = A p (Kn stencil plus the screening blocks of the adjacent occupied cells); partials of p.q
__global__ void __launch_bounds__(PSN_THREADS) psn_apply_kernel(PsnGrid g, const int32_t *__restrict__ cellmap,
                                                                const float *__restrict__ qf,
                                                                const float *__restrict__ p, float *__restrict__ q,
                                                                double *__restrict__ partials, const PsnCG *cg) {
    __shared__ double sPart[PSN_THREADS / 32][2];
    if (cg->done) return;
    const int64_t s1 = g.N1, s2 = (int64_t)g.N1 * g.N1;
    double acc2[2] = {0.0, 0.0};
    for (int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; n < g.nodes; n += (int64_t)gridDim.x * blockDim.x) {
        int i, j, k;
        psn_node(n, g.N1, i, j, k);
        float mz[3], kz[3];
#pragma unroll
        for (int d = 0; d < 3; ++d) mz[d] = psn_m(k, d - 1, g.R), kz[d] = psn_k(k, d - 1, g.R);
        float acc = 0.0f;
#pragma unroll
        for (int di = -1; di <= 1; ++di) {
            if (i + di < 0 || i + di > g.R) continue;
            const float mi = psn_m(i, di, g.R), ki = psn_k(i, di, g.R);
#pragma unroll
            for (int dj = -1; dj <= 1; ++dj) {
                if (j + dj < 0 || j + dj > g.R) continue;
                const float mj = psn_m(j, dj, g.R), kj = psn_k(j, dj, g.R);
                const float ab = ki * mj + mi * kj, mm = mi * mj;
                const float *row = p + n + di * s2 + dj * s1;
#pragma unroll
                for (int dk = -1; dk <= 1; ++dk) {
                    if (k + dk < 0 || k + dk > g.R) continue;
                    acc += (ab * mz[dk + 1] + mm * kz[dk + 1]) * row[dk];
                }
            }
        }
        for (int qc = 0; qc < 8; ++qc) {
            int64_t c;
            const int a = psn_adjacent(i, j, k, qc, g.R, c);
            if (a < 0) continue;
            const int idx = cellmap[c];
            if (idx < 0) continue;
            const float *blk = qf + (int64_t)idx * 64 + a * 8;
            const int64_t base = n - ((a >> 2) & 1) * s2 - ((a >> 1) & 1) * s1 - (a & 1);   // the cell's corner 0
#pragma unroll
            for (int b = 0; b < 8; ++b) acc += blk[b] * p[base + ((b >> 2) & 1) * s2 + ((b >> 1) & 1) * s1 + (b & 1)];
        }
        q[n] = acc;
        acc2[0] += (double)p[n] * acc;
    }
    const double v = block_sum(acc2, sPart);
    if (threadIdx.x < 2) partials[blockIdx.x * 2 + threadIdx.x] = v;
}

// r = b - q (r holds b); p = r / diag; partials {r.z, r.r}
__global__ void __launch_bounds__(PSN_THREADS) psn_start_kernel(int64_t nodes, const float *__restrict__ q,
                                                                const float *__restrict__ inv, float *__restrict__ r,
                                                                float *__restrict__ p, double *__restrict__ partials) {
    __shared__ double sPart[PSN_THREADS / 32][2];
    double acc[2] = {0.0, 0.0};
    for (int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; n < nodes; n += (int64_t)gridDim.x * blockDim.x) {
        const float rn = r[n] - q[n], z = rn * inv[n];
        r[n] = rn, p[n] = z;
        acc[0] += (double)rn * z, acc[1] += (double)rn * rn;
    }
    const double v = block_sum(acc, sPart);
    if (threadIdx.x < 2) partials[blockIdx.x * 2 + threadIdx.x] = v;
}

// x += alpha p; r -= alpha q; partials {r.z, r.r} of the new residual
__global__ void __launch_bounds__(PSN_THREADS) psn_update_kernel(int64_t nodes, const float *__restrict__ p,
                                                                 const float *__restrict__ q,
                                                                 const float *__restrict__ inv, float *__restrict__ x,
                                                                 float *__restrict__ r, double *__restrict__ partials,
                                                                 const PsnCG *cg) {
    __shared__ double sPart[PSN_THREADS / 32][2];
    if (cg->done) return;
    const float alpha = (float)cg->alpha;
    double acc[2] = {0.0, 0.0};
    for (int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; n < nodes; n += (int64_t)gridDim.x * blockDim.x) {
        x[n] = x[n] + alpha * p[n];
        const float rn = r[n] - alpha * q[n];
        r[n] = rn;
        acc[0] += (double)rn * (rn * inv[n]), acc[1] += (double)rn * rn;
    }
    const double v = block_sum(acc, sPart);
    if (threadIdx.x < 2) partials[blockIdx.x * 2 + threadIdx.x] = v;
}

// p = r / diag + beta p
__global__ void __launch_bounds__(PSN_THREADS) psn_direction_kernel(int64_t nodes, const float *__restrict__ r,
                                                                    const float *__restrict__ inv,
                                                                    float *__restrict__ p, const PsnCG *cg) {
    if (cg->done) return;
    const float beta = (float)cg->beta;
    for (int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; n < nodes; n += (int64_t)gridDim.x * blockDim.x)
        p[n] = r[n] * inv[n] + beta * p[n];
}

// The fixed-order finish of the partials, one block.  MODE 0: |b|^2.  1: the start's {r.z, r.r}.  2: p.q -> alpha.
// 3: an iteration's {r.z, r.r} -> the convergence test and beta.
template <int MODE>
__global__ void __launch_bounds__(PSN_THREADS) psn_finish_kernel(const double *__restrict__ partials, int blocks,
                                                                 PsnCG *cg, double tol, int max_iter) {
    __shared__ double sPart[PSN_THREADS / 32][2];
    __shared__ double sTot[2];
    if (MODE >= 2 && cg->done) return;
    double acc[2] = {0.0, 0.0};
    for (int b = threadIdx.x; b < blocks; b += blockDim.x) acc[0] += partials[b * 2], acc[1] += partials[b * 2 + 1];
    const double v = block_sum(acc, sPart);
    if (threadIdx.x < 2) sTot[threadIdx.x] = v;
    __syncthreads();
    if (threadIdx.x != 0) return;
    if (MODE == 0) {
        cg->bb = sTot[0];
    } else if (MODE == 2) {
        if (sTot[0] > 0.0) cg->alpha = cg->rz / sTot[0];
        else cg->done = 1;     // p = 0 (an exact solution) or a breakdown: stop with the current iterate
    } else {
        const double rz = sTot[0], rr = sTot[1];
        if (MODE == 3) cg->iter += 1;
        cg->rr = rr;
        cg->rel = cg->bb > 0.0 ? sqrt(rr / cg->bb) : 0.0;
        if (cg->rel <= tol || cg->iter >= max_iter || !(rz > 0.0)) cg->done = 1;
        cg->beta = MODE == 3 && cg->rz != 0.0 ? rz / cg->rz : 0.0;
        cg->rz = rz;
    }
}

// chi of level R from level R/2 (coarse, nodes (R/2 + 1)^3): the trilinear interpolant at the fine nodes
__global__ void __launch_bounds__(PSN_THREADS) psn_prolong_kernel(const float *__restrict__ coarse, PsnGrid g,
                                                                  float *__restrict__ x) {
    const int Nc = g.R / 2 + 1;
    for (int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; n < g.nodes; n += (int64_t)gridDim.x * blockDim.x) {
        int i, j, k;
        psn_node(n, g.N1, i, j, k);
        float v = 0.0f;
        const float wi = (i & 1) ? 0.5f : 1.0f, wj = (j & 1) ? 0.5f : 1.0f, wk = (k & 1) ? 0.5f : 1.0f;
        for (int a = i >> 1; a <= (i + 1) >> 1; ++a)
            for (int b = j >> 1; b <= (j + 1) >> 1; ++b)
                for (int c = k >> 1; c <= (k + 1) >> 1; ++c) v += wi * wj * wk * coarse[((int64_t)a * Nc + b) * Nc + c];
        x[n] = v;
    }
}

// ---- marching tetrahedra ----------------------------------------------------------------------------------------

// The 6 Kuhn tetrahedra of a cube around its corner 0 - corner 7 diagonal (corner bits x = 4, y = 2, z = 1), one per
// order of the axes (xyz, xzy, yxz, yzx, zxy, zyx), each listed with a positive orientation.
__constant__ int8_t MT_TETS[6][4] = {{0, 4, 6, 7}, {0, 5, 4, 7}, {0, 6, 2, 7}, {0, 2, 3, 7}, {0, 1, 5, 7}, {0, 3, 1, 7}};
// for local vertex i, the other three ordered so that (i, j, k, l) is an even permutation: (j, k, l) faces away from i
__constant__ int8_t MT_OPP[4][3] = {{1, 2, 3}, {0, 3, 2}, {0, 1, 3}, {0, 2, 1}};

struct MtTotals {
    unsigned long long verts, faces;
};

__device__ __forceinline__ int mt_tet_faces(int inside4) {
    const int c = __popc(inside4);
    return c == 2 ? 2 : (c == 1 || c == 3) ? 1 : 0;
}

// inside bits of a cube's 8 corners -> its triangle count
__device__ __forceinline__ int mt_cube_faces(int inside8) {
    if (inside8 == 0 || inside8 == 255) return 0;
    int f = 0;
#pragma unroll
    for (int t = 0; t < 6; ++t) {
        int m = 0;
#pragma unroll
        for (int v = 0; v < 4; ++v) m |= ((inside8 >> MT_TETS[t][v]) & 1) << v;
        f += mt_tet_faces(m);
    }
    return f;
}

// per node: the crossing mask of its 7 directions (bit m, m = 4 dx + 2 dy + dz) and their number; per cube (the node
// its corner 0): the triangle count.  64-bit totals.
__global__ void __launch_bounds__(PSN_THREADS) mt_count_kernel(const float *__restrict__ chi, int R,
                                                               uint8_t *__restrict__ mask, int32_t *__restrict__ vcnt,
                                                               int32_t *__restrict__ fcnt, MtTotals *tot) {
    const int N1 = R + 1;
    const int64_t nodes = (int64_t)N1 * N1 * N1, s1 = N1, s2 = (int64_t)N1 * N1;
    unsigned long long tv = 0, tf = 0;
    for (int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; n < nodes; n += (int64_t)gridDim.x * blockDim.x) {
        int i, j, k;
        psn_node(n, N1, i, j, k);
        int in8 = 0, valid = 0;
#pragma unroll
        for (int a = 0; a < 8; ++a) {
            const int dx = a >> 2, dy = (a >> 1) & 1, dz = a & 1;
            if (i + dx > R || j + dy > R || k + dz > R) continue;
            valid |= 1 << a;
            in8 |= (chi[n + dx * s2 + dy * s1 + dz] < 0.0f ? 1 : 0) << a;
        }
        const int a0 = in8 & 1;
        int m = 0;
#pragma unroll
        for (int d = 1; d < 8; ++d)
            if (((valid >> d) & 1) && ((in8 >> d) & 1) != a0) m |= 1 << d;
        mask[n] = (uint8_t)m;
        vcnt[n] = __popc(m);
        tv += __popc(m);
        if (i < R && j < R && k < R) {
            const int f = mt_cube_faces(in8);
            fcnt[((int64_t)i * R + j) * R + k] = f;
            tf += f;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        tv += __shfl_xor_sync(0xffffffffu, tv, o);
        tf += __shfl_xor_sync(0xffffffffu, tf, o);
    }
    if ((threadIdx.x & 31) == 0) {
        if (tv) atomicAdd(&tot->verts, tv);
        if (tf) atomicAdd(&tot->faces, tf);
    }
}

// one vertex per crossing edge (a, a + d), at t = (0 - chi_a) / (chi_b - chi_a) from a:
//   g = i + t along the axes of d (i elsewhere);  world = c + (g h - 0.5) L,  every operation rounded on its own
__global__ void __launch_bounds__(PSN_THREADS) mt_verts_kernel(const float *__restrict__ chi, int R,
                                                               const uint8_t *__restrict__ mask,
                                                               const int32_t *__restrict__ vbase, float cx, float cy,
                                                               float cz, float L, float *__restrict__ verts) {
    const int N1 = R + 1;
    const int64_t nodes = (int64_t)N1 * N1 * N1, s1 = N1, s2 = (int64_t)N1 * N1;
    const float h = 1.0f / (float)R, c[3] = {cx, cy, cz};
    for (int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; n < nodes; n += (int64_t)gridDim.x * blockDim.x) {
        const int m = mask[n];
        if (!m) continue;
        int ijk[3];
        psn_node(n, N1, ijk[0], ijk[1], ijk[2]);
        const float ca = chi[n];
        int64_t out = vbase[n];
        for (int d = 1; d < 8; ++d) {
            if (!((m >> d) & 1)) continue;
            const int dd[3] = {d >> 2, (d >> 1) & 1, d & 1};
            const float cb = chi[n + dd[0] * s2 + dd[1] * s1 + dd[2]];
            const float t = __fdiv_rn(__fsub_rn(0.0f, ca), __fsub_rn(cb, ca));
#pragma unroll
            for (int a = 0; a < 3; ++a) {
                const float g = dd[a] ? __fadd_rn((float)ijk[a], t) : (float)ijk[a];
                verts[out * 3 + a] = __fadd_rn(c[a], __fmul_rn(__fsub_rn(__fmul_rn(g, h), 0.5f), L));
            }
            ++out;
        }
    }
}

// vertex of the crossing edge between cube corners a and b (comparable corners: the start is a & b, d = a ^ b)
__device__ __forceinline__ int32_t mt_vid(int64_t n0, int a, int b, int64_t s2, int64_t s1,
                                          const uint8_t *__restrict__ mask, const int32_t *__restrict__ vbase) {
    const int s = a & b, d = a ^ b;
    const int64_t node = n0 + ((s >> 2) & 1) * s2 + ((s >> 1) & 1) * s1 + (s & 1);
    return vbase[node] + __popc(mask[node] & ((1 << d) - 1));
}

__global__ void __launch_bounds__(PSN_THREADS) mt_faces_kernel(const float *__restrict__ chi, int R,
                                                               const uint8_t *__restrict__ mask,
                                                               const int32_t *__restrict__ vbase,
                                                               const int32_t *__restrict__ fbase,
                                                               int32_t *__restrict__ faces) {
    const int N1 = R + 1;
    const int64_t cubes = (int64_t)R * R * R, s1 = N1, s2 = (int64_t)N1 * N1;
    for (int64_t cu = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; cu < cubes; cu += (int64_t)gridDim.x * blockDim.x) {
        const int i = (int)(cu / ((int64_t)R * R)), j = (int)((cu / R) % R), k = (int)(cu % R);
        const int64_t n0 = ((int64_t)i * N1 + j) * N1 + k;
        int in8 = 0;
#pragma unroll
        for (int a = 0; a < 8; ++a) in8 |= (chi[n0 + ((a >> 2) & 1) * s2 + ((a >> 1) & 1) * s1 + (a & 1)] < 0.0f) << a;
        if (in8 == 0 || in8 == 255) continue;
        int64_t out = fbase[cu];
        for (int t = 0; t < 6; ++t) {
            int cv[4], m = 0;
#pragma unroll
            for (int v = 0; v < 4; ++v) cv[v] = MT_TETS[t][v], m |= ((in8 >> cv[v]) & 1) << v;
            const int cnt = __popc(m);
            if (cnt == 0 || cnt == 4) continue;
            int32_t tri[2][3];
            int ntri = 1;
            if (cnt == 1 || cnt == 3) {
                // the lone vertex o; (j, k, l) faces away from it: keep that order when o is inside, reverse it else
                const int o = __ffs(cnt == 1 ? m : (~m & 15)) - 1;
                const int j0 = MT_OPP[o][0], j1 = cnt == 1 ? MT_OPP[o][1] : MT_OPP[o][2],
                          j2 = cnt == 1 ? MT_OPP[o][2] : MT_OPP[o][1];
                tri[0][0] = mt_vid(n0, cv[o], cv[j0], s2, s1, mask, vbase);
                tri[0][1] = mt_vid(n0, cv[o], cv[j1], s2, s1, mask, vbase);
                tri[0][2] = mt_vid(n0, cv[o], cv[j2], s2, s1, mask, vbase);
            } else {
                // inside i0 < i1, outside o0 < o1, swapped when (i0, i1, o0, o1) is an odd permutation; the quad
                // (i0o0, i0o1, i1o1, i1o0) is split along i0o0 - i1o1
                int ins[2], outs[2], ni = 0, no = 0;
#pragma unroll
                for (int v = 0; v < 4; ++v) {
                    if ((m >> v) & 1) ins[ni++] = v;
                    else outs[no++] = v;
                }
                const int perm[4] = {ins[0], ins[1], outs[0], outs[1]};
                int inv = 0;
#pragma unroll
                for (int a = 0; a < 4; ++a)
#pragma unroll
                    for (int b = a + 1; b < 4; ++b) inv += perm[a] > perm[b];
                if (inv & 1) {
                    const int tmp = outs[0];
                    outs[0] = outs[1], outs[1] = tmp;
                }
                const int32_t q0 = mt_vid(n0, cv[ins[0]], cv[outs[0]], s2, s1, mask, vbase);
                const int32_t q1 = mt_vid(n0, cv[ins[0]], cv[outs[1]], s2, s1, mask, vbase);
                const int32_t q2 = mt_vid(n0, cv[ins[1]], cv[outs[1]], s2, s1, mask, vbase);
                const int32_t q3 = mt_vid(n0, cv[ins[1]], cv[outs[0]], s2, s1, mask, vbase);
                tri[0][0] = q0, tri[0][1] = q1, tri[0][2] = q2;
                tri[1][0] = q0, tri[1][1] = q2, tri[1][2] = q3;
                ntri = 2;
            }
            for (int f = 0; f < ntri; ++f, ++out)
#pragma unroll
                for (int a = 0; a < 3; ++a) faces[out * 3 + a] = tri[f][a];
        }
    }
}

}  // namespace dss

extern "C" {

int dss_poisson_solve(dss_ctx *ctx, const float *points, const float *normals, int64_t P, int depth, float *chi,
                      float *center, float *side, int *iterations, double *residual, int *level_iterations,
                      float *level_ms, void *stream) {
    using namespace dss;
    cudaStream_t st = (cudaStream_t)stream;
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    DSS_REQUIRE(depth >= 2 && depth <= DSS_POISSON_MAX_DEPTH, "depth must lie in [2, 9]");
    DSS_REQUIRE(P >= 0 && P <= (int64_t)INT32_MAX, "P out of range");
    DSS_REQUIRE(chi && center && side, "null output");
    DSS_REQUIRE(P == 0 || (points && normals), "null points or normals");
    const int Rf = 1 << depth;
    const int64_t NU = (int64_t)(Rf + 1) * (Rf + 1) * (Rf + 1);
    const int first = depth < DSS_POISSON_FIRST_DEPTH ? depth : DSS_POISSON_FIRST_DEPTH;
    if (iterations) *iterations = 0;
    if (residual) *residual = 0.0;
    if (level_iterations)
        for (int l = 0; l <= depth; ++l) level_iterations[l] = 0;
    if (level_ms)
        for (int l = 0; l < 2 * (depth + 1); ++l) level_ms[l] = 0.0f;
    center[0] = center[1] = center[2] = 0.0f;
    *side = 0.0f;

    // the state slot: the domain, the CG state, then the partials
    const unsigned nb = grid_blocks(NU, PSN_THREADS, ctx->sm_count, 4);
    const size_t state_bytes = 256 + (size_t)nb * 2 * sizeof(double);
    char *state = nullptr;
    int rc;
    if ((rc = ctx_get(ctx, BUF_PSN_STATE, state_bytes, &state))) return rc;
    PsnDomain *dom = reinterpret_cast<PsnDomain *>(state);
    PsnCG *cg = reinterpret_cast<PsnCG *>(state + 64);
    double *partials = reinterpret_cast<double *>(state + 256);

    // 1. the domain (host synchronisation 1: the box and the number of usable samples)
    psn_domain_init_kernel<<<1, 32, 0, st>>>(dom);
    DSS_LAUNCH_CHECK(ctx);
    const unsigned pb = grid_blocks(P, PSN_THREADS, ctx->sm_count, 8);
    if (P > 0) {
        psn_bbox_kernel<<<pb, PSN_THREADS, 0, st>>>(points, normals, P, dom);
        DSS_LAUNCH_CHECK(ctx);
    }
    PsnDomain *h_dom = reinterpret_cast<PsnDomain *>(ctx->h_pinned + 40);
    DSS_CUDA_TRY(cudaMemcpyAsync(h_dom, dom, sizeof(PsnDomain), cudaMemcpyDeviceToHost, st));
    DSS_CUDA_TRY(cudaStreamSynchronize(st));
    const PsnDomain d = *h_dom;
    double ext = 0.0;
    float cf[3] = {0.0f, 0.0f, 0.0f};
    if (d.usable > 0) {
        for (int k = 0; k < 3; ++k) {
            int lo = d.lo[k], hi = d.hi[k];
            float flo, fhi;
            lo = lo >= 0 ? lo : lo ^ 0x7fffffff, hi = hi >= 0 ? hi : hi ^ 0x7fffffff;
            memcpy(&flo, &lo, 4), memcpy(&fhi, &hi, 4);
            cf[k] = (float)(0.5 * ((double)flo + (double)fhi));
            ext = fmax(ext, (double)fhi - (double)flo);
        }
    }
    const float Lf = (float)(1.1 * ext);
    center[0] = cf[0], center[1] = cf[1], center[2] = cf[2];
    *side = Lf;
    const unsigned gb = grid_blocks(NU, PSN_THREADS, ctx->sm_count, 8);
    if (d.usable == 0 || !(Lf > 0.0f)) {
        // no usable sample, or all of them one point: everything is outside, the surface is empty
        psn_fill_kernel<<<gb, PSN_THREADS, 0, st>>>(chi, NU, 1.0f);
        DSS_LAUNCH_CHECK(ctx);
        return DSS_OK;
    }

    // workspace: 8 node arrays of the finest level (cellmap, r, then S over 6 of them: p, q, 1 / diag once S is used)
    float *grid = nullptr, *coarse = nullptr;
    char *cells = nullptr;
    const int64_t ncap = (int64_t)d.usable < (int64_t)Rf * Rf * Rf ? (int64_t)d.usable : (int64_t)Rf * Rf * Rf;
    if ((rc = ctx_get(ctx, BUF_PSN_GRID, (size_t)NU * 8, &grid))) return rc;
    if ((rc = ctx_get(ctx, BUF_PSN_COARSE, (size_t)(Rf / 2 + 1) * (Rf / 2 + 1) * (Rf / 2 + 1), &coarse))) return rc;
    if ((rc = ctx_get(ctx, BUF_PSN_CELLS, (size_t)ncap * (36 * 8 + 64 * 4), &cells))) return rc;
    int32_t *cellmap = reinterpret_cast<int32_t *>(grid);
    float *r = grid + NU;
    unsigned long long *S = reinterpret_cast<unsigned long long *>(grid + 2 * NU);
    float *p = grid + 2 * NU, *q = grid + 3 * NU, *inv = grid + 4 * NU;
    unsigned long long *qfix = reinterpret_cast<unsigned long long *>(cells);
    float *qf = reinterpret_cast<float *>(cells + (size_t)ncap * 36 * 8);
    PsnCG *h_cg = reinterpret_cast<PsnCG *>(ctx->h_pinned + 48);

    PsnEvents events;
    cudaEvent_t *ev = events.e;
    if (level_ms)
        for (int e = 0; e < 3; ++e) DSS_CUDA_TRY(cudaEventCreate(&ev[e]));
    rc = DSS_OK;
    for (int l = first; l <= depth && rc == DSS_OK; ++l) {
        PsnGrid g;
        for (int k = 0; k < 3; ++k) g.c[k] = cf[k];
        g.L = Lf, g.R = 1 << l, g.N1 = g.R + 1;
        g.nodes = (int64_t)g.N1 * g.N1 * g.N1, g.cells = (int64_t)g.R * g.R * g.R;
        const double h = 1.0 / g.R;
        const unsigned nbl = grid_blocks(g.nodes, PSN_THREADS, ctx->sm_count, 4);
        if (level_ms) DSS_CUDA_TRY(cudaEventRecord(ev[0], st));
        // 1. occupied cells
        DSS_CUDA_TRY(cudaMemsetAsync(cellmap, 0, (size_t)g.cells * sizeof(int32_t), st));
        psn_mark_kernel<<<pb, PSN_THREADS, 0, st>>>(points, normals, P, g, cellmap);
        DSS_LAUNCH_CHECK(ctx);
        int32_t *scan = reinterpret_cast<int32_t *>(r);
        if ((rc = exclusive_scan_i32(ctx, cellmap, scan, g.cells, st))) break;
        psn_compact_kernel<<<grid_blocks(g.cells, PSN_THREADS, ctx->sm_count, 8), PSN_THREADS, 0, st>>>(cellmap, scan,
                                                                                                        g.cells);
        DSS_LAUNCH_CHECK(ctx);
        psn_level_init_kernel<<<1, 1, 0, st>>>(cg, cellmap, scan, g.cells);
        DSS_LAUNCH_CHECK(ctx);
        // 2. S and the blocks of Q
        DSS_CUDA_TRY(cudaMemsetAsync(S, 0, (size_t)g.nodes * 3 * sizeof(unsigned long long), st));
        DSS_CUDA_TRY(cudaMemsetAsync(qfix, 0, (size_t)ncap * 36 * sizeof(unsigned long long), st));
        psn_splat_kernel<<<pb, PSN_THREADS, 0, st>>>(points, normals, P, g, cellmap, S, qfix);
        DSS_LAUNCH_CHECK(ctx);
        // 3. b, the float blocks, 1 / diag
        psn_cells_kernel<<<grid_blocks(ncap * 64, PSN_THREADS, ctx->sm_count, 8), PSN_THREADS, 0, st>>>(
            qfix, qf, cg, d.usable, h);
        DSS_LAUNCH_CHECK(ctx);
        psn_rhs_kernel<<<nbl, PSN_THREADS, 0, st>>>(S, g, cg, d.usable, r, partials);
        DSS_LAUNCH_CHECK(ctx);
        psn_finish_kernel<0><<<1, PSN_THREADS, 0, st>>>(partials, (int)nbl, cg, 0.0, 0);
        DSS_LAUNCH_CHECK(ctx);
        psn_diag_kernel<<<nbl, PSN_THREADS, 0, st>>>(g, cellmap, qf, inv);
        DSS_LAUNCH_CHECK(ctx);
        // 4. the start
        if (l == first) {
            DSS_CUDA_TRY(cudaMemsetAsync(chi, 0, (size_t)g.nodes * sizeof(float), st));
        } else {
            psn_prolong_kernel<<<nbl, PSN_THREADS, 0, st>>>(coarse, g, chi);
            DSS_LAUNCH_CHECK(ctx);
        }
        psn_apply_kernel<<<nbl, PSN_THREADS, 0, st>>>(g, cellmap, qf, chi, q, partials, cg);
        DSS_LAUNCH_CHECK(ctx);
        psn_start_kernel<<<nbl, PSN_THREADS, 0, st>>>(g.nodes, q, inv, r, p, partials);
        DSS_LAUNCH_CHECK(ctx);
        psn_finish_kernel<1><<<1, PSN_THREADS, 0, st>>>(partials, (int)nbl, cg, DSS_POISSON_TOLERANCE,
                                                        DSS_POISSON_MAX_ITERATIONS);
        DSS_LAUNCH_CHECK(ctx);
        if (level_ms) DSS_CUDA_TRY(cudaEventRecord(ev[1], st));
        // 5. CG; the host reads the state once every DSS_POISSON_CHECK_EVERY iterations
        for (;;) {
            for (int s = 0; s < DSS_POISSON_CHECK_EVERY; ++s) {
                psn_apply_kernel<<<nbl, PSN_THREADS, 0, st>>>(g, cellmap, qf, p, q, partials, cg);
                DSS_LAUNCH_CHECK(ctx);
                psn_finish_kernel<2><<<1, PSN_THREADS, 0, st>>>(partials, (int)nbl, cg, DSS_POISSON_TOLERANCE,
                                                                DSS_POISSON_MAX_ITERATIONS);
                DSS_LAUNCH_CHECK(ctx);
                psn_update_kernel<<<nbl, PSN_THREADS, 0, st>>>(g.nodes, p, q, inv, chi, r, partials, cg);
                DSS_LAUNCH_CHECK(ctx);
                psn_finish_kernel<3><<<1, PSN_THREADS, 0, st>>>(partials, (int)nbl, cg, DSS_POISSON_TOLERANCE,
                                                                DSS_POISSON_MAX_ITERATIONS);
                DSS_LAUNCH_CHECK(ctx);
                psn_direction_kernel<<<nbl, PSN_THREADS, 0, st>>>(g.nodes, r, inv, p, cg);
                DSS_LAUNCH_CHECK(ctx);
            }
            DSS_CUDA_TRY(cudaMemcpyAsync(h_cg, cg, sizeof(PsnCG), cudaMemcpyDeviceToHost, st));
            DSS_CUDA_TRY(cudaStreamSynchronize(st));
            if (h_cg->done) break;
        }
        if (level_ms) {
            DSS_CUDA_TRY(cudaEventRecord(ev[2], st));
            DSS_CUDA_TRY(cudaEventSynchronize(ev[2]));
            DSS_CUDA_TRY(cudaEventElapsedTime(&level_ms[2 * l], ev[0], ev[1]));
            DSS_CUDA_TRY(cudaEventElapsedTime(&level_ms[2 * l + 1], ev[1], ev[2]));
        }
        if (level_iterations) level_iterations[l] = h_cg->iter;
        if (iterations) *iterations = h_cg->iter;
        if (residual) *residual = h_cg->rel;
        if (l < depth)
            DSS_CUDA_TRY(cudaMemcpyAsync(coarse, chi, (size_t)g.nodes * sizeof(float), cudaMemcpyDeviceToDevice, st));
    }
    return rc;
}

int dss_marching_tetrahedra(dss_ctx *ctx, const float *chi, int R, const float *center, float side, float *verts,
                            int64_t max_verts, int32_t *faces, int64_t max_faces, int64_t *n_verts, int64_t *n_faces,
                            void *stream) {
    using namespace dss;
    cudaStream_t st = (cudaStream_t)stream;
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    DSS_REQUIRE(R >= 1 && R <= 1289, "R must lie in [1, 1289]");
    DSS_REQUIRE(chi && center && n_verts && n_faces, "null pointer");
    DSS_REQUIRE(max_verts >= 0 && max_faces >= 0, "negative capacity");
    DSS_REQUIRE((max_verts == 0 || verts) && (max_faces == 0 || faces), "null output with a capacity");
    *n_verts = 0, *n_faces = 0;
    const int64_t N1 = R + 1, nodes = N1 * N1 * N1, cubes = (int64_t)R * R * R;
    // one slot: totals, vertex counts / bases (nodes), face counts / bases (cubes + 1), masks (nodes bytes)
    char *buf = nullptr;
    int rc;
    const size_t bytes = 256 + (size_t)nodes * 4 + (size_t)(cubes + 1) * 4 + (size_t)nodes;
    if ((rc = ctx_get(ctx, BUF_MT, bytes, &buf))) return rc;
    MtTotals *tot = reinterpret_cast<MtTotals *>(buf);
    int32_t *vcnt = reinterpret_cast<int32_t *>(buf + 256);
    int32_t *fcnt = vcnt + nodes;
    uint8_t *mask = reinterpret_cast<uint8_t *>(fcnt + cubes + 1);
    DSS_CUDA_TRY(cudaMemsetAsync(tot, 0, sizeof(MtTotals), st));
    const unsigned nb = grid_blocks(nodes, PSN_THREADS, ctx->sm_count, 8);
    mt_count_kernel<<<nb, PSN_THREADS, 0, st>>>(chi, R, mask, vcnt, fcnt, tot);
    DSS_LAUNCH_CHECK(ctx);
    // the call's one host synchronisation: the output sizes
    MtTotals *h_tot = reinterpret_cast<MtTotals *>(ctx->h_pinned + 60);
    DSS_CUDA_TRY(cudaMemcpyAsync(h_tot, tot, sizeof(MtTotals), cudaMemcpyDeviceToHost, st));
    DSS_CUDA_TRY(cudaStreamSynchronize(st));
    const MtTotals t = *h_tot;
    *n_verts = (int64_t)t.verts, *n_faces = (int64_t)t.faces;
    if (t.verts > (unsigned long long)INT32_MAX || t.faces > (unsigned long long)INT32_MAX) {
        set_error("dss_marching_tetrahedra: %llu vertices and %llu faces; at most 2^31 - 1 of each", t.verts, t.faces);
        return DSS_E_CAPACITY;
    }
    if ((int64_t)t.verts > max_verts || (int64_t)t.faces > max_faces) {
        set_error("dss_marching_tetrahedra: the surface has %llu vertices and %llu faces, the outputs hold %lld and "
                  "%lld", t.verts, t.faces, (long long)max_verts, (long long)max_faces);
        return DSS_E_CAPACITY;
    }
    if (t.verts == 0) return DSS_OK;   // no crossing edge: no triangle either
    if ((rc = exclusive_scan_i32(ctx, vcnt, vcnt, nodes, st))) return rc;
    if ((rc = exclusive_scan_i32(ctx, fcnt, fcnt, cubes, st))) return rc;
    mt_verts_kernel<<<nb, PSN_THREADS, 0, st>>>(chi, R, mask, vcnt, center[0], center[1], center[2], side, verts);
    DSS_LAUNCH_CHECK(ctx);
    mt_faces_kernel<<<grid_blocks(cubes, PSN_THREADS, ctx->sm_count, 8), PSN_THREADS, 0, st>>>(chi, R, mask, vcnt,
                                                                                                fcnt, faces);
    DSS_LAUNCH_CHECK(ctx);
    return DSS_OK;
}

}  // extern "C"
