// normals.cu -- oriented point normals of clouds that carry none: PCA over the k nearest neighbours, then the sign of
// each normal propagated along a minimum spanning forest of the k-NN graph (Hoppe et al. 1992; meshlab's "Compute
// normals for point sets", the step of the reference's scripts/poisson_sampling_pca.mlx, and
// PointClouds3D.estimate_normals, DSS/core/cloud.py:210-258).  The rules are in include/dss_b200.h and DESIGN.md.
//
// Stages, all on the device and without a host synchronisation:
//   1. PCA, one thread per row: the population covariance of the row's k neighbours in float64, sym3_eigen.cuh's
//      solve, the eigenvector of the smallest eigenvalue rounded once, then the canonical sign.
//   2. Boruvka: in every round each component takes its lightest outgoing edge under the key (w, min(i,j), max(i,j))
//      -- a 64-bit atomicMin on (w, min), then a 32-bit atomicMin on max among the edges that attained it -- and hooks
//      to the component across it (of two components that chose the same edge, the one with the larger label hooks);
//      pointer jumping then flattens the hooks.  The key is a strict total order, so the forest is the unique minimum
//      spanning forest and does not depend on thread order.
//   3. The root of each component (largest z, then smallest index) by a 64-bit atomicMax.
//   4. Rooting: an Euler tour of every tree (each vertex's arcs in an atomicExch-linked list; the order of that list
//      does not matter, only which of an edge's two arcs comes first), cut at the root and ranked by pointer jumping
//      (Wyllie).  An edge's first arc runs from the parent to the child.
//   5. Signs: each vertex's sign is a function of its parent's (keep, flip, or +1 when the dot product is zero, which
//      does not flip); ancestor doubling composes these functions up to the root, whose sign is fixed.
// Every loop of rounds has a fixed length (ceil(log2 P) + 1, enough for any input) and reads an early-out flag that
// the previous round wrote on the device, so the launches are fixed and the call can be captured in a CUDA graph.
// Indices inside are rows of the packed input; clouds are never connected, since every neighbour lies in its cloud.
//
// dss_outlier_ratio (remove_outliers, DSS/core/cloud.py:363-378) runs the same PCA (knn_pca) and keeps the row when
// its smallest eigenvalue is less than `tolerance` of the three's sum.
#include <math_constants.h>

#include "common.cuh"
#include "sym3_eigen.cuh"

namespace dss {

constexpr int NRM_THREADS = 256;
constexpr int NRM_MAX_LOG = 32;   // rounds of a loop at most: ceil(log2(2P)) + 1 with P < 2^30
// flag words: Boruvka rounds, their jump iterations, the list-ranking and the sign-doubling iterations
constexpr int NRM_F_ROUND = 0;
constexpr int NRM_F_JUMP = NRM_F_ROUND + NRM_MAX_LOG;
constexpr int NRM_F_RANK = NRM_F_JUMP + NRM_MAX_LOG * NRM_MAX_LOG;
constexpr int NRM_F_SIGN = NRM_F_RANK + NRM_MAX_LOG;
constexpr int NRM_FLAGS = NRM_F_SIGN + NRM_MAX_LOG;

// sign functions of stage 5: bit 1 set = a constant (bit 0 the sign: 1 = flipped), clear = the parent's sign xor bit 0
constexpr int SIGN_CONST = 2;

struct NormalArgs {
    const float *points;       // (P,3)
    const int64_t *first_idx;  // (N,)
    const int64_t *num_points; // (N,)
    const int32_t *knn_idx;    // (P,k) local to the cloud, -1 missing
    int k;
    int64_t P;
    float *normals;            // (P,3) out
    int32_t *root;             // (P,) out, local
    int32_t *parent;           // (P,) out, local
    // scratch, indexed by row (arcs by 2 row + {0, 1})
    float4 *nrm;               // unoriented normal, w = 1 on a valid row
    int32_t *label, *hook;
    unsigned long long *best;  // (ord(w) << 32 | min row) of the component's lightest outgoing edge
    uint32_t *best_max;        //   and its max row
    int32_t *edge_a, *edge_b;  // the tree edge row c's component added when it hooked, -1 none
    unsigned long long *root_key;
    int32_t *head, *next_arc, *succ;
    int32_t *rank[2], *jump[2];
    int32_t *gparent;
    int32_t *sfun[2], *anc[2];
    int *flags;
};

// order-preserving map of a float to an unsigned integer
__device__ __forceinline__ uint32_t ord_u32(float f) {
    const uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// n_i . n_j in float32, rounded after every operation in the order x, y, z
__device__ __forceinline__ float dot_rn(float4 a, float4 b) {
    return __fadd_rn(__fadd_rn(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)), __fmul_rn(a.z, b.z));
}

#define NRM_ROWS(a)                                                                                          \
    const ViewRange cr = view_range((a).first_idx, (a).num_points, blockIdx.y, (a).P);                       \
    for (int64_t i_ = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i_ < cr.count;                        \
         i_ += (int64_t)gridDim.x * blockDim.x)

// The PCA of one row, shared by the normals and the outlier ratio: the population covariance of the row's k
// neighbours nb (local to the cloud starting at row `first`) about their mean in float64, and sym3_eigen's solve of it.
// False, with nothing solved, when a neighbour is -1.
__device__ __forceinline__ bool knn_pca(const float *points, int64_t first, const int32_t *nb, int k, double &l0,
                                        double &l1, double &l2, double (&f0)[3], double (&f1)[3], double (&f2)[3]) {
    bool ok = true;
    double m[3] = {0.0, 0.0, 0.0};
    for (int s = 0; s < k; ++s) {
        const int32_t j = nb[s];
        ok = ok && j >= 0;
        const int64_t src = first + (j >= 0 ? j : 0);
#pragma unroll
        for (int e = 0; e < 3; ++e) m[e] += (double)points[src * 3 + e];
    }
    if (!ok) return false;
    const double inv_k = 1.0 / k;
#pragma unroll
    for (int e = 0; e < 3; ++e) m[e] *= inv_k;
    double A[3][3] = {{0.0, 0.0, 0.0}, {0.0, 0.0, 0.0}, {0.0, 0.0, 0.0}};
    for (int s = 0; s < k; ++s) {
        const int64_t src = first + nb[s];
        const double d0 = (double)points[src * 3] - m[0], d1 = (double)points[src * 3 + 1] - m[1],
                     d2 = (double)points[src * 3 + 2] - m[2];
        A[0][0] = fma(d0, d0, A[0][0]);
        A[0][1] = fma(d0, d1, A[0][1]);
        A[0][2] = fma(d0, d2, A[0][2]);
        A[1][1] = fma(d1, d1, A[1][1]);
        A[1][2] = fma(d1, d2, A[1][2]);
        A[2][2] = fma(d2, d2, A[2][2]);
    }
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = r; c < 3; ++c) A[r][c] *= inv_k;
    sym3_eigen(A, l0, l1, l2, f0, f1, f2);
    return true;
}

// 1. PCA, canonical sign, and the initial state of every later stage
__global__ void __launch_bounds__(NRM_THREADS) normals_pca_kernel(const __grid_constant__ NormalArgs a) {
    NRM_ROWS(a) {
        const int32_t row = (int32_t)(cr.first + i_);
        float4 n = make_float4(CUDART_NAN_F, CUDART_NAN_F, CUDART_NAN_F, 0.0f);
        double l0, l1, l2, f0[3], f1[3], f2[3];
        if (knn_pca(a.points, cr.first, a.knn_idx + (int64_t)row * a.k, a.k, l0, l1, l2, f0, f1, f2)) {
            // degenerate rows: the normal is sym3_fix_degenerate's f1 (collinear: perpendicular to the line;
            // duplicates: e_z)
            const bool flat = l1 - l0 <= SYM3_DEGENERATE * fabs(l2);
            sym3_fix_degenerate(l0, l1, l2, f1, f2);
            n = make_float4((float)(flat ? f1[0] : f0[0]), (float)(flat ? f1[1] : f0[1]), (float)(flat ? f1[2] : f0[2]),
                            1.0f);
            // canonical sign: the component of largest |n_k| (the first such axis) positive, on the rounded values
            const float ax = fabsf(n.x), ay = fabsf(n.y), az = fabsf(n.z);
            const float big = (ax >= ay && ax >= az) ? n.x : (ay >= az ? n.y : n.z);
            if (big < 0.0f) n.x = -n.x, n.y = -n.y, n.z = -n.z;
        }
        a.nrm[row] = n;
        a.normals[(int64_t)row * 3] = n.x, a.normals[(int64_t)row * 3 + 1] = n.y, a.normals[(int64_t)row * 3 + 2] = n.z;
        a.root[row] = -1, a.parent[row] = -1;
        if (a.label) {
            a.label[row] = row, a.hook[row] = row;
            a.best[row] = ~0ull, a.best_max[row] = ~0u;
            a.edge_a[row] = -1, a.edge_b[row] = -1;
            a.root_key[row] = 0ull, a.head[row] = -1, a.gparent[row] = -1;
        }
    }
}

// The outlier ratio of every row: l0 / ((l0 + l1) + l2) of the same PCA, NaN on an invalid row (and 0 / 0 on a row of
// duplicates), and keep = ratio < tolerance, both in float64 (NaN is not kept)
__global__ void __launch_bounds__(NRM_THREADS)
outlier_ratio_kernel(const float *__restrict__ points, const int64_t *__restrict__ first_idx,
                     const int64_t *__restrict__ num_points, const int32_t *__restrict__ knn_idx, int k, int64_t P,
                     double tolerance, double *__restrict__ ratio, uint8_t *__restrict__ keep) {
    const ViewRange cr = view_range(first_idx, num_points, blockIdx.y, P);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < cr.count; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t row = cr.first + i;
        double l0, l1, l2, f0[3], f1[3], f2[3];
        double r = CUDART_NAN;
        if (knn_pca(points, cr.first, knn_idx + row * k, k, l0, l1, l2, f0, f1, f2)) r = __ddiv_rn(l0, __dadd_rn(__dadd_rn(l0, l1), l2));
        ratio[row] = r;
        keep[row] = r < tolerance ? 1 : 0;
    }
}

// a round (or iteration) runs when the one before it recorded work
__device__ __forceinline__ bool nrm_active(const int *flags, int f, int t) { return t == 0 || flags[f + t - 1] != 0; }

// 2a/2b. per edge {row, j} of a valid row's list with j in another component: the (w, min) minimum of both components
// (pass 0), then the max minimum among the edges that attained it (pass 1)
template <int PASS>
__global__ void __launch_bounds__(NRM_THREADS) normals_edges_kernel(const __grid_constant__ NormalArgs a, int round) {
    if (!nrm_active(a.flags, NRM_F_ROUND, round)) return;
    NRM_ROWS(a) {
        const int32_t row = (int32_t)(cr.first + i_);
        const float4 ni = a.nrm[row];
        if (ni.w == 0.0f) continue;
        const int32_t li = a.label[row];
        const int32_t *nb = a.knn_idx + (int64_t)row * a.k;
        for (int s = 0; s < a.k; ++s) {
            const int32_t j = (int32_t)cr.first + nb[s];
            if (j == row) continue;
            const int32_t lj = a.label[j];
            if (lj == li) continue;
            const float4 nj = a.nrm[j];
            if (nj.w == 0.0f) continue;
            const float w = __fsub_rn(1.0f, fabsf(dot_rn(ni, nj)));
            const uint32_t lo = (uint32_t)min(row, j), hi = (uint32_t)max(row, j);
            const unsigned long long key = ((unsigned long long)ord_u32(w) << 32) | lo;
            if (PASS == 0) {
                atomicMin(a.best + li, key);
                atomicMin(a.best + lj, key);
            } else {
                if (a.best[li] == key) atomicMin(a.best_max + li, hi);
                if (a.best[lj] == key) atomicMin(a.best_max + lj, hi);
            }
        }
    }
}

// 2c. every component with an outgoing edge hooks across it, except the smaller label of a pair that chose the same
// edge; the hooking component records the edge
__global__ void __launch_bounds__(NRM_THREADS) normals_hook_kernel(const __grid_constant__ NormalArgs a, int round) {
    if (!nrm_active(a.flags, NRM_F_ROUND, round)) return;
    NRM_ROWS(a) {
        const int32_t c = (int32_t)(cr.first + i_);
        if (a.nrm[c].w == 0.0f || a.label[c] != c || a.best[c] == ~0ull) continue;
        const int32_t ea = (int32_t)(uint32_t)a.best[c], eb = (int32_t)a.best_max[c];
        const int32_t la = a.label[ea], d = la == c ? a.label[eb] : la;
        if (a.best[d] == a.best[c] && a.best_max[d] == a.best_max[c] && c < d) continue;
        a.hook[c] = d;
        a.edge_a[c] = ea, a.edge_b[c] = eb;
        a.flags[NRM_F_ROUND + round] = 1;
    }
}

// 2d. pointer jumping over the hooks of the round's components (in place: every value read is an ancestor)
__global__ void __launch_bounds__(NRM_THREADS) normals_jump_kernel(const __grid_constant__ NormalArgs a, int round,
                                                                   int t) {
    if (!nrm_active(a.flags, NRM_F_ROUND, round + 1)) return;   // no hook this round
    int *const jf = a.flags + NRM_F_JUMP + round * NRM_MAX_LOG;
    if (t > 0 && jf[t - 1] == 0) return;
    NRM_ROWS(a) {
        const int32_t c = (int32_t)(cr.first + i_);
        if (a.nrm[c].w == 0.0f || a.label[c] != c) continue;
        volatile int32_t *hook = a.hook;
        const int32_t h = hook[c], hh = hook[h];
        if (hh != h) {
            hook[c] = hh;
            jf[t] = 1;
        }
    }
}

// 2e. every row takes its component's new label; the minima are reset for the next round
__global__ void __launch_bounds__(NRM_THREADS) normals_relabel_kernel(const __grid_constant__ NormalArgs a, int round) {
    if (!nrm_active(a.flags, NRM_F_ROUND, round + 1)) return;
    NRM_ROWS(a) {
        const int32_t row = (int32_t)(cr.first + i_);
        if (a.nrm[row].w == 0.0f) continue;
        a.label[row] = a.hook[a.label[row]];
        a.best[row] = ~0ull, a.best_max[row] = ~0u;
    }
}

// 3 and 4a. the component's root key; every tree edge's two arcs (2c: a -> b, 2c + 1: b -> a) linked into their
// tails' lists
__global__ void __launch_bounds__(NRM_THREADS) normals_root_arcs_kernel(const __grid_constant__ NormalArgs a) {
    NRM_ROWS(a) {
        const int32_t row = (int32_t)(cr.first + i_);
        if (a.nrm[row].w == 0.0f) continue;
        const float z = a.points[(int64_t)row * 3 + 2];
        atomicMax(a.root_key + a.label[row], ((unsigned long long)ord_u32(z) << 32) | (0xffffffffu - (uint32_t)row));
        const int32_t ea = a.edge_a[row];
        if (ea >= 0) {
            a.next_arc[2 * row] = atomicExch(a.head + ea, 2 * row);
            a.next_arc[2 * row + 1] = atomicExch(a.head + a.edge_b[row], 2 * row + 1);
        }
    }
}

__device__ __forceinline__ int32_t root_of(const NormalArgs &a, int32_t row) {
    return (int32_t)(0xffffffffu - (uint32_t)a.root_key[a.label[row]]);
}

// 4b. the tour's successor of every arc u -> v: the arc after v -> u in v's list, wrapping to its head, except at the
// root, where the wrap ends the tour; the ranks' first iteration
__global__ void __launch_bounds__(NRM_THREADS) normals_succ_kernel(const __grid_constant__ NormalArgs a) {
    NRM_ROWS(a) {
        const int32_t row = (int32_t)(cr.first + i_);
        if (a.nrm[row].w == 0.0f || a.edge_a[row] < 0) continue;
#pragma unroll
        for (int side = 0; side < 2; ++side) {
            const int32_t arc = 2 * row + side, v = side ? a.edge_a[row] : a.edge_b[row];
            int32_t s = a.next_arc[arc ^ 1];
            if (s < 0) s = root_of(a, v) == v ? -1 : a.head[v];
            a.succ[arc] = s;
            a.rank[0][arc] = s >= 0 ? 1 : 0;
            a.jump[0][arc] = s;
        }
    }
}

// the buffer a ping-pong loop left its result in: the first iteration that found nothing left to do ran last
__device__ __forceinline__ int nrm_last(const int *flags, int f) {
    int t = 0;
    while (t < NRM_MAX_LOG - 1 && flags[f + t] != 0) ++t;
    return (t + 1) & 1;
}

// 4c. list ranking (Wyllie): rank = arcs after this one in the tour
__global__ void __launch_bounds__(NRM_THREADS) normals_rank_kernel(const __grid_constant__ NormalArgs a, int t) {
    if (!nrm_active(a.flags, NRM_F_RANK, t)) return;
    const int src = t & 1;
    NRM_ROWS(a) {
        const int32_t row = (int32_t)(cr.first + i_);
        if (a.nrm[row].w == 0.0f || a.edge_a[row] < 0) continue;
#pragma unroll
        for (int side = 0; side < 2; ++side) {
            const int32_t arc = 2 * row + side, nx = a.jump[src][arc];
            int32_t r = a.rank[src][arc], j = -1;
            if (nx >= 0) {
                r += a.rank[src][nx];
                j = a.jump[src][nx];
                if (j >= 0) a.flags[NRM_F_RANK + t] = 1;
            }
            a.rank[src ^ 1][arc] = r;
            a.jump[src ^ 1][arc] = j;
        }
    }
}

// 4d and 5a. an edge's earlier arc (the larger rank) runs from the parent to the child; each row's sign function
__global__ void __launch_bounds__(NRM_THREADS) normals_parent_kernel(const __grid_constant__ NormalArgs a) {
    const int buf = nrm_last(a.flags, NRM_F_RANK);
    NRM_ROWS(a) {
        const int32_t row = (int32_t)(cr.first + i_);
        if (a.nrm[row].w == 0.0f || a.edge_a[row] < 0) continue;
        const bool a_first = a.rank[buf][2 * row] > a.rank[buf][2 * row + 1];
        a.gparent[a_first ? a.edge_b[row] : a.edge_a[row]] = a_first ? a.edge_a[row] : a.edge_b[row];
    }
}

__global__ void __launch_bounds__(NRM_THREADS) normals_sign_init_kernel(const __grid_constant__ NormalArgs a) {
    NRM_ROWS(a) {
        const int32_t row = (int32_t)(cr.first + i_);
        const float4 n = a.nrm[row];
        if (n.w == 0.0f) continue;
        const int32_t p = a.gparent[row];
        int f;
        if (p < 0) {
            f = SIGN_CONST | (n.z < 0.0f ? 1 : 0);   // n_z == 0 keeps the canonical sign
        } else {
            const float d = dot_rn(n, a.nrm[p]);
            f = d == 0.0f ? SIGN_CONST : (d < 0.0f ? 1 : 0);
        }
        a.sfun[0][row] = f;
        a.anc[0][row] = p;
    }
}

// 5b. ancestor doubling: f_row <- f_row o f_anc, anc <- anc(anc), until every function is a constant
__global__ void __launch_bounds__(NRM_THREADS) normals_sign_kernel(const __grid_constant__ NormalArgs a, int t) {
    if (!nrm_active(a.flags, NRM_F_SIGN, t)) return;
    const int src = t & 1;
    NRM_ROWS(a) {
        const int32_t row = (int32_t)(cr.first + i_);
        if (a.nrm[row].w == 0.0f) continue;
        int f = a.sfun[src][row];
        int32_t p = a.anc[src][row];
        if (!(f & SIGN_CONST)) {
            const int g = a.sfun[src][p];
            f = (g & SIGN_CONST) | ((f ^ g) & 1);
            p = (g & SIGN_CONST) ? -1 : a.anc[src][p];
            if (!(f & SIGN_CONST)) a.flags[NRM_F_SIGN + t] = 1;
        }
        a.sfun[src ^ 1][row] = f;
        a.anc[src ^ 1][row] = p;
    }
}

// 6. the oriented normals, the roots and the parents (local to the cloud)
__global__ void __launch_bounds__(NRM_THREADS) normals_out_kernel(const __grid_constant__ NormalArgs a) {
    const int buf = nrm_last(a.flags, NRM_F_SIGN);
    NRM_ROWS(a) {
        const int32_t row = (int32_t)(cr.first + i_);
        const float4 n = a.nrm[row];
        if (n.w == 0.0f) continue;
        const float s = (a.sfun[buf][row] & 1) ? -1.0f : 1.0f;
        a.normals[(int64_t)row * 3] = s * n.x, a.normals[(int64_t)row * 3 + 1] = s * n.y;
        a.normals[(int64_t)row * 3 + 2] = s * n.z;
        a.root[row] = root_of(a, row) - (int32_t)cr.first;
        const int32_t p = a.gparent[row];
        a.parent[row] = p < 0 ? -1 : p - (int32_t)cr.first;
    }
}

int ceil_log2(int64_t x) {
    int l = 0;
    while (((int64_t)1 << l) < x) ++l;
    return l;
}

}  // namespace dss

extern "C" {

int dss_estimate_normals(dss_ctx *ctx, const float *points, const int64_t *first_idx, const int64_t *num_points, int N,
                         int64_t P, const int32_t *knn_idx, int k, int orient, float *normals, int32_t *root,
                         int32_t *parent, void *stream) {
    using namespace dss;
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    DSS_REQUIRE(P >= 0 && P < ((int64_t)1 << 30), "P out of range");
    DSS_REQUIRE(first_idx && num_points, "first_idx and num_points are required");
    DSS_REQUIRE(N >= 1 && N <= 65535, "N out of range");
    DSS_REQUIRE(k >= 3 && k <= 32, "k must lie in [3, 32]");
    if (P == 0) return DSS_OK;
    DSS_REQUIRE(points && knn_idx && normals && root && parent, "null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    NormalArgs a = {};
    a.points = points, a.first_idx = first_idx, a.num_points = num_points, a.knn_idx = knn_idx, a.k = k, a.P = P;
    a.normals = normals, a.root = root, a.parent = parent;
    // scratch: the normals (16 bytes per row); to orient, two 64-bit and 11 32-bit words per row, 6 32-bit words per
    // arc (two per row), and the flags
    const size_t rows = (size_t)P;
    const size_t bytes = rows * 16 + (orient ? rows * (2 * 8 + 11 * 4) + 2 * rows * 6 * 4 : 0) + NRM_FLAGS * sizeof(int);
    char *s = nullptr;
    if (int rc = ctx_get(ctx, BUF_NORMALS, bytes, &s)) return rc;
    a.nrm = reinterpret_cast<float4 *>(s), s += rows * 16;
    if (orient) {
        a.best = reinterpret_cast<unsigned long long *>(s), s += rows * 8;
        a.root_key = reinterpret_cast<unsigned long long *>(s), s += rows * 8;
        auto words = [&](size_t n) {
            int32_t *w = reinterpret_cast<int32_t *>(s);
            s += n * sizeof(int32_t);
            return w;
        };
        a.label = words(rows), a.hook = words(rows), a.best_max = reinterpret_cast<uint32_t *>(words(rows));
        a.edge_a = words(rows), a.edge_b = words(rows), a.head = words(rows), a.gparent = words(rows);
        a.sfun[0] = words(rows), a.sfun[1] = words(rows), a.anc[0] = words(rows), a.anc[1] = words(rows);
        a.next_arc = words(2 * rows), a.succ = words(2 * rows);
        a.rank[0] = words(2 * rows), a.rank[1] = words(2 * rows), a.jump[0] = words(2 * rows), a.jump[1] = words(2 * rows);
    }
    a.flags = reinterpret_cast<int *>(s);
    const dim3 grid(grid_blocks(P, NRM_THREADS, ctx->sm_count, 8), N);
    StageScope prof(ctx, ST_KNN, st);
    if (orient) DSS_CUDA_TRY(cudaMemsetAsync(a.flags, 0, NRM_FLAGS * sizeof(int), st));
    normals_pca_kernel<<<grid, NRM_THREADS, 0, st>>>(a);
    DSS_LAUNCH_CHECK(ctx);
    if (!orient) return DSS_OK;
    // components at least halve every round and a chain of hooks at most halves in length every jump
    const int rounds = ceil_log2(P) + 1, ranks = ceil_log2(2 * P) + 1;
    for (int r = 0; r < rounds; ++r) {
        normals_edges_kernel<0><<<grid, NRM_THREADS, 0, st>>>(a, r);
        DSS_LAUNCH_CHECK(ctx);
        normals_edges_kernel<1><<<grid, NRM_THREADS, 0, st>>>(a, r);
        DSS_LAUNCH_CHECK(ctx);
        normals_hook_kernel<<<grid, NRM_THREADS, 0, st>>>(a, r);
        DSS_LAUNCH_CHECK(ctx);
        for (int t = 0; t < rounds; ++t) {
            normals_jump_kernel<<<grid, NRM_THREADS, 0, st>>>(a, r, t);
            DSS_LAUNCH_CHECK(ctx);
        }
        normals_relabel_kernel<<<grid, NRM_THREADS, 0, st>>>(a, r);
        DSS_LAUNCH_CHECK(ctx);
    }
    normals_root_arcs_kernel<<<grid, NRM_THREADS, 0, st>>>(a);
    DSS_LAUNCH_CHECK(ctx);
    normals_succ_kernel<<<grid, NRM_THREADS, 0, st>>>(a);
    DSS_LAUNCH_CHECK(ctx);
    for (int t = 0; t < ranks; ++t) {
        normals_rank_kernel<<<grid, NRM_THREADS, 0, st>>>(a, t);
        DSS_LAUNCH_CHECK(ctx);
    }
    normals_parent_kernel<<<grid, NRM_THREADS, 0, st>>>(a);
    DSS_LAUNCH_CHECK(ctx);
    normals_sign_init_kernel<<<grid, NRM_THREADS, 0, st>>>(a);
    DSS_LAUNCH_CHECK(ctx);
    for (int t = 0; t < rounds; ++t) {
        normals_sign_kernel<<<grid, NRM_THREADS, 0, st>>>(a, t);
        DSS_LAUNCH_CHECK(ctx);
    }
    normals_out_kernel<<<grid, NRM_THREADS, 0, st>>>(a);
    DSS_LAUNCH_CHECK(ctx);
    return DSS_OK;
}

int dss_outlier_ratio(dss_ctx *ctx, const float *points, const int64_t *first_idx, const int64_t *num_points, int N,
                      int64_t P, const int32_t *knn_idx, int k, double tolerance, double *ratio, uint8_t *keep,
                      void *stream) {
    using namespace dss;
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    DSS_REQUIRE(P >= 0 && P < ((int64_t)1 << 30), "P out of range");
    DSS_REQUIRE(first_idx && num_points, "first_idx and num_points are required");
    DSS_REQUIRE(N >= 1 && N <= 65535, "N out of range");
    DSS_REQUIRE(k >= 3 && k <= 32, "k must lie in [3, 32]");
    if (P == 0) return DSS_OK;
    DSS_REQUIRE(points && knn_idx && ratio && keep, "null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    const dim3 grid(grid_blocks(P, NRM_THREADS, ctx->sm_count, 8), N);
    StageScope prof(ctx, ST_KNN, st);
    outlier_ratio_kernel<<<grid, NRM_THREADS, 0, st>>>(points, first_idx, num_points, knn_idx, k, P, tolerance, ratio,
                                                       keep);
    DSS_LAUNCH_CHECK(ctx);
    return DSS_OK;
}

}  // extern "C"
