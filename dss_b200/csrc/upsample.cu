// upsample.cu -- densify point clouds: in every round each cloud inserts a point next to each of its sparsest
// neighbourhoods (upsample, DSS/core/cloud.py:555-632).  The rules are in include/dss_b200.h and DESIGN.md.
//
// The caller lays the output out once: cloud n owns rows [first[n], first[n] + n_n) of the packed buffers, holds its
// input rows at the start of that range, and in round r occupies the prefix of sizes[r][n] rows.  Each round appends
// the round's new points behind that prefix, so no row ever moves.  Per round, all on the device:
//   1. dss_knn_points at K = k + 1 over the clouds that grow this round (knn_num[r]: their current size, 0 otherwise).
//   2. ups_sparsity_kernel, one thread per row: the neighbours are the row's K-NN row less its own index (less the
//      last entry when its own index is not in it); candidates c_j = (q_j + 2 p) / 3; s_j = min_k |c_j - q_k|;
//      s = max_j s_j at the first j attaining it.  The key (bits(s) << 32 | ~i) orders rows by (s desc, i asc).
//   3. An MSB-first radix select, 8 bits a pass, of the key of ascending rank c - m in every cloud (m = the round's new
//      points): ups_hist_kernel once per byte, then ups_thresh_kernel.  Exactly the m keys >= that threshold are the
//      round's parents, since the keys of a cloud are distinct.
//   4. ups_flags_kernel, exclusive_scan_i32 over all rows, then ups_write_kernel: parent i (local) writes its
//      candidate, normal, feature and (i, j*) to row first[n] + c + (its rank among the cloud's parents).
// Histogram counts are integers, so every call gives the same bits; nothing waits on the host.
#include <math_constants.h>

#include "common.cuh"
#include "kernels.cuh"

namespace dss {

constexpr int UPS_THREADS = 128;
constexpr int UPS_PASSES = 8;        // bytes of the 64-bit select key
constexpr int UPS_MAX_K = 31;        // the K-NN runs at k + 1 <= 32

struct UpsampleArgs {
    float *points;               // (M,3), rows [first, first + c) of every cloud valid on entry to the round
    float *normals;              // (M,3) or null
    float *features;             // (M,D) or null
    int D;
    const int64_t *first;        // (N,)
    const int64_t *cur;          // (N,) sizes at the start of the round
    const int64_t *next;         // (N,) sizes at its end
    const int32_t *knn_idx;      // (M, k + 1), local to the cloud
    int k;
    int32_t *parents;            // (M,2) out
    // scratch
    unsigned long long *key;     // (M,) select key of every current row
    int32_t *jstar;              // (M,) local index of the row's chosen neighbour
    int32_t *flags, *pos;        // (M,) parent flags and their exclusive scan
    unsigned int *hist;          // (N, UPS_PASSES, 256)
    unsigned long long *thresh;  // (N,) the smallest parent key of each cloud
};

// a + 2 b over 3, rounded after every operation: the candidate between neighbour a and point b, and the child's feature
__device__ __forceinline__ float third_rn(float a, float b) { return __fdiv_rn(__fadd_rn(a, __fmul_rn(2.0f, b)), 3.0f); }

// |v|^2 as (x x + y y) + z z, rounded after every operation
__device__ __forceinline__ float norm2_rn(float x, float y, float z) {
    return __fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z));
}

__device__ __forceinline__ float3 normalize_rn(float3 v) {
    const float l = __fsqrt_rn(norm2_rn(v.x, v.y, v.z));
    return make_float3(__fdiv_rn(v.x, l), __fdiv_rn(v.y, l), __fdiv_rn(v.z, l));
}

__device__ __forceinline__ float3 load3(const float *p, int64_t row) {
    return make_float3(p[row * 3], p[row * 3 + 1], p[row * 3 + 2]);
}

// the rows of cloud blockIdx.y that take part in the round: its current rows when it grows this round
#define UPS_ROWS(a, i_)                                                                                      \
    const int n_ = blockIdx.y;                                                                               \
    const int64_t f_ = (a).first[n_], c_ = (a).cur[n_], m_ = (a).next[n_] - c_;                              \
    for (int64_t i_ = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; m_ > 0 && i_ < c_;                     \
         i_ += (int64_t)gridDim.x * blockDim.x)

// 2. the sparsity of every row, its chosen neighbour and its select key; the neighbours' positions are staged in
// dynamic shared memory, [coordinate * k + s][thread]
__global__ void __launch_bounds__(UPS_THREADS) ups_sparsity_kernel(const __grid_constant__ UpsampleArgs a) {
    extern __shared__ float sq[];
    const int k = a.k, T = blockDim.x, t = threadIdx.x;
    UPS_ROWS(a, i) {
        const int64_t row = f_ + i;
        const int32_t *nb = a.knn_idx + row * (k + 1);
        // the K-NN row less the row's own index, or less its last entry when the index is not in it
        const int own = knn_own_entry(nb, k, (int32_t)i);
        for (int s = 0; s < k; ++s) {
            const int64_t q = f_ + nb[knn_other(s, own)];
            sq[(0 * k + s) * T + t] = a.points[q * 3];
            sq[(1 * k + s) * T + t] = a.points[q * 3 + 1];
            sq[(2 * k + s) * T + t] = a.points[q * 3 + 2];
        }
        const float3 p = load3(a.points, row);
        float best = -1.0f;
        int jb = 0;
        for (int j = 0; j < k; ++j) {
            const float cx = third_rn(sq[(0 * k + j) * T + t], p.x), cy = third_rn(sq[(1 * k + j) * T + t], p.y),
                        cz = third_rn(sq[(2 * k + j) * T + t], p.z);
            float d2 = CUDART_INF_F;
            for (int s = 0; s < k; ++s)
                d2 = fminf(d2, norm2_rn(__fsub_rn(cx, sq[(0 * k + s) * T + t]), __fsub_rn(cy, sq[(1 * k + s) * T + t]),
                                        __fsub_rn(cz, sq[(2 * k + s) * T + t])));
            // sqrt is monotone, so the square root of the minimum is the minimum of the square roots
            const float sj = __fsqrt_rn(d2);
            if (sj > best) best = sj, jb = j;
        }
        // s >= 0, so its bit pattern orders like its value
        a.key[row] = ((unsigned long long)__float_as_uint(best) << 32) | (0xffffffffu - (uint32_t)i);
        a.jstar[row] = nb[knn_other(jb, own)];
    }
}

// Walk the histograms of passes [0, upto) of one cloud: the key prefix they fix and the rank left inside it.  One warp;
// each lane owns 8 consecutive bins.
__device__ void ups_resolve(const unsigned int *hist_n, int upto, unsigned long long rank, unsigned long long &prefix,
                            unsigned long long &rank_left) {
    const int lane = threadIdx.x & 31;
    prefix = 0;
    for (int pass = 0; pass < upto; ++pass) {
        const unsigned int *h = hist_n + pass * 256;
        unsigned int c[8];
        unsigned long long s = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            c[j] = h[lane * 8 + j];
            s += c[j];
        }
        unsigned long long incl = s;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const unsigned long long u = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d) incl += u;
        }
        unsigned long long excl = incl - s;
        int found = -1;
        unsigned long long found_excl = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            if (found < 0 && rank >= excl && rank < excl + c[j]) found = lane * 8 + j, found_excl = excl;
            excl += c[j];
        }
        const unsigned int who = __ballot_sync(0xffffffffu, found >= 0);
        const int src = who ? __ffs(who) - 1 : 0;
        const int digit = __shfl_sync(0xffffffffu, found, src);
        const unsigned long long dexcl = __shfl_sync(0xffffffffu, found_excl, src);
        prefix = (prefix << 8) | (unsigned int)(who ? digit : 0);
        rank -= who ? dexcl : 0;
    }
    rank_left = rank;
}

// 3a. one radix-select pass: the keys that match the prefix of the earlier passes, counted by their next byte
__global__ void __launch_bounds__(256) ups_hist_kernel(const __grid_constant__ UpsampleArgs a, int pass) {
    __shared__ unsigned int s_hist[256];
    __shared__ unsigned long long s_prefix;
    const int n = blockIdx.y;
    const int64_t c = a.cur[n], m = a.next[n] - c;
    if (m <= 0) return;
    unsigned int *hist_n = a.hist + (int64_t)n * UPS_PASSES * 256;
    s_hist[threadIdx.x] = 0;
    if (threadIdx.x < 32) {
        unsigned long long prefix, left;
        ups_resolve(hist_n, pass, (unsigned long long)(c - m), prefix, left);
        if (threadIdx.x == 0) s_prefix = prefix;
    }
    __syncthreads();
    const unsigned long long prefix = s_prefix;
    const int shift = 56 - 8 * pass;
    const unsigned long long *key = a.key + a.first[n];
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < c; i += (int64_t)gridDim.x * blockDim.x) {
        const unsigned long long kk = key[i];
        if (pass == 0 || (kk >> (shift + 8)) == prefix) atomicAdd(&s_hist[(kk >> shift) & 255u], 1u);
    }
    __syncthreads();
    const unsigned int v = s_hist[threadIdx.x];
    if (v) atomicAdd(&hist_n[pass * 256 + threadIdx.x], v);
}

// 3b. the key of ascending rank c - m: the smallest of the m largest
__global__ void ups_thresh_kernel(const __grid_constant__ UpsampleArgs a) {
    const int n = blockIdx.x;
    const int64_t c = a.cur[n], m = a.next[n] - c;
    unsigned long long prefix = ~0ull, left;
    if (m > 0) ups_resolve(a.hist + (int64_t)n * UPS_PASSES * 256, UPS_PASSES, (unsigned long long)(c - m), prefix, left);
    if (threadIdx.x == 0) a.thresh[n] = prefix;
}

// 4a. the parent flags over every row a cloud owns this round or later (0 outside its current rows)
__global__ void __launch_bounds__(UPS_THREADS) ups_flags_kernel(const __grid_constant__ UpsampleArgs a,
                                                                const int64_t *__restrict__ final_num) {
    const int n = blockIdx.y;
    const int64_t f = a.first[n], c = a.cur[n], m = a.next[n] - c, total = final_num[n];
    const unsigned long long th = a.thresh[n];
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x)
        a.flags[f + i] = (m > 0 && i < c && a.key[f + i] >= th) ? 1 : 0;
}

// 4b. every parent writes its child behind the cloud's current rows, in the order of the parents' indices
__global__ void __launch_bounds__(UPS_THREADS) ups_write_kernel(const __grid_constant__ UpsampleArgs a) {
    UPS_ROWS(a, i) {
        const int64_t row = f_ + i;
        if (!a.flags[row]) continue;
        const int64_t dst = f_ + c_ + (a.pos[row] - a.pos[f_]);
        const int32_t j = a.jstar[row];
        const int64_t q = f_ + j;
        const float3 p = load3(a.points, row), qj = load3(a.points, q);
        a.points[dst * 3] = third_rn(qj.x, p.x);
        a.points[dst * 3 + 1] = third_rn(qj.y, p.y);
        a.points[dst * 3 + 2] = third_rn(qj.z, p.z);
        if (a.normals) {
            const float3 ni = normalize_rn(load3(a.normals, row)), nj = normalize_rn(load3(a.normals, q));
            const float3 nn = normalize_rn(make_float3(__fadd_rn(__fmul_rn(2.0f, ni.x), nj.x),
                                                       __fadd_rn(__fmul_rn(2.0f, ni.y), nj.y),
                                                       __fadd_rn(__fmul_rn(2.0f, ni.z), nj.z)));
            a.normals[dst * 3] = nn.x, a.normals[dst * 3 + 1] = nn.y, a.normals[dst * 3 + 2] = nn.z;
        }
        for (int d = 0; d < (a.features ? a.D : 0); ++d)
            a.features[dst * a.D + d] = third_rn(a.features[q * a.D + d], a.features[row * a.D + d]);
        a.parents[dst * 2] = (int32_t)i;
        a.parents[dst * 2 + 1] = j;
    }
}

}  // namespace dss

extern "C" {

int dss_upsample_points(dss_ctx *ctx, float *points, float *normals, float *features, int D, const int64_t *first_idx,
                        const int64_t *sizes, const int64_t *knn_num, int N, int64_t M, int rounds, int k,
                        int32_t *parents, void *stream) {
    using namespace dss;
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    DSS_REQUIRE(M >= 0 && M < (int64_t)INT32_MAX, "M out of range");
    DSS_REQUIRE(N >= 1 && N <= 65535, "N out of range");
    DSS_REQUIRE(k >= 3 && k <= UPS_MAX_K, "k must lie in [3, 31]");
    DSS_REQUIRE(rounds >= 0, "negative number of rounds");
    DSS_REQUIRE(features == nullptr || D >= 1, "features need D >= 1");
    if (M == 0 || rounds == 0) return DSS_OK;
    DSS_REQUIRE(points && first_idx && sizes && knn_num && parents, "null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    UpsampleArgs a = {};
    a.points = points, a.normals = normals, a.features = features, a.D = D, a.first = first_idx, a.k = k;
    a.parents = parents;
    // scratch: the K-NN rows and distances, 8 + 3 x 4 bytes of round state per row, the histograms and thresholds
    const size_t rows = (size_t)M, K = (size_t)k + 1;
    const size_t bytes = rows * K * 8 + rows * 20 + (size_t)N * UPS_PASSES * 256 * 4 + (size_t)N * 8;
    char *s = nullptr;
    if (int rc = ctx_get(ctx, BUF_UPSAMPLE, bytes, &s)) return rc;
    a.key = reinterpret_cast<unsigned long long *>(s), s += rows * 8;
    a.thresh = reinterpret_cast<unsigned long long *>(s), s += (size_t)N * 8;
    float *knn_d = reinterpret_cast<float *>(s);
    s += rows * K * 4;
    int32_t *knn_idx = reinterpret_cast<int32_t *>(s);
    s += rows * K * 4;
    a.knn_idx = knn_idx;
    a.jstar = reinterpret_cast<int32_t *>(s), s += rows * 4;
    a.flags = reinterpret_cast<int32_t *>(s), s += rows * 4;
    a.pos = reinterpret_cast<int32_t *>(s), s += rows * 4;
    a.hist = reinterpret_cast<unsigned int *>(s);
    const int64_t *final_num = sizes + (int64_t)rounds * N;
    const dim3 grid(grid_blocks(M, UPS_THREADS, ctx->sm_count, 8), N);
    const dim3 hgrid(grid_blocks(M, 256, ctx->sm_count, 4), N);
    const size_t smem = (size_t)3 * k * UPS_THREADS * sizeof(float);
    for (int r = 0; r < rounds; ++r) {
        a.cur = sizes + (int64_t)r * N, a.next = sizes + (int64_t)(r + 1) * N;
        if (int rc = dss_knn_points(ctx, nullptr, nullptr, nullptr, points, first_idx, knn_num + (int64_t)r * N, N, M, M,
                                    k + 1, -1.0f, knn_d, knn_idx, stream))
            return rc;
        ups_sparsity_kernel<<<grid, UPS_THREADS, smem, st>>>(a);
        DSS_LAUNCH_CHECK(ctx);
        DSS_CUDA_TRY(cudaMemsetAsync(a.hist, 0, (size_t)N * UPS_PASSES * 256 * sizeof(unsigned int), st));
        for (int pass = 0; pass < UPS_PASSES; ++pass) {
            ups_hist_kernel<<<hgrid, 256, 0, st>>>(a, pass);
            DSS_LAUNCH_CHECK(ctx);
        }
        ups_thresh_kernel<<<N, 32, 0, st>>>(a);
        DSS_LAUNCH_CHECK(ctx);
        ups_flags_kernel<<<grid, UPS_THREADS, 0, st>>>(a, final_num);
        DSS_LAUNCH_CHECK(ctx);
        if (int rc = exclusive_scan_i32(ctx, a.flags, a.pos, M, st)) return rc;
        ups_write_kernel<<<grid, UPS_THREADS, 0, st>>>(a);
        DSS_LAUNCH_CHECK(ctx);
    }
    return DSS_OK;
}

}  // extern "C"
