// l0_smooth.cu -- L0 gradient-minimisation smoothing of images (Xu et al. 2011; the reference's L0Smooth,
// DSS/misc/imageFilters.py:133-180), in float64 on periodic boundaries.  The rules are in include/dss_b200.h and
// DESIGN.md.
//
// The images live as float64 planes (N, C, H, W) in the context's scratch: I (the input) and S (the estimate).  Per
// round, with beta = 0.1 2^r:
//   1. l0_keep_kernel, one thread per pixel: keep = !(sum_c(hp^2 + vp^2) < lmd / beta) of S's periodic forward
//      differences.
//   2. l0_rows_forward_kernel: its load pass forms T = I + beta hv, hv the adjoint difference of the kept (hp, vp),
//      then every row of T is transformed along x.
//   3. l0_columns_kernel: every column is transformed along y, divided by 1 + beta D(u, v) and transformed back.
//   4. l0_rows_inverse_kernel: every row is transformed back along x; S = real part / (H W).
// fft2(I) + beta fft2(hv) = fft2(I + beta hv), so one forward 2-D transform per round suffices.  The transforms are a
// mixed-radix (4, 2, 3, 5) Stockham autosort FFT in shared memory (fft_lines): a CTA owns whole lines (2048 / L of
// them), ping-pongs them between two shared buffers stage by stage, and reads its twiddles exp(-2 pi i m / L) from a
// table built once per call.  Every value is computed by one thread in a fixed order: the same bits on every call, no
// atomics, no host synchronisation.
#include <cmath>

#include "common.cuh"

namespace dss {

constexpr int L0_THREADS = 256;
constexpr int L0_LINE_ELEMS = DSS_L0_MAX_SIZE;   // complex values a CTA transforms at once (64 KB, two buffers)
constexpr int L0_MAX_STAGES = 12;
constexpr double L0_BETA0 = 0.1, L0_BETA_MAX = 1e5;
constexpr int L0_MAX_ROUNDS = 40;

struct FftPlan {
    int n_stages;
    int radix[L0_MAX_STAGES];
};

struct L0Args {
    int N, C, H, W;
    int64_t plane;            // H W
    double *I, *S;            // (N, C, H, W)
    double2 *Z;               // (N, C, H, W) complex: the rows' transforms
    uint8_t *keep;            // (N, H, W)
    const double2 *twW, *twH; // exp(-2 pi i m / W), m < W; the same for H
    FftPlan pw, ph;
    int rows_per_cta, cols_per_cta;
};

__device__ __forceinline__ double2 cmul(double2 a, double2 b) {
    return make_double2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}

// cos and sin of 2 pi m / R, m < R, R in {2, 3, 4, 5}; exact where they are 0 or +-1
__device__ __forceinline__ constexpr double root_cos(int R, int m) {
    return R == 2 ? (m == 0 ? 1.0 : -1.0)
         : R == 4 ? (m == 0 ? 1.0 : m == 2 ? -1.0 : 0.0)
         : R == 3 ? (m == 0 ? 1.0 : -0.5)
         : (m == 0 ? 1.0 : (m == 1 || m == 4) ? 0.30901699437494742410 : -0.80901699437494742410);
}
__device__ __forceinline__ constexpr double root_sin(int R, int m) {
    return R == 2 ? 0.0
         : R == 4 ? (m == 1 ? 1.0 : m == 3 ? -1.0 : 0.0)
         : R == 3 ? (m == 0 ? 0.0 : m == 1 ? 0.86602540378443864676 : -0.86602540378443864676)
         : (m == 0 ? 0.0 : m == 1 ? 0.95105651629515357212 : m == 2 ? 0.58778525229247312917
            : m == 3 ? -0.58778525229247312917 : -0.95105651629515357212);
}

// one Stockham stage of radix R over nl lines of length L (SIGN -1 forward, +1 inverse): butterfly j of a line reads
// x[j + r L / R], twiddles it by w^(r k), k = j mod Ns, takes the R-point DFT and writes y[(j / Ns) Ns R + k + r Ns]
template <int R, int SIGN>
__device__ __forceinline__ void fft_stage(const double2 *__restrict__ x, double2 *__restrict__ y, int nl, int L,
                                          int Ns, const double2 *__restrict__ tw) {
    const int M = L / R, step = L / (Ns * R);
    for (int e = threadIdx.x; e < nl * M; e += blockDim.x) {
        const int line = e / M, j = e - line * M, k = j % Ns;
        const double2 *xl = x + line * L;
        double2 v[R];
#pragma unroll
        for (int r = 0; r < R; ++r) v[r] = xl[j + r * M];
#pragma unroll
        for (int r = 1; r < R; ++r) {
            double2 w = __ldg(tw + r * k * step);
            if (SIGN > 0) w.y = -w.y;
            v[r] = cmul(v[r], w);
        }
        double2 out[R];
#pragma unroll
        for (int q = 0; q < R; ++q) {
            double2 acc = v[0];
#pragma unroll
            for (int r = 1; r < R; ++r) {
                const int m = (r * q) % R;
                if (m == 0) {
                    acc.x += v[r].x, acc.y += v[r].y;
                } else {
                    const double2 w = make_double2(root_cos(R, m), SIGN * root_sin(R, m));
                    const double2 p = cmul(v[r], w);
                    acc.x += p.x, acc.y += p.y;
                }
            }
            out[q] = acc;
        }
        double2 *yl = y + line * L + (j / Ns) * Ns * R + k;
#pragma unroll
        for (int r = 0; r < R; ++r) yl[r * Ns] = out[r];
    }
}

// the DFT (SIGN -1) or unscaled inverse DFT (SIGN +1) of nl lines of length L held in a; b is the other buffer.
// Returns the buffer that holds the result.  Every thread of the CTA calls it; it ends with a barrier.
template <int SIGN>
__device__ double2 *fft_lines(double2 *a, double2 *b, int nl, int L, const FftPlan &p, const double2 *tw) {
    int Ns = 1;
    for (int s = 0; s < p.n_stages; ++s) {
        const int R = p.radix[s];
        if (R == 4) fft_stage<4, SIGN>(a, b, nl, L, Ns, tw);
        else if (R == 2) fft_stage<2, SIGN>(a, b, nl, L, Ns, tw);
        else if (R == 3) fft_stage<3, SIGN>(a, b, nl, L, Ns, tw);
        else fft_stage<5, SIGN>(a, b, nl, L, Ns, tw);
        __syncthreads();
        double2 *t = a;
        a = b, b = t;
        Ns *= R;
    }
    return a;
}

__global__ void l0_twiddle_kernel(double2 *tw, int W, int H) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < W + H; i += gridDim.x * blockDim.x) {
        const int L = i < W ? W : H, m = i < W ? i : i - W;
        double s, c;
        sincospi(2.0 * m / L, &s, &c);
        tw[i] = make_double2(c, -s);
    }
}

// images (N, H, W, C) at the given element strides, float32 or float64 -> I and S
__global__ void l0_load_kernel(const L0Args a, const void *__restrict__ in, int f64, int64_t s0, int64_t s1, int64_t s2,
                               int64_t s3) {
    const int64_t total = (int64_t)a.N * a.C * a.plane;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int x = (int)(i % a.W);
        const int64_t r = i / a.W;
        const int y = (int)(r % a.H);
        const int64_t nc = r / a.H;
        const int c = (int)(nc % a.C), n = (int)(nc / a.C);
        const int64_t off = n * s0 + y * s1 + x * s2 + c * s3;
        const double v = f64 ? static_cast<const double *>(in)[off] : (double)static_cast<const float *>(in)[off];
        a.I[i] = v;
        a.S[i] = v;
    }
}

// S -> out (N, H, W, C) contiguous, float32 (rounded once) or float64
__global__ void l0_store_kernel(const L0Args a, void *__restrict__ out, int f64) {
    const int64_t total = (int64_t)a.N * a.C * a.plane;
    for (int64_t o = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; o < total; o += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(o % a.C);
        const int64_t pix = o / a.C, n = pix / a.plane;
        const double v = a.S[(n * a.C + c) * a.plane + pix % a.plane];
        if (f64) static_cast<double *>(out)[o] = v;
        else static_cast<float *>(out)[o] = (float)v;
    }
}

// 1. keep = !(sum_c(hp^2 + vp^2) < thr), the channels summed in order, each operation rounded on its own
__global__ void l0_keep_kernel(const L0Args a, double thr) {
    const int64_t total = (int64_t)a.N * a.plane;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t n = i / a.plane, p = i % a.plane;
        const int y = (int)(p / a.W), x = (int)(p % a.W);
        const int64_t right = (int64_t)y * a.W + (x + 1 == a.W ? 0 : x + 1);
        const int64_t down = (int64_t)(y + 1 == a.H ? 0 : y + 1) * a.W + x;
        double e = 0.0;
        for (int c = 0; c < a.C; ++c) {
            const double *s = a.S + (n * a.C + c) * a.plane;
            const double v = s[p], hp = __dsub_rn(s[right], v), vp = __dsub_rn(s[down], v);
            e = __dadd_rn(e, __dadd_rn(__dmul_rn(hp, hp), __dmul_rn(vp, vp)));
        }
        a.keep[i] = !(e < thr);
    }
}

// 2. the rows of T = I + beta hv, hv = (hp(x-1, y) - hp(x, y)) + (vp(x, y-1) - vp(x, y)) of the kept differences,
// transformed along x into Z
__global__ void __launch_bounds__(L0_THREADS) l0_rows_forward_kernel(const L0Args a, double beta) {
    extern __shared__ double2 smem[];
    double2 *buf0 = smem, *buf1 = smem + L0_LINE_ELEMS;
    const int W = a.W, H = a.H;
    const int64_t lines = (int64_t)a.N * a.C * H, q0 = (int64_t)blockIdx.x * a.rows_per_cta;
    const int nl = (int)min((int64_t)a.rows_per_cta, lines - q0);
    for (int e = threadIdx.x; e < nl * W; e += blockDim.x) {
        const int l = e / W, x = e - l * W;
        const int64_t q = q0 + l, nc = q / H;
        const int y = (int)(q % H);
        const int n = (int)(nc / a.C);
        const double *s = a.S + nc * a.plane;
        const uint8_t *keep = a.keep + (int64_t)n * a.plane;
        const int xl = x == 0 ? W - 1 : x - 1, xr = x + 1 == W ? 0 : x + 1;
        const int yu = y == 0 ? H - 1 : y - 1, yd = y + 1 == H ? 0 : y + 1;
        const int64_t row = (int64_t)y * W;
        const double v = s[row + x];
        const double hp = keep[row + x] ? s[row + xr] - v : 0.0;
        const double vp = keep[row + x] ? s[(int64_t)yd * W + x] - v : 0.0;
        const double hpl = keep[row + xl] ? v - s[row + xl] : 0.0;
        const double vpu = keep[(int64_t)yu * W + x] ? v - s[(int64_t)yu * W + x] : 0.0;
        const double hv = (hpl - hp) + (vpu - vp);
        buf0[l * W + x] = make_double2(a.I[nc * a.plane + row + x] + beta * hv, 0.0);
    }
    __syncthreads();
    const double2 *res = fft_lines<-1>(buf0, buf1, nl, W, a.pw, a.twW);
    for (int e = threadIdx.x; e < nl * W; e += blockDim.x) a.Z[q0 * W + e] = res[e];
}

// 3. the columns of Z: transformed along y, divided by 1 + beta D(u, v), D = (2 - 2 cos 2 pi u / W) + (2 - 2 cos 2 pi
// v / H), transformed back (unscaled).  Adjacent threads load adjacent columns.
__global__ void __launch_bounds__(L0_THREADS) l0_columns_kernel(const L0Args a, double beta) {
    extern __shared__ double2 smem[];
    double2 *buf0 = smem, *buf1 = smem + L0_LINE_ELEMS;
    const int W = a.W, H = a.H;
    const int64_t lines = (int64_t)a.N * a.C * W, q0 = (int64_t)blockIdx.x * a.cols_per_cta;
    const int nl = (int)min((int64_t)a.cols_per_cta, lines - q0);
    for (int e = threadIdx.x; e < nl * H; e += blockDim.x) {
        const int l = e % nl, y = e / nl;
        const int64_t q = q0 + l;
        buf0[l * H + y] = a.Z[((q / W) * H + y) * W + q % W];
    }
    __syncthreads();
    double2 *res = fft_lines<-1>(buf0, buf1, nl, H, a.ph, a.twH);
    double2 *other = res == buf0 ? buf1 : buf0;
    for (int e = threadIdx.x; e < nl * H; e += blockDim.x) {
        const int l = e / H, v = e - l * H;
        const int u = (int)((q0 + l) % W);
        const double D = (2.0 - 2.0 * __ldg(&a.twW[u].x)) + (2.0 - 2.0 * __ldg(&a.twH[v].x));
        const double den = 1.0 + beta * D;
        res[e] = make_double2(res[e].x / den, res[e].y / den);
    }
    __syncthreads();
    res = fft_lines<1>(res, other, nl, H, a.ph, a.twH);
    for (int e = threadIdx.x; e < nl * H; e += blockDim.x) {
        const int l = e % nl, y = e / nl;
        const int64_t q = q0 + l;
        a.Z[((q / W) * H + y) * W + q % W] = res[l * H + y];
    }
}

// 4. the rows of Z transformed back along x: S = real part / (H W)
__global__ void __launch_bounds__(L0_THREADS) l0_rows_inverse_kernel(const L0Args a) {
    extern __shared__ double2 smem[];
    double2 *buf0 = smem, *buf1 = smem + L0_LINE_ELEMS;
    const int W = a.W;
    const int64_t lines = (int64_t)a.N * a.C * a.H, q0 = (int64_t)blockIdx.x * a.rows_per_cta;
    const int nl = (int)min((int64_t)a.rows_per_cta, lines - q0);
    for (int e = threadIdx.x; e < nl * W; e += blockDim.x) buf0[e] = a.Z[q0 * W + e];
    __syncthreads();
    const double2 *res = fft_lines<1>(buf0, buf1, nl, W, a.pw, a.twW);
    const double scale = (double)a.plane;
    for (int e = threadIdx.x; e < nl * W; e += blockDim.x) a.S[q0 * W + e] = res[e].x / scale;
}

// radices 4, then 2, 3 and 5; false when L has another prime factor
static bool make_plan(int L, FftPlan *p) {
    p->n_stages = 0;
    for (int r : {4, 2, 3, 5})
        while (L % r == 0 && p->n_stages < L0_MAX_STAGES) p->radix[p->n_stages++] = r, L /= r;
    return L == 1;
}

}  // namespace dss

extern "C" {

int dss_l0_smooth(dss_ctx *ctx, const void *images, int f64, const int64_t *strides, int N, int H, int W, int C,
                  double lmd, void *out, void *stream) {
    using namespace dss;
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    DSS_REQUIRE(N >= 0, "negative N");
    DSS_REQUIRE(C == 1 || C == 3, "C must be 1 or 3");
    DSS_REQUIRE(H >= 2 && H <= DSS_L0_MAX_SIZE && W >= 2 && W <= DSS_L0_MAX_SIZE, "H and W must lie in [2, 2048]");
    DSS_REQUIRE(std::isfinite(lmd) && lmd >= 0.0, "lmd must be finite and >= 0");
    L0Args a = {};
    DSS_REQUIRE(make_plan(W, &a.pw) && make_plan(H, &a.ph), "H and W must have no prime factor above 5");
    if (N == 0) return DSS_OK;
    DSS_REQUIRE(images && strides && out, "null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    a.N = N, a.C = C, a.H = H, a.W = W, a.plane = (int64_t)H * W;
    const size_t T = (size_t)N * C * a.plane;
    const size_t bytes = T * 32 + (size_t)(W + H) * 16 + (size_t)N * a.plane;
    char *s = nullptr;
    if (int rc = ctx_get(ctx, BUF_L0, bytes, &s)) return rc;
    a.Z = reinterpret_cast<double2 *>(s), s += T * 16;
    double2 *tw = reinterpret_cast<double2 *>(s);
    s += (size_t)(W + H) * 16;
    a.twW = tw, a.twH = tw + W;
    a.I = reinterpret_cast<double *>(s), s += T * 8;
    a.S = reinterpret_cast<double *>(s), s += T * 8;
    a.keep = reinterpret_cast<uint8_t *>(s);
    a.rows_per_cta = L0_LINE_ELEMS / W, a.cols_per_cta = L0_LINE_ELEMS / H;
    const size_t smem = 2 * (size_t)L0_LINE_ELEMS * sizeof(double2);
    DSS_CUDA_TRY(cudaFuncSetAttribute(l0_rows_forward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    DSS_CUDA_TRY(cudaFuncSetAttribute(l0_columns_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    DSS_CUDA_TRY(cudaFuncSetAttribute(l0_rows_inverse_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int64_t row_lines = (int64_t)N * C * H, col_lines = (int64_t)N * C * W;
    const unsigned int row_grid = (unsigned int)((row_lines + a.rows_per_cta - 1) / a.rows_per_cta);
    const unsigned int col_grid = (unsigned int)((col_lines + a.cols_per_cta - 1) / a.cols_per_cta);
    l0_twiddle_kernel<<<grid_blocks(W + H, 256, ctx->sm_count, 4), 256, 0, st>>>(tw, W, H);
    DSS_LAUNCH_CHECK(ctx);
    const unsigned int pix_grid = grid_blocks((int64_t)T, 256, ctx->sm_count, 8);
    l0_load_kernel<<<pix_grid, 256, 0, st>>>(a, images, f64, strides[0], strides[1], strides[2], strides[3]);
    DSS_LAUNCH_CHECK(ctx);
    const unsigned int keep_grid = grid_blocks((int64_t)N * a.plane, 256, ctx->sm_count, 8);
    // beta = 0.1 2^r while beta <= 1e5 (20 rounds), as the reference's loop runs it
    double beta = L0_BETA0;
    for (int r = 0; r < L0_MAX_ROUNDS; ++r) {
        l0_keep_kernel<<<keep_grid, 256, 0, st>>>(a, lmd / beta);
        DSS_LAUNCH_CHECK(ctx);
        l0_rows_forward_kernel<<<row_grid, L0_THREADS, smem, st>>>(a, beta);
        DSS_LAUNCH_CHECK(ctx);
        l0_columns_kernel<<<col_grid, L0_THREADS, smem, st>>>(a, beta);
        DSS_LAUNCH_CHECK(ctx);
        l0_rows_inverse_kernel<<<row_grid, L0_THREADS, smem, st>>>(a);
        DSS_LAUNCH_CHECK(ctx);
        beta *= 2.0;
        if (beta > L0_BETA_MAX) break;
    }
    l0_store_kernel<<<pix_grid, 256, 0, st>>>(a, out, f64);
    DSS_LAUNCH_CHECK(ctx);
    return DSS_OK;
}

}  // extern "C"
