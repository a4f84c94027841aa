// render.cu -- fused renderer path: per-(point,view) preprocess, forward orchestration, backward
// orchestration (gradient clip + chain to world space).
#include <math_constants.h>

#include "binning.cuh"
#include "common.cuh"
#include "kernels.cuh"
#include "shading.cuh"

namespace dss {

// Every kernel of this file takes the call's dss_render_args as it is (`g`, a __grid_constant__ parameter), plus only
// what the call does not hold: context scratch and, for the chain, what the host decided from the call.

// light rows and ambient of view n
__device__ __forceinline__ const float *view_lights(const dss_render_args &g, int n) {
    return g.lights_per_view ? g.lights + (int64_t)n * g.n_lights * 9 : g.lights;
}
__device__ __forceinline__ const float *view_ambient(const dss_render_args &g, int n) {
    return g.lights_per_view ? g.ambient + (int64_t)n * 3 : g.ambient;
}
// stages view n's shading rows into sL[DSS_MAX_LIGHTS * 9 + 6]: lights, then ambient (3) and camera centre (3) at
// DSS_MAX_LIGHTS * 9 (the caller synchronises)
__device__ __forceinline__ void stage_view_shading(float *sL, const dss_render_args &g, int n) {
    if (threadIdx.x < g.n_lights * 9) sL[threadIdx.x] = view_lights(g, n)[threadIdx.x];
    if (threadIdx.x < 3) {
        sL[DSS_MAX_LIGHTS * 9 + threadIdx.x] = view_ambient(g, n)[threadIdx.x];
        sL[DSS_MAX_LIGHTS * 9 + 3 + threadIdx.x] = g.cam_centres[n * 3 + threadIdx.x];
    }
}

// Fast reciprocal (rcp_approx, common.cuh) and square root (MUFU based, <= 2 ulp): the per-splat quantities are compared
// with the float64 oracle at 2e-5 .. 2e-3 relative, IEEE-exact division and sqrt were a third of this kernel's instructions.
__device__ __forceinline__ float fast_sqrt(float x) {
    float y;
    asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// Python-side eps helpers of the reference (DSS/utils/mathHelper.py:10-22), zero counts as positive.
__device__ __forceinline__ float py_eps_denom(float d) { return eps_denom(d, 1e-17f); }
__device__ __forceinline__ float py_eps_sqrt(float s) { return fmaxf(fabsf(s), 1e-17f); }

// View-space depth of world point p in view n (sV: the view's matrix) after the preprocess's filters
// (rasterizer.py:187-192, :152): the depth range and, with backface culling, the normal n facing the camera.  A filtered
// point gets -1.  The preprocess and the depth-range pre-pass of the fused route both call this, so that the pre-pass
// finds exactly the depths the records will hold.
__device__ __forceinline__ float kept_view_depth(const dss_render_args &g, const float *sV, float p0, float p1, float p2,
                                                 float n0, float n1, float n2) {
    const float zv = fmaf(p0, sV[2], fmaf(p1, sV[6], fmaf(p2, sV[10], sV[14])));
    bool keep = (zv >= g.znear) && (zv <= g.zfar);
    if (g.backface_culling) {
        const float nz = n0 * sV[2] + n1 * sV[6] + n2 * sV[10];
        keep = keep && (nz < 0.0f);
    }
    return keep ? zv : -1.0f;
}

// Counting inputs and outputs of the fused route's preprocess (BIN != 0 below).
struct PreprocessBins {
    const float *zrange;        // (N,2) depth ranges of the views (depth_range_kernel)
    int32_t *counts;            // (N*B*B*NS) list sizes, zeroed by the caller
    unsigned int *rects;        // (P,) packed tile rectangle + depth slice of every splat
    int32_t *block_offsets;     // (N, gridDim.x, B*B*NS) each block's offset inside the bins it touches
    int B, NS;
};

// ---------------------------------------------------------------------------------------------
// One thread per (view, point).  Fuses DSS/core/rasterizer.py:183-217 (depth filter), :148-181
// (backface filter), :443-496 (_compute_WJk), :293-342 (global/isotropic Vrk with Sk^T Sk = I - n n^T),
// :404-441 (variance + detMk), :525-565 (conic, radii, scaler) and the pytorch3d transform of :614
// (x/t, y/t, view-space z) -- about 40 ATen launches incl. batched det/inverse in the reference.
// Filtered points keep their slot but get z = -1, which every later stage treats as "not renderable"
// exactly like the reference treats points behind the camera (rasterize_points.cu:87-88).
// rec: the (P,2) records (g.records or context scratch); zrange: (N,2) float bits, min / max view depth of the
// renderable splats, or null.  SHADE: write the shaded colour of every (view, point) to g.shaded.
// FRAMES (anisotropic splats, rasterizer.py:256-291, 425-439): the world variance is l1 f1 f1^T + l2 f2 f2^T from the
// g.frames record of the point instead of h (I - n n^T); with u = (f1.J0, f1.J1), v = (f2.J0, f2.J1):
//   Vk = l1 u u^T + l2 v v^T,   |det Mk| = |u0 v1 - u1 v0|
// and the rest (G = Vk + aa I, conic, radii, scaler, filters, shading) is shared.  The body is one inlined function
// so that the two kernels without frames keep the code they had.
// BIN (the fused route, 1: S a power of two, 2: any S): the thread also bins the splat it has just written, with the
// binning's own functions on the same register values (bin_count_kernel reads them back from the record), stores the
// packed rectangle and counts it in the block's histogram of the B*B*NS bins (dynamic shared memory).  At the end each
// non-empty bin is added to the view's count with one atomic, whose return value -- the block's offset inside the bin --
// goes to the block's row of pb.block_offsets for bin_scatter_counted.  The depth slices need the view's depth range
// before the first record exists: pb.zrange comes from depth_range_kernel, and the kernel makes no zrange atomics.
// ---------------------------------------------------------------------------------------------
constexpr int FLUSH_BATCH = 8;   // histogram bins per thread whose flush atomics are in flight together

template <bool SHADE, bool FRAMES, int BIN>
__device__ __forceinline__ void preprocess_splats(const dss_render_args &g, float4 *rec, int32_t *zrange,
                                                  const PreprocessBins &pb) {
    __shared__ float sM[16], sV[16];
    __shared__ float sL[DSS_MAX_LIGHTS * 9 + 6];   // lights, ambient (3), camera centre (3)
    extern __shared__ int32_t s_hist[];            // BIN: B*B*NS counters
    const int n = blockIdx.y;
    if (threadIdx.x < 16) {
        sM[threadIdx.x] = g.proj[n * 16 + threadIdx.x];
        sV[threadIdx.x] = g.view[n * 16 + threadIdx.x];
    }
    constexpr bool shade = SHADE;
    if (shade) stage_view_shading(sL, g, n);
    const int nt = pb.B * pb.B * pb.NS;
    if (BIN)
        for (int t = threadIdx.x; t < nt; t += PREPROCESS_THREADS) s_hist[t] = 0;
    __syncthreads();
    const SliceMap slices = make_slice_map(BIN ? pb.zrange : nullptr, n, pb.NS);
    const ViewRange vr = view_range(g.shared_cloud ? nullptr : g.first_idx, g.num_points, n, g.P0);
    const float pix = 2.0f / (float)g.image_size;
    const float aa = g.antialiasing_sigma * pix * pix;
    int zlo = 0x7f7fffff, zhi = 0;   // depth range of this thread's renderable splats (float bits)
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < vr.count;
         i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t s = vr.first + i;                     // packed slot
        const int64_t src = g.shared_cloud ? i : s;         // where the world-space point lives
        const float p0 = g.points_world[src * 3 + 0], p1 = g.points_world[src * 3 + 1], p2 = g.points_world[src * 3 + 2];
        const float n0 = g.normals_world[src * 3 + 0], n1 = g.normals_world[src * 3 + 1],
                    n2 = g.normals_world[src * 3 + 2];
        // [p 1] . M  (row-vector convention, rasterizer.py:465-476)
        const float x = fmaf(p0, sM[0], fmaf(p1, sM[4], fmaf(p2, sM[8], sM[12])));
        const float y = fmaf(p0, sM[1], fmaf(p1, sM[5], fmaf(p2, sM[9], sM[13])));
        const float t = fmaf(p0, sM[3], fmaf(p1, sM[7], fmaf(p2, sM[11], sM[15])));
        const float te = py_eps_denom(t);
        const float t2 = py_eps_denom(t * t);
        const float it = rcp_approx(te), it2 = rcp_approx(t2);
        // J = d(ndc xy)/d(world xyz), 3x2 (Mk = W @ Jk, rasterizer.py:483-494)
        float J0[3], J1[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            J0[k] = sM[k * 4 + 0] * it - sM[k * 4 + 3] * x * it2;
            J1[k] = sM[k * 4 + 1] * it - sM[k * 4 + 3] * y * it2;
        }
        float G00, G01, G11;
        float T00, T01, T11;        // without frames: T = J^T (I - n n^T) J
        float u0, u1, v0, v1;       // with frames: Sk WJk = [u; v]
        if (FRAMES) {
            // u_k = f1.J_k, v_k = f2.J_k (rasterizer.py:289-291, 428-439)
            const float4 fa = reinterpret_cast<const float4 *>(g.frames)[2 * src];
            const float4 fb = reinterpret_cast<const float4 *>(g.frames)[2 * src + 1];
            u0 = fa.x * J0[0] + fa.y * J0[1] + fa.z * J0[2];
            u1 = fa.x * J1[0] + fa.y * J1[1] + fa.z * J1[2];
            v0 = fb.x * J0[0] + fb.y * J0[1] + fb.z * J0[2];
            v1 = fb.x * J1[0] + fb.y * J1[1] + fb.z * J1[2];
            G00 = fmaf(fa.w * u0, u0, fmaf(fb.w * v0, v0, aa));
            G01 = fmaf(fa.w * u0, u1, fb.w * v0 * v1);
            G11 = fmaf(fa.w * u1, u1, fmaf(fb.w * v1, v1, aa));
        } else {
            const float nj0 = n0 * J0[0] + n1 * J0[1] + n2 * J0[2];
            const float nj1 = n0 * J1[0] + n1 * J1[1] + n2 * J1[2];
            T00 = (J0[0] * J0[0] + J0[1] * J0[1] + J0[2] * J0[2]) - nj0 * nj0;
            T01 = (J0[0] * J1[0] + J0[1] * J1[1] + J0[2] * J1[2]) - nj0 * nj1;
            T11 = (J1[0] * J1[0] + J1[1] * J1[1] + J1[2] * J1[2]) - nj1 * nj1;
            const float hh = g.h_per_splat ? g.h[s] : g.h[n];
            G00 = fmaf(hh, T00, aa), G01 = hh * T01, G11 = fmaf(hh, T11, aa);
        }
        const float detG = G00 * G11 - G01 * G01;
        const float idet = rcp_approx(detG);
        const float ea = G11 * idet, eb = -2.0f * G01 * idet, ec = G00 * idet;   // rasterizer.py:543-551
        const float den = py_eps_denom(4.0f * ea * ec - eb * eb);                 // :509-519
        const float iden = rcp_approx(den);
        const float ry = fast_sqrt(py_eps_sqrt(4.0f * ea * g.cutoff_threshold * iden));
        const float rx = fast_sqrt(py_eps_sqrt(4.0f * ec * g.cutoff_threshold * iden));
        // |det Mk|: sqrt(det T) = |det(Sk WJk)| for the orthonormal tangent frame of I - n n^T
        const float detM = FRAMES ? fabsf(u0 * v1 - u1 * v0) : fast_sqrt(fmaxf(T00 * T11 - T01 * T01, 0.0f));
        const float sc = detM *
                         rcp_approx(py_eps_denom(fast_sqrt(py_eps_sqrt(detG * (4.0f * CUDART_PI_F * CUDART_PI_F)))));  // :558-559
        const float zv = kept_view_depth(g, sV, p0, p1, p2, n0, n1, n2);
        if (zv >= 0.0f && zv < 3.0e38f) {
            const int zb = __float_as_int(zv + 0.0f);
            zlo = min(zlo, zb);
            zhi = max(zhi, zb);
        }
        const float irt = rcp_approx(t);
        const float xn = x * irt, yn = y * irt;
        rec[2 * s] = make_float4(xn, yn, zv, rx);
        rec[2 * s + 1] = make_float4(ry, ea, eb, ec);
        if (g.scaler) g.scaler[s] = sc;
        if (g.ndc) {
            g.ndc[s * 3 + 0] = xn;
            g.ndc[s * 3 + 1] = yn;
            g.ndc[s * 3 + 2] = zv;
        }
        if (g.ellipse) {
            g.ellipse[s * 3 + 0] = ea;
            g.ellipse[s * 3 + 1] = eb;
            g.ellipse[s * 3 + 2] = ec;
        }
        if (g.radii) {
            g.radii[s * 2 + 0] = rx;
            g.radii[s * 2 + 1] = ry;
        }
        if (shade) {
            V3 ga, gn, gp;
            const float *amb = sL + DSS_MAX_LIGHTS * 9;
            const V3 c = shade_point<false>(sL, g.n_lights, g.light_type, g.shininess, v3(amb[0], amb[1], amb[2]),
                                            v3(p0, p1, p2), v3(n0, n1, n2),
                                            v3(g.albedo[src * 3], g.albedo[src * 3 + 1], g.albedo[src * 3 + 2]),
                                            v3(amb[3], amb[4], amb[5]), v3(0.f, 0.f, 0.f), ga, gn, gp);
            g.shaded[s * 3 + 0] = c.x;
            g.shaded[s * 3 + 1] = c.y;
            g.shaded[s * 3 + 2] = c.z;
        }
        if (BIN) {
            const BinRect r = splat_bin_rect<BIN == 1>(make_float4(xn, yn, zv, rx), ry, RASTER_TILE, g.image_size, pb.B);
            const int sl = r.empty ? 0 : depth_slice(slices, zv);
            pb.rects[s] = pack_rect(r, sl);
            if (!r.empty)
                for (int by = r.y0; by <= r.y1; ++by)
                    for (int bx = r.x0; bx <= r.x1; ++bx) atomicAdd(&s_hist[(by * pb.B + bx) * pb.NS + sl], 1);
        }
    }
    if (BIN) {
        __syncthreads();
        int32_t *cnt = pb.counts + (int64_t)n * nt;
        int32_t *own = pb.block_offsets + ((int64_t)n * gridDim.x + blockIdx.x) * nt;
        // the atomics of a batch are issued before their results are stored (a store between two atomics would make
        // each one wait for the previous one's round trip)
        for (int t0 = threadIdx.x; t0 < nt; t0 += FLUSH_BATCH * PREPROCESS_THREADS) {
            int v[FLUSH_BATCH], r[FLUSH_BATCH];
#pragma unroll
            for (int j = 0; j < FLUSH_BATCH; ++j) {
                const int t = t0 + j * PREPROCESS_THREADS;
                v[j] = t < nt ? s_hist[t] : 0;
                r[j] = v[j] ? atomicAdd(&cnt[t], v[j]) : 0;
            }
#pragma unroll
            for (int j = 0; j < FLUSH_BATCH; ++j)
                if (v[j]) own[t0 + j * PREPROCESS_THREADS] = r[j];
        }
    }
    if (zrange) {   // one pair of atomics per block
        __shared__ int s_lo[8], s_hi[8];
        zlo = __reduce_min_sync(0xffffffffu, zlo);
        zhi = __reduce_max_sync(0xffffffffu, zhi);
        if ((threadIdx.x & 31) == 0) {
            s_lo[threadIdx.x >> 5] = zlo;
            s_hi[threadIdx.x >> 5] = zhi;
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            for (int w = 1; w < 8; ++w) {
                zlo = min(zlo, s_lo[w]);
                zhi = max(zhi, s_hi[w]);
            }
            atomicMin(&zrange[2 * n], zlo);
            atomicMax(&zrange[2 * n + 1], zhi);
        }
    }
}

template <bool SHADE, int BIN>
__global__ void __launch_bounds__(PREPROCESS_THREADS)
preprocess_kernel(const __grid_constant__ dss_render_args g, float4 *rec, int32_t *zrange, const PreprocessBins pb) {
    preprocess_splats<SHADE, false, BIN>(g, rec, zrange, pb);
}

template <bool SHADE, int BIN>
__global__ void __launch_bounds__(PREPROCESS_THREADS)
preprocess_frames_kernel(const __grid_constant__ dss_render_args g, float4 *rec, int32_t *zrange, const PreprocessBins pb) {
    preprocess_splats<SHADE, true, BIN>(g, rec, zrange, pb);
}

typedef void (*PreprocessKernel)(const dss_render_args, float4 *, int32_t *, const PreprocessBins);
template <int BIN>
static PreprocessKernel preprocess_kernel_for(bool frames, bool shade) {
    if (frames) return shade ? preprocess_frames_kernel<true, BIN> : preprocess_frames_kernel<false, BIN>;
    return shade ? preprocess_kernel<true, BIN> : preprocess_kernel<false, BIN>;
}

// Depth range pre-pass of the fused route: zrange[n] = {min, max} (float bits) of kept_view_depth over the renderable
// points of view n -- what the preprocess's own zrange atomics find, before the preprocess runs.  zrange must hold
// {0x7f7fffff, 0} per view (init_zrange).  A shared cloud is read once: one thread per world point takes it through all
// the views (grid (blocks, 1)); a packed cloud has a range per view (grid (blocks, N)).  Each warp folds its depths of a
// view into the block's shared pair, each block folds its pairs into zrange.
__global__ void __launch_bounds__(256) depth_range_kernel(const __grid_constant__ dss_render_args g, int32_t *zrange) {
    extern __shared__ float s_view[];   // nv view matrices (16 floats each), then {min, max} per view
    const int v0 = g.shared_cloud ? 0 : blockIdx.y, nv = g.shared_cloud ? g.n_views : 1;
    int32_t *s_z = reinterpret_cast<int32_t *>(s_view + nv * 16);
    for (int i = threadIdx.x; i < nv * 16; i += blockDim.x) s_view[i] = g.view[v0 * 16 + i];
    for (int i = threadIdx.x; i < nv; i += blockDim.x) {
        s_z[2 * i] = 0x7f7fffff;
        s_z[2 * i + 1] = 0;
    }
    __syncthreads();
    const ViewRange vr = view_range(g.shared_cloud ? nullptr : g.first_idx, g.num_points, v0, g.P0);
    const int lane = threadIdx.x & 31;
    for (int64_t w = (int64_t)blockIdx.x * blockDim.x + (threadIdx.x - lane); w < vr.count;
         w += (int64_t)gridDim.x * blockDim.x) {   // warp-uniform trip count: the reductions below take all lanes
        const int64_t i = w + lane, src = vr.first + i;
        const bool in = i < vr.count;
        float p0 = 0.f, p1 = 0.f, p2 = 0.f, n0 = 0.f, n1 = 0.f, n2 = 0.f;
        if (in) {
            p0 = g.points_world[src * 3 + 0];
            p1 = g.points_world[src * 3 + 1];
            p2 = g.points_world[src * 3 + 2];
            if (g.backface_culling) {
                n0 = g.normals_world[src * 3 + 0];
                n1 = g.normals_world[src * 3 + 1];
                n2 = g.normals_world[src * 3 + 2];
            }
        }
        for (int v = 0; v < nv; ++v) {
            const float zv = in ? kept_view_depth(g, s_view + v * 16, p0, p1, p2, n0, n1, n2) : -1.0f;
            int zlo = 0x7f7fffff, zhi = 0;
            if (zv >= 0.0f && zv < 3.0e38f) zlo = zhi = __float_as_int(zv + 0.0f);
            zlo = __reduce_min_sync(0xffffffffu, zlo);
            zhi = __reduce_max_sync(0xffffffffu, zhi);
            if (lane == 0 && zlo <= zhi) {
                atomicMin(&s_z[2 * v], zlo);
                atomicMax(&s_z[2 * v + 1], zhi);
            }
        }
    }
    __syncthreads();
    for (int v = threadIdx.x; v < nv; v += blockDim.x) {
        if (s_z[2 * v] > s_z[2 * v + 1]) continue;   // no renderable point of view v in this block
        atomicMin(&zrange[2 * (v0 + v)], s_z[2 * v]);
        atomicMax(&zrange[2 * (v0 + v) + 1], s_z[2 * v + 1]);
    }
}

// d L / d shaded (N*P0,3) -> d albedo, d normal, d position (through the shading) per world point, summed over the views:
// one thread per point loops over the views (deterministic, no atomics) and re-evaluates the lighting of the
// (view, point) pairs that received a colour gradient (the visible ones, ~18 %).
__global__ void __launch_bounds__(256) shade_backward_kernel(const __grid_constant__ dss_render_args g) {
    // lights (L*9) and ambient (3), once or (per_view) for every view, then the camera centres (N*3)
    extern __shared__ float sS[];
    const int nl9 = g.n_lights * 9, stride = nl9 + 3, rows = g.lights_per_view ? g.n_views : 1;
    for (int i = threadIdx.x; i < rows * nl9; i += blockDim.x) sS[(i / nl9) * stride + i % nl9] = g.lights[i];
    for (int i = threadIdx.x; i < rows * 3; i += blockDim.x) sS[(i / 3) * stride + nl9 + i % 3] = g.ambient[i];
    float *sC = sS + rows * stride;
    for (int i = threadIdx.x; i < g.n_views * 3; i += blockDim.x) sC[i] = g.cam_centres[i];
    __syncthreads();
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < g.P0; i += (int64_t)gridDim.x * blockDim.x) {
        const V3 p = v3(g.points_world[i * 3], g.points_world[i * 3 + 1], g.points_world[i * 3 + 2]);
        const V3 nrm = v3(g.normals_world[i * 3], g.normals_world[i * 3 + 1], g.normals_world[i * 3 + 2]);
        const V3 alb = v3(g.albedo[i * 3], g.albedo[i * 3 + 1], g.albedo[i * 3 + 2]);
        V3 ga = v3(0.f, 0.f, 0.f), gn = v3(0.f, 0.f, 0.f), gp = v3(0.f, 0.f, 0.f);
        for (int n = 0; n < g.n_views; ++n) {
            const float *gs = g.grad_colours + ((int64_t)n * g.P0 + i) * 3;
            const V3 gc = v3(gs[0], gs[1], gs[2]);
            if (gc.x == 0.0f && gc.y == 0.0f && gc.z == 0.0f) continue;
            const float *c = sC + n * 3, *L = sS + (g.lights_per_view ? n * stride : 0);
            shade_point<true>(L, g.n_lights, g.light_type, g.shininess, v3(L[nl9], L[nl9 + 1], L[nl9 + 2]), p, nrm, alb,
                              v3(c[0], c[1], c[2]), gc, ga, gn, gp);
        }
        store3(g.grad_albedo + i * 3, ga);
        store3(g.grad_normals_world + i * 3, gn);
        store3(g.grad_points_shading + i * 3, gp);
    }
}

// Packed clouds: every packed row is its own (view, point), so d albedo / d normal / d position are per row.  Grid
// (point blocks, views), one thread per row of view n's range (as the packed branch of chain_kernel); each row is
// written once, by its view (deterministic, no atomics).  Rows outside every range are left to the caller.
__global__ void __launch_bounds__(256) shade_backward_packed_kernel(const __grid_constant__ dss_render_args g) {
    __shared__ float sL[DSS_MAX_LIGHTS * 9 + 6];   // lights, ambient (3), camera centre (3)
    const int n = blockIdx.y;
    stage_view_shading(sL, g, n);
    __syncthreads();
    const float *amb = sL + DSS_MAX_LIGHTS * 9;
    const ViewRange vr = view_range(g.first_idx, g.num_points, n, g.P0);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < vr.count; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t s = vr.first + i;
        const V3 gc = v3(g.grad_colours[s * 3], g.grad_colours[s * 3 + 1], g.grad_colours[s * 3 + 2]);
        V3 ga = v3(0.f, 0.f, 0.f), gn = v3(0.f, 0.f, 0.f), gp = v3(0.f, 0.f, 0.f);
        if (gc.x != 0.0f || gc.y != 0.0f || gc.z != 0.0f)
            shade_point<true>(sL, g.n_lights, g.light_type, g.shininess, v3(amb[0], amb[1], amb[2]),
                              v3(g.points_world[s * 3], g.points_world[s * 3 + 1], g.points_world[s * 3 + 2]),
                              v3(g.normals_world[s * 3], g.normals_world[s * 3 + 1], g.normals_world[s * 3 + 2]),
                              v3(g.albedo[s * 3], g.albedo[s * 3 + 1], g.albedo[s * 3 + 2]),
                              v3(amb[3], amb[4], amb[5]), gc, ga, gn, gp);
        store3(g.grad_albedo + s * 3, ga);
        store3(g.grad_normals_world + s * 3, gn);
        store3(g.grad_points_shading + s * 3, gp);
    }
}

// Fork/join of the context's side stream: once work has been forked, EVERY return path makes the caller's stream wait
// for it (an error return that skipped the join would let the caller free tensors the side stream still writes).
struct SideJoin {
    dss_ctx *ctx;
    cudaStream_t st;
    bool forked = false, joined = false;
    SideJoin(dss_ctx *c, cudaStream_t s) : ctx(c), st(s) {}
    int fork() {
        DSS_CUDA_TRY(cudaEventRecord(ctx->ev_fork, st));
        DSS_CUDA_TRY(cudaStreamWaitEvent(ctx->side, ctx->ev_fork, 0));
        forked = true;
        return DSS_OK;
    }
    int join() {
        if (!forked || joined) return DSS_OK;
        joined = true;
        DSS_CUDA_TRY(cudaEventRecord(ctx->ev_join, ctx->side));
        DSS_CUDA_TRY(cudaStreamWaitEvent(st, ctx->ev_join, 0));
        return DSS_OK;
    }
    ~SideJoin() {
        if (forked && !joined) {
            cudaEventRecord(ctx->ev_join, ctx->side);
            cudaStreamWaitEvent(st, ctx->ev_join, 0);
        }
    }
};

static int run_colour_backward(dss_ctx *ctx, const dss_render_args *g, cudaStream_t on) {
    const int N = g->n_views, S = g->image_size, K = g->points_per_pixel;
    const int64_t npix = (int64_t)N * S * S;
    const int64_t cP0 = (g->shared_cloud && g->shared_colours && !g->shade) ? g->P0 : 0;
    int rc;
    if (g->shade && g->deterministic_colours) {
        // the training step's d shaded: summed in fixed point, the same bits every run
        rc = colour_backward_fixed(ctx, g->idx, g->weights, g->grad_image, npix, K, g->grad_colours, g->P,
                                   (int64_t)S * S, on);
    } else {
        DSS_CUDA_TRY(cudaMemsetAsync(g->grad_colours, 0, (size_t)(cP0 > 0 ? cP0 : g->P) * 3 * sizeof(float), on));
        rc = colour_backward(ctx, g->idx, g->weights, g->grad_image, npix, K, g->grad_colours, cP0, (int64_t)S * S, on);
    }
    if (rc || !g->shade) return rc;
    // shading backward: d shaded (P,3) -> d albedo, d normal, d position, per world point (shared cloud) or packed row
    DSS_REQUIRE(g->grad_albedo && g->grad_normals_world && g->grad_points_shading && g->points_world,
                "shading backward needs grad_albedo, grad_normals_world, grad_points_shading");
    if (!g->shared_cloud) {
        StageScope prof(ctx, ST_COLOUR_BWD, on);
        shade_backward_packed_kernel<<<dim3(grid_blocks(g->P0, 256, ctx->sm_count, 8), N), 256, 0, on>>>(*g);
        DSS_LAUNCH_CHECK(ctx);
        return DSS_OK;
    }
    // per-view lights at the limits (256 views x 8 lights) take 78 KB: more than the default 48 KB of dynamic shared memory
    const size_t smem = (size_t)((g->n_lights * 9 + 3) * (g->lights_per_view ? N : 1) + N * 3) * sizeof(float);
    if (smem > 48 * 1024)
        DSS_CUDA_TRY(cudaFuncSetAttribute(shade_backward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    StageScope prof(ctx, ST_COLOUR_BWD, on);
    shade_backward_kernel<<<grid_blocks(g->P0, 256, ctx->sm_count, 8), 256, smem, on>>>(*g);
    DSS_LAUNCH_CHECK(ctx);
    return DSS_OK;
}

static int check_common(const dss_render_args *g) {
    DSS_REQUIRE(g != nullptr, "args is null");
    DSS_REQUIRE(g->n_views > 0, "n_views must be positive");
    DSS_REQUIRE(g->P0 >= 0 && g->P >= 0, "negative size");
    DSS_REQUIRE(g->P < (int64_t)INT32_MAX, "more than 2^31-1 packed points");
    DSS_REQUIRE(g->image_size > 0, "image_size must be positive");
    DSS_REQUIRE(g->points_per_pixel > 0 && g->points_per_pixel <= DSS_MAX_POINTS_PER_PIXEL,
                "points_per_pixel must be in [1, 64]");
    DSS_REQUIRE(g->shared_cloud || (g->first_idx && g->num_points), "first_idx/num_points required");
    DSS_REQUIRE(!g->shared_cloud || g->P == (int64_t)g->n_views * g->P0, "P != n_views * P0");
    DSS_REQUIRE(!g->shared_cloud || g->n_views <= DSS_MAX_SHARED_VIEWS, "a shared cloud takes at most 256 views per call");
    if (g->shade) {
        DSS_REQUIRE(g->n_lights >= 1 && g->n_lights <= DSS_MAX_LIGHTS, "n_lights must be in [1, 8]");
        DSS_REQUIRE(g->albedo && g->lights && g->ambient && g->cam_centres && g->normals_world, "shading needs albedo, lights, ambient, cam_centres, normals");
        DSS_REQUIRE(g->light_type == 0 || g->light_type == 1, "light_type must be 0 (directional) or 1 (point)");
    }
    DSS_REQUIRE(g->lights_per_view == 0 || g->lights_per_view == 1, "lights_per_view must be 0 or 1");
    DSS_REQUIRE(!g->lights_per_view || g->shade, "lights_per_view needs the fused shading (shade != 0)");
    return DSS_OK;
}

static int check_preprocess_inputs(const dss_render_args *g) {
    DSS_REQUIRE(g->points_world && g->normals_world && g->proj && g->view && (g->h || g->frames), "null input array");
    DSS_REQUIRE(!(g->h && g->frames), "pass exactly one of h and frames");
    DSS_REQUIRE(!g->frames || (reinterpret_cast<uintptr_t>(g->frames) & 15) == 0, "frames must be 16-byte aligned");
    return DSS_OK;
}

static int run_preprocess(dss_ctx *ctx, const dss_render_args *g, float4 *rec, cudaStream_t st, float *zrange = nullptr) {
    if (zrange) {
        int rc = init_zrange(ctx, zrange, g->n_views, st);
        if (rc) return rc;
    }
    if (g->P == 0 || g->P0 == 0) return DSS_OK;
    int rc = check_preprocess_inputs(g);
    if (rc) return rc;
    dim3 grid(grid_blocks(g->P0, PREPROCESS_THREADS, ctx->sm_count, 8), g->n_views);
    StageScope prof(ctx, ST_PREPROCESS, st);
    preprocess_kernel_for<0>(g->frames != nullptr, g->shade && g->shaded)<<<grid, PREPROCESS_THREADS, 0, st>>>(
        *g, rec, reinterpret_cast<int32_t *>(zrange), PreprocessBins{});
    DSS_LAUNCH_CHECK(ctx);
    return DSS_OK;
}

// The fused route's preprocess, which also counts the forward tile lists of `plan` (packed): the depth-range pre-pass,
// then the counting preprocess.  Fills zrange, the list sizes in BUF_TILE_COUNTS, the packed rectangles and the block
// offsets, and describes them in *out for bin_and_raster.  The grid is COUNTING_WAVES waves of the counting kernel over
// all views (at the occupancy its B*B*NS-counter histogram allows), at most one block per 256 points of a view.
// Every block flushes its whole histogram, so fewer blocks make a cheaper preprocess; but bin_scatter_counted runs on
// the same grid, and its id stores -- most of its time -- fill each block's slots of a list over the block's whole
// lifetime: long-lived blocks leave partly written sectors of the (larger than L2) id buffer to be evicted and merged
// in DRAM.  On the 1M-point / 8 x 512^2 workload (bench.py, H100 SXM, 700 W) 1, 2, 3, 4, 6 and 8 waves gave
// preprocess + scatter 0.561, 0.524, 0.484, 0.490, 0.513, 0.533 ms and 3 waves the best step (DESIGN.md section 6).
constexpr int COUNTING_WAVES = 3;

static int run_counting_preprocess(dss_ctx *ctx, const dss_render_args *g, const TilePlan &plan, float4 *rec,
                                   float *zrange, CountedBins *out, cudaStream_t st) {
    int rc = check_preprocess_inputs(g);
    if (rc) return rc;
    const int N = g->n_views;
    const int64_t nt = (int64_t)plan.B * plan.B * plan.NS;
    const int S = g->image_size;
    PreprocessKernel kern = (S & (S - 1)) == 0 ? preprocess_kernel_for<1>(g->frames != nullptr, g->shade && g->shaded)
                                               : preprocess_kernel_for<2>(g->frames != nullptr, g->shade && g->shaded);
    const size_t smem = (size_t)nt * sizeof(int32_t);
    if (smem > 48 * 1024)
        DSS_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    DSS_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, PREPROCESS_THREADS, smem));
    int64_t blocks = (int64_t)COUNTING_WAVES * (per_sm > 0 ? per_sm : 1) * ctx->sm_count / N;
    const int64_t need = (g->P0 + PREPROCESS_THREADS - 1) / PREPROCESS_THREADS;
    if (blocks > need) blocks = need;
    if (blocks < 1) blocks = 1;
    PreprocessBins pb;
    pb.zrange = zrange;
    pb.B = plan.B;
    pb.NS = plan.NS;
    if ((rc = ctx_get(ctx, BUF_TILE_COUNTS, (size_t)(N * nt + 1), &pb.counts))) return rc;
    if ((rc = ctx_get(ctx, BUF_BIN_RECTS, (size_t)g->P, &pb.rects))) return rc;
    if ((rc = ctx_get(ctx, BUF_BIN_BLOCK_OFFSETS, (size_t)(N * blocks * nt), &pb.block_offsets))) return rc;
    DSS_CUDA_TRY(cudaMemsetAsync(pb.counts, 0, (size_t)(N * nt + 1) * sizeof(int32_t), st));
    {
        StageScope prof(ctx, ST_BIN_COUNT, st);
        if ((rc = init_zrange(ctx, zrange, N, st))) return rc;
        const int nv = g->shared_cloud ? N : 1;
        dim3 grid(grid_blocks(g->P0, 256, ctx->sm_count, 4), g->shared_cloud ? 1 : N);
        depth_range_kernel<<<grid, 256, (size_t)nv * 18 * sizeof(float), st>>>(*g, reinterpret_cast<int32_t *>(zrange));
        DSS_LAUNCH_CHECK(ctx);
    }
    {
        StageScope prof(ctx, ST_PREPROCESS, st);
        kern<<<dim3((unsigned int)blocks, N), PREPROCESS_THREADS, smem, st>>>(*g, rec, nullptr, pb);
        DSS_LAUNCH_CHECK(ctx);
    }
    out->rects = pb.rects;
    out->block_offsets = pb.block_offsets;
    out->blocks = (unsigned int)blocks;
    return DSS_OK;
}

// ---------------------------------------------------------------------------------------------
// Backward tail: per-point gradient clip (rasterizer.py:667-673) and chain through
// ndc = (X/T, Y/T, z_view) to world space: d ndc_xy / d p = J (the same Jacobian as the forward
// pass), d z_view / d p = V[:3, 2].  shared_cloud: one thread per world point loops over the views
// and writes the sum (deterministic, no atomics); otherwise one thread per packed splat.
//   grad_xy:    (P,2) occupancy gradient
//   grad_z:     (P,) z gradient or null
//   grad_shade: position gradient through the shading, shaped like grad_points_world and added to it, or null
// ---------------------------------------------------------------------------------------------

__device__ __forceinline__ void chain_one(const float *M, const float *V, float p0, float p1, float p2,
                                          float gx, float gy, float gz, float &w0, float &w1, float &w2) {
    const float x = fmaf(p0, M[0], fmaf(p1, M[4], fmaf(p2, M[8], M[12])));
    const float y = fmaf(p0, M[1], fmaf(p1, M[5], fmaf(p2, M[9], M[13])));
    const float t = fmaf(p0, M[3], fmaf(p1, M[7], fmaf(p2, M[11], M[15])));
    const float it = 1.0f / t, it2 = it * it;
    float w[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float j0 = M[k * 4 + 0] * it - M[k * 4 + 3] * x * it2;
        const float j1 = M[k * 4 + 1] * it - M[k * 4 + 3] * y * it2;
        w[k] = j0 * gx + j1 * gy + V[k * 4 + 2] * gz;
    }
    w0 = w[0];
    w1 = w[1];
    w2 = w[2];
}

__device__ __forceinline__ void clip_grad(float clip, float &gx, float &gy, float &gz) {
    if (clip > 0.0f) {
        // grad.norm().clamp(0, clip) * normalize(grad)  (F.normalize eps = 1e-12)
        const float nrm = sqrtf(gx * gx + gy * gy + gz * gz);
        const float s = fminf(nrm, clip) / fmaxf(nrm, 1e-12f);
        gx *= s;
        gy *= s;
        gz *= s;
    }
}

__global__ void __launch_bounds__(256) chain_kernel(const __grid_constant__ dss_render_args g, const float2 *grad_xy,
                                                    const float *grad_z, const float *grad_shade) {
    extern __shared__ float sMat[];  // N * 32 floats: proj then view per view (shared_cloud) or 32 (packed)
    if (g.shared_cloud) {
        for (int i = threadIdx.x; i < g.n_views * 16; i += blockDim.x) {
            sMat[(i / 16) * 32 + (i % 16)] = g.proj[i];
            sMat[(i / 16) * 32 + 16 + (i % 16)] = g.view[i];
        }
        __syncthreads();
        for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < g.P0;
             i += (int64_t)gridDim.x * blockDim.x) {
            const float p0 = g.points_world[i * 3], p1 = g.points_world[i * 3 + 1], p2 = g.points_world[i * 3 + 2];
            float acc0 = 0.f, acc1 = 0.f, acc2 = 0.f;
            // views in batches of four: the (independent) gradient loads of a batch are issued together
            for (int n0 = 0; n0 < g.n_views; n0 += 4) {
                float2 g4[4];
                float gz4[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int64_t s = (int64_t)(n0 + j) * g.P0 + i;
                    g4[j] = (n0 + j < g.n_views) ? grad_xy[s] : make_float2(0.f, 0.f);
                    gz4[j] = (grad_z && n0 + j < g.n_views) ? grad_z[s] : 0.0f;
                }
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int n = n0 + j;
                    if (n >= g.n_views) break;
                    const int64_t s = (int64_t)n * g.P0 + i;
                    float gx = g4[j].x, gy = g4[j].y, gz = gz4[j];
                    clip_grad(g.clip_pts_grad, gx, gy, gz);
                    if (g.grad_ndc) {
                        g.grad_ndc[s * 3 + 0] = gx;
                        g.grad_ndc[s * 3 + 1] = gy;
                        g.grad_ndc[s * 3 + 2] = gz;
                    }
                    if (gx != 0.0f || gy != 0.0f || gz != 0.0f) {
                        float w0, w1, w2;
                        chain_one(sMat + n * 32, sMat + n * 32 + 16, p0, p1, p2, gx, gy, gz, w0, w1, w2);
                        acc0 += w0;
                        acc1 += w1;
                        acc2 += w2;
                    }
                }
            }
            if (grad_shade) {
                acc0 += grad_shade[i * 3 + 0];
                acc1 += grad_shade[i * 3 + 1];
                acc2 += grad_shade[i * 3 + 2];
            }
            g.grad_points_world[i * 3 + 0] = acc0;
            g.grad_points_world[i * 3 + 1] = acc1;
            g.grad_points_world[i * 3 + 2] = acc2;
        }
    } else {
        const int n = blockIdx.y;
        if (threadIdx.x < 16) {
            sMat[threadIdx.x] = g.proj[n * 16 + threadIdx.x];
            sMat[16 + threadIdx.x] = g.view[n * 16 + threadIdx.x];
        }
        __syncthreads();
        const ViewRange vr = view_range(g.first_idx, g.num_points, n, g.P0);
        for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < vr.count;
             i += (int64_t)gridDim.x * blockDim.x) {
            const int64_t s = vr.first + i;
            const float2 gxy = grad_xy[s];
            float gx = gxy.x, gy = gxy.y, gz = grad_z ? grad_z[s] : 0.0f;
            clip_grad(g.clip_pts_grad, gx, gy, gz);
            if (g.grad_ndc) {
                g.grad_ndc[s * 3 + 0] = gx;
                g.grad_ndc[s * 3 + 1] = gy;
                g.grad_ndc[s * 3 + 2] = gz;
            }
            float w0 = 0.f, w1 = 0.f, w2 = 0.f;
            if (gx != 0.0f || gy != 0.0f || gz != 0.0f)
                chain_one(sMat, sMat + 16, g.points_world[s * 3], g.points_world[s * 3 + 1], g.points_world[s * 3 + 2],
                          gx, gy, gz, w0, w1, w2);
            if (grad_shade) {
                w0 += grad_shade[s * 3 + 0];
                w1 += grad_shade[s * 3 + 1];
                w2 += grad_shade[s * 3 + 2];
            }
            g.grad_points_world[s * 3 + 0] = w0;
            g.grad_points_world[s * 3 + 1] = w1;
            g.grad_points_world[s * 3 + 2] = w2;
        }
    }
}

// ---------------------------------------------------------------------------------------------
// Camera gradients (the reference differentiates through pytorch3d's transform, rasterizer.py:614, and the shading
// reads cameras.get_camera_center()).  Per (view, point) slot with the clipped NDC gradient g = (gx, gy, gz) and
// p_h = [p 1], clip = p_h M, w = clip3, (x, y) = clip01 / w:
//   d L / d clip = (gx / w, gy / w, 0, -(gx x + gy y) / w)
//   grad_proj[n][r][c] = sum_p p_h[r] dclip[c]        (column 2 stays zero: screen z is the view depth)
//   grad_view[n][r][2] = sum_p p_h[r] gz
// and with fused shading grad_cam[n] = sum_p normalize_bwd(v, g_v), v = normalize(cam - p).
// Pass 1: grid (point blocks, views), every block writes its CAM_SUMS sums (fp64) to a partials array.  Pass 2: one
// block per view adds its partials in block order.  Fixed grid and fixed reduction order: bit-reproducible.
// ---------------------------------------------------------------------------------------------
constexpr int CAM_SUMS = 19;   // 12 proj (rows 0..3 x columns 0, 1, 3), 4 view (rows 0..3, column 2), 3 camera centre

constexpr int CAM_BATCH = 4;   // slots per thread whose loads are issued together

// partials: (N, gridDim.x, CAM_SUMS).  SHADE: also the camera-centre sums, from d L / d shaded in g.grad_colours.
template <bool SHADE>
__global__ void __launch_bounds__(256) camera_partials_kernel(const __grid_constant__ dss_render_args g,
                                                              double *partials) {
    __shared__ float sM[16];
    __shared__ float sL[DSS_MAX_LIGHTS * 9 + 6];   // lights, ambient (3), camera centre (3)
    __shared__ double sPart[8][CAM_SUMS];
    const int n = blockIdx.y;
    if (threadIdx.x < 16) sM[threadIdx.x] = g.proj[n * 16 + threadIdx.x];
    if (SHADE) stage_view_shading(sL, g, n);
    __syncthreads();
    double acc[CAM_SUMS];
#pragma unroll
    for (int k = 0; k < CAM_SUMS; ++k) acc[k] = 0.0;
    const ViewRange vr = view_range(g.shared_cloud ? nullptr : g.first_idx, g.num_points, n, g.P0);
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i0 < vr.count; i0 += CAM_BATCH * stride) {
        float gd[CAM_BATCH][3], gs[CAM_BATCH][3];
#pragma unroll
        for (int j = 0; j < CAM_BATCH; ++j) {
            const int64_t i = i0 + j * stride, s = vr.first + i;
            const bool in = i < vr.count;
#pragma unroll
            for (int e = 0; e < 3; ++e) {
                gd[j][e] = in ? g.grad_ndc[s * 3 + e] : 0.0f;
                gs[j][e] = (SHADE && in) ? g.grad_colours[s * 3 + e] : 0.0f;
            }
        }
#pragma unroll
        for (int j = 0; j < CAM_BATCH; ++j) {
            const int64_t i = i0 + j * stride, s = vr.first + i;
            const int64_t src = g.shared_cloud ? i : s;
            const float gx = gd[j][0], gy = gd[j][1], gz = gd[j][2];
            if (gx != 0.0f || gy != 0.0f || gz != 0.0f) {
                const float ph[4] = {g.points_world[src * 3], g.points_world[src * 3 + 1], g.points_world[src * 3 + 2],
                                     1.0f};
                const float x = fmaf(ph[0], sM[0], fmaf(ph[1], sM[4], fmaf(ph[2], sM[8], sM[12])));
                const float y = fmaf(ph[0], sM[1], fmaf(ph[1], sM[5], fmaf(ph[2], sM[9], sM[13])));
                const float t = fmaf(ph[0], sM[3], fmaf(ph[1], sM[7], fmaf(ph[2], sM[11], sM[15])));
                const float it = 1.0f / t;
                const float d0 = gx * it, d1 = gy * it, d3 = -(gx * (x * it) + gy * (y * it)) * it;
#pragma unroll
                for (int r = 0; r < 4; ++r) {
                    const double pr = (double)ph[r];
                    acc[3 * r + 0] = fma(pr, (double)d0, acc[3 * r + 0]);
                    acc[3 * r + 1] = fma(pr, (double)d1, acc[3 * r + 1]);
                    acc[3 * r + 2] = fma(pr, (double)d3, acc[3 * r + 2]);
                    acc[12 + r] = fma(pr, (double)gz, acc[12 + r]);
                }
            }
            const V3 gc = v3(gs[j][0], gs[j][1], gs[j][2]);
            if (SHADE && (gc.x != 0.0f || gc.y != 0.0f || gc.z != 0.0f)) {
                const float *amb = sL + DSS_MAX_LIGHTS * 9;
                V3 ga = v3(0.f, 0.f, 0.f), gn = v3(0.f, 0.f, 0.f), gp = v3(0.f, 0.f, 0.f), gcam = v3(0.f, 0.f, 0.f);
                shade_point<true, true>(
                    sL, g.n_lights, g.light_type, g.shininess, v3(amb[0], amb[1], amb[2]),
                    v3(g.points_world[src * 3], g.points_world[src * 3 + 1], g.points_world[src * 3 + 2]),
                    v3(g.normals_world[src * 3], g.normals_world[src * 3 + 1], g.normals_world[src * 3 + 2]),
                    v3(g.albedo[src * 3], g.albedo[src * 3 + 1], g.albedo[src * 3 + 2]), v3(amb[3], amb[4], amb[5]), gc,
                    ga, gn, gp, &gcam);
                acc[16] += (double)gcam.x;
                acc[17] += (double)gcam.y;
                acc[18] += (double)gcam.z;
            }
        }
    }
    const double v = block_sum(acc, sPart);
    if (threadIdx.x < CAM_SUMS) partials[((int64_t)n * gridDim.x + blockIdx.x) * CAM_SUMS + threadIdx.x] = v;
}

// output rows of the camera gradients: view m's (4,4) / (4,4) / (3,) rows from its CAM_SUMS totals
struct CamRows {
    float *grad_proj, *grad_view, *grad_cam;
    __device__ __forceinline__ void operator()(const double *tot, int l, int m, int k) const {
        if (k < 16) {
            const int r = k >> 2, c = k & 3;
            grad_proj[m * 16 + k] = c == 2 ? 0.0f : (float)tot[3 * r + (c == 3 ? 2 : c)];
            grad_view[m * 16 + k] = c == 2 ? (float)tot[12 + r] : 0.0f;
        }
        if (grad_cam && k < 3) grad_cam[m * 3 + k] = (float)tot[16 + k];
    }
};

// ---------------------------------------------------------------------------------------------
// Light gradients (the reference's lights are tensors that autograd reaches through lighting.py:10-172).  Light l's
// share of the gradient depends only on its own terms and the normalised normal and view direction of the
// (view, point); with gc = d L / d shaded:
//   g_vec = normalize_bwd(d, g_d)   (direction; for point lights the location: d = normalize(loc - p))
//   g_cd = gc * alb * relu(n.d),   g_cs = gc * pw,   g_amb = gc * alb   (ambient: summed over the lights' terms)
// Pass 1: grid (point blocks, views, lights), every block writes its LIGHT_SUMS sums (fp64) to a partials array, the
// ambient ones from the l = 0 slice.  Pass 2: one block per (light, output row) adds the partials in a fixed order.
// ---------------------------------------------------------------------------------------------
constexpr int LIGHT_SUMS = 12;   // direction or location (3), diffuse rgb (3), specular rgb (3), ambient rgb (3)

// partials: (N, gridDim.z, gridDim.x, LIGHT_SUMS)
__global__ void __launch_bounds__(256) light_partials_kernel(const __grid_constant__ dss_render_args g,
                                                             double *partials) {
    __shared__ float sL[9 + 3];   // the light's row, camera centre
    __shared__ double sPart[8][LIGHT_SUMS];
    const int n = blockIdx.y, l = blockIdx.z;
    if (threadIdx.x < 9) sL[threadIdx.x] = view_lights(g, n)[l * 9 + threadIdx.x];
    if (threadIdx.x < 3) sL[9 + threadIdx.x] = g.cam_centres[n * 3 + threadIdx.x];
    __syncthreads();
    const V3 cam = v3(sL[9], sL[10], sL[11]);
    double acc[LIGHT_SUMS];
#pragma unroll
    for (int k = 0; k < LIGHT_SUMS; ++k) acc[k] = 0.0;
    // view n's rows of d L / d shaded: n*P0 .. n*P0+P0 (shared cloud, world point i) or its packed range (row s)
    const ViewRange vr = view_range(g.shared_cloud ? nullptr : g.first_idx, g.num_points, n, g.P0);
    const float *gsh = g.grad_colours + vr.first * 3;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i0 < vr.count; i0 += CAM_BATCH * stride) {
        float gs[CAM_BATCH][3];
#pragma unroll
        for (int j = 0; j < CAM_BATCH; ++j) {
            const int64_t i = i0 + j * stride;
#pragma unroll
            for (int e = 0; e < 3; ++e) gs[j][e] = i < vr.count ? gsh[i * 3 + e] : 0.0f;
        }
#pragma unroll
        for (int j = 0; j < CAM_BATCH; ++j) {
            const V3 gc = v3(gs[j][0], gs[j][1], gs[j][2]);
            if (gc.x == 0.0f && gc.y == 0.0f && gc.z == 0.0f) continue;
            const int64_t i = i0 + j * stride, src = g.shared_cloud ? i : vr.first + i;
            const V3 p = v3(g.points_world[src * 3], g.points_world[src * 3 + 1], g.points_world[src * 3 + 2]);
            const V3 alb = v3(g.albedo[src * 3], g.albedo[src * 3 + 1], g.albedo[src * 3 + 2]);
            float nlen, vlen;
            const V3 nh =
                normalize3(v3(g.normals_world[src * 3], g.normals_world[src * 3 + 1], g.normals_world[src * 3 + 2]), nlen);
            const V3 v = normalize3(sub3(cam, p), vlen);
            V3 diff = v3(0.f, 0.f, 0.f), spec = v3(0.f, 0.f, 0.f), g_nh = v3(0.f, 0.f, 0.f), g_v = v3(0.f, 0.f, 0.f);
            const LightTerm t = shade_light<true>(sL, g.light_type, g.shininess, p, nh, v, alb, gc, diff, spec, g_nh, g_v);
            const V3 gvec = normalize3_bwd(t.d, t.dlen, t.draw, t.g_d);
            const V3 ga = v3(gc.x * alb.x, gc.y * alb.y, gc.z * alb.z);
            acc[0] += (double)gvec.x;
            acc[1] += (double)gvec.y;
            acc[2] += (double)gvec.z;
            acc[3] += (double)(ga.x * t.lam);
            acc[4] += (double)(ga.y * t.lam);
            acc[5] += (double)(ga.z * t.lam);
            acc[6] += (double)(gc.x * t.pw);
            acc[7] += (double)(gc.y * t.pw);
            acc[8] += (double)(gc.z * t.pw);
            if (l == 0) {
                acc[9] += (double)ga.x;
                acc[10] += (double)ga.y;
                acc[11] += (double)ga.z;
            }
        }
    }
    const double v = block_sum(acc, sPart);
    if (threadIdx.x < LIGHT_SUMS)
        partials[(((int64_t)n * gridDim.z + l) * gridDim.x + blockIdx.x) * LIGHT_SUMS + threadIdx.x] = v;
}

// output rows of the light gradients: light l's row of output row m, and the ambient row from the l = 0 slice
struct LightRows {
    float *grad_lights, *grad_ambient;
    __device__ __forceinline__ void operator()(const double *tot, int l, int m, int k) const {
        if (grad_lights && k < 9) grad_lights[((int64_t)m * gridDim.x + l) * 9 + k] = (float)tot[k];
        if (grad_ambient && l == 0 && k < 3) grad_ambient[m * 3 + k] = (float)tot[9 + k];
    }
};

// point blocks per slice of the partials kernels: one wave over all slices at two blocks per SM (95-122 registers per
// thread), and no more blocks than the points need
static unsigned int wave_blocks(const dss_ctx *ctx, int64_t slices, int64_t P0) {
    const int64_t want = ((int64_t)ctx->sm_count * 2 + slices - 1) / slices, need = (P0 + 255) / 256;
    return (unsigned int)(want < need ? want : need);
}

}  // namespace dss

extern "C" {

int dss_preprocess(dss_ctx *ctx, const dss_render_args *g, void *stream) {
    using namespace dss;
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    int rc = check_common(g);
    if (rc) return rc;
    float4 *rec = reinterpret_cast<float4 *>(g->records);
    if (!rec && (rc = ctx_get(ctx, BUF_RECORDS, (size_t)(2 * (g->P > 0 ? g->P : 1)), &rec))) return rc;
    return run_preprocess(ctx, g, rec, (cudaStream_t)stream);
}

int dss_render_forward(dss_ctx *ctx, const dss_render_args *g, void *stream) {
    using namespace dss;
    cudaStream_t st = (cudaStream_t)stream;
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    int rc = check_common(g);
    if (rc) return rc;
    DSS_REQUIRE(g->image && g->idx && g->scaler && (g->shade ? (const void *)g->shaded : (const void *)g->colours),
                "forward needs image, idx, scaler and colours (or, with shade, the shaded output)");
    float4 *rec = reinterpret_cast<float4 *>(g->records);
    if (!rec && (rc = ctx_get(ctx, BUF_RECORDS, (size_t)(2 * (g->P > 0 ? g->P : 1)), &rec))) return rc;
    DSS_REQUIRE((reinterpret_cast<uintptr_t>(rec) & 15) == 0, "records must be 16-byte aligned");
    float *zrange = nullptr;
    if ((rc = ctx_get(ctx, BUF_ZRANGE, (size_t)(2 * g->n_views), &zrange))) return rc;
    // the preprocess counts the tile lists itself wherever the binning would use block histograms and packed rectangles
    TilePlan plan;
    if ((rc = plan_tiles(ctx, g->n_views, g->image_size, g->points_per_pixel, &plan))) return rc;
    CountedBins counted;
    const bool count_here = plan.packed && g->P > 0 && g->P0 > 0;
    if (count_here) rc = run_counting_preprocess(ctx, g, plan, rec, zrange, &counted, st);
    else rc = run_preprocess(ctx, g, rec, st, zrange);
    if (rc) return rc;
    if (g->visible) DSS_CUDA_TRY(cudaMemsetAsync(g->visible, 0, (size_t)g->P, st));
    // fused count pass of the backward's binning (see RasterArgs::cell_counts)
    int32_t *cell_counts = nullptr;
    if (g->cell_counts && g->visible && (reinterpret_cast<uintptr_t>(g->visible) & 3) == 0) {
        cell_counts = g->cell_counts;
        DSS_CUDA_TRY(cudaMemsetAsync(cell_counts, 0, (size_t)occ_cell_count(g->n_views, g->image_size) * sizeof(int32_t), st));
    }
    RasterArgs a;
    memset(&a, 0, sizeof(a));
    a.rec = rec;
    a.cutoff = nullptr;
    a.cutoff_uniform = g->cutoff_threshold;
    a.N = g->n_views;
    a.S = g->image_size;
    a.K = g->points_per_pixel;
    a.depth_merge = g->depth_merging_threshold;
    a.idx = g->idx;
    a.zbuf = g->zbuf;
    a.qvalue = g->qvalue;
    a.occ = nullptr;
    a.scaler = g->scaler;
    a.colours = g->shade ? g->shaded : g->colours;
    a.colour_P0 = (g->shared_cloud && g->shared_colours && !g->shade) ? g->P0 : 0;
    a.image = g->image;
    a.weights = g->weights;
    a.visible = g->visible;
    a.cell_counts = cell_counts;
    a.zrange = zrange;   // already filled by the preprocess or its pre-pass
    rc = bin_and_raster(ctx, a, g->shared_cloud ? nullptr : g->first_idx, g->num_points, g->P0, st,
                        count_here ? &counted : nullptr);
    if (rc || !g->depth) return rc;
    return depth_forward(ctx, g, rec, st);
}

int dss_colour_backward(dss_ctx *ctx, const dss_render_args *g, void *stream) {
    using namespace dss;
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    int rc = check_common(g);
    if (rc) return rc;
    DSS_REQUIRE(g->grad_image && g->idx && g->weights && g->grad_colours, "colour backward needs grad_image, idx, weights, grad_colours");
    if (g->P == 0) return DSS_OK;
    return run_colour_backward(ctx, g, (cudaStream_t)stream);
}

int dss_render_backward(dss_ctx *ctx, const dss_render_args *g, void *stream) {
    using namespace dss;
    cudaStream_t st = (cudaStream_t)stream;
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    int rc = check_common(g);
    if (rc) return rc;
    DSS_REQUIRE(g->grad_image && g->idx && g->weights && g->visible, "backward needs grad_image, idx, weights, visible");
    DSS_REQUIRE(g->records || (g->ndc && g->radii), "backward needs the records (or ndc and radii) saved by the forward pass");
    DSS_REQUIRE(g->grad_points_world && g->points_world && g->proj && g->view, "null pointer");
    const int N = g->n_views, S = g->image_size, K = g->points_per_pixel;
    const int64_t P = g->P, npix = (int64_t)N * S * S;
    const int64_t *fi = g->shared_cloud ? nullptr : g->first_idx;
    if (P == 0) return DSS_OK;
    float4 *rec = reinterpret_cast<float4 *>(g->records);
    float *rs = nullptr, *gxy = nullptr;
    if (!rec) {
        // rebuild from the tensors the caller saved (another forward may have reused the scratch)
        if ((rc = ctx_get(ctx, BUF_RECORDS, (size_t)(2 * P), &rec))) return rc;
        if ((rc = pack_records(ctx, g->ndc, g->radii, nullptr, P, rec, st))) return rc;
    }
    if ((rc = ctx_get(ctx, BUF_RS, (size_t)N, &rs))) return rc;
    if ((rc = ctx_get(ctx, BUF_GRADXY, (size_t)(2 * P), &gxy))) return rc;
    // The colour scatter does not depend on the occupancy path: fork it onto the context's side stream so that its
    // atomics overlap the (latency-bound) binning / median kernels, join before the chain kernel (and on every return).
    SideJoin side(ctx, st);
    if (g->grad_colours != nullptr) {
        if ((rc = side.fork())) return rc;
        if ((rc = run_colour_backward(ctx, g, ctx->side))) return rc;
    }
    if ((rc = occ_backward(ctx, rec, g->visible, rs, g->radii_backward_scaler, g->grad_image, 4, 3, fi, g->num_points, N,
                           g->P0, S, gxy,
                           (g->cell_counts && (reinterpret_cast<uintptr_t>(g->visible) & 3) == 0) ? g->cell_counts : nullptr,
                           st)))
        return rc;
    if (g->search_radius)
        DSS_CUDA_TRY(cudaMemcpyAsync(g->search_radius, rs, (size_t)N * sizeof(float), cudaMemcpyDeviceToDevice, st));
    if ((rc = side.join())) return rc;
    float *gz = nullptr;
    if (g->grad_zbuf || g->grad_depth) {
        if ((rc = ctx_get(ctx, BUF_MISC, (size_t)P, &gz))) return rc;
        DSS_CUDA_TRY(cudaMemsetAsync(gz, 0, (size_t)P * sizeof(float), st));
        if (g->grad_zbuf && (rc = zbuf_backward(ctx, g->idx, g->grad_zbuf, npix, K, gz, 1, st))) return rc;
        if (g->grad_depth && (rc = depth_backward(ctx, g, gz, st))) return rc;
    }
    const float2 *grad_xy = reinterpret_cast<const float2 *>(gxy);
    // the shading's position gradient exists only when this call ran the colour half
    const float *grad_shade = (g->shade && g->grad_colours != nullptr) ? g->grad_points_shading : nullptr;
    StageScope prof(ctx, ST_CHAIN, st);
    if (g->shared_cloud) {
        chain_kernel<<<grid_blocks(g->P0, 256, ctx->sm_count, 8), 256, (size_t)N * 32 * sizeof(float), st>>>(
            *g, grad_xy, gz, grad_shade);
    } else {
        dim3 grid(grid_blocks(g->P0, 256, ctx->sm_count, 8), N);
        chain_kernel<<<grid, 256, 32 * sizeof(float), st>>>(*g, grad_xy, gz, grad_shade);
    }
    DSS_LAUNCH_CHECK(ctx);
    return DSS_OK;
}

int dss_camera_backward(dss_ctx *ctx, const dss_render_args *g, float *grad_proj, float *grad_view,
                        float *grad_cam_centres, void *stream) {
    using namespace dss;
    cudaStream_t st = (cudaStream_t)stream;
    // every argument check comes before the first use of the context
    int rc = check_common(g);
    if (rc) return rc;
    DSS_REQUIRE(grad_proj && grad_view, "camera backward needs grad_proj and grad_view");
    DSS_REQUIRE(g->grad_ndc, "camera backward reads the grad_ndc that dss_render_backward wrote");
    DSS_REQUIRE(g->points_world && g->proj, "camera backward needs points_world and proj");
    if (grad_cam_centres) {
        DSS_REQUIRE(g->shade, "grad_cam_centres needs the fused shading inputs (shade != 0)");
        DSS_REQUIRE(g->grad_colours, "grad_cam_centres reads d L / d shaded from grad_colours");
    }
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    const int N = g->n_views;
    const bool shade = grad_cam_centres != nullptr;
    if (g->P == 0 || g->P0 == 0) {
        DSS_CUDA_TRY(cudaMemsetAsync(grad_proj, 0, (size_t)N * 16 * sizeof(float), st));
        DSS_CUDA_TRY(cudaMemsetAsync(grad_view, 0, (size_t)N * 16 * sizeof(float), st));
        if (shade) DSS_CUDA_TRY(cudaMemsetAsync(grad_cam_centres, 0, (size_t)N * 3 * sizeof(float), st));
        return DSS_OK;
    }
    const unsigned int blocks = wave_blocks(ctx, N, g->P0);
    double *partials = nullptr;
    if ((rc = ctx_get(ctx, BUF_CAMERA, (size_t)N * blocks * CAM_SUMS, &partials))) return rc;
    StageScope prof(ctx, ST_CAMERA_BWD, st);
    if (shade) camera_partials_kernel<true><<<dim3(blocks, N), 256, 0, st>>>(*g, partials);
    else camera_partials_kernel<false><<<dim3(blocks, N), 256, 0, st>>>(*g, partials);
    DSS_LAUNCH_CHECK(ctx);
    grad_finish_kernel<CAM_SUMS><<<dim3(1, N), 256, 0, st>>>(partials, (int)blocks, N, 1,
                                                             CamRows{grad_proj, grad_view, grad_cam_centres});
    DSS_LAUNCH_CHECK(ctx);
    return DSS_OK;
}

int dss_light_backward(dss_ctx *ctx, const dss_render_args *g, float *grad_lights, float *grad_ambient, void *stream) {
    using namespace dss;
    cudaStream_t st = (cudaStream_t)stream;
    // every argument check comes before the first use of the context
    int rc = check_common(g);
    if (rc) return rc;
    DSS_REQUIRE(g->shade, "light backward needs the fused shading inputs (shade != 0)");
    DSS_REQUIRE(g->grad_colours, "light backward reads d L / d shaded from grad_colours");
    DSS_REQUIRE(g->points_world, "light backward needs points_world");
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    const int N = g->n_views, L = g->n_lights, rows = g->lights_per_view ? N : 1;
    if (!grad_lights && !grad_ambient) return DSS_OK;
    if (g->P0 == 0) {
        if (grad_lights) DSS_CUDA_TRY(cudaMemsetAsync(grad_lights, 0, (size_t)rows * L * 9 * sizeof(float), st));
        if (grad_ambient) DSS_CUDA_TRY(cudaMemsetAsync(grad_ambient, 0, (size_t)rows * 3 * sizeof(float), st));
        return DSS_OK;
    }
    // the ambient sums live in the l = 0 slice: without grad_lights that slice is all that is needed
    const int nl = grad_lights ? L : 1;
    const unsigned int blocks = wave_blocks(ctx, (int64_t)N * nl, g->P0);
    double *partials = nullptr;
    if ((rc = ctx_get(ctx, BUF_LIGHT, (size_t)N * nl * blocks * LIGHT_SUMS, &partials))) return rc;
    StageScope prof(ctx, ST_LIGHT_BWD, st);
    light_partials_kernel<<<dim3(blocks, N, nl), 256, 0, st>>>(*g, partials);
    DSS_LAUNCH_CHECK(ctx);
    grad_finish_kernel<LIGHT_SUMS><<<dim3(nl, rows), 256, 0, st>>>(partials, (int)blocks, N, g->lights_per_view,
                                                                    LightRows{grad_lights, grad_ambient});
    DSS_LAUNCH_CHECK(ctx);
    return DSS_OK;
}

}  // extern "C"
