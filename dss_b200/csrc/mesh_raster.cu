// mesh_raster.cu -- opaque triangle meshes: the closest face per pixel, and flat shading (dss_rasterize_mesh).
//
// pytorch3d's rasterize_meshes with the settings of the reference's data script (blur_radius 0, no perspective-correct
// barycentrics, no back-face culling, front fragment only) followed by HardFlatShader, for one shared mesh seen by N
// cameras.  The rules are restated in include/dss_b200.h and DESIGN.md; every value the coverage test and the depth
// depend on is formed with explicit round-to-nearest operations, so the result is the same bits as the float32 oracle.
//
// Per chunk of views:
//   1. screen_kernel : one thread per (view, vertex): NDC x, y as the splat preprocess forms them, view-space z.
//   2. count_kernel  : one thread per (view, face): the rectangle of pixel centres inside the face's closed bounding
//                      box (exact, by the pixel-centre expression itself) and its size; 0 for skipped faces.
//   3. a 64-bit exclusive scan of the sizes (exclusive_scan_i64, 3 launches).
//   4. item_kernel   : one thread per (face, pixel) item, found by binary search over the scan: the coverage test and
//                      a 64-bit atomicMin of (depth bits << 32 | face) into the pixel's key.  Faces of any size spread
//                      evenly over the grid; the minimum does not depend on the order of the atomics.
//   5. resolve_kernel: one thread per pixel writes pix_to_face, zbuf and (optionally) the shaded RGBA.
// No float atomics, no host synchronisation (the item kernel reads the total from the device).
#include "common.cuh"
#include "kernels.cuh"
#include "shading.cuh"

namespace dss {

constexpr int MESH_THREADS = 256;
constexpr int64_t MESH_CHUNK_ENTRIES = (int64_t)1 << 23;             // (view, face) entries per chunk
constexpr int64_t MESH_CHUNK_PIXELS = (int64_t)1 << 25;              // pixel keys per chunk
constexpr unsigned long long MESH_EMPTY = ~0ull;

// E(p, a, b) = (p.x - a.x)(b.y - a.y) - (p.y - a.y)(b.x - a.x), every operation rounded on its own (no contraction)
__device__ __forceinline__ float edge_fn(float px, float py, float ax, float ay, float bx, float by) {
    return __fsub_rn(__fmul_rn(__fsub_rn(px, ax), __fsub_rn(by, ay)), __fmul_rn(__fsub_rn(py, ay), __fsub_rn(bx, ax)));
}

// first pixel index i in [0, S] whose centre pix_to_ndc(i) >= lo (S: none), lo not NaN
__device__ __forceinline__ int first_centre_at_or_above(float lo, int S) {
    const float e = ceilf(((lo + 1.0f) * (float)S - 1.0f) * 0.5f);
    int i = (int)fminf(fmaxf(e, 0.0f), (float)S);
    while (i > 0 && pix_to_ndc(i - 1, S) >= lo) --i;
    while (i < S && pix_to_ndc(i, S) < lo) ++i;
    return i;
}
// last pixel index i in [-1, S-1] whose centre pix_to_ndc(i) <= hi (-1: none), hi not NaN
__device__ __forceinline__ int last_centre_at_or_below(float hi, int S) {
    const float e = floorf(((hi + 1.0f) * (float)S - 1.0f) * 0.5f);
    int i = (int)fminf(fmaxf(e, -1.0f), (float)(S - 1));
    while (i < S - 1 && pix_to_ndc(i + 1, S) <= hi) ++i;
    while (i >= 0 && pix_to_ndc(i, S) > hi) --i;
    return i;
}

// the face's vertex indices, or false when one lies outside [0, V) (the face then covers nothing)
__device__ __forceinline__ bool face_verts(const int32_t *faces, int64_t f, int64_t V, int &i0, int &i1, int &i2) {
    i0 = faces[f * 3 + 0];
    i1 = faces[f * 3 + 1];
    i2 = faces[f * 3 + 2];
    return (uint64_t)(int64_t)i0 < (uint64_t)V && (uint64_t)(int64_t)i1 < (uint64_t)V &&
           (uint64_t)(int64_t)i2 < (uint64_t)V;
}

// 1. Grid (vertex blocks, chunk views).  The expressions of the splat preprocess (render.cu, preprocess_splats) for a
//    splat centre: x = [p 1] . M[:,0], t = [p 1] . M[:,3] as nested fmaf, NDC x = x * rcp(t); z = [p 1] . V[:,2].
__global__ void __launch_bounds__(MESH_THREADS) mesh_screen_kernel(const float *verts, int64_t V, const float *proj,
                                                                   const float *view, int n0, float4 *screen) {
    __shared__ float sM[16], sV[16];
    const int c = blockIdx.y, n = n0 + c;
    if (threadIdx.x < 16) {
        sM[threadIdx.x] = proj[n * 16 + threadIdx.x];
        sV[threadIdx.x] = view[n * 16 + threadIdx.x];
    }
    __syncthreads();
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < V; i += (int64_t)gridDim.x * blockDim.x) {
        const float p0 = verts[i * 3 + 0], p1 = verts[i * 3 + 1], p2 = verts[i * 3 + 2];
        const float x = fmaf(p0, sM[0], fmaf(p1, sM[4], fmaf(p2, sM[8], sM[12])));
        const float y = fmaf(p0, sM[1], fmaf(p1, sM[5], fmaf(p2, sM[9], sM[13])));
        const float t = fmaf(p0, sM[3], fmaf(p1, sM[7], fmaf(p2, sM[11], sM[15])));
        const float zv = fmaf(p0, sV[2], fmaf(p1, sV[6], fmaf(p2, sV[10], sV[14])));
        const float irt = rcp_approx(t);
        screen[(int64_t)c * V + i] = make_float4(x * irt, y * irt, zv, 0.0f);
    }
}

// 2. One thread per (chunk view, face): counts[e] = pixel centres inside the closed bounding box, 0 when the face is
//    skipped (max z < 0, |E(v0, v1, v2)| <= 1e-8, an index out of range, or a NaN box).  rects[e] = {column lo, row lo,
//    width, 0} in pixel-index space (pix_to_ndc order, before the image flip).
__global__ void __launch_bounds__(MESH_THREADS) mesh_count_kernel(const int32_t *faces, int64_t F, int64_t V,
                                                                  const float4 *screen, int64_t M, int S,
                                                                  int64_t *counts, int4 *rects) {
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < M; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t c = e / F, f = e - c * F;
        int i0, i1, i2;
        int64_t cnt = 0;
        int4 r = make_int4(0, 0, 0, 0);
        if (face_verts(faces, f, V, i0, i1, i2)) {
            const float4 a = screen[c * V + i0], b = screen[c * V + i1], d = screen[c * V + i2];
            const float zmax = fmaxf(fmaxf(a.z, b.z), d.z);
            const float area = edge_fn(a.x, a.y, b.x, b.y, d.x, d.y);
            const float xmin = fminf(fminf(a.x, b.x), d.x), xmax = fmaxf(fmaxf(a.x, b.x), d.x);
            const float ymin = fminf(fminf(a.y, b.y), d.y), ymax = fmaxf(fmaxf(a.y, b.y), d.y);
            const bool skip = zmax < 0.0f || (area <= 1e-8f && area >= -1e-8f);
            // a NaN bound contains no pixel centre (the comparisons of the box test are false)
            if (!skip && xmin == xmin && xmax == xmax && ymin == ymin && ymax == ymax) {
                const int cx0 = first_centre_at_or_above(xmin, S), cx1 = last_centre_at_or_below(xmax, S);
                const int cy0 = first_centre_at_or_above(ymin, S), cy1 = last_centre_at_or_below(ymax, S);
                if (cx1 >= cx0 && cy1 >= cy0) {
                    r = make_int4(cx0, cy0, cx1 - cx0 + 1, 0);
                    cnt = (int64_t)(cx1 - cx0 + 1) * (cy1 - cy0 + 1);
                }
            }
        }
        counts[e] = cnt;
        rects[e] = r;
    }
}

// 4. One thread per (face, pixel-centre) item of the chunk.  Coverage and depth, with p the pixel centre:
//      den = E(v2, v0, v1) + 1e-8,  w0 = E(p, v1, v2) / den,  w1 = E(p, v2, v0) / den,  w2 = E(p, v0, v1) / den
//      pz  = (w0 z0 + w1 z1) + w2 z2;   covered: w0 > 0 && w1 > 0 && w2 > 0 && pz >= 0
//    The key (bits of pz + 0 << 32 | face) orders by depth, then by face index: atomicMin keeps the closest face.
__global__ void __launch_bounds__(MESH_THREADS) mesh_item_kernel(const int32_t *faces, int64_t F, const float4 *screen,
                                                                 int64_t V, const int64_t *offsets, const int4 *rects,
                                                                 int64_t M, int S, unsigned long long *keys) {
    const int64_t total = offsets[M];
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
        // the last entry whose range starts at or before t (entries of empty faces share their successor's offset)
        int64_t lo = 0, hi = M;
        while (hi - lo > 1) {
            const int64_t mid = (lo + hi) >> 1;
            if (offsets[mid] <= t) lo = mid;
            else hi = mid;
        }
        const int64_t e = lo, c = e / F, f = e - c * F;
        const int4 r = rects[e];
        const int k = (int)(t - offsets[e]);
        const int xi = r.x + k % r.z, yi = r.y + k / r.z;
        const float px = pix_to_ndc(xi, S), py = pix_to_ndc(yi, S);
        int i0, i1, i2;
        face_verts(faces, f, V, i0, i1, i2);   // in range: the face has items
        const float4 a = screen[c * V + i0], b = screen[c * V + i1], d = screen[c * V + i2];
        const float den = __fadd_rn(edge_fn(d.x, d.y, a.x, a.y, b.x, b.y), 1e-8f);
        const float w0 = __fdiv_rn(edge_fn(px, py, b.x, b.y, d.x, d.y), den);
        const float w1 = __fdiv_rn(edge_fn(px, py, d.x, d.y, a.x, a.y), den);
        const float w2 = __fdiv_rn(edge_fn(px, py, a.x, a.y, b.x, b.y), den);
        const float pz = __fadd_rn(__fadd_rn(__fmul_rn(w0, a.z), __fmul_rn(w1, b.z)), __fmul_rn(w2, d.z));
        if (w0 > 0.0f && w1 > 0.0f && w2 > 0.0f && pz >= 0.0f) {
            const unsigned long long key =
                ((unsigned long long)__float_as_uint(__fadd_rn(pz, 0.0f)) << 32) | (unsigned long long)(uint32_t)f;
            // image row S-1-yi, column S-1-xi (the point rasterizer's flip, raster_fwd.cu pixel_epilogue)
            atomicMin(&keys[((c * S) + (S - 1 - yi)) * (int64_t)S + (S - 1 - xi)], key);
        }
    }
}

struct MeshShading {
    int n_lights, light_type, lights_per_view;
    float shininess;
    const float *lights, *ambient, *cam_centres;
};

// 5. Grid (pixel blocks, chunk views).  pix_to_face / zbuf from the key (-1 / -1 where no face covers the pixel); with
//    rgba, flat shading of the face (pytorch3d flat_shading + hard_rgb_blend, white vertex colours, materials of ones):
//    shade_point at the face centroid with normal normalize(cross(v1 - v0, v2 - v0)); background (1, 1, 1, 0).
__global__ void __launch_bounds__(MESH_THREADS) mesh_resolve_kernel(const unsigned long long *keys, int n0, int S,
                                                                    const float *verts, const int32_t *faces,
                                                                    int32_t *pix_to_face, float *zbuf, float *rgba,
                                                                    const MeshShading sh) {
    __shared__ float sL[DSS_MAX_LIGHTS * 9 + 6];   // lights, ambient (3), camera centre (3)
    const int c = blockIdx.y, n = n0 + c;
    if (rgba) {
        const float *L = sh.lights_per_view ? sh.lights + (int64_t)n * sh.n_lights * 9 : sh.lights;
        const float *A = sh.lights_per_view ? sh.ambient + (int64_t)n * 3 : sh.ambient;
        if (threadIdx.x < sh.n_lights * 9) sL[threadIdx.x] = L[threadIdx.x];
        if (threadIdx.x < 3) {
            sL[DSS_MAX_LIGHTS * 9 + threadIdx.x] = A[threadIdx.x];
            sL[DSS_MAX_LIGHTS * 9 + 3 + threadIdx.x] = sh.cam_centres[n * 3 + threadIdx.x];
        }
        __syncthreads();
    }
    const int64_t npix = (int64_t)S * S;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < npix; i += (int64_t)gridDim.x * blockDim.x) {
        const unsigned long long key = keys[c * npix + i];
        const int64_t out = (int64_t)n * npix + i;
        const bool hit = key != MESH_EMPTY;
        const int f = hit ? (int)(uint32_t)key : -1;
        pix_to_face[out] = f;
        zbuf[out] = hit ? __uint_as_float((uint32_t)(key >> 32)) : -1.0f;
        if (rgba) {
            float4 o = make_float4(1.0f, 1.0f, 1.0f, 0.0f);
            if (hit) {
                const int64_t i0 = faces[(int64_t)f * 3], i1 = faces[(int64_t)f * 3 + 1], i2 = faces[(int64_t)f * 3 + 2];
                const V3 p0 = v3(verts[i0 * 3], verts[i0 * 3 + 1], verts[i0 * 3 + 2]);
                const V3 p1 = v3(verts[i1 * 3], verts[i1 * 3 + 1], verts[i1 * 3 + 2]);
                const V3 p2 = v3(verts[i2 * 3], verts[i2 * 3 + 1], verts[i2 * 3 + 2]);
                const V3 sum = add3(add3(p0, p1), p2);
                const V3 centroid = v3(sum.x / 3.0f, sum.y / 3.0f, sum.z / 3.0f);   // faces_verts.mean(-2)
                const V3 e1 = sub3(p1, p0), e2 = sub3(p2, p0);
                float len;
                const V3 nrm = normalize3(v3(e1.y * e2.z - e1.z * e2.y, e1.z * e2.x - e1.x * e2.z,
                                             e1.x * e2.y - e1.y * e2.x), len);
                const float *amb = sL + DSS_MAX_LIGHTS * 9;
                V3 ga, gn, gp;
                const V3 col = shade_point<false>(sL, sh.n_lights, sh.light_type, sh.shininess,
                                                  v3(amb[0], amb[1], amb[2]), centroid, nrm, v3(1.0f, 1.0f, 1.0f),
                                                  v3(amb[3], amb[4], amb[5]), v3(0.f, 0.f, 0.f), ga, gn, gp);
                o = make_float4(col.x, col.y, col.z, 1.0f);
            }
            reinterpret_cast<float4 *>(rgba)[out] = o;
        }
    }
}

}  // namespace dss

extern "C" {

int dss_rasterize_mesh(dss_ctx *ctx, const float *verts, int64_t V, const int32_t *faces, int64_t F, const float *proj,
                       const float *view, int N, int image_size, int n_lights, int light_type, int lights_per_view,
                       float shininess, const float *lights, const float *ambient, const float *cam_centres,
                       int32_t *pix_to_face, float *zbuf, float *rgba, void *stream) {
    using namespace dss;
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    DSS_REQUIRE(N >= 1, "N must be positive");
    DSS_REQUIRE(image_size >= 1 && image_size <= 32768, "image_size must be in [1, 32768]");
    DSS_REQUIRE(V >= 0 && V <= (int64_t)INT32_MAX && F >= 0 && F <= (int64_t)INT32_MAX, "V and F must be in [0, 2^31)");
    DSS_REQUIRE(proj && view && pix_to_face && zbuf, "null input or output array");
    DSS_REQUIRE(V == 0 || verts, "verts is null");
    DSS_REQUIRE(F == 0 || faces, "faces is null");
    if (rgba) {
        DSS_REQUIRE(n_lights >= 1 && n_lights <= DSS_MAX_LIGHTS, "n_lights must be in [1, 8]");
        DSS_REQUIRE(light_type == 0 || light_type == 1, "light_type must be 0 (directional) or 1 (point)");
        DSS_REQUIRE(lights_per_view == 0 || lights_per_view == 1, "lights_per_view must be 0 or 1");
        DSS_REQUIRE(lights && ambient && cam_centres, "shading needs lights, ambient and cam_centres");
    }
    cudaStream_t st = (cudaStream_t)stream;
    const int S = image_size;
    const int64_t npix = (int64_t)S * S;
    // views per chunk: bounded by the (view, face) table, the pixel keys and the grid's y extent
    int64_t C = MESH_CHUNK_ENTRIES / (F > 0 ? F : 1);
    const int64_t Cpix = MESH_CHUNK_PIXELS / npix;
    if (Cpix < C) C = Cpix;
    if (C > N) C = N;
    if (C > 65535) C = 65535;
    if (C < 1) C = 1;
    const bool have_faces = F > 0 && V > 0;
    float4 *screen = nullptr;
    int64_t *offsets = nullptr, *tile_sums = nullptr;
    int4 *rects = nullptr;
    unsigned long long *keys = nullptr;
    int rc;
    if ((rc = ctx_get(ctx, BUF_MESH_KEYS, (size_t)(C * npix), &keys))) return rc;
    if (have_faces) {
        const int64_t Mmax = C * F, tiles = scan_i64_tiles(Mmax);
        if ((rc = ctx_get(ctx, BUF_MESH_SCREEN, (size_t)(C * V), &screen))) return rc;
        if ((rc = ctx_get(ctx, BUF_MESH_OFFSETS, (size_t)(Mmax + 1), &offsets))) return rc;
        if ((rc = ctx_get(ctx, BUF_MESH_RECTS, (size_t)Mmax, &rects))) return rc;
        if ((rc = ctx_get(ctx, BUF_MESH_BLOCKS, (size_t)tiles, &tile_sums))) return rc;
    }
    MeshShading sh{n_lights, light_type, lights_per_view, shininess, lights, ambient, cam_centres};
    for (int n0 = 0; n0 < N; n0 += (int)C) {
        const int Cn = (int)(N - n0 < C ? N - n0 : C);
        DSS_CUDA_TRY(cudaMemsetAsync(keys, 0xff, (size_t)(Cn * npix) * sizeof(unsigned long long), st));
        if (have_faces) {
            const int64_t M = (int64_t)Cn * F;
            mesh_screen_kernel<<<dim3(grid_blocks(V, MESH_THREADS, ctx->sm_count, 8), Cn), MESH_THREADS, 0, st>>>(
                verts, V, proj, view, n0, screen);
            DSS_LAUNCH_CHECK(ctx);
            mesh_count_kernel<<<grid_blocks(M, MESH_THREADS, ctx->sm_count, 8), MESH_THREADS, 0, st>>>(
                faces, F, V, screen, M, S, offsets, rects);
            DSS_LAUNCH_CHECK(ctx);
            if ((rc = exclusive_scan_i64(ctx, offsets, M, tile_sums, st))) return rc;
            // the item total is on the device: a full grid strides over it
            mesh_item_kernel<<<grid_blocks(INT64_MAX / 2, MESH_THREADS, ctx->sm_count, 8), MESH_THREADS, 0, st>>>(
                faces, F, screen, V, offsets, rects, M, S, keys);
            DSS_LAUNCH_CHECK(ctx);
        }
        mesh_resolve_kernel<<<dim3(grid_blocks(npix, MESH_THREADS, ctx->sm_count, 8), Cn), MESH_THREADS, 0, st>>>(
            keys, n0, S, verts, faces, pix_to_face, zbuf, rgba, sh);
        DSS_LAUNCH_CHECK(ctx);
    }
    return DSS_OK;
}

}  // extern "C"
