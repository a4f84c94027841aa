// shading.cuh -- per-point shading device code shared by the fused splatting path (render.cu) and the mesh
// rasterizer's flat shading (mesh_raster.cu).
#pragma once
#include "common.cuh"

namespace dss {

// ---------------------------------------------------------------------------------------------
// Per-point shading (SURVEY.md 8(f)3): DSS/core/texture.py:74-127 (LightingTexture.forward:
// shaded = rgb * (ambient + diffuse) + specular) over DSS/core/lighting.py:10-172 (diffuse: Lambert with the
// renormalised normal and light direction, :62-69; specular: reflected ray against the view direction, masked where
// the light is behind the surface, :139-172).  Lights sit in shared memory as rows of 9 floats.
// ---------------------------------------------------------------------------------------------
struct V3 {
    float x, y, z;
};
__device__ __forceinline__ V3 v3(float x, float y, float z) { return V3{x, y, z}; }
__device__ __forceinline__ float dot3(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ V3 add3(V3 a, V3 b) { return v3(a.x + b.x, a.y + b.y, a.z + b.z); }
__device__ __forceinline__ V3 sub3(V3 a, V3 b) { return v3(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ V3 mul3(V3 a, float s) { return v3(a.x * s, a.y * s, a.z * s); }
__device__ __forceinline__ void store3(float *p, V3 a) { p[0] = a.x, p[1] = a.y, p[2] = a.z; }
// F.normalize(x, p=2, dim=-1, eps=1e-6): x / max(|x|, eps); returns the clamped norm through `len` and, for the
// backward, the unclamped one through `raw`
__device__ __forceinline__ V3 normalize3(V3 a, float &len, float &raw) {
    raw = sqrtf(dot3(a, a));
    len = fmaxf(raw, 1e-6f);
    return mul3(a, 1.0f / len);
}
__device__ __forceinline__ V3 normalize3(V3 a, float &len) {
    float raw;
    return normalize3(a, len, raw);
}
// gradient of y = normalize(x) given dL/dy: the backward of x / clamp_min(|x|, eps), which passes the gradient through
// the norm where |x| >= eps, at equality too (float32 F.normalize); only below eps is the map linear: g / eps
__device__ __forceinline__ V3 normalize3_bwd(V3 y, float len, float raw, V3 gy) {
    if (raw < 1e-6f) return mul3(gy, 1.0f / len);
    return mul3(sub3(gy, mul3(y, dot3(y, gy))), 1.0f / len);
}

// One light's share of the shading of one (view, point): L is the light's row of 9 floats, nh / v the normalised
// normal and view direction.  Adds the light's diffuse and specular terms to diff / spec; with BACKWARD (gc = d L / d
// colour) also its share of d nh and d v to g_nh / g_v, and returns in g_d the gradient w.r.t. the normalised light
// direction d.  Every user of the shading (forward, shading backward, camera and light gradients) goes through here.
struct LightTerm {
    V3 d;          // normalised light direction (direction, or location - p)
    float dlen;    // clamped norm of the un-normalised one
    float draw;    // its unclamped norm
    float lam;     // relu(n.d): factor of the diffuse colour
    float pw;      // (relu(v.r) [n.d > 0])^shininess: factor of the specular colour
    V3 g_d;        // BACKWARD: d L / d d
};
template <bool BACKWARD>
__device__ __forceinline__ LightTerm shade_light(const float *L, int light_type, float shininess, V3 p, V3 nh, V3 v,
                                                 V3 alb, V3 gc, V3 &diff, V3 &spec, V3 &g_nh, V3 &g_v) {
    LightTerm t;
    const V3 draw = light_type ? sub3(v3(L[0], L[1], L[2]), p) : v3(L[0], L[1], L[2]);
    t.d = normalize3(draw, t.dlen, t.draw);
    const V3 d = t.d;
    const V3 cd = v3(L[3], L[4], L[5]), cs = v3(L[6], L[7], L[8]);
    const float cosang = dot3(nh, d);
    const float lam = fmaxf(cosang, 0.0f);                           // lighting.py:65
    diff = add3(diff, mul3(cd, lam));
    const float mask = cosang > 0.0f ? 1.0f : 0.0f;                   // :158
    const V3 r = add3(mul3(d, -1.0f), mul3(nh, 2.0f * cosang));       // :163
    const float vr = dot3(v, r);
    const float alpha = fmaxf(vr, 0.0f) * mask;                       // :166-167
    const float pw = alpha > 0.0f ? powf(alpha, shininess) : 0.0f;    // :169
    spec = add3(spec, mul3(cs, pw));
    t.lam = lam;
    t.pw = pw;
    if (BACKWARD) {
        // diffuse: d/d cos = sum_c (gc*alb)_c cd_c  where cos > 0
        float g_cos = (cosang > 0.0f) ? (gc.x * alb.x * cd.x + gc.y * alb.y * cd.y + gc.z * alb.z * cd.z) : 0.0f;
        V3 g_d = v3(0.f, 0.f, 0.f);
        if (alpha > 0.0f) {
            const float g_alpha = dot3(gc, cs) * shininess * powf(alpha, shininess - 1.0f);
            const float g_vr = g_alpha;                                // alpha = vr where vr > 0 and mask = 1
            const V3 g_r = mul3(v, g_vr);
            g_v = add3(g_v, mul3(r, g_vr));
            g_cos += 2.0f * dot3(g_r, nh);
            g_nh = add3(g_nh, mul3(g_r, 2.0f * cosang));
            g_d = sub3(g_d, g_r);
        }
        g_nh = add3(g_nh, mul3(d, g_cos));
        t.g_d = add3(g_d, mul3(nh, g_cos));
    }
    return t;
}

// forward (and, with gc != nullptr, backward) of the shading of one (view, point).  sL: the view's lights.
//   colour = albedo * (ambient + diffuse) + specular
// backward: accumulates d albedo, d normal (un-normalised input normal), d position into g_alb / g_nrm / g_pos, and
// with CAM_GRAD the camera-centre gradient (the view-direction half of d position, opposite sign) into *g_cam.
template <bool BACKWARD, bool CAM_GRAD = false>
__device__ __forceinline__ V3 shade_point(const float *sL, int n_lights, int light_type, float shininess, V3 amb, V3 p,
                                          V3 nrm, V3 alb, V3 cam, V3 gc, V3 &g_alb, V3 &g_nrm, V3 &g_pos,
                                          V3 *g_cam = nullptr) {
    float nlen, vlen, nraw, vraw;
    const V3 nh = normalize3(nrm, nlen, nraw);
    const V3 v = normalize3(sub3(cam, p), vlen, vraw);
    V3 diff = v3(0.f, 0.f, 0.f), spec = v3(0.f, 0.f, 0.f);
    V3 g_nh = v3(0.f, 0.f, 0.f), g_v = v3(0.f, 0.f, 0.f);
    for (int l = 0; l < n_lights; ++l) {
        const LightTerm t = shade_light<BACKWARD>(sL + l * 9, light_type, shininess, p, nh, v, alb, gc, diff, spec, g_nh,
                                                  g_v);
        if (BACKWARD && light_type) g_pos = sub3(g_pos, normalize3_bwd(t.d, t.dlen, t.draw, t.g_d));   // d = normalize(loc - p)
    }
    if (BACKWARD) {
        g_alb = add3(g_alb, v3(gc.x * (amb.x + diff.x), gc.y * (amb.y + diff.y), gc.z * (amb.z + diff.z)));
        g_nrm = add3(g_nrm, normalize3_bwd(nh, nlen, nraw, g_nh));
        const V3 g_cam_v = normalize3_bwd(v, vlen, vraw, g_v);           // v = normalize(cam - p)
        g_pos = sub3(g_pos, g_cam_v);
        if (CAM_GRAD) *g_cam = add3(*g_cam, g_cam_v);
    }
    return v3(alb.x * (amb.x + diff.x) + spec.x, alb.y * (amb.y + diff.y) + spec.y, alb.z * (amb.z + diff.z) + spec.z);
}

}  // namespace dss
