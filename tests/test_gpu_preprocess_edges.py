"""The per-splat preprocess (dss_preprocess: csrc/render.cu, preprocess_kernel) against float64 at its edges, every slot
within the error bound of tests/test_preprocess_bound.py; the fused renderer at a cutoff and an antialiasing sigma
other than 1 (the uniform-cutoff raster instantiations the renderer runs); and the fused shading per slot against
float64 `apply_lighting` at its eps branches.

Preprocess: every kept slot's ndc, view depth, radii, conic and scaler within the bound; slots the depth filter (or
backface culling) removes, away from the filter's boundary by the depth's own bound, get z = -1 exactly, and their
other outputs are finite wherever float64's are.  Families: sphere clouds at S = 64 .. 2048 and h = 5e-5, 1e-3, 1e-2,
exactly edge-on normals, normals of length 1 ± a few ulp, the near-plane cloud of test_gpu_raster_edges.py, a camera
0.05 and 0.005 from the surface with znear 1e-3, points far off-screen, on the camera plane and behind it, cutoff 0.5 /
2 and sigma 0.25 / 4, per-splat h, and the packed layouts of test_gpu_backward_f64.py (ragged, empty and uncovered
views), a view range that is not a multiple of 256, one that needs the grid-stride loop, and 256 shared views."""
import ctypes as C

import numpy as np
import pytest
import torch

from dss_b200 import _lib, ops
from dss_b200.core.camera import FoVPerspectiveCameras, camera_matrices
from dss_b200.core.lighting import DirectionalLights, PointLights, pack_lights
from dss_b200.core.texture import apply_lighting, camera_centres
from dss_b200.ops import Shading, SplatParams, preprocess_points
from tests.test_gpu_backward_f64 import _packed_layout, _render_and_check
from tests.test_gpu_raster_edges import _check_render
from tests.test_preprocess_bound import (FAMILIES, QUANTITIES, REF_FACTOR, U, exempt_ratios, exempt_slots, family,
                                         preprocess_bound, ratios, reference_errors, slots, unbounded)
from tests.util import random_cameras, scene, sphere_cloud

pytestmark = pytest.mark.gpu


def _np(t):
    return t.detach().cpu().numpy()


def _preprocess(dev, pts, nrm, proj, view, h, prm, first=None, num=None):
    shared = first is None
    t = lambda a: torch.as_tensor(np.ascontiguousarray(a)).to(dev)
    pre = preprocess_points(t(pts), t(nrm), t(proj), t(view), t(h), prm, first_idx=None if shared else t(first),
                            num_points=None if shared else t(num), shared_cloud=shared)
    ndc, ell, rad, sc = (_np(pre[k]).astype(np.float64) for k in ("ndc", "ellipse_params", "radii", "scaler"))
    return dict(x=ndc[:, 0], y=ndc[:, 1], z=ndc[:, 2], rx=rad[:, 0], ry=rad[:, 1], a=ell[:, 0], b=ell[:, 1],
                c=ell[:, 2], scaler=sc)


def _check_slots(got, want, bnd, znear, zfar, covered, nz=None, label="", ref=None):
    """every covered slot against the bound / the filter; where the bound is infinite (and the splat reaches the
    image) the conic and the scaler against REF_FACTOR x the reference route's error on the same slots, `ref` =
    dict(proj, pts, nrm, h, vidx, cutoff, sigma, S) of the slots; -> worst ratio per quantity"""
    z, ez = want["z"], bnd["z"]
    inside = (z >= znear + ez) & (z <= zfar - ez)
    outside = (z < znear - ez) | (z > zfar + ez) | ~np.isfinite(z)
    if nz is not None:    # backface culling: n . V[:3, 2] < 0 keeps the slot
        cull = np.abs(nz) > 4 * U * np.abs(nz).max()
        inside &= (nz < 0) & cull
        outside |= (nz > 0) & cull
    inside &= covered
    outside &= covered
    finite = np.ones_like(covered)
    for k in QUANTITIES:
        finite &= np.isfinite(want[k])
    kept = inside & finite
    assert kept.sum() > 0, label
    r = ratios(got, want, bnd, kept)
    for k, (worst, over) in r.items():
        assert over == 0, (label, k, worst, over)
    ex = exempt_slots(want, bnd, kept)
    assert ref is not None or not ex.any(), label
    rr = exempt_ratios(got, want, reference_errors(ref, want), ex) if ex.any() else {}
    for k, v in rr.items():
        assert v <= 1, (label, "exempt", k, v)
    # filtered slots: z = -1 exactly; the rest finite where float64 is
    assert (got["z"][outside] == -1.0).all(), (label, int((got["z"][outside] != -1.0).sum()))
    for k in QUANTITIES:
        if k != "z":
            m = outside & np.isfinite(want[k])
            assert np.isfinite(got[k][m]).all(), (label, k)
    print("%s: %d kept (%d with an infinite bound, %d of them on screen: error / (%g x reference) %s), %d filtered; "
          "worst ratio %s" % (label, kept.sum(), unbounded(bnd, kept), ex.sum(), REF_FACTOR,
                              {k: "%.3g" % v for k, v in rr.items()}, outside.sum(),
                              {k: "%.3g" % v[0] for k, v in r.items()}))
    return r


# ---- 1. families, shared cloud --------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", FAMILIES)
def test_preprocess_families_within_the_bound(cuda_device, name):
    f = family(name)
    prm = SplatParams(image_size=f["S"], cutoff_threshold=f["cutoff"], antialiasing_sigma=f["sigma"],
                      znear=f["znear"], zfar=f["zfar"])
    got = _preprocess(cuda_device, f["pts"], f["nrm"], f["proj"], f["view"], f["h"], prm)
    pts, nrm, h, vidx = slots(f)
    want, bnd = preprocess_bound(f["proj"], f["view"], pts, nrm, h, vidx, f["cutoff"], f["sigma"], f["S"])
    ref = dict(proj=f["proj"], pts=pts, nrm=nrm, h=h, vidx=vidx, cutoff=f["cutoff"], sigma=f["sigma"], S=f["S"])
    _check_slots(got, want, bnd, f["znear"], f["zfar"], np.ones(len(vidx), bool), label=name, ref=ref)


def test_preprocess_backface_culling_and_depth_range(cuda_device):
    f = family("sphere/512,1e-3")
    prm = SplatParams(image_size=512, znear=1.45, zfar=1.6, backface_culling=True)
    got = _preprocess(cuda_device, f["pts"], f["nrm"], f["proj"], f["view"], f["h"], prm)
    pts, nrm, h, vidx = slots(f)
    want, bnd = preprocess_bound(f["proj"], f["view"], pts, nrm, h, vidx, 1.0, 1.0, 512)
    nz = (nrm.astype(np.float64) * f["view"][vidx, :3, 2]).sum(1)
    _check_slots(got, want, bnd, 1.45, 1.6, np.ones(len(vidx), bool), nz=nz, label="culling")
    assert (got["z"] == -1).sum() > len(vidx) // 2 and (got["z"] > 0).sum() > 1000


# ---- 2. packed layouts and launch shapes -----------------------------------------------------------------------------
def _packed_check(dev, rows, first, num, pts_w, nrm_w, proj, view, h, S=256, label=""):
    P = len(rows)
    vidx = np.full(P, -1)
    for n, (f0, m) in enumerate(zip(first, num)):
        vidx[f0:f0 + m] = n
    covered = vidx >= 0
    pts, nrm = pts_w[rows], nrm_w[rows]
    prm = SplatParams(image_size=S, znear=0.1)
    got = _preprocess(dev, pts, nrm, proj, view, h, prm, first, num)
    hs = h if h.size == P else h[np.maximum(vidx, 0)]
    want, bnd = preprocess_bound(proj, view, pts, nrm, hs, np.maximum(vidx, 0), 1.0, 1.0, S)
    _check_slots(got, want, bnd, 0.1, 100.0, covered, label=label)


@pytest.mark.parametrize("P0", [6000, 1001])
@pytest.mark.parametrize("per_splat_h", [False, True])
def test_preprocess_packed_layouts(cuda_device, P0, per_splat_h):
    pts, nrm, _, proj, view, _ = scene(P0 + 150, 4, seed=P0)
    rows, first, num = _packed_layout(P0)
    rng = np.random.default_rng(P0)
    h = (np.exp(rng.uniform(np.log(5e-5), np.log(1e-2), len(rows))) if per_splat_h else np.full(4, 1e-3)).astype(
        np.float32)
    _packed_check(cuda_device, rows, first, num, _np(pts), _np(nrm), _np(proj), _np(view), h,
                  label="packed P0=%d per_splat_h=%s" % (P0, per_splat_h))


def test_preprocess_grid_stride_and_256_views(cuda_device):
    d = cuda_device
    # one view of 300 001 points: more than the preprocess grid (8 blocks of 256 per SM) covers in one pass
    P0 = 300001
    pts, nrm, _ = sphere_cloud(P0, seed=5)
    proj, view = camera_matrices(random_cameras(1, 5, dist=(1.5, 1.5)))
    prm = SplatParams(image_size=1024, znear=0.1)
    h = np.full(1, 1e-3, np.float32)
    got = _preprocess(d, _np(pts), _np(nrm), _np(proj), _np(view), h, prm)
    want, bnd = preprocess_bound(_np(proj), _np(view), _np(pts), _np(nrm), np.full(P0, 1e-3, np.float32),
                                 np.zeros(P0, int), 1.0, 1.0, 1024)
    _check_slots(got, want, bnd, 0.1, 100.0, np.ones(P0, bool), label="grid-stride")
    # 256 shared views of a small cloud
    P0, N = 300, 256
    pts, nrm, _ = sphere_cloud(P0, seed=6)
    proj, view = camera_matrices(random_cameras(N, 6, dist=(1.0, 3.0)))
    h = np.random.default_rng(6).uniform(5e-5, 1e-2, N).astype(np.float32)
    got = _preprocess(d, _np(pts), _np(nrm), _np(proj), _np(view), h, SplatParams(image_size=128, znear=0.1))
    vidx = np.repeat(np.arange(N), P0)
    want, bnd = preprocess_bound(_np(proj), _np(view), np.tile(_np(pts), (N, 1)), np.tile(_np(nrm), (N, 1)), h[vidx],
                                 vidx, 1.0, 1.0, 128)
    _check_slots(got, want, bnd, 0.1, 100.0, np.ones(N * P0, bool), label="256 views")


# ---- 3. the fused renderer at cutoff 0.5 and sigma != 1 --------------------------------------------------------------
@pytest.mark.parametrize("K", [5, 8, 12])
@pytest.mark.parametrize("cutoff,sigma", [(0.5, 1.0), (0.5, 0.25), (2.0, 4.0)])
def test_render_at_cutoff_and_sigma(cuda_device, K, cutoff, sigma):
    P0, N, S = 8000, 2, 128
    pts, nrm, col, proj, view, _ = scene(P0, N, seed=K)
    prm = SplatParams(image_size=S, points_per_pixel=K, znear=0.1, cutoff_threshold=cutoff, antialiasing_sigma=sigma)
    h = torch.full((N,), 3e-4)
    out, _ = _check_render(cuda_device, pts, nrm, col.repeat(N, 1), proj, view, h, prm)
    # the render's own records are the preprocess at this cutoff and sigma
    rec = _np(out.records).astype(np.float64)
    got = dict(x=rec[:, 0], y=rec[:, 1], z=rec[:, 2], rx=rec[:, 3], ry=rec[:, 4], a=rec[:, 5], b=rec[:, 6],
               c=rec[:, 7], scaler=_np(out.scaler).astype(np.float64))
    vidx = np.repeat(np.arange(N), P0)
    want, bnd = preprocess_bound(_np(proj), _np(view), np.tile(_np(pts), (N, 1)), np.tile(_np(nrm), (N, 1)),
                                 np.full(N * P0, 3e-4, np.float32), vidx, cutoff, sigma, S)
    _check_slots(got, want, bnd, 0.1, 100.0, np.ones(N * P0, bool), label="render K=%d cutoff=%g sigma=%g" % (K, cutoff, sigma))


@pytest.mark.parametrize("layout", ["shared", "packed"])
def test_render_backward_at_cutoff_half(cuda_device, layout):
    d = cuda_device
    if layout == "packed":
        P0 = 6000
        pts, nrm, col, proj, view, _ = scene(P0 + 150, 4, seed=61)
        rows, first, num = _packed_layout(P0)
        prm = SplatParams(image_size=128, points_per_pixel=5, znear=0.1, clip_pts_grad=0.05, cutoff_threshold=0.5,
                          antialiasing_sigma=0.25)
        leaf = pts.to(d).requires_grad_(True)
        ridx = torch.as_tensor(rows).to(d)
        _render_and_check(leaf[ridx], nrm.to(d)[ridx], col.to(d)[ridx], proj.to(d), view.to(d),
                          torch.full((4,), 3e-4, device=d), prm, first=first, num=num, seed=61, world_rows=rows,
                          pts_leaf=leaf)
    else:
        P0, N = 8000, 3
        pts, nrm, col, proj, view, _ = scene(P0, N, seed=62)
        prm = SplatParams(image_size=128, points_per_pixel=5, znear=0.1, clip_pts_grad=0.05, cutoff_threshold=0.5,
                          antialiasing_sigma=4.0)
        leaf = pts.to(d).requires_grad_(True)
        _render_and_check(leaf, nrm.to(d), col.to(d), proj.to(d), view.to(d), torch.full((N,), 3e-4, device=d), prm,
                          seed=62, world_rows=np.arange(P0), pts_leaf=leaf)


def test_render_fronto_parallel_plane_and_a_single_splat_view(cuda_device):
    """a plane facing view 0 (R = I: every splat it keeps at one view depth, so its depth range is one value) and a
    view 1 looking the other way whose only renderable splat is one point behind view 0 (the plane lies behind it)"""
    g = torch.Generator().manual_seed(7)
    P0 = 3000
    xy = (torch.rand(P0, 2, generator=g) * 2 - 1) * 1.1
    pts = torch.cat([xy, torch.full((P0, 1), 2.0)], 1).contiguous()
    nrm = torch.tensor([0.0, 0.0, -1.0]).repeat(P0, 1).contiguous()
    col = torch.rand(P0, 3, generator=g)
    # view 0 at the origin looks down +z at the plane (z = 2); view 1 at z = -1 looks down -z (R = diag(-1, 1, -1)):
    # point 0 at z = -3 is behind view 0 and 2 in front of view 1, the plane is behind view 1
    pts[0] = torch.tensor([0.01, -0.02, -3.0])
    R = torch.stack([torch.eye(3), torch.diag(torch.tensor([-1.0, 1.0, -1.0]))])
    T = torch.tensor([[0.0, 0.0, 0.0], [0.0, 0.0, -1.0]])
    proj, view = camera_matrices(FoVPerspectiveCameras(znear=0.1, zfar=100.0, R=R, T=T))
    for K in (5, 12):
        prm = SplatParams(image_size=96, points_per_pixel=K, znear=0.1, cutoff_threshold=0.5)
        out, want = _check_render(cuda_device, pts, nrm, col.repeat(2, 1), proj, view, torch.full((2,), 1e-3), prm)
        rec = _np(out.records)
        z0 = rec[:P0, 2]
        assert z0[0] == -1 and (z0[1:] >= 0).all() and len(np.unique(z0[1:])) == 1
        assert (rec[P0:, 2] >= 0).sum() == 1 and rec[P0, 2] == 2.0
        assert (_np(out.idx[1]) >= 0).any() and set(np.unique(_np(out.idx[1]))) <= {-1, P0}


# ---- 4. fused shading per slot ---------------------------------------------------------------------------------------
def _shade_lib(dev, pts, nrm, alb, proj, view, sh):
    """dss_preprocess with `shade` and `shaded` set (preprocess_kernel<true>) -> (N*P0,3) shaded colours"""
    N, P0 = proj.shape[0], pts.shape[0]
    a = _lib.RenderArgs()
    h = torch.full((N,), 1e-3, device=dev)
    ops._fill_common(a, pts, nrm, None, proj, view, h, None, None, True, N, P0, N * P0, SplatParams(image_size=64))
    ops._fill_shading(a, sh, alb)
    shaded = torch.full((N * P0, 3), float("nan"), device=dev)
    a.shaded = _lib.ptr(shaded)
    _lib.check(_lib.load().dss_preprocess(_lib.ctx(dev), C.byref(a), _lib.stream_ptr(dev)), "dss_preprocess")
    torch.cuda.synchronize(dev)
    return shaded


def _shade_bound(p, n, alb, rows, amb, cam, light_type, shin):
    """float64 shading of every slot and its bound.  p, n, alb, cam (P,3) float64 per slot; rows (P,L,9) the slot's
    lights; amb (P,3).  Per light: the normalised vectors carry 6 ulp (+ the rounding of the difference relative to
    its length), n.d 3 ulp of Σ|terms| plus theirs, the reflected ray and v.r likewise; pw = alpha^shin is bounded by
    its value at alpha + e_alpha; the specular mask may flip where 0 < |n.d| <= e_cos.  Colour: (L + 3) ulp of Σ|terms|."""
    nl = lambda v, eps=1e-6: v / np.maximum(np.linalg.norm(v, axis=-1, keepdims=True), eps)
    nh = nl(n)
    vraw = cam - p
    vlen = np.maximum(np.linalg.norm(vraw, axis=1), 1e-6)
    v = nl(vraw)
    e_n = 6 * U * np.ones(len(p))
    e_v = 6 * U + U * (np.abs(cam) + np.abs(p)).sum(1) / vlen
    col = alb * amb
    err = np.zeros_like(col)
    mag = alb * amb
    for l in range(rows.shape[1]):
        L = rows[:, l]
        draw = L[:, :3] - p if light_type else L[:, :3]
        dlen = np.maximum(np.linalg.norm(draw, axis=1), 1e-6)
        d = nl(draw)
        e_d = 6 * U + (U * (np.abs(L[:, :3]) + np.abs(p)).sum(1) / dlen if light_type else 0)
        cos = (nh * d).sum(1)
        e_cos = 3 * U + 3 * (e_n + e_d)
        lam = np.maximum(cos, 0)
        r = -d + 2 * cos[:, None] * nh
        e_r = e_d + 2 * (e_cos + e_n) + 3 * U
        vr = (v * r).sum(1)
        e_al = 3 * e_r + 9 * e_v + 9 * U
        alpha = np.where(cos > 0, np.maximum(vr, 0), 0.0)
        pw = np.where(alpha > 0, alpha ** shin, 0.0)
        e_pw = (alpha + e_al) ** shin - alpha ** shin + 3 * U * pw
        flip = (cos != 0) & (np.abs(cos) <= e_cos)
        e_pw = np.where(flip, (np.maximum(vr, 0) + e_al) ** shin, e_pw)
        cd, cs = L[:, 3:6], L[:, 6:9]
        col = col + alb * cd * lam[:, None] + cs * pw[:, None]
        mag = mag + alb * cd * lam[:, None] + cs * pw[:, None]
        err = err + alb * cd * e_cos[:, None] + cs * e_pw[:, None]
    return col, err + (rows.shape[1] + 3) * U * mag


def _light_rows(kind, N, L, per_view, seed):
    g = torch.Generator().manual_seed(seed)
    shape = (N, L) if per_view else (1, L)
    vec = torch.randn(*shape, 3, generator=g) * (1.0 if kind == "sun" else 1.5)
    kw = dict(ambient_color=0.2 * torch.rand(*shape, 3, generator=g), diffuse_color=0.6 * torch.rand(*shape, 3, generator=g),
              specular_color=0.5 * torch.rand(*shape, 3, generator=g))
    return DirectionalLights(direction=vec, **kw) if kind == "sun" else PointLights(location=vec, **kw)


def _edge_points(P0, seed, light_pos):
    """a sphere cloud with the edge cases in front: zero and sub-1e-6 normals, a point at a point light, n.d = 0
    exactly against a directional light along +x (normal +z), and a point at the first camera centre"""
    pts, nrm, alb = (t.numpy().astype(np.float32) for t in sphere_cloud(P0, seed=seed))
    nrm = nrm * np.random.default_rng(seed).uniform(0.5, 2.0, (P0, 1)).astype(np.float32)
    nrm[0] = 0
    nrm[1] = nrm[1] / np.linalg.norm(nrm[1]) * 3e-7
    nrm[2] = [1e-7, -2e-7, 0]
    if light_pos is not None:
        pts[3] = light_pos
    nrm[4] = [0, 0, 1]
    return pts, nrm, alb


@pytest.mark.parametrize("kind", ["sun", "point"])
@pytest.mark.parametrize("per_view", [False, True])
@pytest.mark.parametrize("L,shin", [(1, 1.0), (8, 13.5), (2, 64.0)])
def test_fused_shading_per_slot_within_its_bound(cuda_device, kind, per_view, L, shin):
    d = cuda_device
    P0, N = 5000, 3
    lights = _light_rows(kind, N, L, per_view, seed=L)
    rows, ambient, lt = pack_lights(lights)
    rows = rows.detach().clone()
    if kind == "sun":   # light 0 along +x: n.d = 0 exactly for the normal +z of point 4
        rows[..., 0, 0:3] = torch.tensor([1.0, 0.0, 0.0])
    pts, nrm, alb = _edge_points(P0, L, rows.reshape(-1, 9)[0, :3].numpy() if kind == "point" else None)
    proj, view = camera_matrices(random_cameras(N, L, dist=(1.2, 2.2)))
    cams = camera_centres(view).float()
    pts[5] = cams[0].numpy()
    # point 4 seen from the mirror direction of the light (v = -d, v.r = 1): the mask alone decides its highlight
    cams[1] = torch.as_tensor(pts[4]) + torch.tensor([-1.0, 0.0, 0.0])
    sh = Shading(rows.to(d), ambient.float().to(d), cams.to(d), lt, shin)
    got = _np(_shade_lib(d, torch.as_tensor(pts).to(d), torch.as_tensor(nrm).to(d), torch.as_tensor(alb).to(d),
                         proj.to(d), view.to(d), sh)).astype(np.float64)
    vidx = np.repeat(np.arange(N), P0)
    r64 = rows.double().numpy()
    rows_s = r64[vidx] if per_view else np.broadcast_to(r64, (N * P0,) + r64.shape[-2:])
    amb64 = ambient.double().numpy()
    amb_s = amb64[vidx] if per_view else np.broadcast_to(amb64.reshape(1, 3), (N * P0, 3))
    p64, n64, a64 = (np.tile(x.astype(np.float64), (N, 1)) for x in (pts, nrm, alb))
    want, bnd = _shade_bound(p64, n64, a64, rows_s, amb_s, cams.double().numpy()[vidx], lt, shin)
    # float64 apply_lighting (the torch shading) is the arbiter of the values
    idx = torch.as_tensor(vidx)
    vec = (rows if per_view else rows[None]).double()[..., :3]
    l64 = type(lights)(**{k: getattr(lights, k).double() for k in ("ambient_color", "diffuse_color",
                                                                   "specular_color")},
                       **({"direction": vec} if kind == "sun" else {"location": vec}))
    A, D, Sp = apply_lighting(torch.as_tensor(p64), torch.as_tensor(n64), l64, torch.as_tensor(cams.double().numpy()[vidx]),
                              shininess=shin, view_idx=idx if per_view else None)
    ref = (torch.as_tensor(a64) * (A + D) + Sp).numpy()
    # (the light objects hold float32 buffers, so the torch shading agrees to float32 rounding: a check of the formula)
    np.testing.assert_allclose(want, ref, rtol=4e-6, atol=1e-7)
    e = np.abs(got - want)
    assert np.isfinite(got).all()
    assert (e <= bnd).all(), (kind, per_view, L, shin, float((e / np.maximum(bnd, 1e-300)).max()))
    print("shading %s per_view=%s L=%d shin=%g: worst ratio %.3g" % (kind, per_view, L, shin, float((e / bnd).max())))
    # the edge slots: a zero normal gives albedo * ambient, one rounding; n.d = 0 exactly gives no highlight although
    # the camera sits in the mirror direction (a highlight there would be cs itself, far outside the bound)
    z = np.arange(N) * P0
    assert (np.abs(got[z] - a64[z] * amb_s[z]) <= U * a64[z] * amb_s[z]).all()
    if kind == "sun":
        d0 = rows_s[P0 + 4, 0, :3]
        v = cams.double().numpy()[1] - p64[P0 + 4]
        assert d0 @ n64[P0 + 4] == 0 and v @ -d0 > 0


# ---- 5. shading gradients at the same edges (shade_backward_kernel) -------------------------------------------------
def _shade64_torch(p, n, alb, rows, amb, cam, light_type, shin):
    """the shading in float64 torch, autograd-differentiable (the formula of _shade_bound)"""
    nl = lambda v: v / v.norm(dim=-1, keepdim=True).clamp_min(1e-6)
    nh, v = nl(n), nl(cam - p)
    col = alb * amb
    for l in range(rows.shape[1]):
        L = rows[:, l]
        d = nl(L[:, :3] - p if light_type else L[:, :3])
        cos = (nh * d).sum(1)
        r = -d + 2 * cos[:, None] * nh
        alpha = torch.where(cos > 0, torch.relu((v * r).sum(1)), torch.zeros_like(cos))
        pw = torch.where(alpha > 0, alpha.clamp_min(1e-300) ** shin, torch.zeros_like(alpha))
        col = col + alb * L[:, 3:6] * torch.relu(cos)[:, None] + L[:, 6:9] * pw[:, None]   # relu'(0) = 0
    return col


@pytest.mark.parametrize("kind", ["sun", "point"])
@pytest.mark.parametrize("L,shin", [(1, 1.0), (2, 64.0)])
def test_shading_gradients_at_the_edges_match_float64_autograd(cuda_device, kind, L, shin):
    """grad albedo / normal / position of shade_backward_kernel (shared cloud, per-view lights off) against float64
    autograd, per point, within c·u·Σ|terms|: Σ over the views of |d L / d colour| times the magnitudes of the
    colour's terms (ambient, diffuse, and shin·alpha^(shin-1) of the specular), over the clamped lengths the
    gradient divides by (|n| for the normal, |c - p| and |l - p| for the position); c = 256.  The edges: zero and
    sub-1e-6 normals, a point at the point light, a point at a camera centre (normalize3_bwd's eps branch)."""
    from tests.test_gpu_light_grad import _shading_backward_via_lib
    d = cuda_device
    P0, N, S2 = 5000, 3, 72
    lights = _light_rows(kind, N, L, False, seed=L)
    rows, ambient, lt = pack_lights(lights)
    rows = rows.detach().clone()
    pts, nrm, alb = _edge_points(P0, L, rows[0, :3].numpy() if kind == "point" else None)
    proj, view = camera_matrices(random_cameras(N, L, dist=(1.2, 2.2)))
    cams = camera_centres(view).float()
    pts[5] = cams[0].numpy()
    sh = Shading(rows.to(d), ambient.float().to(d), cams.to(d), lt, shin)
    gi = torch.randn(N, S2, S2, 4, generator=torch.Generator().manual_seed(L))
    tp, tn, ta = (torch.as_tensor(x).to(d) for x in (pts, nrm, alb))
    ga, gn, gp, _ = _shading_backward_via_lib(sh, tp, tn, ta, gi.to(d), S2, torch.empty(L, 9, device=d),
                                              torch.empty(3, device=d), repeat=0)
    gc = gi.reshape(N, S2 * S2, 4)[:, :P0, :3].double().reshape(N * P0, 3)
    p64, n64, a64 = (torch.as_tensor(x).double().repeat(N, 1).requires_grad_(True) for x in (pts, nrm, alb))
    vidx = torch.arange(N).repeat_interleave(P0)
    r64 = rows.double()[None].expand(N * P0, -1, -1)
    c64 = cams.double()[vidx]
    col = _shade64_torch(p64, n64, a64, r64, ambient.double()[None], c64, lt, shin)
    want = [g.detach().reshape(N, P0, 3).sum(0).numpy() for g in torch.autograd.grad(col, [a64, n64, p64], gc)]
    assert all(np.isfinite(w).all() for w in want)
    # term magnitudes per (view, point)
    with torch.no_grad():
        nlen = n64.norm(dim=1).clamp_min(1e-6)
        vlen = (c64 - p64).norm(dim=1).clamp_min(1e-6)
        nh = n64 / nlen[:, None]
        v = (c64 - p64) / vlen[:, None]
        g = gc.abs()
        m_alb = g * ambient.double()[None]
        m_geo = torch.zeros(N * P0, dtype=torch.float64)
        inv_d = torch.zeros(N * P0, dtype=torch.float64)
        for l in range(L):
            Lr = r64[:, l]
            draw = Lr[:, :3] - p64 if lt else Lr[:, :3].expand(N * P0, 3)
            dl = draw.norm(dim=1).clamp_min(1e-6)
            dd = draw / dl[:, None]
            cos = (nh * dd).sum(1)
            vr = (v * (-dd + 2 * cos[:, None] * nh)).sum(1).clamp_min(0)
            spec = shin * (vr + 1e-4) ** (shin - 1) * (1 + shin * 1e-4)
            m_alb = m_alb + g * Lr[:, 3:6] * (cos.clamp_min(0) + 64 * U)[:, None]
            m_geo = m_geo + (g * (a64 * Lr[:, 3:6] + Lr[:, 6:9] * spec[:, None])).sum(1)
            if lt:
                inv_d = inv_d + (g * (a64 * Lr[:, 3:6] + Lr[:, 6:9] * spec[:, None])).sum(1) / dl
        m_n = (m_geo / nlen).reshape(N, P0).sum(0).numpy()
        m_p = (m_geo / vlen + inv_d).reshape(N, P0).sum(0).numpy()
        m_a = m_alb.reshape(N, P0, 3).sum(0).numpy()
    c = 256 * U
    res = {}
    for name, got, w, m in (("albedo", ga, want[0], m_a), ("normals", gn, want[1], m_n[:, None]),
                            ("points", gp, want[2], m_p[:, None])):
        e = np.abs(_np(got).astype(np.float64) - w)
        assert np.isfinite(_np(got)).all(), name
        res[name] = float((e / (c * m)).max())
        assert (e <= c * m).all(), (name, res[name])
    print("shading gradients %s L=%d shin=%g: worst ratio %s" % (kind, L, shin, {k: "%.3g" % v for k, v in res.items()}))
    # the eps branches were reached and give the float64 gradients: zero / tiny normals (g / 1e-6), camera at point 5
    assert np.abs(want[1][:3]).max() > 0 and (np.abs(want[1][:3]) > 1e3 * np.abs(want[1][6:]).max()).any()
