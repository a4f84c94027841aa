"""Camera gradients through the fused renderer (dss_camera_backward): R / T gradients equal the unfused route's,
grad_proj / grad_view equal the float64 sums over the NDC gradient the same backward wrote, the shading's camera
centres get the float64 autograd route's gradient, results are reproducible, and cameras that do not require grad
cost nothing."""
import os
from collections import namedtuple

import pytest
import torch

from dss_b200 import _C, _lib
from dss_b200.core.camera import FoVPerspectiveCameras, camera_matrices, look_at_view_transform
from dss_b200.core.cloud import PointClouds3D
from dss_b200.core.lighting import pack_lights
from dss_b200.core.rasterizer import PointsRasterizationSettings, SurfaceSplatting, _splat_params
from dss_b200.core.renderer import NormWeightedCompositor, SurfaceSplattingRenderer
from dss_b200.core.texture import apply_lighting, camera_centres
from dss_b200.ops import Shading, SplatParams, make_shading, render_points
from dss_b200.utils.io import read_ply
from tests.test_camera_grad import camera_grads64
from tests.test_shading import _lights, _shade64
from tests.util import GOLDEN_DIR, backward_via_lib, scene, sphere_cloud

pytestmark = pytest.mark.gpu


# ---- 3. fused vs unfused SurfaceSplattingRenderer -------------------------------------------------------------------
def _cameras(dev, N=3):
    R, T = look_at_view_transform(dist=[1.5, 1.8, 2.1][:N], elev=[10, -30, 60][:N], azim=[0, 120, -70][:N])
    return FoVPerspectiveCameras(znear=0.1, zfar=100.0, R=R, T=T, device=dev)


@pytest.mark.parametrize("clip", [0.05, -1.0])
@pytest.mark.parametrize("vrk,layout", [("invariant", "shared"), ("isotropic", "shared"), ("invariant", "packed")])
def test_R_T_gradients_match_unfused_route(cuda_device, clip, vrk, layout):
    dev, S = cuda_device, 96
    pts, nrm, col = (t.to(dev) for t in sphere_cloud(4000, seed=3))
    settings = PointsRasterizationSettings(backface_culling=False, cutoff_threshold=1.0, depth_merging_threshold=0.05,
                                           Vrk_invariant=vrk == "invariant", Vrk_isotropic=vrk == "isotropic",
                                           radii_backward_scaler=5, image_size=S, points_per_pixel=5, bin_size=None,
                                           clip_pts_grad=clip)
    renderer = SurfaceSplattingRenderer(SurfaceSplatting(cameras=_cameras(dev), raster_settings=settings),
                                        NormWeightedCompositor())
    g = torch.randn(3, S, S, 4, generator=torch.Generator().manual_seed(1)).to(dev) * 1e-3
    slices = [slice(0, 4000)] * 3 if layout == "shared" else [slice(0, 3000), slice(500, 4000), slice(1000, 2500)]

    def run(fused, cam_grad):
        cams = _cameras(dev)
        cams.R.requires_grad_(cam_grad)
        cams.T.requires_grad_(cam_grad)
        p = pts.clone().requires_grad_(True)
        c = col.clone().requires_grad_(True)
        if layout == "shared":
            cloud = PointClouds3D([p], normals=[nrm], features=[c])
        else:
            cloud = PointClouds3D([p[s] for s in slices], normals=[nrm[s] for s in slices], features=[c[s] for s in slices])
        renderer(cloud, cameras=cams, fused=fused).backward(g)
        return cams.R.grad, cams.T.grad, p.grad, c.grad

    # the library sizes some of its work from the previous call: warm it up with this shape so that the two fused runs
    # compared below take the same paths
    run(True, False)
    Rf, Tf, pf, cf = run(True, True)
    _, _, p0, c0 = run(True, False)
    Ru, Tu, _, _ = run(False, True)
    for got, want in ((Rf, Ru), (Tf, Tu)):
        scale = want.abs().max()
        assert scale > 0 and (got - want).abs().max() <= 2e-4 * scale, ((got - want).abs().max(), scale)
    # the camera gradients leave the point gradients alone (the occupancy path is a gather: bit-reproducible; the colour
    # scatter adds with float atomics, so its sums may round in another order from run to run)
    assert torch.equal(pf, p0)
    torch.testing.assert_close(cf, c0, rtol=1e-5, atol=1e-9)


def test_packed_isotropic_routes_part_only_through_ndc_rounding(cuda_device):
    """Packed clouds with Vrk_isotropic (the default settings): the two routes rasterize the same fragments, but their
    screen positions differ in the last bits -- the preprocess kernel computes x * rcp(t) with fused multiply-adds, the
    differentiable transform of the unfused route divides after a matmul.  The occupancy gradient has hard edges (the
    search disc, and the splat's box for positive pixel gradients), so a pixel within those bits of an edge is counted by
    one route and not by the other: that moves one point's NDC gradient by one pixel's term, up to 7e-2 of the largest
    position gradient once the clip at 0.05 shrinks the rest.  Each route matches float64 on its own records
    (test_gpu_backward_f64.py); here the unfused route's records and fragments, fed to the fused backward and camera
    backward, give the unfused route's position and R / T gradients."""
    dev, S, clip = cuda_device, 96, 0.05
    pts, nrm, col = (t.to(dev) for t in sphere_cloud(4000, seed=3))
    settings = PointsRasterizationSettings(backface_culling=False, cutoff_threshold=1.0, depth_merging_threshold=0.05,
                                           Vrk_invariant=False, Vrk_isotropic=True, radii_backward_scaler=5,
                                           image_size=S, points_per_pixel=5, bin_size=None, clip_pts_grad=clip)
    renderer = SurfaceSplattingRenderer(SurfaceSplatting(cameras=_cameras(dev), raster_settings=settings),
                                        NormWeightedCompositor())
    g = torch.randn(3, S, S, 4, generator=torch.Generator().manual_seed(1)).to(dev) * 1e-3
    slices = [slice(0, 3000), slice(500, 4000), slice(1000, 2500)]
    rows = torch.cat([torch.arange(4000)[s] for s in slices]).to(dev)

    def run(fused):
        cams = _cameras(dev)
        cams.R.requires_grad_(True)
        cams.T.requires_grad_(True)
        p = pts.clone().requires_grad_(True)
        cloud = PointClouds3D([p[s] for s in slices], normals=[nrm[s] for s in slices], features=[col[s] for s in slices])
        img, frags = renderer(cloud, cameras=cams, fused=fused, verbose=True)
        img.backward(g)
        return cams, cloud, frags, p.grad

    run(True)
    _, _, frags_f, p_f = run(True)
    cams, cloud, frags_u, p_u = run(False)
    rast = renderer.rasterizer
    with torch.no_grad():
        info = rast._get_per_point_info(cloud, cameras=cams)      # the preprocess kernel: the fused route's records
        t = rast.transform(cloud, cameras=cams)
        ndc_u = torch.cat([t[:, :2], torch.where(info["ndc"][:, 2:] >= 0, t[:, 2:], info["ndc"][:, 2:])], 1)
    P = ndc_u.shape[0]
    # 1. the forwards: the same fragments, screen positions apart by rounding only
    pix_differ = int((frags_f.idx != frags_u.idx).any(-1).sum())
    vis_u = _C.visibility_from_idx(frags_u.idx, P)
    vis_differ = int((_C.visibility_from_idx(frags_f.idx, P) != vis_u).sum())
    dndc = (info["ndc"] - ndc_u).abs()
    assert pix_differ <= 1e-3 * frags_u.idx[..., 0].numel() and vis_differ <= 1e-3 * P, (pix_differ, vis_differ)
    assert dndc.max() <= 1e-6 and (dndc > 0).any(), dndc.max()
    # 2. the unfused route's records and fragments through the fused backward + camera backward
    rec = torch.zeros((P, 8), device=dev)
    rec[:, :3], rec[:, 3:5] = ndc_u, info["radii"]
    frag = namedtuple("Fragments", "records idx weights visible")(rec, frags_u.idx.contiguous(),
                                                                  torch.zeros_like(frags_u.qvalue), vis_u)
    proj, view = camera_matrices(cams)
    _, g_rows, [(gP, gV)] = backward_via_lib(frag, cloud.points_packed().detach().contiguous(), proj.detach(),
                                             view.detach(), cloud.cloud_to_packed_first_idx(),
                                             cloud.num_points_per_cloud(), False, _splat_params(settings, cams), g, None)
    R, T = cams.R.detach().clone().requires_grad_(True), cams.T.detach().clone().requires_grad_(True)
    torch.autograd.backward(camera_matrices(FoVPerspectiveCameras(znear=0.1, zfar=100.0, R=R, T=T, device=dev)),
                            [gP, gV])
    p_x = torch.zeros_like(p_u).index_add_(0, rows, g_rows)
    for name, got, want in (("points", p_x, p_u), ("R", R.grad, cams.R.grad), ("T", T.grad, cams.T.grad)):
        scale = want.abs().max()
        assert scale > 0 and (got - want).abs().max() <= 2e-4 * scale, (name, (got - want).abs().max(), scale)
    # (the routes' own position gradients, for the record: apart by far more than 2e-4 here)
    gap = ((p_f - p_u).abs().max() / p_u.abs().max()).item()
    print("differing fragments %d, visible %d, NDC slots %d (max %.3g); fused vs unfused position gradient %.3g"
          % (pix_differ, vis_differ, int((dndc > 0).any(1).sum()), dndc.max().item(), gap))


# ---- 4. grad_proj / grad_view against the float64 sums over the same grad_ndc --------------------------------------
def _check_against_float64(pts, proj, view, grad_ndc, first, num, gP, gV):
    wP, wV, aP, aV = camera_grads64(pts, proj, view, grad_ndc, first, num)
    assert torch.isfinite(gP).all() and torch.isfinite(gV).all()
    assert ((gP.double() - wP).abs() <= 1e-5 * aP).all(), ((gP.double() - wP).abs() / aP.clamp(min=1e-30)).max()
    assert ((gV.double() - wV).abs() <= 1e-5 * aV).all(), ((gV.double() - wV).abs() / aV.clamp(min=1e-30)).max()
    assert wP.abs().max() > 0


@pytest.mark.parametrize("clip", [0.05, -1.0])
@pytest.mark.parametrize("shared", [True, False])
def test_proj_view_gradients_equal_float64_sums(cuda_device, clip, shared):
    d = cuda_device
    P0, N, S, K = 20000, 3, 128, 5
    pts, nrm, col, proj, view, _ = scene(P0, N, seed=21)
    prm = SplatParams(image_size=S, points_per_pixel=K, znear=0.1, clip_pts_grad=clip)
    gen = torch.Generator().manual_seed(5)
    if shared:
        p, n, c, first, num = pts.to(d), nrm.to(d), col.repeat(N, 1).to(d), None, None
    else:   # a different cloud per view, packed
        keep = [torch.randperm(P0, generator=gen)[: P0 - 3000 * k] for k in range(N)]
        p, n, c = (torch.cat([t[k] for k in keep]).to(d) for t in (pts, nrm, col))
        first = torch.tensor([0] + [len(k) for k in keep[:-1]]).cumsum(0).to(d)
        num = torch.tensor([len(k) for k in keep]).to(d)
    h = torch.full((N,), 3e-4, device=d)
    projd, viewd = proj.to(d), view.to(d)
    out = render_points(p, n, c, projd, viewd, h, prm, first_idx=first, num_points=num, shared_cloud=shared,
                        return_fragments=True)
    gi = (torch.randn(N, S, S, 4, generator=gen) * 1e-3).to(d)
    gz = (torch.randn(N, S, S, K, generator=gen) * 1e-3).to(d) * (out.idx >= 0)     # loss on the z-buffer too
    grad_ndc, _, res = backward_via_lib(out, p, projd, viewd, first, num, shared, prm, gi, gz, repeat_camera=2)
    gP, gV = res[0]
    _check_against_float64(p, projd, viewd, grad_ndc, first, num, gP, gV)
    assert gV[:, :, 2].abs().sum() > 0                              # the z-buffer gradient reaches view[:, :, 2]
    assert (gP[:, :, 2] == 0).all() and (gV[:, :, [0, 1, 3]] == 0).all()
    # 6. the camera kernels are deterministic: the same inputs give the same bits
    assert torch.equal(res[1][0], gP) and torch.equal(res[1][1], gV)


# ---- 5. fused shading: camera centres, and the view matrices through make_shading ----------------------------------
def _shade64_cam(p, n, alb, lights, cam, shininess):
    """_shade64 of tests/test_shading.py with the camera centres as the input"""
    N, P0 = cam.shape[0], p.shape[0]
    l64 = lights.double()
    outs = []
    for v in range(N):
        amb, dif, spe = apply_lighting(p, n, l64, cam[v].expand(P0, 3), shininess=shininess)
        outs.append(alb * (amb + dif) + spe)
    return torch.cat(outs, 0)


@pytest.mark.parametrize("kind", ["sun", "point"])
def test_shading_camera_gradients_match_float64_autograd(cuda_device, kind):
    d = cuda_device
    P0, N, S, shin = 20000, 3, 96, 24.0
    pts, nrm, col, proj, view, _ = scene(P0, N, seed=12)
    g = torch.Generator().manual_seed(1)
    nrm = nrm * (0.85 + 0.15 * torch.rand(P0, 1, generator=g))
    lights = _lights(kind, d)
    prm = SplatParams(image_size=S, znear=0.1, clip_pts_grad=-1.0)
    h = torch.full((N,), 3e-4, device=d)
    gi = (torch.randn(N, S, S, 4, generator=g) * 1e-3).to(d)
    projd, viewd = proj.to(d), view.to(d)
    p2, n2, a2 = (t.to(d).double().requires_grad_(True) for t in (pts, nrm, col))

    def unfused(shaded, *leaves):
        o = render_points(p2.float(), n2.float().detach(), shaded.float(), projd, viewd, h, prm)
        return torch.autograd.grad(o.image, leaves, gi)

    # camera centres as a leaf
    cam = camera_centres(viewd).detach().requires_grad_(True)
    sh = make_shading(lights, viewd, shininess=shin)._replace(cam_centres=cam)
    render_points(pts.to(d), nrm.to(d), col.to(d), projd, viewd, h, prm, shading=sh).image.backward(gi)
    cam64 = cam.detach().double().requires_grad_(True)
    (want_cam,) = unfused(_shade64_cam(p2, n2, a2, lights, cam64, shin), cam64)
    # the view matrices through make_shading (no z-buffer loss: the geometry adds nothing to view)
    view_f = viewd.clone().requires_grad_(True)
    sh = make_shading(lights, view_f, shininess=shin)
    render_points(pts.to(d), nrm.to(d), col.to(d), projd, view_f, h, prm, shading=sh).image.backward(gi)
    view64 = viewd.double().requires_grad_(True)
    (want_view,) = unfused(_shade64(p2, n2, a2, lights, view64, shin), view64)
    for name, got, want in (("cam_centres", cam.grad, want_cam), ("view", view_f.grad, want_view)):
        scale = want.abs().max().item()
        assert scale > 0, name
        err = (got.double() - want).abs().max().item()
        assert err <= 2e-4 * scale, (name, err, scale)


# ---- 6. determinism, and the data-parallel backward of one rank ---------------------------------------------------
def test_camera_gradients_reproducible_and_equal_through_grad_sync(cuda_device):
    from dss_b200.parallel import GradSync
    d = cuda_device
    P0, N, S = 12000, 2, 64
    pts, nrm, col, proj, view, _ = scene(P0, N, seed=5)
    prm = SplatParams(image_size=S, znear=0.1, clip_pts_grad=0.05)
    h = torch.full((N,), 3e-4, device=d)
    gi = (torch.randn(N, S, S, 4, generator=torch.Generator().manual_seed(2)) * 1e-3).to(d)
    rows, amb, kind = pack_lights(_lights("point", d))
    res = []
    for sync in (None, None, GradSync()):
        pr, vw = proj.to(d).requires_grad_(True), view.to(d).requires_grad_(True)
        cam = camera_centres(view.to(d)).requires_grad_(True)
        sh = Shading(rows.to(d), amb.to(d), cam, kind, 64.0)
        p, n, a = (t.to(d).requires_grad_(True) for t in (pts, nrm, col))
        render_points(p, n, a, pr, vw, h, prm, shading=sh, grad_sync=sync).image.backward(gi)
        torch.cuda.synchronize()
        res.append((pr.grad, vw.grad, cam.grad, p.grad))
    for other in res[1:]:
        # proj / view come from the occupancy gather (no atomics): the same bits.  The camera centres read d L / d shaded,
        # which the colour scatter sums with float atomics
        assert torch.equal(other[0], res[0][0]) and torch.equal(other[1], res[0][1])
        torch.testing.assert_close(other[2], res[0][2], rtol=1e-5, atol=1e-9)
        torch.testing.assert_close(other[3], res[0][3], rtol=1e-5, atol=1e-9)
    assert res[0][0].abs().max() > 0 and res[0][2].abs().max() > 0


# ---- 7. launches: nothing new unless a camera requires grad --------------------------------------------------------
def test_camera_gradients_add_only_their_own_launches(cuda_device):
    d = cuda_device
    P0, N, S = 8000, 2, 64
    pts, nrm, col, proj, view, _ = scene(P0, N, seed=6)
    prm = SplatParams(image_size=S, znear=0.1)
    h = torch.full((N,), 3e-4, device=d)
    gi = (torch.randn(N, S, S, 4, generator=torch.Generator().manual_seed(3)) * 1e-3).to(d)
    rows, amb, kind = pack_lights(_lights("sun", d))

    def launches(cam_grad, shading):
        pr, vw = proj.to(d).requires_grad_(cam_grad), view.to(d).requires_grad_(cam_grad)
        sh = Shading(rows.to(d), amb.to(d), camera_centres(view.to(d)).requires_grad_(cam_grad), kind, 64.0) \
            if shading else None
        p = pts.to(d).requires_grad_(True)
        c = col.to(d).requires_grad_(True)
        out = render_points(p, nrm.to(d), c, pr, vw, h, prm, shading=sh)
        torch.cuda.synchronize()
        _lib.profile_reset(d)
        n0 = _lib.launch_count(d)
        out.image.backward(gi)
        torch.cuda.synchronize()
        return _lib.launch_count(d) - n0, _lib.profile_read(d)["camera_backward"][1]

    _lib.profile_enable(True, d)
    try:
        for shading in (False, True):
            launches(False, shading)                       # warm-up: scratch sizes
            base, base_brackets = launches(False, shading)
            with_cam, brackets = launches(True, shading)
            assert base_brackets == 0 and brackets == 1
            assert with_cam == base + 2                    # partial sums + per-view totals
            assert launches(False, shading) == (base, 0)
    finally:
        _lib.profile_enable(False, d)


# ---- 8. the headline size ----------------------------------------------------------------------------------------
def test_headline_size_camera_gradients_equal_float64_sums(cuda_device):
    d = cuda_device
    P0, N, S, K = 1_000_000, 8, 512, 5
    pts, nrm, col, proj, view, _ = scene(P0, N, seed=0)
    prm = SplatParams(image_size=S, points_per_pixel=K, znear=0.1, clip_pts_grad=0.05)
    h = torch.full((N,), 5e-5, device=d)
    p, projd, viewd = pts.to(d), proj.to(d), view.to(d)
    out = render_points(p, nrm.to(d), col.to(d), projd, viewd, h, prm, return_fragments=True)
    gen = torch.Generator().manual_seed(4)
    gi = (torch.randn(N, S, S, 4, generator=gen) * 1e-3).to(d)
    gz = (torch.randn(N, S, S, K, generator=gen) * 1e-4).to(d) * (out.idx >= 0)
    grad_ndc, _, res = backward_via_lib(out, p, projd, viewd, None, None, True, prm, gi, gz)
    _check_against_float64(p, projd, viewd, grad_ndc, None, None, *res[0])


# ---- 9. usefulness: recover a camera translation from silhouettes -------------------------------------------------
def test_silhouette_l1_recovers_translation_offset(cuda_device):
    dev, S, N, steps = cuda_device, 128, 4, 60
    ply = read_ply(os.path.join(GOLDEN_DIR, "ply", "bunny-8000.ply"))
    pts = torch.as_tensor(ply["points"], dtype=torch.float32)
    pts = (pts - pts.mean(0)) / (pts - pts.mean(0)).norm(dim=1).max() * 0.6
    nrm = torch.nn.functional.normalize(torch.as_tensor(ply["normals"], dtype=torch.float32), dim=1)
    cloud = PointClouds3D([pts.to(dev)], normals=[nrm.to(dev)], features=[torch.ones_like(pts).to(dev)])
    R, T_true = look_at_view_transform(dist=2.0, elev=[20, -10, 35, 0], azim=[0, 90, 200, 300])
    settings = PointsRasterizationSettings(backface_culling=False, Vrk_invariant=False, Vrk_isotropic=True,
                                           radii_backward_scaler=5, image_size=S, points_per_pixel=5,
                                           clip_pts_grad=-1.0)
    cams = FoVPerspectiveCameras(znear=0.1, zfar=100.0, R=R, T=T_true, device=dev)
    renderer = SurfaceSplattingRenderer(SurfaceSplatting(cameras=cams, raster_settings=settings))
    with torch.no_grad():
        target = renderer(cloud, cameras=cams)[..., 3]
    offset = torch.tensor([[0.04, -0.03, 0.02], [-0.03, 0.03, -0.02], [0.02, 0.04, 0.03], [-0.04, -0.02, -0.03]])
    T = (T_true + offset).to(dev).requires_grad_(True)
    opt = torch.optim.Adam([T], lr=5e-3)
    T_true = T_true.to(dev)
    dist0 = (T.detach() - T_true).norm().item()
    for _ in range(steps):
        opt.zero_grad()
        cams.T = T
        (renderer(cloud, cameras=cams)[..., 3] - target).abs().mean().backward()
        assert torch.isfinite(T.grad).all() and T.grad.abs().max() > 0
        opt.step()
    dist = (T.detach() - T_true).norm().item()
    assert dist <= 0.5 * dist0, (dist0, dist)
