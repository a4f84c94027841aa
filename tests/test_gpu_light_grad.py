"""Per-view lights and light gradients through the fused shading (dss_light_backward): images and the albedo / normal /
position / camera-centre / light gradients equal the float64 autograd route for shared and per-view lights, shared
lights expanded per view give the shared path's bits, the light kernels are deterministic and cost nothing unless a
light requires grad, the ABI limits (256 views x 8 per-view lights) run, a captured step replays per-view lights, and
Adam on the per-view light directions recovers them from rendered images."""
import ctypes as C
import os

import pytest
import torch

from dss_b200 import _lib, ops
from dss_b200.core.camera import FoVPerspectiveCameras, camera_matrices, look_at_view_transform
from dss_b200.core.lighting import DirectionalLights, PointLights
from dss_b200.core.texture import apply_lighting, camera_centres
from dss_b200.ops import SplatParams, make_shading, render_points
from dss_b200.utils.io import read_ply
from tests.test_shading import _lights
from tests.util import GOLDEN_DIR, scene

pytestmark = pytest.mark.gpu

_PROPS = ("_vec", "diffuse_color", "specular_color", "ambient_color")


def _per_view_lights(kind, dev, N=3):
    """two lights per view: the directions / locations and the diffuse colours vary per view, the specular colours are
    shared (batch 1, broadcast), two ambient terms per view (summed)"""
    base = _lights(kind)
    g = torch.Generator().manual_seed(11)
    vec = base._vec + 0.4 * torch.randn(N, 2, 3, generator=g)
    dif = base.diffuse_color * (0.7 + 0.6 * torch.rand(N, 2, 3, generator=g))
    amb = base.ambient_color * (0.5 + torch.rand(N, 2, 3, generator=g))
    kw = dict(ambient_color=amb, diffuse_color=dif, specular_color=base.specular_color, device=dev)
    return DirectionalLights(direction=vec, **kw) if kind == "sun" else PointLights(location=vec, **kw)


def _leaf_lights(lights, dtype):
    """a copy of `lights` whose four property tensors are fresh leaves of `dtype` that require grad"""
    out = type(lights)(device=lights.device)
    for name in _PROPS:
        setattr(out, name, getattr(lights, name).detach().to(dtype).clone().requires_grad_(True))
    return out


def _shade64(p, n, alb, lights, cam, shininess):
    """(N*P0,3) shaded colours of every (view, point) through the torch shading, lights gathered per view"""
    N, P0 = cam.shape[0], p.shape[0]
    idx = torch.arange(N, device=p.device).repeat_interleave(P0)
    amb, dif, spe = apply_lighting(p.repeat(N, 1), n.repeat(N, 1), lights, cam[idx], shininess=shininess, view_idx=idx)
    return alb.repeat(N, 1) * (amb + dif) + spe


def _close(name, got, want, rel=2e-4):
    scale = want.abs().max().item()
    assert scale > 0, name
    err = (got.double() - want.double()).abs().max().item()
    assert err <= rel * scale, (name, err, scale)


# ---- 1, 3, 4. fused vs the float64 autograd route: image, point, camera-centre and light gradients ------------------
@pytest.mark.parametrize("layout", ["shared", "per_view"])
@pytest.mark.parametrize("kind", ["sun", "point"])
def test_fused_light_and_shading_gradients_match_float64_autograd(cuda_device, kind, layout):
    d = cuda_device
    P0, N, S, shin = 20000, 3, 96, 13.5                 # non-integer shininess
    pts, nrm, col, proj, view, _ = scene(P0, N, seed=12)
    g = torch.Generator().manual_seed(1)
    nrm = nrm * (0.85 + 0.15 * torch.rand(P0, 1, generator=g))
    # every light of a sphere's cloud is behind part of its surface
    lights = _lights(kind, d) if layout == "shared" else _per_view_lights(kind, d, N)
    prm = SplatParams(image_size=S, znear=0.1, clip_pts_grad=-1.0)
    h = torch.full((N,), 3e-4, device=d)
    gi = (torch.randn(N, S, S, 4, generator=g) * 1e-3).to(d)
    projd, viewd = proj.to(d), view.to(d)
    # ---- fused ----
    l32 = _leaf_lights(lights, torch.float32)
    cam = camera_centres(viewd).detach().requires_grad_(True)
    p1, n1, a1 = (t.to(d).requires_grad_(True) for t in (pts, nrm, col))
    sh = make_shading(l32, viewd, shininess=shin)._replace(cam_centres=cam)
    assert sh.lights.dim() == (2 if layout == "shared" else 3)
    o1 = render_points(p1, n1, a1, projd, viewd, h, prm, shading=sh)
    o1.image.backward(gi)
    # ---- float64 torch shading feeding the per-(view, point) colour path ----
    l64 = _leaf_lights(lights, torch.float64)
    cam64 = cam.detach().double().requires_grad_(True)
    p2, n2, a2 = (t.to(d).double().requires_grad_(True) for t in (pts, nrm, col))
    shaded = _shade64(p2, n2, a2, l64, cam64, shin)
    o2 = render_points(p2.float(), n2.float().detach(), shaded.float(), projd, viewd, h, prm)
    leaves64 = [p2, n2, a2, cam64] + [getattr(l64, k) for k in _PROPS]
    want = torch.autograd.grad(o2.image, leaves64, gi)
    assert torch.equal(o1.idx, o2.idx)
    torch.testing.assert_close(o1.image, o2.image, rtol=1e-4, atol=2e-6)
    got = [p1.grad, n1.grad, a1.grad, cam.grad] + [getattr(l32, k).grad for k in _PROPS]
    names = ["points", "normals", "albedo", "cam_centres", "direction/location", "diffuse", "specular", "ambient"]
    for name, gt, wt in zip(names, got, want):
        assert gt is not None and gt.shape == wt.shape, name
        _close(name, gt, wt)


# ---- 2. shared lights expanded per view give the shared path's bits -----------------------------------------------
def _shading_backward_via_lib(sh, pts, nrm, alb, grad_image, S, grad_lights, grad_amb, repeat=1):
    """dss_colour_backward over an idx that gives every (view, point) slot exactly one pixel (so that d L / d shaded has
    no atomics to reorder), then dss_light_backward `repeat` times -> (albedo, normal, position grads, light grads)"""
    dev = pts.device
    N, P0 = sh.cam_centres.shape[0], pts.shape[0]
    idx = torch.full((N, S * S), -1, dtype=torch.int32, device=dev)
    idx[:, :P0] = (torch.arange(N, device=dev)[:, None] * P0 + torch.arange(P0, device=dev)[None]).int()
    idx = idx.view(N, S, S, 1)
    weights = torch.ones((N, S, S, 1), device=dev)
    a = _lib.RenderArgs()
    prm = SplatParams(image_size=S, points_per_pixel=1)
    ops._fill_common(a, pts, nrm, None, None, None, None, None, None, True, N, P0, N * P0, prm)
    ops._fill_shading(a, sh, alb)
    grad_colours = torch.empty((N * P0, 3), device=dev)
    ga, gn, gp = (torch.empty_like(pts) for _ in range(3))
    a.idx, a.weights, a.grad_image, a.grad_colours = (_lib.ptr(t) for t in (idx, weights, grad_image, grad_colours))
    a.grad_albedo, a.grad_normals_world, a.grad_points_shading = _lib.ptr(ga), _lib.ptr(gn), _lib.ptr(gp)
    lib, ctx, st = _lib.load(), _lib.ctx(dev), _lib.stream_ptr(dev)
    _lib.check(lib.dss_colour_backward(ctx, C.byref(a), st), "dss_colour_backward")
    res = []
    for _ in range(repeat):
        gl, gam = torch.full_like(grad_lights, float("nan")), torch.full_like(grad_amb, float("nan"))
        _lib.check(lib.dss_light_backward(ctx, C.byref(a), _lib.ptr(gl), _lib.ptr(gam), st), "dss_light_backward")
        res.append((gl, gam))
    torch.cuda.synchronize(dev)
    return ga, gn, gp, res


@pytest.mark.parametrize("kind", ["sun", "point"])
def test_shared_lights_expanded_per_view_equal_the_shared_path_bit_for_bit(cuda_device, kind):
    d = cuda_device
    P0, N, S = 20000, 3, 96
    pts, nrm, col, proj, view, _ = scene(P0, N, seed=14)
    prm = SplatParams(image_size=S, znear=0.1, clip_pts_grad=-1.0)
    h = torch.full((N,), 3e-4, device=d)
    p, n, a, projd, viewd = pts.to(d), nrm.to(d), col.to(d), proj.to(d), view.to(d)
    shared = make_shading(_lights(kind, d), viewd, shininess=24.0)
    expanded = shared._replace(lights=shared.lights.expand(N, -1, -1).contiguous(),
                               ambient=shared.ambient.expand(N, 3).contiguous())
    o = [render_points(p, n, a, projd, viewd, h, prm, shading=s) for s in (shared, expanded)]
    assert torch.equal(o[0].image, o[1].image) and torch.equal(o[0].idx, o[1].idx)
    # the backward kernels on the same d L / d shaded (one pixel per slot: no atomics to reorder)
    S2 = 160                                             # S2^2 >= P0
    g2 = torch.randn(N, S2, S2, 4, generator=torch.Generator().manual_seed(3)).to(d)
    L = shared.lights.shape[0]
    rs = _shading_backward_via_lib(shared, p, n, a, g2, S2, torch.empty(L, 9, device=d), torch.empty(3, device=d), 2)
    re = _shading_backward_via_lib(expanded, p, n, a, g2, S2, torch.empty(N, L, 9, device=d), torch.empty(N, 3, device=d), 2)
    for name, x, y in zip(("albedo", "normals", "points"), rs[:3], re[:3]):
        assert torch.equal(x, y), name
        assert x.abs().max() > 0, name
    # 5. the light kernels reproduce run to run; the per-view rows add up to the shared ones
    for r in (rs, re):
        assert torch.equal(r[3][0][0], r[3][1][0]) and torch.equal(r[3][0][1], r[3][1][1])
    (gl_s, gam_s), (gl_e, gam_e) = rs[3][0], re[3][0]
    assert torch.isfinite(gl_e).all() and gl_e[..., 0:3].abs().max() > 0
    torch.testing.assert_close(gl_e.double().sum(0), gl_s.double(), rtol=1e-5, atol=1e-6 * gl_s.abs().max().item())
    torch.testing.assert_close(gam_e.double().sum(0), gam_s.double(), rtol=1e-5, atol=1e-6)


# ---- 5. the GradSync path gives the same light gradients --------------------------------------------------------------
def test_light_gradients_reproducible_and_equal_through_grad_sync(cuda_device):
    from dss_b200.parallel import GradSync
    d = cuda_device
    P0, N, S = 12000, 3, 64
    pts, nrm, col, proj, view, _ = scene(P0, N, seed=5)
    prm = SplatParams(image_size=S, znear=0.1, clip_pts_grad=0.05)
    h = torch.full((N,), 3e-4, device=d)
    gi = (torch.randn(N, S, S, 4, generator=torch.Generator().manual_seed(2)) * 1e-3).to(d)
    res = []
    for sync in (None, None, GradSync()):
        lights = _leaf_lights(_per_view_lights("point", d, N), torch.float32)
        sh = make_shading(lights, view.to(d))
        p, n, a = (t.to(d).requires_grad_(True) for t in (pts, nrm, col))
        render_points(p, n, a, proj.to(d), view.to(d), h, prm, shading=sh, grad_sync=sync).image.backward(gi)
        torch.cuda.synchronize()
        res.append([getattr(lights, k).grad for k in _PROPS] + [p.grad])
    for other in res[1:]:
        # the light kernels are deterministic; d L / d shaded comes from the colour scatter's float atomics
        for x, y in zip(other, res[0]):
            torch.testing.assert_close(x, y, rtol=1e-5, atol=1e-9)
    assert all(t.abs().max() > 0 for t in res[0])


# ---- 6. launches: nothing new unless a light requires grad -------------------------------------------------------
def test_light_gradients_add_only_their_own_launches(cuda_device):
    d = cuda_device
    P0, N, S = 8000, 2, 64
    pts, nrm, col, proj, view, _ = scene(P0, N, seed=6)
    prm = SplatParams(image_size=S, znear=0.1)
    h = torch.full((N,), 3e-4, device=d)
    gi = (torch.randn(N, S, S, 4, generator=torch.Generator().manual_seed(3)) * 1e-3).to(d)

    def launches(layout, light_grad, amb_grad, cam_grad):
        lights = _lights("sun", d) if layout == "shared" else _per_view_lights("sun", d, N)
        sh = make_shading(lights, view.to(d))
        sh = sh._replace(lights=sh.lights.detach().requires_grad_(light_grad),
                         ambient=sh.ambient.detach().requires_grad_(amb_grad),
                         cam_centres=sh.cam_centres.detach().requires_grad_(cam_grad))
        p = pts.to(d).requires_grad_(True)
        out = render_points(p, nrm.to(d), col.to(d), proj.to(d), view.to(d), h, prm, shading=sh)
        torch.cuda.synchronize()
        _lib.profile_reset(d)
        n0 = _lib.launch_count(d)
        out.image.backward(gi)
        torch.cuda.synchronize()
        st = _lib.profile_read(d)
        assert (sh.lights.grad is not None) == light_grad and (sh.ambient.grad is not None) == amb_grad
        return _lib.launch_count(d) - n0, st["light_backward"][1], st["camera_backward"][1]

    _lib.profile_enable(True, d)
    try:
        for layout in ("shared", "per_view"):
            launches(layout, False, False, False)                          # warm-up: scratch sizes
            base = launches(layout, False, False, False)
            assert base[1:] == (0, 0)
            assert launches(layout, True, False, False) == (base[0] + 2, 1, 0)      # partial sums + finish
            assert launches(layout, False, True, False) == (base[0] + 2, 1, 0)
            assert launches(layout, True, True, True) == (base[0] + 4, 1, 1)        # both sets
            assert launches(layout, False, False, False) == base
    finally:
        _lib.profile_enable(False, d)


# ---- 7. the ABI limits: 256 views x 8 per-view lights --------------------------------------------------------------
def test_256_views_with_8_lights_each_match_float64_autograd(cuda_device):
    d = cuda_device
    P0, N, L, S, shin = 3000, 256, 8, 32, 20.0
    pts, nrm, col, proj, view, _ = scene(P0, N, seed=31)
    g = torch.Generator().manual_seed(4)
    lights = DirectionalLights(ambient_color=0.1 * torch.rand(N, L, 3, generator=g),
                               diffuse_color=0.15 * torch.rand(N, L, 3, generator=g),
                               specular_color=0.1 * torch.rand(N, L, 3, generator=g),
                               direction=torch.randn(N, L, 3, generator=g), device=d)
    prm = SplatParams(image_size=S, znear=0.1, clip_pts_grad=-1.0)
    h = torch.full((N,), 1e-3, device=d)
    gi = (torch.randn(N, S, S, 4, generator=g) * 1e-3).to(d)
    projd, viewd = proj.to(d), view.to(d)
    l32 = _leaf_lights(lights, torch.float32)
    a1 = col.to(d).requires_grad_(True)
    sh = make_shading(l32, viewd, shininess=shin)
    assert sh.lights.shape == (N, L, 9)
    o1 = render_points(pts.to(d), nrm.to(d), a1, projd, viewd, h, prm, shading=sh)
    o1.image.backward(gi)
    l64 = _leaf_lights(lights, torch.float64)
    a2 = col.to(d).double().requires_grad_(True)
    shaded = _shade64(pts.to(d).double(), nrm.to(d).double(), a2, l64, camera_centres(viewd.double()), shin)
    o2 = render_points(pts.to(d), nrm.to(d), shaded.float(), projd, viewd, h, prm)
    want = torch.autograd.grad(o2.image, [a2] + [getattr(l64, k) for k in _PROPS], gi)
    torch.testing.assert_close(o1.image, o2.image, rtol=1e-4, atol=2e-6)
    _close("albedo", a1.grad, want[0])
    views = torch.randperm(N, generator=torch.Generator().manual_seed(5))[:24].to(d)
    for name, k, wt in zip(("direction", "diffuse", "specular", "ambient"), _PROPS, want[1:]):
        gt = getattr(l32, k).grad
        assert gt.shape == (N, L, 3) and torch.isfinite(gt).all(), name
        scale = wt.abs().max().item()
        err = (gt[views].double() - wt[views]).abs().max().item()
        assert scale > 0 and err <= 2e-4 * scale, (name, err, scale)


# ---- 8. a captured step with per-view lights ------------------------------------------------------------------------
def test_graphed_step_with_per_view_lights_replays_the_eager_step(cuda_device):
    from dss_b200.graph import GraphedRenderStep
    d = cuda_device
    P0, N, S = 20000, 3, 96
    pts, nrm, col, proj, view, _ = scene(P0, N, seed=23)
    prm = SplatParams(image_size=S, znear=0.1, clip_pts_grad=0.05)
    h = torch.full((N,), 3e-4, device=d)
    g = (torch.randn(N, S, S, 4, generator=torch.Generator().manual_seed(8)) * 1e-3).to(d)
    lights = _leaf_lights(_per_view_lights("point", d, N), torch.float32)
    sh = make_shading(lights, view.to(d))
    step = GraphedRenderStep(pts.to(d), nrm.to(d), col.to(d), proj.to(d), view.to(d), h, prm, g, shading=sh)
    step.replay()
    torch.cuda.synchronize()
    assert all(getattr(lights, k).grad is None for k in _PROPS)       # the lights are constants of the captured step
    const = sh._replace(lights=sh.lights.detach(), ambient=sh.ambient.detach())
    for it in range(2):
        img = step.replay()
        torch.cuda.synchronize()
        pe, ne, ce = (t.detach().clone().requires_grad_(True) for t in (step.points, step.normals, step.colours))
        o = render_points(pe, ne, ce, proj.to(d), view.to(d), h, prm, shading=const)
        o.image.backward(g)
        assert torch.equal(img, o.image.detach())
        for got, want in ((step.grad_points, pe.grad), (step.grad_normals, ne.grad), (step.grad_colours, ce.grad)):
            torch.testing.assert_close(got, want, rtol=1e-4, atol=1e-9)     # float atomics in the colour scatter
        with torch.no_grad():
            step.colours.mul_(0.9)


# ---- 9. usefulness: recover per-view light directions from images --------------------------------------------------
def test_adam_on_per_view_light_directions_recovers_them(cuda_device):
    dev, S, N, steps = cuda_device, 128, 4, 60
    ply = read_ply(os.path.join(GOLDEN_DIR, "ply", "bunny-8000.ply"))
    pts = torch.as_tensor(ply["points"], dtype=torch.float32)
    pts = ((pts - pts.mean(0)) / (pts - pts.mean(0)).norm(dim=1).max() * 0.6).to(dev)
    nrm = torch.nn.functional.normalize(torch.as_tensor(ply["normals"], dtype=torch.float32), dim=1).to(dev)
    alb = torch.full_like(pts, 0.8)
    R, T = look_at_view_transform(dist=2.0, elev=[20, -10, 35, 0], azim=[0, 90, 200, 300])
    proj, view = (m.to(dev) for m in camera_matrices(FoVPerspectiveCameras(znear=0.1, zfar=100.0, R=R, T=T)))
    prm = SplatParams(image_size=S, points_per_pixel=5, znear=0.1, clip_pts_grad=-1.0)
    h = torch.full((N,), 1e-3, device=dev)
    # a light from the camera's side of each view, as the reference's data draws one in each camera's frame
    true_dir = torch.nn.functional.normalize(camera_centres(view) + torch.tensor([[0.5, 1.0, 0.3]], device=dev), dim=1)
    colours = dict(ambient_color=(((0.3, 0.3, 0.3),),), diffuse_color=(((0.6, 0.6, 0.6),),),
                   specular_color=(((0.2, 0.2, 0.2),),), device=dev)

    def render(direction):
        sh = make_shading(DirectionalLights(direction=direction[:, None, :], **colours), view, shininess=20.0)
        return render_points(pts, nrm, alb, proj, view, h, prm, shading=sh).image[..., :3]

    def angle(a):
        cos = (torch.nn.functional.normalize(a, dim=1) * true_dir).sum(1).clamp(-1, 1)
        return torch.rad2deg(torch.acos(cos)).mean().item()

    with torch.no_grad():
        target = render(true_dir)
    offset = torch.tensor([[0.3, -0.1, 0.1], [-0.2, 0.2, -0.1], [0.1, 0.25, -0.2], [-0.25, -0.15, 0.15]], device=dev)
    direction = (true_dir + offset).requires_grad_(True)
    opt = torch.optim.Adam([direction], lr=2e-2)
    err0 = angle(direction.detach())
    for _ in range(steps):
        opt.zero_grad()
        ((render(direction) - target) ** 2).mean().backward()
        assert torch.isfinite(direction.grad).all() and direction.grad.abs().max() > 0
        opt.step()
    err = angle(direction.detach())
    assert err <= 0.5 * err0, (err0, err)
