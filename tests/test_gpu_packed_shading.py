"""Fused shading of packed clouds: every packed row is shaded with the lights and camera centre of the view whose range
holds it, and its albedo / normal / position gradients are written per row.  Checked against the float64 torch shading
(ragged and empty views, duplicated world points, rows no view covers), against the shared-cloud kernels on a shared
cloud laid out as N packed copies, for run-to-run reproducibility, and for the operator's input checks."""
import ctypes as C

import numpy as np
import pytest
import torch

from dss_b200 import _lib, ops
from dss_b200.core.texture import apply_lighting, camera_centres
from dss_b200.ops import SplatParams, make_shading, render_points
from tests.test_gpu_backward_f64 import _packed_layout
from tests.test_gpu_light_grad import _PROPS, _leaf_lights, _per_view_lights
from tests.test_shading import _lights
from tests.util import scene

pytestmark = pytest.mark.gpu

_NAMES = ("direction/location", "diffuse", "specular", "ambient")


def _close(name, got, want, rel):
    scale = want.abs().max().item()
    assert scale > 0, name
    err = (got.double() - want.double()).abs().max().item()
    assert err <= rel * scale, (name, err, scale)


def _packed_case(d, kind, layout, P0=6000, seed=12):
    """the layout of test_gpu_backward_f64._packed_layout over a sphere cloud: 4 views (ragged, one empty, duplicated
    world points, 150 uncovered rows) -> packed points, normals, albedo, proj, view, first, num, view index per row,
    covered-row mask and the lights"""
    pts, nrm, col, proj, view, _ = scene(P0 + 150, 4, seed=seed)
    g = torch.Generator().manual_seed(seed)
    nrm = nrm * (0.85 + 0.15 * torch.rand(P0 + 150, 1, generator=g))   # un-normalised normals
    rows, first, num = _packed_layout(P0)
    ridx = torch.as_tensor(rows)
    vidx = torch.zeros(len(rows), dtype=torch.int64)
    covered = torch.zeros(len(rows), dtype=torch.bool)
    for n, (f, k) in enumerate(zip(first, num)):
        vidx[f:f + k] = n
        covered[f:f + k] = True
    lights = _lights(kind, d) if layout == "shared" else _per_view_lights(kind, d, 4)
    return dict(pts=pts[ridx].to(d), nrm=nrm[ridx].to(d), alb=col[ridx].to(d), proj=proj.to(d), view=view.to(d),
                first=torch.as_tensor(first).to(d), num=torch.as_tensor(num).to(d), vidx=vidx.to(d),
                covered=covered.to(d), lights=lights)


# ---- 1. fused packed shading vs the float64 torch shading feeding the (P,3) colour route ----------------------------
@pytest.mark.parametrize("layout", ["shared", "per_view"])
@pytest.mark.parametrize("kind", ["sun", "point"])
def test_packed_shading_gradients_match_float64_autograd(cuda_device, kind, layout):
    d = cuda_device
    c = _packed_case(d, kind, layout)
    N, S, shin = 4, 128, 13.5                             # non-integer shininess
    prm = SplatParams(image_size=S, znear=0.1, clip_pts_grad=-1.0)
    h = torch.full((N,), 3e-4, device=d)
    gi = (torch.randn(N, S, S, 4, generator=torch.Generator().manual_seed(1)) * 1e-3).to(d)
    fi, npts = c["first"], c["num"]
    # ---- fused: the view matrices reach the shading through make_shading's camera centres ----
    l32 = _leaf_lights(c["lights"], torch.float32)
    v1 = c["view"].clone().requires_grad_(True)
    p1, n1, a1 = (c[k].clone().requires_grad_(True) for k in ("pts", "nrm", "alb"))
    sh = make_shading(l32, v1, shininess=shin)
    sh.cam_centres.retain_grad()
    o1 = render_points(p1, n1, a1, c["proj"], v1, h, prm, first_idx=fi, num_points=npts, shared_cloud=False,
                       shading=sh)
    o1.image.backward(gi)
    # ---- float64 torch shading of every packed row with its view's lights and camera ----
    l64 = _leaf_lights(c["lights"], torch.float64)
    v2 = c["view"].double().requires_grad_(True)
    p2, n2, a2 = (c[k].double().requires_grad_(True) for k in ("pts", "nrm", "alb"))
    cam64 = camera_centres(v2)
    vidx = c["vidx"]
    amb, dif, spe = apply_lighting(p2, n2, l64, cam64[vidx], shininess=shin, view_idx=vidx)
    shaded = a2 * (amb + dif) + spe
    o2 = render_points(p2.float(), n2.float().detach(), shaded.float(), c["proj"], v2.float(), h, prm, first_idx=fi,
                       num_points=npts, shared_cloud=False)
    leaves64 = [p2, n2, a2, cam64, v2] + [getattr(l64, k) for k in _PROPS]
    want = torch.autograd.grad(o2.image, leaves64, gi)
    assert torch.equal(o1.idx, o2.idx)
    torch.testing.assert_close(o1.image, o2.image, rtol=1e-4, atol=2e-6)
    got = [p1.grad, n1.grad, a1.grad, sh.cam_centres.grad, v1.grad] + [getattr(l32, k).grad for k in _PROPS]
    names = ["points", "normals", "albedo", "cam_centres", "view"] + list(_NAMES)
    for name, gt, wt in zip(names, got, want):
        assert gt is not None and gt.shape == wt.shape, name
        _close(name, gt, wt, 2e-4)
    # rows no view covers and the empty view (2) get exactly zero; everything else receives a gradient
    cov = c["covered"]
    for name, gt in zip(names[:3], got[:3]):
        assert (gt[~cov] == 0).all(), name
        assert gt[cov].abs().max() > 0, name
    for name, gt in zip(names[3:5], got[3:5]):
        assert (gt[2] == 0).all(), name
        assert all(gt[n].abs().max() > 0 for n in (0, 1, 3)), name
    for name, k, gt in zip(_NAMES, _PROPS, got[5:]):
        if layout == "per_view" and gt.shape[0] == N:
            assert (gt[2] == 0).all(), name
            assert all(gt[n].abs().max() > 0 for n in (0, 1, 3)), name
        else:
            assert gt.abs().max() > 0, name


# ---- the shading kernels behind an atomics-free colour gradient ------------------------------------------------------
def _shading_kernels(sh, pts, nrm, alb, first, num, grad_image, grad_ndc, S):
    """dss_colour_backward over an idx that gives every slot of view n's range exactly one pixel of view n (d L / d
    shaded then has no atomics to reorder), then dss_camera_backward (with the given grad_ndc) and dss_light_backward.
    first / num None: a shared cloud.  -> dict of the library's outputs"""
    dev = pts.device
    N = sh.cam_centres.shape[0]
    shared = first is None
    P = pts.shape[0] * (N if shared else 1)
    P0 = pts.shape[0]
    fr = [n * P0 for n in range(N)] if shared else first.tolist()
    nr = [P0] * N if shared else num.tolist()
    idx = torch.full((N, S * S), -1, dtype=torch.int32, device=dev)
    for n, (f, k) in enumerate(zip(fr, nr)):
        idx[n, :k] = torch.arange(f, f + k, dtype=torch.int32, device=dev)
    idx = idx.view(N, S, S, 1)
    weights = torch.ones((N, S, S, 1), device=dev)
    a = _lib.RenderArgs()
    prm = SplatParams(image_size=S, points_per_pixel=1)
    proj = torch.eye(4, device=dev).repeat(N, 1, 1)
    proj[:, 3, 3] = 2.0
    ops._fill_common(a, pts, nrm, None, proj, proj, None, None if shared else first, None if shared else num, shared,
                     N, P0, P, prm)
    ops._fill_shading(a, sh, alb)
    grad_colours = torch.empty((P, 3), device=dev)
    out = {k: torch.zeros_like(pts) for k in ("albedo", "normals", "points")}
    out.update(proj=torch.empty(N, 4, 4, device=dev), view=torch.empty(N, 4, 4, device=dev),
               cam=torch.empty(N, 3, device=dev), lights=torch.empty_like(sh.lights), ambient=torch.empty_like(sh.ambient))
    a.idx, a.weights, a.grad_image, a.grad_colours = (_lib.ptr(t) for t in (idx, weights, grad_image, grad_colours))
    a.grad_ndc = _lib.ptr(grad_ndc)
    a.grad_albedo, a.grad_normals_world = _lib.ptr(out["albedo"]), _lib.ptr(out["normals"])
    a.grad_points_shading = _lib.ptr(out["points"])
    lib, ctx, st = _lib.load(), _lib.ctx(dev), _lib.stream_ptr(dev)
    _lib.check(lib.dss_colour_backward(ctx, C.byref(a), st), "dss_colour_backward")
    _lib.check(lib.dss_camera_backward(ctx, C.byref(a), _lib.ptr(out["proj"]), _lib.ptr(out["view"]),
                                       _lib.ptr(out["cam"]), st), "dss_camera_backward")
    _lib.check(lib.dss_light_backward(ctx, C.byref(a), _lib.ptr(out["lights"]), _lib.ptr(out["ambient"]), st),
               "dss_light_backward")
    torch.cuda.synchronize(dev)
    return out


# ---- 2. a shared cloud laid out as N packed copies gives the shared fused shading -----------------------------------
@pytest.mark.parametrize("layout", ["shared", "per_view"])
@pytest.mark.parametrize("kind", ["sun", "point"])
def test_duplicated_packed_layout_equals_the_shared_cloud(cuda_device, kind, layout):
    d = cuda_device
    P0, N, S = 12000, 3, 96
    pts, nrm, col, proj, view, _ = scene(P0, N, seed=14)
    p, n, a, projd, viewd = pts.to(d), nrm.to(d), col.to(d), proj.to(d), view.to(d)
    sh = make_shading(_lights(kind, d) if layout == "shared" else _per_view_lights(kind, d, N), viewd, shininess=24.0)
    first = torch.arange(N, device=d) * P0
    num = torch.full((N,), P0, dtype=torch.int64, device=d)
    pp, npk, ap = p.repeat(N, 1), n.repeat(N, 1), a.repeat(N, 1)
    prm = SplatParams(image_size=S, znear=0.1)
    h = torch.full((N,), 3e-4, device=d)
    os_ = render_points(p, n, a, projd, viewd, h, prm, shading=sh)
    op = render_points(pp, npk, ap, projd, viewd, h, prm, first_idx=first, num_points=num, shared_cloud=False,
                       shading=sh)
    for name in ("image", "idx", "weights"):
        assert torch.equal(getattr(os_, name), getattr(op, name)), name
    # gradients of the shading kernels on the same d L / d shaded
    S2 = 112                                                # S2^2 >= P0
    g = torch.Generator().manual_seed(3)
    gi = torch.randn(N, S2, S2, 4, generator=g).to(d)
    gndc = torch.randn(N * P0, 3, generator=g).to(d)
    rs = _shading_kernels(sh, p, n, a, None, None, gi, gndc, S2)
    rp = _shading_kernels(sh, pp, npk, ap, first, num, gi, gndc, S2)
    # each view's rows are that view's term of the shared kernel's sum bit for bit: the shared kernel given the colour
    # gradient of view m alone computes exactly that term
    for m in range(N):
        gm = torch.zeros_like(gi)
        gm[m] = gi[m]
        rm = _shading_kernels(sh, p, n, a, None, None, gm, gndc, S2)
        for name in ("albedo", "normals"):
            assert torch.equal(rp[name][m * P0:(m + 1) * P0], rm[name]), (name, m)
    # the rows added over the views in view order give the shared sums; the shared kernel accumulates them with fused
    # multiply-adds, so the two differ by the rounding of the products (and the positions by the order of their terms)
    for name in ("albedo", "normals", "points"):
        tot = rp[name][:P0].clone()
        for m in range(1, N):
            tot += rp[name][m * P0:(m + 1) * P0]
        assert rs[name].abs().max() > 0, name
        _close(name, tot, rs[name], 1e-6)
    # camera and light gradients: fp64 sums over a different block partition
    for name in ("proj", "view", "cam", "lights", "ambient"):
        assert rs[name].abs().max() > 0, name
        _close(name, rp[name], rs[name], 1e-6)


# ---- 3. reproducibility ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["sun", "point"])
def test_packed_shading_backward_is_bit_reproducible(cuda_device, kind):
    d = cuda_device
    c = _packed_case(d, kind, "per_view", seed=21)
    sh = make_shading(c["lights"], c["view"], shininess=13.5)
    S = 80                                                  # S^2 >= the largest view range (4500)
    g = torch.Generator().manual_seed(4)
    gi = torch.randn(4, S, S, 4, generator=g).to(d)
    gndc = torch.randn(c["pts"].shape[0], 3, generator=g).to(d)
    runs = [_shading_kernels(sh, c["pts"], c["nrm"], c["alb"], c["first"], c["num"], gi, gndc, S) for _ in range(2)]
    cov = c["covered"]
    for name in runs[0]:
        assert torch.equal(runs[0][name], runs[1][name]), name
        assert torch.isfinite(runs[0][name]).all() and runs[0][name].abs().max() > 0, name
    for name in ("albedo", "normals", "points"):
        assert (runs[0][name][~cov] == 0).all(), name


# ---- 4. input checks ---------------------------------------------------------------------------------------------------
def test_packed_shading_input_checks(cuda_device):
    from dss_b200.parallel import GradSync
    d = cuda_device
    c = _packed_case(d, "sun", "shared", P0=600)
    sh = make_shading(c["lights"], c["view"])
    h = torch.full((4,), 3e-4, device=d)
    prm = SplatParams(image_size=32, znear=0.1)
    kw = dict(first_idx=c["first"], num_points=c["num"], shared_cloud=False, shading=sh)
    P = c["pts"].shape[0]
    for bad in (c["alb"][:600], c["alb"].repeat(4, 1), torch.ones(P, 4, device=d)):
        with pytest.raises(RuntimeError, match="albedo"):
            render_points(c["pts"], c["nrm"], bad, c["proj"], c["view"], h, prm, **kw)
    with pytest.raises(RuntimeError, match="grad_sync"):
        render_points(c["pts"], c["nrm"], c["alb"], c["proj"], c["view"], h, prm, grad_sync=GradSync(), **kw)
    # the right shape renders
    out = render_points(c["pts"], c["nrm"], c["alb"], c["proj"], c["view"], h, prm, **kw)
    assert torch.isfinite(out.image).all()
