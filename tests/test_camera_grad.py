"""Camera gradients, host side: the float64 closed form that dss_camera_backward evaluates (the gradient of the
pytorch3d transform of rasterizer.py:614 with respect to the full projection and the world-to-view matrix) against
torch autograd through SurfaceSplatting.transform, and the argument checks of the entry point (no device needed)."""
import ctypes as C

import torch

import dss_b200.core.rasterizer as rasterizer
from dss_b200 import _lib
from dss_b200.core.camera import camera_matrices
from dss_b200.core.cloud import PointClouds3D
from dss_b200.core.rasterizer import PointsRasterizationSettings, SurfaceSplatting
from tests.util import random_cameras, sphere_cloud


def camera_grads64(pts, proj, view, grad_ndc, first, num):
    """float64 (grad_proj, grad_view, |terms| sums of grad_proj, |terms| sums of grad_view) of the views' packed slots.
    pts: (P0,3) shared by every view (first is None) or packed (P,3) with view n at rows first[n] .. + num[n]."""
    N = proj.shape[0]
    f64 = dict(dtype=torch.float64, device=proj.device)
    gP, gV, aP, aV = (torch.zeros((N, 4, 4), **f64) for _ in range(4))
    P0 = pts.shape[0]
    for n in range(N):
        s0, cnt = (n * P0, P0) if first is None else (int(first[n]), int(num[n]))
        p = pts if first is None else pts[s0:s0 + cnt]
        ph = torch.cat([p.double(), torch.ones((cnt, 1), **f64)], 1)
        g = grad_ndc[s0:s0 + cnt].double()
        clip = ph @ proj[n].double()
        w = clip[:, 3]
        x, y = clip[:, 0] / w, clip[:, 1] / w
        dclip = torch.stack([g[:, 0] / w, g[:, 1] / w, torch.zeros_like(w), -(g[:, 0] * x + g[:, 1] * y) / w], 1)
        gP[n] = ph.t() @ dclip
        aP[n] = ph.abs().t() @ dclip.abs()
        gV[n, :, 2] = ph.t() @ g[:, 2]
        aV[n, :, 2] = ph.abs().t() @ g[:, 2].abs()
    return gP, gV, aP, aV


class _MatrixCameras:
    """just enough of a camera for SurfaceSplatting.transform once camera_matrices is bypassed"""

    def __init__(self, proj, view):
        self.proj, self.view = proj, view


def test_closed_form_equals_autograd_through_transform_float64(monkeypatch):
    N, P0 = 3, 400
    pts, nrm, _ = sphere_cloud(P0, seed=7)
    cams = random_cameras(N, seed=7)
    proj, view = camera_matrices(cams)
    proj64, view64 = proj.double().requires_grad_(True), view.double().requires_grad_(True)
    # camera_matrices returns float32 by contract; hand the float64 leaves straight to transform
    monkeypatch.setattr(rasterizer, "camera_matrices", lambda cameras, **kw: (cameras.proj, cameras.view))
    rast = SurfaceSplatting(cameras=_MatrixCameras(proj64, view64), raster_settings=PointsRasterizationSettings())
    for shared in (True, False):
        if shared:
            cloud, first, num, p_in = PointClouds3D([pts.double()], normals=[nrm.double()]).extend(N), None, None, pts
        else:
            sl = [slice(0, 400), slice(50, 300), slice(100, 350)]
            cloud = PointClouds3D([pts[s].double() for s in sl], normals=[nrm[s].double() for s in sl])
            first, num = cloud.cloud_to_packed_first_idx(), cloud.num_points_per_cloud()
            p_in = cloud.points_packed()
        screen = rast.transform(cloud)
        G = torch.randn(screen.shape, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
        gp, gv = torch.autograd.grad((screen * G).sum(), (proj64, view64))
        wP, wV, _, _ = camera_grads64(p_in, proj64.detach(), view64.detach(), G, first, num)
        torch.testing.assert_close(gp, wP, rtol=1e-12, atol=1e-12)
        torch.testing.assert_close(gv, wV, rtol=1e-12, atol=1e-12)
        assert (wP[:, :, 2] == 0).all() and (wV[:, :, [0, 1, 3]] == 0).all()


def test_closed_form_chains_to_R_and_T_like_autograd():
    """the fused route hands (grad_proj, grad_view) to autograd, which chains them through camera_matrices to R / T:
    that must equal autograd through the unfused transform end to end"""
    N, P0 = 3, 600
    pts, nrm, _ = sphere_cloud(P0, seed=8)
    cams = random_cameras(N, seed=8)
    cams.R.requires_grad_(True)
    cams.T.requires_grad_(True)
    rast = SurfaceSplatting(cameras=cams, raster_settings=PointsRasterizationSettings())
    cloud = PointClouds3D([pts], normals=[nrm]).extend(N)
    screen = rast.transform(cloud)
    G = torch.randn(screen.shape, generator=torch.Generator().manual_seed(2))
    gR, gT = torch.autograd.grad((screen * G).sum(), (cams.R, cams.T))
    proj, view = camera_matrices(cams)
    wP, wV, _, _ = camera_grads64(pts, proj.detach(), view.detach(), G, None, None)
    cR, cT = torch.autograd.grad((proj, view), (cams.R, cams.T), (wP.float(), wV.float()))
    for got, want in ((cR, gR), (cT, gT)):
        assert (got - want).abs().max() <= 1e-5 * want.abs().max(), (got, want)


def _args(**kw):
    a = _lib.RenderArgs()
    fake = C.c_void_p(256)          # never dereferenced: every case fails an argument check first
    for f in ("points_world", "proj", "view", "grad_ndc"):
        setattr(a, f, fake)
    a.n_views, a.shared_cloud, a.P0, a.P, a.image_size, a.points_per_pixel = 2, 1, 10, 20, 16, 5
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def test_camera_backward_rejects_bad_arguments_without_a_device():
    lib = _lib.load()
    out = C.c_void_p(512)
    null = C.c_void_p(0)

    def call(a, gp=out, gv=out, gc=null):
        rc = lib.dss_camera_backward(null, None if a is None else C.byref(a), gp, gv, gc, null)
        return rc, _lib.last_error()

    cases = [
        (None, {}, "args is null"),
        (_args(grad_ndc=null), {}, "grad_ndc"),
        (_args(), {"gp": null}, "grad_proj"),
        (_args(), {"gv": null}, "grad_view"),
        (_args(points_world=null), {}, "points_world"),
        (_args(proj=null), {}, "proj"),
        (_args(P=21), {}, "P != n_views * P0"),
        (_args(n_views=0), {}, "n_views"),
        (_args(shared_cloud=0), {}, "first_idx/num_points"),
        (_args(), {"gc": out}, "shade"),
        (_args(shade=1, n_lights=1), {"gc": out}, "shading needs"),
        (_args(shade=1, n_lights=1, albedo=out, lights=out, ambient=out, cam_centres=out, normals_world=out),
         {"gc": out}, "grad_colours"),
        (_args(), {}, "ctx is null"),           # consistent arguments: only the missing context is left
    ]
    for a, kw, msg in cases:
        rc, err = call(a, **kw)
        assert rc == -1 and msg in err, (msg, rc, err)
