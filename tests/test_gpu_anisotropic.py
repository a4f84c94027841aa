"""GPU tests of the anisotropic splat kernel (Vrk_invariant = Vrk_isotropic = false): dss_local_frames
(csrc/local_frames.cu) row by row against float64 on its own neighbour indices, the preprocess with frames slot by slot
against the bound of tests/test_local_frames.py, the render against the oracle and the float64 backward, the layers and
the training step."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import oracle
from dss_b200 import _lib
from dss_b200.core.camera import FoVPerspectiveCameras, camera_matrices, look_at_view_transform
from dss_b200.core.cloud import PointClouds3D, PointCloudsFilters
from dss_b200.core.rasterizer import PointsRasterizationSettings, SurfaceSplatting
from dss_b200.core.renderer import NormWeightedCompositor, SurfaceSplattingRenderer
from dss_b200.frnn_grid import knn_points_packed
from dss_b200.ops import SplatParams, local_frames, make_shading, point_filters, preprocess_points, render_points
from dss_b200.training.losses import ProjectionLoss, image_loss
from dss_b200.training.step import GraphedTrainStep, TrainStep
from dss_b200.utils.io import read_ply
from tests.test_local_frames import ANISO_FAMILIES, aniso_bound, aniso_family, slots
from tests.test_preprocess_bound import kept_mask, ratios
from tests.util import assert_fragments_exact, render_backward_f64_of, scene, sphere_cloud

pytestmark = pytest.mark.gpu

U = 2.0 ** -24


def _np(t):
    return t.detach().cpu().numpy()


# ---- 1. dss_local_frames against float64 ---------------------------------------------------------------------------
def frames_check(pts, fr, idx, first=None, num=None):
    """rows of `fr` against the float64 eigenproblem of the covariance of the neighbours `idx` names (the kernel's own
    K-NN): λ1, λ2 within 1.25 u λ2 on every row (the one rounding to float32, at most u |λ|, and float64's noise), and
    where λ1 - λ0 >= 2^-20 λ2 the rebuilt Vr within 4 u λ2 (three roundings per term) and |det(F^T J)| within
    16 u (1 + λ2 / (λ1 - λ0)) |J0| |J1| for random J.  A float32 solve misses the λ bound by 3x.  Rows with a -1
    neighbour must be all NaN, the others finite.  Returns the number of rows checked against the tight bounds."""
    pts, fr, idx = np.asarray(pts, np.float64), _np(fr).astype(np.float64), _np(idx)
    P = pts.shape[0]
    base = np.zeros(P, np.int64)
    if first is not None:
        for f, m in zip(_np(first), _np(num)):
            base[f:f + m] = f
    missing = (idx < 0).any(1)
    assert np.isnan(fr[missing]).all() and np.isfinite(fr[~missing]).all()
    rows = np.nonzero(~missing)[0]
    nb = pts[base[rows, None] + idx[rows]]
    D = nb - nb.mean(1, keepdims=True)
    C = np.einsum("pki,pkj->pij", D, D) / 8
    lam, vec = np.linalg.eigh(C)
    l2 = np.maximum(np.abs(lam[:, 2]), 1e-300)
    good = lam[:, 1] - lam[:, 0] >= 2.0 ** -20 * lam[:, 2]
    g = fr[rows]
    el = np.maximum(np.abs(g[:, 3] - lam[:, 1]), np.abs(g[:, 7] - lam[:, 2])) / (U * l2)
    assert (el <= 1.25).all(), float(el.max())
    Vr = (g[:, 3, None, None] * g[:, 0:3, None] * g[:, None, 0:3] + g[:, 7, None, None] * g[:, 4:7, None] * g[:, None, 4:7])
    want = np.einsum("pia,pa,pja->pij", vec[:, :, 1:], lam[:, 1:], vec[:, :, 1:])
    err = np.abs(Vr - want).max((1, 2))
    assert (err <= 4 * U * l2)[good].all(), float((err / l2)[good].max() / U)
    J = np.random.default_rng(0).normal(size=(rows.size, 3, 2))
    det = np.abs(np.linalg.det(np.einsum("pia,pib->pab", np.stack([g[:, 0:3], g[:, 4:7]], 2), J)))
    wdet = np.abs(np.linalg.det(np.einsum("pia,pib->pab", vec[:, :, 1:], J)))
    nJ = np.linalg.norm(J[:, :, 0], axis=1) * np.linalg.norm(J[:, :, 1], axis=1)
    with np.errstate(all="ignore"):
        cond = 1 + lam[:, 2] / (lam[:, 1] - lam[:, 0])
    assert (np.abs(det - wdet) <= 16 * U * cond * nJ)[good].all()
    return int(good.sum())


def knn_of(pts_t, first=None, num=None):
    if first is None:
        first = torch.zeros(1, dtype=torch.int64, device=pts_t.device)
        num = torch.full((1,), pts_t.shape[0], dtype=torch.int64, device=pts_t.device)
    return knn_points_packed(pts_t, first, num, 8, -1.0)[1]


def frame_cloud(name, dev):
    if name == "bunny":
        pts = read_ply(os.path.join(os.path.dirname(__file__), "golden", "ply", "bunny-8000.ply"))["points"]
        return torch.as_tensor(np.asarray(pts, np.float32)).to(dev)
    kind, _, arg = name.partition("/")
    rng = np.random.default_rng(7)
    if kind == "sphere":
        return sphere_cloud(int(arg), seed=3)[0].to(dev)
    if kind == "plane":   # λ0 = 0 exactly: z = 0
        xy = rng.uniform(-0.5, 0.5, (20000, 2))
        return torch.as_tensor(np.concatenate([xy, np.zeros((20000, 1))], 1), dtype=torch.float32).to(dev)
    if kind == "ellipsoid":
        return (sphere_cloud(20000, seed=4)[0] * torch.tensor([1.0, 0.2, 0.02])).to(dev)
    if kind == "scale":
        return (sphere_cloud(20000, seed=5)[0] * float(arg)).to(dev)
    if kind == "odd":   # not a multiple of the block size
        return sphere_cloud(5003, seed=6)[0].to(dev)
    raise ValueError(name)


@pytest.mark.parametrize("name", ["bunny", "sphere/5000", "sphere/100000", "sphere/1000000", "plane", "ellipsoid",
                                  "scale/1e-3", "scale/1e3", "odd"])
def test_local_frames_match_float64(cuda_device, name):
    pts = frame_cloud(name, cuda_device)
    fr = local_frames(pts)
    idx = knn_of(pts)
    n = frames_check(_np(pts), fr, idx)
    assert n >= 0.5 * pts.shape[0]
    assert torch.equal(local_frames(pts), fr)       # same bits on every run
    print("%s: %d of %d rows checked against float64" % (name, n, pts.shape[0]))


def test_local_frames_degenerate_rows(cuda_device):
    """collinear neighbours (λ0 = λ1) along an axis and along a general direction (float32-rounded, so only nearly
    collinear) and clusters of duplicates (all λ = 0): finite, deterministic, the documented frame; for all λ = 0 the
    radii are the antialiasing-only radii"""
    d = cuda_device
    line = torch.zeros(40, 3)
    line[:, 0] = torch.arange(40) * 0.01
    dup = torch.full((30, 3), 0.25)
    other = sphere_cloud(200, seed=9)[0] + 3.0
    pts = torch.cat([line, dup, other]).to(d)
    fr = local_frames(pts)
    assert torch.isfinite(fr).all() and torch.equal(local_frames(pts), fr)
    e = lambda *v: torch.tensor(v, device=d).expand(fr.shape[0], 3)
    assert torch.equal(fr[:40, 4:7], e(1.0, 0, 0)[:40]) and torch.equal(fr[:40, 0:3], e(0, 0, 1.0)[:40])
    assert (fr[:40, 3] == 0).all() and (fr[:40, 7] > 0).all()
    assert (fr[40:70, [3, 7]] == 0).all()
    assert torch.equal(fr[40:70, 4:7], e(1.0, 0, 0)[:30]) and torch.equal(fr[40:70, 0:3], e(0, 0, 1.0)[:30])
    # a line in a general direction, rounded to float32: nearly collinear neighbourhoods (λ1 - λ0 <= 3e-13 λ2 in
    # float64, 2^-40 = 9e-13), where the Jacobi sweeps do rotate; f2 along the line, f1 by the rule from f2
    dirn = torch.tensor([1.0, 2.0, 3.0], dtype=torch.float64) / 14 ** 0.5
    oblique = (torch.tensor([-0.3, 0.2, 0.05], dtype=torch.float64) + (0.1 + 0.01 * torch.arange(40.0))[:, None] * dirn)
    pts2 = torch.cat([oblique.float(), other]).to(d)
    fr2 = local_frames(pts2)
    assert torch.isfinite(fr2).all() and torch.equal(local_frames(pts2), fr2)
    idx2 = _np(knn_of(pts2))[:40]
    nb = _np(pts2).astype(np.float64)[idx2]
    D = nb - nb.mean(1, keepdims=True)
    lam = np.linalg.eigvalsh(np.einsum("pki,pkj->pij", D, D) / 8)
    assert ((lam[:, 1] - lam[:, 0]) <= 2.0 ** -41 * lam[:, 2]).all()        # inside the degenerate rule, 2x margin
    g2 = _np(fr2[:40]).astype(np.float64)
    f2 = g2[:, 4:7]
    assert (np.abs(f2 @ dirn.numpy()) >= 1 - 1e-6).all()
    k = np.argmin(np.abs(f2), axis=1)
    rule = np.cross(f2, np.eye(3)[k])
    rule /= np.linalg.norm(rule, axis=1, keepdims=True)
    assert np.abs(g2[:, 0:3] - rule).max() <= 4 * U, np.abs(g2[:, 0:3] - rule).max()
    assert (np.abs(g2[:, 3]) <= 2.0 ** -38 * g2[:, 7]).all()
    # all λ = 0: G = aa I, as for the isotropic kernel with h = 0
    _, _, _, proj, view, _ = scene(10, 2, seed=1)
    proj, view = proj.to(d), view.to(d)
    prm = SplatParams(image_size=128, znear=0.1)
    nrm = torch.nn.functional.normalize(torch.randn(pts.shape, generator=torch.Generator().manual_seed(0)), dim=1).to(d)
    a = preprocess_points(pts, nrm, proj, view, None, prm, frames=fr)
    b = preprocess_points(pts, nrm, proj, view, torch.zeros(2 * pts.shape[0], device=d), prm)
    rows = torch.cat([torch.arange(40, 70), torch.arange(40, 70) + pts.shape[0]]).to(d)
    assert torch.equal(a["radii"][rows], b["radii"][rows]) and torch.equal(a["ellipse_params"][rows],
                                                                          b["ellipse_params"][rows])


def test_local_frames_packed_ragged_and_nan(cuda_device):
    """packed ragged clouds (one of exactly 9 points, one of fewer than 8: NaN rows) equal the clouds one by one; a NaN
    point gets a NaN row and is nobody's neighbour"""
    d = cuda_device
    sizes = [9, 5, 3001, 1234]
    parts = [sphere_cloud(m, seed=20 + i)[0] * (1 + i) for i, m in enumerate(sizes)]
    parts[3][17] = float("nan")
    pts = torch.cat(parts).to(d)
    num = torch.tensor(sizes, dtype=torch.int64, device=d)
    first = torch.cumsum(num, 0) - num
    fr = local_frames(pts, first, num)
    idx = knn_of(pts, first, num)
    frames_check(_np(pts), fr, idx, first, num)
    assert torch.isnan(fr[9:14]).all() and torch.isnan(fr[int(first[3]) + 17]).all()
    for i, m in enumerate(sizes):
        f0 = int(first[i])
        if m > 8 and i != 3:
            assert torch.equal(local_frames(pts[f0:f0 + m]), fr[f0:f0 + m]), i
    with pytest.raises(ValueError):
        local_frames(pts[:8])


# ---- 2. the preprocess with frames against the float64 bound ---------------------------------------------------------
def _preprocess_case(f, dev, backface=False, views=None):
    """the preprocess with frames of a shared cloud, its float64 values and bound -> (got, want, bound, kept slots).
    The (P0,8) frames are the first rows of an (N*P0,8) buffer whose other rows are NaN: a kernel that read view n's
    record at the packed slot n*P0 + i instead of the point's row i reads valid memory and breaks the bound."""
    pts = torch.as_tensor(f["pts"]).to(dev)
    fr = local_frames(pts)
    proj, view = torch.as_tensor(f["proj"]), torch.as_tensor(f["view"])
    if views is not None:
        proj, view = proj[torch.arange(views) % proj.shape[0]], view[torch.arange(views) % view.shape[0]]
    N, P0 = proj.shape[0], pts.shape[0]
    buf = torch.full((N * P0, 8), float("nan"), device=dev)
    buf[:P0] = fr
    prm = SplatParams(image_size=f["S"], cutoff_threshold=f["cutoff"], antialiasing_sigma=f["sigma"], znear=f["znear"],
                      zfar=f["zfar"], backface_culling=backface)
    nrm = torch.nn.functional.normalize(pts, dim=1)
    out = preprocess_points(pts, nrm, proj.to(dev), view.to(dev), None, prm, frames=buf[:P0])
    g = {"x": out["ndc"][:, 0], "y": out["ndc"][:, 1], "z": out["ndc"][:, 2], "rx": out["radii"][:, 0],
         "ry": out["radii"][:, 1], "a": out["ellipse_params"][:, 0], "b": out["ellipse_params"][:, 1],
         "c": out["ellipse_params"][:, 2], "scaler": out["scaler"]}
    g = {k: _np(v).astype(np.float64) for k, v in g.items()}
    ff = dict(f, proj=_np(proj), view=_np(view))
    p, frs, vidx = slots(ff, _np(fr))
    want, bnd = aniso_bound(ff["proj"], ff["view"], p, frs, vidx, f["cutoff"], f["sigma"], f["S"])
    keep = kept_mask(want, f)
    if backface:
        # view-space normal z away from 0 (the kernel's float32 sign decides at 0)
        nz = np.einsum("pk,pk->p", np.tile(_np(nrm), (ff["proj"].shape[0], 1)).astype(np.float64),
                       ff["view"][vidx, :3, 2].astype(np.float64))
        assert (g["z"][keep & (nz > 1e-5)] == -1).all()
        keep &= nz < -1e-5
    return g, want, bnd, keep


@pytest.mark.parametrize("name", ANISO_FAMILIES + ["backface", "views/256"])
def test_preprocess_with_frames_meets_the_bound(cuda_device, name):
    backface = name == "backface"
    views = 256 if name == "views/256" else None
    f = aniso_family("sphere" if name in ("backface", "views/256") else name)
    g, want, bnd, keep = _preprocess_case(f, cuda_device, backface, views)
    assert keep.sum() > 1000
    r = ratios(g, want, bnd, keep)
    print(name, {k: "%.3g" % v[0] for k, v in r.items()})
    for k, (worst, over) in r.items():
        assert over == 0, (name, k, worst, over)


def _near_plane_cloud(P0, seed):
    """points just past znear = 0.1 and far off to the side of the view axis (huge splats, centres at |ndc| >> 1),
    with an ordinary cloud behind them; two cameras looking down +z from slightly different places"""
    g = torch.Generator().manual_seed(seed)
    m = P0 // 3
    z_near = 0.1 + torch.rand(m, generator=g) * 0.05
    xy_near = (torch.rand(m, 2, generator=g) * 2 - 1) * z_near[:, None] * 4.0
    z_far = 1.0 + torch.rand(P0 - m, generator=g)
    xy_far = (torch.rand(P0 - m, 2, generator=g) * 2 - 1) * z_far[:, None] * 0.6
    pts = torch.cat([torch.cat([xy_near, z_near[:, None]], 1), torch.cat([xy_far, z_far[:, None]], 1)]).contiguous()
    R = torch.eye(3).repeat(2, 1, 1)
    T = torch.tensor([[0.0, 0.0, 0.0], [0.01, -0.005, 0.0]])
    proj, view = camera_matrices(FoVPerspectiveCameras(znear=0.1, zfar=100.0, R=R, T=T))
    return pts, proj, view


def test_preprocess_with_frames_near_plane(cuda_device):
    pts, proj, view = _near_plane_cloud(3000, 0)
    f = dict(pts=_np(pts).astype(np.float32), proj=_np(proj).astype(np.float32), view=_np(view).astype(np.float32),
             S=128, cutoff=1.0, sigma=1.0, znear=0.1, zfar=100.0)
    g, want, bnd, keep = _preprocess_case(f, cuda_device)
    assert keep.sum() > 100
    r = ratios(g, want, bnd, keep)
    print("near plane", {k: "%.3g" % v[0] for k, v in r.items()})
    for k, (worst, over) in r.items():
        assert over == 0, (k, worst, over)


def test_preprocess_refuses_h_with_frames(cuda_device):
    d = cuda_device
    pts, nrm, _, proj, view, _ = scene(100, 2, seed=2)
    pts, nrm, proj, view = pts.to(d), nrm.to(d), proj.to(d), view.to(d)
    fr = local_frames(pts)
    with pytest.raises(RuntimeError, match="exactly one of h"):
        preprocess_points(pts, nrm, proj, view, torch.full((2,), 1e-3, device=d), SplatParams(), frames=fr)
    with pytest.raises(RuntimeError, match="frames must have shape"):
        preprocess_points(pts, nrm, proj, view, None, SplatParams(), frames=fr[:50])


# ---- 3. the render: fragments against the oracle, backward against float64 -------------------------------------------
@pytest.mark.parametrize("shade", [False, True])
def test_render_with_frames_matches_oracle_and_float64_backward(cuda_device, shade):
    d = cuda_device
    P0, N, S, K = 20000, 3, 128, 5
    pts, nrm, col, proj, view, cams = scene(P0, N, seed=31)
    pts, nrm, col, proj, view = pts.to(d), nrm.to(d), col.to(d), proj.to(d), view.to(d)
    prm = SplatParams(image_size=S, points_per_pixel=K, cutoff_threshold=0.5, znear=0.1, clip_pts_grad=0.05,
                      radii_backward_scaler=5.0)
    fr = local_frames(pts)
    p = pts.clone().requires_grad_(True)
    n = nrm.clone().requires_grad_(True)
    c = col.clone().requires_grad_(True)
    shading = None
    if shade:
        from dss_b200.core.lighting import DirectionalLights
        lights = DirectionalLights(direction=torch.tensor([[0.3, -0.5, 1.0]]), device=d)
        shading = make_shading(lights, view)
    out = render_points(p, n, c if shade else c.repeat(N, 1), proj, view, None, prm, return_fragments=True,
                        shading=shading, frames=fr)
    rec = _np(out.records)
    first = np.arange(N, dtype=np.int64) * P0
    num = np.full(N, P0, np.int64)
    want = oracle.splat_points_binned(np.ascontiguousarray(rec[:, :3]), np.ascontiguousarray(rec[:, 5:8]),
                                      np.full(N * P0, 0.5, np.float32), np.ascontiguousarray(rec[:, 3:5]), first, num,
                                      prm.depth_merging_threshold, S, K, 16, fma_mode=1)
    rim, same = assert_fragments_exact((out.idx, out.zbuf, out.qvalue, out.image[..., 3]), want,
                                       np.full(N * P0, 0.5, np.float32))
    assert same.mean() > 0.999
    gi = (torch.randn(N, S, S, 4, generator=torch.Generator().manual_seed(3)) * 1e-3).to(d)
    out.image.backward(gi)
    if not shade:
        # the position and colour gradients against the float64 backward on the forward's own fragments
        ref = render_backward_f64_of(out, pts, proj, view, prm, gi)
        wrow = ref["world"]
        scale = np.abs(wrow).max()
        gp = _np(p.grad).astype(np.float64)
        assert scale > 0 and np.abs(gp - wrow).max() <= 2e-4 * scale, (np.abs(gp - wrow).max(), scale)
        np.testing.assert_allclose(_np(c.grad), ref["colours"].reshape(N, P0, 3).sum(0), rtol=2e-4, atol=1e-7)
        assert n.grad is None                        # without shading the normals get nothing
    else:
        # the normals' gradient is the shading's alone (the frames are constants): zero wherever no view's colour
        # gradient reached the point
        assert n.grad is not None and torch.isfinite(n.grad).all() and n.grad.abs().sum() > 0
        reached = (out.visible.view(N, P0) != 0).any(0)
        assert (n.grad[~reached] == 0).all()
    print("anisotropic render (shade=%s): %d rim pixels" % (shade, rim))


# ---- 4. the layers --------------------------------------------------------------------------------------------------
def _default_yaml_renderer(dev, S=96, N=3):
    R, T = look_at_view_transform(dist=[1.5, 1.8, 2.1][:N], elev=[10, -30, 60][:N], azim=[0, 120, -70][:N])
    cams = FoVPerspectiveCameras(znear=0.1, zfar=100.0, R=R, T=T, device=dev)
    # configs/default.yaml:20-30 (image size reduced)
    settings = PointsRasterizationSettings(backface_culling=False, Vrk_isotropic=False, bin_size=None,
                                           clip_pts_grad=0.05, cutoff_threshold=0.5, depth_merging_threshold=0.05,
                                           image_size=S, max_points_per_bin=None, points_per_pixel=5,
                                           radii_backward_scaler=5)
    rast = SurfaceSplatting(cameras=cams, raster_settings=settings)
    return cams, rast, SurfaceSplattingRenderer(rast, NormWeightedCompositor())


def test_renderer_with_default_yaml_settings_fused_matches_unfused(cuda_device):
    d = cuda_device
    cams, rast, renderer = _default_yaml_renderer(d)
    pts, nrm, col = (t.to(d) for t in sphere_cloud(6000, seed=8))
    N = len(cams)
    g = torch.randn(N, 96, 96, 4, generator=torch.Generator().manual_seed(1)).to(d) * 1e-3

    def run(fused):
        p = pts.clone().requires_grad_(True)
        c = col.clone().requires_grad_(True)
        img = renderer(PointClouds3D([p], normals=[nrm], features=[c]), cameras=cams, fused=fused)
        img.backward(g)
        return img.detach(), p.grad.clone(), c.grad.clone()

    img_f, gp_f, gc_f = run(True)
    img_u, gp_u, gc_u = run(False)
    assert img_f.shape == (N, 96, 96, 4) and img_f[..., 3].sum() > 0
    assert torch.equal(img_f[..., 3], img_u[..., 3])
    assert float(((img_f - img_u) ** 2).mean()) < 1e-10
    torch.testing.assert_close(gc_f, gc_u, rtol=2e-4, atol=1e-8)
    scale = gp_u.abs().max()
    assert scale > 0 and (gp_f - gp_u).abs().max() <= 2e-4 * scale
    # packed clouds of different sizes take the packed route with per-cloud frames
    parts = [sphere_cloud(m, seed=40 + i) for i, m in enumerate((3000, 2000, 4000))]
    cloud = PointClouds3D([q[0].to(d) for q in parts], normals=[q[1].to(d) for q in parts],
                          features=[q[2].to(d) for q in parts])
    a, b = renderer(cloud, cameras=cams, fused=True), renderer(cloud, cameras=cams, fused=False)
    assert torch.equal(a[..., 3], b[..., 3]) and float(((a - b) ** 2).mean()) < 1e-10
    small = PointClouds3D([pts[:8]], normals=[nrm[:8]], features=[col[:8]])
    for fused in (True, False):
        with pytest.raises(ValueError):
            renderer(small, cameras=cams, fused=fused)


# ---- 5. the training step -------------------------------------------------------------------------------------------
def _batch(N, S, dev, seed):
    from dss_b200.core.lighting import DirectionalLights
    _, _, _, proj, view, _ = scene(10, N, seed=seed)
    g = torch.Generator().manual_seed(seed)
    img = torch.rand(N, S, S, 3, generator=g).to(dev)
    mask = (F.interpolate(torch.rand(N, 1, 16, 16, generator=g), size=(S, S), mode="bilinear")[:, 0] > 0.5).float()
    lights = DirectionalLights(ambient_color=0.2 * torch.rand(N, 1, 3, generator=g),
                               diffuse_color=0.5 * torch.rand(N, 1, 3, generator=g),
                               specular_color=0.1 * torch.rand(N, 1, 3, generator=g),
                               direction=torch.randn(N, 1, 3, generator=g), device=dev)
    return img, mask.to(dev), proj.to(dev), view.to(dev), lights


def test_anisotropic_train_step_equals_the_composition(cuda_device):
    d = cuda_device
    P0, N, S = 20000, 4, 128
    pts, nrm, col, _, _, _ = scene(P0, N, seed=61)
    pts, nrm, col = pts.to(d), nrm.to(d), col.to(d)
    prm = SplatParams(image_size=S, points_per_pixel=5, cutoff_threshold=0.5, znear=0.1, clip_pts_grad=0.05,
                      radii_backward_scaler=5.0)
    img, mask, proj, view, lights = _batch(N, S, d, seed=62)
    step = TrainStep(pts, nrm, col, prm, Vrk_invariant=False, Vrk_isotropic=False, lambda_dr_proj=0.01)
    assert step.settings()[2] is False
    loss = step(img, mask, proj, view, lights)
    # the composition: local_frames -> render_points -> image_loss -> point_filters -> regularisers
    p = pts.detach().clone().requires_grad_(True)
    n = nrm.detach().clone().requires_grad_(True)
    normals = F.normalize(n, dim=-1)
    out = render_points(p, normals, col, proj, view, None, prm, shading=make_shading(lights, view),
                        frames=local_frames(p))
    il = image_loss(out.image, img, mask, 1.0, 1.0)
    vis, inm = point_filters(out, mask)
    cloud = PointClouds3D([p], [normals])
    filt = PointCloudsFilters(d, visibility=vis[None], inmask=inm[None])
    lp = ProjectionLoss(reduction="mean", knn_k=12, filter_scale=2.0, sharpness_sigma=0.75)(
        cloud, rebuild_knn=True, points_filter=filt) * 0.01
    total = lp + torch.zeros((), device=d) + il["loss"]
    total.backward()
    assert torch.equal(step.image, out.image.detach()) and torch.equal(step.visibility, vis)
    assert torch.equal(step.inmask, inm)
    assert torch.equal(loss["loss"], total.detach()) and torch.equal(loss["loss_dr_proj"], lp.detach())
    torch.testing.assert_close(step.points.grad, p.grad, rtol=1e-4, atol=1e-9)
    torch.testing.assert_close(step.normals.grad, n.grad, rtol=1e-4, atol=1e-9)
    # launches: the K = 8 search replaces the K = 7 one, and the frames kernel is added
    inv = TrainStep(pts, nrm, col, prm, lambda_dr_proj=0.01)
    counts = []
    for s in (inv, step):
        s(img, mask, proj, view, lights)
        torch.cuda.synchronize()
        c0 = _lib.launch_count()
        s(img, mask, proj, view, lights)
        torch.cuda.synchronize()
        counts.append(_lib.launch_count() - c0)
    print("library launches per step: invariant %d, anisotropic %d" % tuple(counts))
    assert counts[1] == counts[0] + 1
    with pytest.raises(ValueError):
        TrainStep(pts[:8], nrm[:8], col[:8], prm, Vrk_invariant=False, Vrk_isotropic=False)


def test_anisotropic_graphed_train_step_replays_the_eager_step(cuda_device):
    d = cuda_device
    P0, N, S = 20000, 4, 128
    pts, nrm, col, _, _, _ = scene(P0, N, seed=71)
    pts, nrm, col = pts.to(d), nrm.to(d), col.to(d)
    prm = SplatParams(image_size=S, points_per_pixel=5, cutoff_threshold=0.5, znear=0.1, clip_pts_grad=0.05,
                      radii_backward_scaler=5.0)
    a, b = _batch(N, S, d, seed=72), _batch(N, S, d, seed=73)
    kw = dict(Vrk_invariant=False, Vrk_isotropic=False, lambda_dr_repel=0.05)
    eager = TrainStep(pts, nrm, col, prm, **kw)
    keep = lambda s: ({k: v.clone() for k, v in s.loss.items()}, s.image.clone(), s.visibility.clone(),
                      s.inmask.clone(), s.points.grad.clone(), s.normals.grad.clone())
    eager(*a)
    want_a = keep(eager)
    eager(*b)
    want_b = keep(eager)
    step = GraphedTrainStep(pts, nrm, col, prm, *a, **kw)

    def check(want):
        step.replay()
        torch.cuda.synchronize()
        loss, image, vis, inm, gp, gn = want
        assert torch.equal(step.image, image) and torch.equal(step.visibility, vis) and torch.equal(step.inmask, inm)
        for k in loss:
            assert torch.equal(step.loss[k], loss[k]), k
        torch.testing.assert_close(step.points.grad, gp, rtol=1e-4, atol=1e-9)
        torch.testing.assert_close(step.normals.grad, gn, rtol=1e-4, atol=1e-9)

    check(want_a)
    step.load(*b)
    check(want_b)
    print("anisotropic graphed train step: %d kernel nodes per replay" % step.kernel_nodes())


# ---- 6. the view-sharded anisotropic step ----------------------------------------------------------------------------
_SHARDED_WORKER = r'''
import os, sys, torch, torch.distributed as dist
rank, out_dir, port = int(sys.argv[1]), sys.argv[2], int(sys.argv[3])
dev = torch.device("cuda", 0)
torch.cuda.set_device(dev)
dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%d" % port, rank=rank, world_size=2)
# every collective the step issues goes through torch.distributed.all_reduce: count them
n_reduce = [0]
_all_reduce = dist.all_reduce
def counted(*a, **k):
    n_reduce[0] += 1
    return _all_reduce(*a, **k)
dist.all_reduce = counted
from dss_b200 import _lib
from dss_b200.core.lighting import DirectionalLights
from dss_b200.ops import SplatParams, local_frames, render_points
from dss_b200.parallel import GradSync, assign_views, view_costs_from_cameras
from dss_b200.training.step import TrainStep
from dss_b200.utils.io import read_ply
from tests.util import GOLDEN_DIR, camera_matrices, random_cameras

ply = read_ply(os.path.join(GOLDEN_DIR, "ply", "bunny-8000.ply"))
pts = torch.as_tensor(ply["points"], dtype=torch.float32)
pts = (pts - pts.mean(0)) / (pts - pts.mean(0)).norm(dim=1).max() * 0.6
nrm = torch.nn.functional.normalize(torch.as_tensor(ply["normals"], dtype=torch.float32), dim=1)
col = torch.rand(pts.shape, generator=torch.Generator().manual_seed(3))
pts, nrm, col = pts.to(dev), nrm.to(dev), col.to(dev)
S = 256
prm = SplatParams(image_size=S, points_per_pixel=5, cutoff_threshold=0.5, depth_merging_threshold=0.05,
                  radii_backward_scaler=5.0, clip_pts_grad=0.05, znear=0.1)
ANISO = dict(Vrk_invariant=False, Vrk_isotropic=False)
F32 = torch.finfo(torch.float32).eps


def make_batch(N, seed):
    proj, view = (m.to(dev) for m in camera_matrices(random_cameras(N, seed, dist=(1.6, 2.2))))
    g = torch.Generator().manual_seed(seed)
    rows = [0.2 * torch.rand(1, 1, 3, generator=g), 0.5 * torch.rand(1, 1, 3, generator=g),
            0.1 * torch.rand(1, 1, 3, generator=g), torch.randn(1, 1, 3, generator=g)]
    with torch.no_grad():
        tgt = render_points(pts + 0.01 * torch.randn(3, generator=g).to(dev), nrm, col.flip(1), proj, view,
                            torch.full((N,), 1e-3, device=dev), prm).image
    lights = DirectionalLights(ambient_color=rows[0], diffuse_color=rows[1], specular_color=rows[2],
                               direction=rows[3], device=dev)
    return tgt[..., :3].contiguous(), (tgt[..., 3] > 0).float(), proj, view, lights


def views_of(batch, views):
    img, mask, proj, view, lights = batch
    idx = torch.tensor(list(views), dtype=torch.long, device=dev)
    return img[idx], mask[idx], proj[idx], view[idx], lights


saved, report = {}, []
saved["frames"] = {"frames": local_frames(pts).cpu()}
for name, N, seed in (("N=8", 8, 21), ("N=1", 1, 22)):
    batch = make_batch(N, seed)
    mine = assign_views(view_costs_from_cameras(batch[3]).tolist(), 2)[rank]
    single = TrainStep(pts, nrm, col, prm, lambda_dr_repel=0.05, **ANISO)
    single(*views_of(batch, range(N)))
    sharded = TrainStep(pts, nrm, col, prm, grad_sync=GradSync(), lambda_dr_repel=0.05, **ANISO)
    sharded(*views_of(batch, mine))
    torch.cuda.synchronize()
    assert torch.equal(sharded.visibility, single.visibility) and torch.equal(sharded.inmask, single.inmask), name
    assert single.inmask.any(), name
    if mine:
        assert torch.equal(sharded.image, single.image[torch.tensor(mine, device=dev)]), name
    for k, v in single.loss.items():
        w, got = float(v), float(sharded.loss[k])
        tol = 0.0 if k in ("loss_dr_proj", "loss_dr_repel") else 4 * F32 * abs(w)
        assert abs(got - w) <= tol, (name, k, got, w)
    worst = []
    for got, want in ((sharded.points.grad, single.points.grad), (sharded.normals.grad, single.normals.grad)):
        scale, err = float(want.abs().max()), float((got - want).abs().max())
        assert scale > 0 and err <= 1e-5 * scale, (name, err, scale)
        worst.append(err / scale)
    report.append("%s: views %s, d points / d normals within %.2e / %.2e of the largest" % (name, mine, *worst))
    saved[name] = {"loss": torch.stack([v.float() for v in sharded.loss.values()]).cpu(),
                   "vis": sharded.visibility.cpu(), "inm": sharded.inmask.cpu(),
                   "gp": sharded.points.grad.cpu(), "gn": sharded.normals.grad.cpu()}

# the anisotropic sharded step issues the collectives and library launches of the invariant one, plus the frames kernel
batch = make_batch(8, 23)
mine = assign_views(view_costs_from_cameras(batch[3]).tolist(), 2)[rank]
counts = {}
for mode, kw in (("invariant", {}), ("anisotropic", ANISO)):
    for sync in (None, GradSync()):
        st = TrainStep(pts, nrm, col, prm, grad_sync=sync, **kw)
        st(*views_of(batch, mine))
        torch.cuda.synchronize()
        n0, r0 = _lib.launch_count(dev), n_reduce[0]
        st(*views_of(batch, mine))
        torch.cuda.synchronize()
        counts[(mode, sync is not None)] = (_lib.launch_count(dev) - n0, n_reduce[0] - r0)
assert counts[("anisotropic", True)][1] == counts[("invariant", True)][1], counts
assert counts[("anisotropic", False)][1] == counts[("invariant", False)][1] == 0, counts
assert counts[("anisotropic", True)][0] == counts[("invariant", True)][0] + 1, counts
assert counts[("anisotropic", False)][0] == counts[("invariant", False)][0] + 1, counts
report.append("(library launches, all-reduces) per step on %d views: %s" % (len(mine), counts))
torch.save(saved, os.path.join(out_dir, "rank%d.pt" % rank))
dist.destroy_process_group()
print("\n".join(report))
print("rank", rank, "ok")
'''


def test_sharded_anisotropic_train_step_on_two_gloo_ranks(cuda_device):
    """TrainStep(..., Vrk_invariant=False, Vrk_isotropic=False, grad_sync=GradSync()) on 2 gloo ranks on one GPU
    against one anisotropic TrainStep over all the views (the bunny, 8 and 1 views, λ_repel > 0), at the tolerances of
    tests/test_gpu_train_step_sharded.py: filters, per-view render and regularisers bit for bit, the image-loss scalars
    within 4 float32 ulps, d points / d normals within 1e-5 of the largest.  Both ranks compute the same frames bits,
    end with the same bits, and the anisotropic step issues as many all-reduces as the invariant one."""
    import socket
    import subprocess
    import sys
    import tempfile
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    with tempfile.TemporaryDirectory() as d:
        w = os.path.join(d, "worker.py")
        with open(w, "w") as f:
            f.write(_SHARDED_WORKER)
        env = dict(os.environ, PYTHONPATH=root)
        procs = [subprocess.Popen([sys.executable, w, str(r), d, str(port)], stdout=subprocess.PIPE,
                                  stderr=subprocess.STDOUT, text=True, cwd=root, env=env) for r in range(2)]
        try:
            outs = [p.communicate(timeout=900)[0] for p in procs]
        finally:
            for p in procs:
                if p.poll() is None:
                    p.kill()
                    p.wait()
        for r, (p, o) in enumerate(zip(procs, outs)):
            assert p.returncode == 0 and "rank %d ok" % r in o, o
        print(outs[0])
        saved = [torch.load(os.path.join(d, "rank%d.pt" % r)) for r in range(2)]
    assert saved[0].keys() == saved[1].keys()
    for name in saved[0]:
        for k, t in saved[0][name].items():
            assert torch.equal(t, saved[1][name][k]), (name, k)
