"""The whole fused backward (dss_render_backward) against its float64 reference (tests/util.py render_backward_f64) on
the forward's own fragments, in the configurations the operator tests do not reach: packed clouds with ragged and empty
views and rows no view covers, per-splat h (the Vrk_isotropic layout), a z-buffer loss, K > 8 (the pixel-parallel
forward, whose blend epilogue counts the backward's binning cells too), a backward binning of more than 2^25 cells over
more than 96 views, filtered slots, and a staged-window hint left by a different call.

Each case checks the clipped NDC gradient the library writes (grad_ndc), the position gradient per packed row and the
point / colour gradients autograd returns."""
import numpy as np
import pytest
import torch

from dss_b200 import _lib
from dss_b200.core.camera import camera_matrices
from dss_b200.ops import SplatParams, render_points
from tests.util import (backward_via_lib, preprocess_f64_slots, random_cameras, render_backward_f64_of, scene,
                        sphere_cloud, view_ranges)

pytestmark = pytest.mark.gpu


def _np(t):
    return t.detach().cpu().numpy()


def _in_range(P, first, num):
    m = np.zeros(P, bool)
    for f, k in zip(first, num):
        m[f:f + k] = True
    return m


def _packed_layout(P0):
    """Four views over the world points 0..P0-1 of one cloud: ragged and overlapping ranges of the same points, one
    empty view, and packed rows of the world points P0..P0+149 that no view range covers.
    -> (world index of every packed row, first_idx, num_points)"""
    parts = [np.arange(0, 2 * P0 // 3), P0 + np.arange(100), np.arange(P0 // 4, P0), np.arange(P0 // 2, 2 * P0 // 3),
             P0 + 100 + np.arange(50)]
    rows = np.concatenate(parts)
    lens = [len(p) for p in parts]
    starts = np.concatenate([[0], np.cumsum(lens)[:-1]])
    # view 0 = part 0, view 1 = part 2, view 2 = empty (between parts 2 and 3), view 3 = part 3
    first = np.array([starts[0], starts[2], starts[3], starts[3]], np.int64)
    num = np.array([lens[0], lens[2], 0, lens[3]], np.int64)
    return rows, first, num


def _render_and_check(pts, nrm, col, proj, view, h, prm, first=None, num=None, zloss=False, seed=0, world_rows=None,
                      pts_leaf=None, check_records=True):
    """One forward with fragments, the autograd backward (image loss [+ z-buffer loss]) and the library backward with
    grad_ndc set, each checked against the float64 reference on the forward's own fragments.
    pts / col are the tensors render_points receives; pts_leaf / world_rows: the world leaf they were gathered from."""
    d = pts.device
    shared = first is None
    N, S, K = proj.shape[0], prm.image_size, prm.points_per_pixel
    fi = None if shared else torch.as_tensor(first).to(d)
    nm = None if shared else torch.as_tensor(num).to(d)
    col_leaf = col.detach().clone().requires_grad_(True)
    out = render_points(pts, nrm, col_leaf, proj, view, h, prm, first_idx=fi, num_points=nm, shared_cloud=shared,
                        return_fragments=True)
    gen = torch.Generator().manual_seed(seed)
    gi = (torch.randn(N, S, S, 4, generator=gen) * 1e-3).to(d)
    gz = (torch.randn(N, S, S, K, generator=gen) * 1e-3).to(d) if zloss else None
    torch.autograd.backward([out.image] + ([out.zbuf] if zloss else []), [gi] + ([gz] if zloss else []))
    grad_ndc, grad_rows, _ = backward_via_lib(out, pts.detach(), proj, view, fi, nm, shared, prm, gi, gz,
                                              repeat_camera=0)
    ref = render_backward_f64_of(out, pts, proj, view, prm, gi, gz, first, num)
    vis = _np(out.visible)
    in_range = _in_range(vis.shape[0], *view_ranges(N, pts.shape[0], first, num))
    # the forward: visibility as the reference defines it on its own idx, records against the float64 preprocess
    assert np.array_equal(vis, ref["vis"])
    assert vis.any(), "nothing rendered"
    rec = _np(out.records)
    if check_records:
        pre = preprocess_f64_slots(pts, nrm, proj, view, h, prm, first, num)
        kept = in_range & (rec[:, 2] != -1.0)
        np.testing.assert_allclose(rec[kept, :2], pre["ndc"][kept, :2], rtol=2e-5, atol=2e-6)
        np.testing.assert_allclose(rec[kept, 2], pre["ndc"][kept, 2], rtol=2e-5, atol=2e-6)
        np.testing.assert_allclose(rec[in_range, 3:5], pre["radii"][in_range], rtol=2e-4, atol=1e-7)
    # NDC gradient as the library writes it
    got, want = _np(grad_ndc).astype(np.float64), ref["ndc"]
    scale = np.abs(want).max()
    assert scale > 0 and np.abs(got).max() > 0
    err = np.abs(got - want).max()
    assert err <= 2e-5 * scale, (err, scale)
    assert np.linalg.norm(got - want, axis=1).max() <= 4 * ref["ndc_err32"].max() + 1e-6 * scale
    assert (got[vis == 0] == 0).all() and (got[~in_range] == 0).all()
    if zloss:
        assert np.abs(want[:, 2]).max() > 0
    # position gradient per packed row / per world point of a shared cloud
    wrow = ref["world"]
    wscale = np.abs(wrow).max()
    assert wscale > 0
    rows = _np(grad_rows).astype(np.float64)
    assert np.abs(rows - wrow).max() <= 2e-4 * wscale, (np.abs(rows - wrow).max(), wscale)
    if not shared:
        assert (rows[~in_range] == 0).all()
    # what autograd returns: to the leaf the rendered points were gathered from
    if pts_leaf is not None:
        want_leaf = np.zeros(tuple(pts_leaf.shape))
        np.add.at(want_leaf, world_rows, wrow)
        gl = _np(pts_leaf.grad).astype(np.float64)
        assert np.abs(gl - want_leaf).max() <= 2e-4 * wscale, (np.abs(gl - want_leaf).max(), wscale)
        if not shared:
            covered = np.zeros(pts_leaf.shape[0], bool)
            covered[world_rows[in_range]] = True
            assert (gl[~covered] == 0).all()
    wcol = ref["colours"]
    if tuple(col_leaf.shape) != tuple(wcol.shape):     # per-point colours of a shared cloud: summed over the views
        wcol = wcol.reshape(N, -1, 3).sum(0)
    assert np.abs(wcol).max() > 0
    np.testing.assert_allclose(_np(col_leaf.grad), wcol, rtol=2e-4, atol=1e-7)
    return out, ref, grad_ndc


def _packed_case(d, P0=6000, S=128, K=5, per_splat_h=False, clip=0.05, zloss=False, seed=31, **prm_kw):
    pts, nrm, col, proj, view, _ = scene(P0 + 150, 4, seed=seed)
    gen = np.random.default_rng(seed)
    rows, first, num = _packed_layout(P0)
    P = len(rows)
    h = torch.as_tensor(gen.uniform(1e-4, 6e-4, P).astype(np.float32)) if per_splat_h else torch.full((4,), 3e-4)
    prm = SplatParams(image_size=S, points_per_pixel=K, znear=prm_kw.pop("znear", 0.1), clip_pts_grad=clip,
                      **prm_kw)
    leaf = pts.to(d).requires_grad_(True)
    ridx = torch.as_tensor(rows).to(d)
    args = (leaf[ridx], nrm.to(d)[ridx], col.to(d)[ridx], proj.to(d), view.to(d), h.to(d), prm)
    return args, dict(first=first, num=num, zloss=zloss, seed=seed, world_rows=rows, pts_leaf=leaf)


# ---- packed clouds: ragged / empty / uncovered, per-view and per-splat h, clip on and off -----------------------
@pytest.mark.parametrize("clip", [0.05, -1.0])
@pytest.mark.parametrize("per_splat_h", [False, True])
def test_packed_ragged_views_match_float64(cuda_device, per_splat_h, clip):
    args, kw = _packed_case(cuda_device, per_splat_h=per_splat_h, clip=clip)
    _, ref, _ = _render_and_check(*args, **kw)
    nrm = np.linalg.norm(ref["ndc_raw"], axis=1)
    if clip > 0:   # the clip is active on some slots and not on others
        assert (nrm > clip).any() and ((nrm > 0) & (nrm < clip)).any()


# ---- shared cloud with per-splat h (Vrk_isotropic: h of length N * P0), and a non-power-of-two image -----------
@pytest.mark.parametrize("S", [128, 200])
def test_shared_cloud_per_splat_h_matches_float64(cuda_device, S):
    d = cuda_device
    P0, N = 8000, 3
    pts, nrm, col, proj, view, _ = scene(P0, N, seed=41)
    h = torch.as_tensor(np.random.default_rng(41).uniform(1e-4, 6e-4, P0).astype(np.float32)).repeat(N)
    prm = SplatParams(image_size=S, points_per_pixel=5, znear=0.1, clip_pts_grad=0.05)
    leaf = pts.to(d).requires_grad_(True)
    _render_and_check(leaf, nrm.to(d), col.to(d), proj.to(d), view.to(d), h.to(d), prm, seed=S,
                      world_rows=np.arange(P0), pts_leaf=leaf)


# ---- z-buffer loss through the fused path: packed and shared, clip on and off -----------------------------------
@pytest.mark.parametrize("clip", [0.05, -1.0])
@pytest.mark.parametrize("layout", ["packed", "shared"])
def test_zbuffer_loss_matches_float64(cuda_device, layout, clip):
    d = cuda_device
    if layout == "packed":
        args, kw = _packed_case(d, per_splat_h=True, clip=clip, zloss=True, seed=43)
        _render_and_check(*args, **kw)
        return
    P0, N = 8000, 3
    pts, nrm, col, proj, view, _ = scene(P0, N, seed=43)
    prm = SplatParams(image_size=128, points_per_pixel=5, znear=0.1, clip_pts_grad=clip)
    leaf = pts.to(d).requires_grad_(True)
    _render_and_check(leaf, nrm.to(d), col.to(d), proj.to(d), view.to(d), torch.full((N,), 3e-4, device=d), prm,
                      zloss=True, seed=44, world_rows=np.arange(P0), pts_leaf=leaf)


def _backward_launches(d, pts, nrm, col, proj, view, h, prm, first=None, num=None):
    """kernel launches of one autograd backward (image loss) through render_points"""
    shared = first is None
    fi = None if shared else torch.as_tensor(first).to(d)
    nm = None if shared else torch.as_tensor(num).to(d)
    out = render_points(pts.detach().requires_grad_(True), nrm, col, proj, view, h, prm, first_idx=fi, num_points=nm,
                        shared_cloud=shared)
    torch.cuda.synchronize(d)
    n0 = _lib.launch_count(d)
    out.image.backward(torch.ones_like(out.image))
    torch.cuda.synchronize(d)
    return _lib.launch_count(d) - n0


# ---- K > 8: the pixel-parallel forward counts the backward's binning cells like the sliced one (autograd's backward
#      takes those counts; dss_render_backward without them counts on its own), so its backward launches no more
#      kernels than at K = 5 --------------------------------------------------------------------------------------
@pytest.mark.parametrize("layout", ["packed", "shared"])
def test_k12_backward_takes_the_forward_cell_counts(cuda_device, layout):
    d = cuda_device
    if layout == "packed":
        args, kw = _packed_case(d, K=12, per_splat_h=True, clip=0.05, zloss=True, seed=47)
        _render_and_check(*args, **kw)
        launch_args, ranges = args[:6], dict(first=kw["first"], num=kw["num"])
    else:
        P0, N = 8000, 2
        pts, nrm, col, proj, view, _ = scene(P0, N, seed=47)
        prm = SplatParams(image_size=96, points_per_pixel=12, znear=0.1, clip_pts_grad=0.05)
        leaf = pts.to(d).requires_grad_(True)
        h = torch.full((N,), 3e-4, device=d)
        args = (leaf, nrm.to(d), col.to(d).repeat(N, 1), proj.to(d), view.to(d), h, prm)
        _render_and_check(*args, zloss=True, seed=48, world_rows=np.arange(P0), pts_leaf=leaf)
        launch_args, ranges = args[:6], {}
    prm = args[6]
    assert prm.points_per_pixel == 12
    k12 = _backward_launches(d, *launch_args, prm, **ranges)
    k5 = _backward_launches(d, *launch_args, prm._replace(points_per_pixel=5), **ranges)
    assert k12 == k5, (k12, k5)


# ---- 129 shared views at S = 512: a backward binning of N * 16^2 * 1024 > 2^25 cells, and views past the 96 whose
#      radii the staged-window hint reads, with search radii too large for the window it sizes ----------------------
def test_129_views_many_cells_and_unhinted_views(cuda_device):
    d = cuda_device
    P0, S = 300, 512
    pts, nrm, col = sphere_cloud(P0, seed=9)
    pa, va = camera_matrices(random_cameras(96, 9, dist=(2.6, 3.0)))
    pb, vb = camera_matrices(random_cameras(33, 10, dist=(1.0, 1.1)))     # views 97..129: close, large splats
    proj, view = torch.cat([pa, pb]).to(d), torch.cat([va, vb]).to(d)
    N = proj.shape[0]
    h = torch.as_tensor(np.random.default_rng(9).uniform(5e-5, 2e-4, P0).astype(np.float32)).repeat(N).to(d)
    prm = SplatParams(image_size=S, points_per_pixel=3, znear=0.1, clip_pts_grad=0.05)
    for it in range(2):   # the second call runs with the hint the first one left (the far views' radii)
        leaf = pts.to(d).requires_grad_(True)
        _, ref, _ = _render_and_check(leaf, nrm.to(d), col.to(d), proj, view, h, prm, seed=it, world_rows=np.arange(P0),
                                      pts_leaf=leaf, check_records=it == 0)
    # the views past the 96th need a larger window than the first 96 (so they cannot take the hinted one)
    px = ref["rs"] * S / 2
    assert px[96:].min() > 1.5 * px[:96].max(), px


# ---- filtered slots of a packed cloud: depth range inside the cloud, backface culling ---------------------------
@pytest.mark.parametrize("mode", ["znear", "backface"])
def test_packed_filtered_slots_get_zero_and_the_rest_match_float64(cuda_device, mode):
    d = cuda_device
    kw_prm = dict(znear=1.5) if mode == "znear" else dict(backface_culling=True)
    args, kw = _packed_case(d, per_splat_h=True, clip=0.05, zloss=True, seed=53, **kw_prm)
    out, ref, grad_ndc = _render_and_check(*args, **kw)
    rec = _np(out.records)
    first, num = kw["first"], kw["num"]
    in_range = _in_range(rec.shape[0], first, num)
    filt = in_range & (rec[:, 2] == -1.0)
    assert filt.sum() > 100 and (in_range & ~filt & (ref["vis"] == 1)).sum() > 100
    assert (_np(grad_ndc)[filt] == 0).all() and (ref["vis"][filt] == 0).all()
    assert (_np(kw["pts_leaf"].grad) != 0).any()
    # the filter itself, against float64 (away from the boundary)
    pts, nrm, proj, view = (_np(t) for t in (args[0], args[1], args[3], args[4]))
    zv = np.full(rec.shape[0], np.nan)
    nz = np.full(rec.shape[0], np.nan)
    for n, (f, m) in enumerate(zip(first, num)):
        zv[f:f + m] = pts[f:f + m].astype(np.float64) @ view[n, :3, 2] + view[n, 3, 2]
        nz[f:f + m] = nrm[f:f + m].astype(np.float64) @ view[n, :3, 2]
    if mode == "znear":
        want, margin = zv < 1.5, np.abs(zv - 1.5) > 1e-5
    else:
        want, margin = nz >= 0, np.abs(nz) > 1e-5
    sure = in_range & margin
    assert np.array_equal(filt[sure], want[sure])


# ---- history: the staged-window hint comes from the previous call ------------------------------------------------
@pytest.mark.parametrize("prev", ["small", "large"])
def test_result_matches_float64_after_a_call_that_moved_the_hint(cuda_device, prev):
    d = cuda_device
    # a call whose search radii are far smaller (or larger) than the case's: h = 1e-7 leaves the antialiasing
    # footprint only, h = 1e-2 gives splats of tens of pixels
    args, kw = _packed_case(d, per_splat_h=True, clip=0.05, seed=59)
    pts, nrm, col, proj, view, h, prm = args
    hp = torch.full_like(h, 1e-7 if prev == "small" else 1e-2)
    o = render_points(pts.detach(), nrm, col, proj, view, hp, prm, first_idx=torch.as_tensor(kw["first"]).to(d),
                      num_points=torch.as_tensor(kw["num"]).to(d), shared_cloud=False)
    backward_via_lib(o, pts.detach(), proj, view, torch.as_tensor(kw["first"]).to(d),
                     torch.as_tensor(kw["num"]).to(d), False, prm, torch.ones_like(o.image), None, repeat_camera=0)
    for it in range(2):   # right after that call, then after itself
        args, kw = _packed_case(d, per_splat_h=True, clip=0.05, seed=59)
        _render_and_check(*args, **kw)


# ---- SurfaceSplattingRenderer, packed clouds with Vrk_isotropic (the default): both routes on their own fragments --
def _route(dev, fused, clip, S=96):
    """Render the three overlapping clouds of tests/test_gpu_camera_grad.py through one route -> the route's records,
    fragments and gradients, and the float64 reference on them"""
    from dss_b200.core.cloud import PointClouds3D
    from dss_b200.core.rasterizer import PointsRasterizationSettings, SurfaceSplatting, _splat_params
    from dss_b200.core.renderer import NormWeightedCompositor, SurfaceSplattingRenderer
    from tests.test_gpu_camera_grad import _cameras
    from tests.util import render_backward_f64
    pts, nrm, col = (t.to(dev) for t in sphere_cloud(4000, seed=3))
    settings = PointsRasterizationSettings(backface_culling=False, cutoff_threshold=1.0, depth_merging_threshold=0.05,
                                           Vrk_invariant=False, Vrk_isotropic=True, radii_backward_scaler=5,
                                           image_size=S, points_per_pixel=5, bin_size=None, clip_pts_grad=clip)
    cams = _cameras(dev)
    rast = SurfaceSplatting(cameras=cams, raster_settings=settings)
    renderer = SurfaceSplattingRenderer(rast, NormWeightedCompositor())
    slices = [slice(0, 3000), slice(500, 4000), slice(1000, 2500)]
    rows = np.concatenate([np.arange(4000)[s] for s in slices])
    g = (torch.randn(3, S, S, 4, generator=torch.Generator().manual_seed(1)) * 1e-3).to(dev)
    p = pts.clone().requires_grad_(True)
    c = col.clone().requires_grad_(True)
    cloud = PointClouds3D([p[s] for s in slices], normals=[nrm[s] for s in slices], features=[c[s] for s in slices])
    img, frags = renderer(cloud, cameras=cams, fused=fused, verbose=True)
    img.backward(g)
    with torch.no_grad():
        # the screen records each route rasterized: the preprocess kernel's (fused), or the differentiable transform's
        # x, y, z with the kernel's radii (unfused, rasterizer.py:614)
        info = rast._get_per_point_info(cloud)
        ndc = info["ndc"]
        if not fused:
            t = rast.transform(cloud)
            ndc = torch.cat([t[:, :2], torch.where(ndc[:, 2:] >= 0, t[:, 2:], ndc[:, 2:])], 1)
    proj, view = camera_matrices(cams)
    first, num = cloud.cloud_to_packed_first_idx(), cloud.num_points_per_cloud()
    prm = _splat_params(settings, cams)
    ref = render_backward_f64(ndc, info["radii"], frags.idx, frags.qvalue, info["scaler"], cloud.points_packed(), proj,
                              view, prm, g, None, first, num)
    return dict(ndc=ndc, radii=info["radii"], idx=frags.idx, g=g, p=p.grad, c=c.grad, ref=ref, rows=rows, pts=pts,
                first=first, num=num, proj=proj.to(dev), view=view.to(dev), prm=prm, packed=cloud.points_packed())


@pytest.mark.parametrize("clip", [0.05, -1.0])
def test_renderer_routes_each_match_float64_on_their_own_fragments(cuda_device, clip):
    for fused in (True, False):
        r = _route(cuda_device, fused, clip)
        ref, rows = r["ref"], r["rows"]
        want = np.zeros((4000, 3))
        np.add.at(want, rows, ref["world"])
        scale = np.abs(want).max()
        err = np.abs(_np(r["p"]) - want).max()
        assert scale > 0 and err <= 2e-4 * scale, (fused, err, scale)
        wcol = np.zeros((4000, 3))
        np.add.at(wcol, rows, ref["colours"])
        assert np.abs(wcol).max() > 0
        np.testing.assert_allclose(_np(r["c"]), wcol, rtol=2e-4, atol=1e-7)
