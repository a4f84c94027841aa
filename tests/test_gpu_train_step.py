"""GPU tests of the training step on the fused path: dss_point_filters (csrc/point_filter.cu) against the reference's
torch lines and a float64 projection, TrainStep against a composition of the existing public pieces, and
GraphedTrainStep against the eager step."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from dss_b200 import _lib
from dss_b200.core.cloud import PointClouds3D, PointCloudsFilters
from dss_b200.core.knn import knn_sq_dists
from dss_b200.core.lighting import DirectionalLights
from dss_b200.ops import RenderOutput, SplatParams, make_shading, point_filters, render_points, set_point_filters
from dss_b200.training.losses import ProjectionLoss, RepulsionLoss, image_loss_torch
from dss_b200.training.step import GraphedTrainStep, TrainStep
from tests.util import scene

pytestmark = pytest.mark.gpu


def torch_filters(records, visible, mask_img):
    """point_modeling.py:172-173, 198-212 on the render's records: -xy, clamp, grid_sample, .bool(), any, &"""
    N, H, W = mask_img.shape[0], mask_img.shape[-2], mask_img.shape[-1]
    P0 = records.shape[0] // N
    p = -records[:, :2].reshape(N, P0, 2)
    m = mask_img.reshape(N, 1, H, W).float()
    vals = F.grid_sample(m, p.clamp(-1.0, 1.0)[:, None], mode="bilinear", padding_mode="reflection",
                         align_corners=False)[:, 0, 0]
    vis = visible.reshape(N, P0).bool().any(dim=0, keepdim=True)
    return vis[0], (vals.bool().any(dim=0, keepdim=True) & vis)[0]


def make_mask(kind, layout, N, H, W, seed, dev):
    """a seeded mask of blobs (so that it changes across pixel edges in places and not in others)"""
    g = torch.Generator().manual_seed(seed)
    low = torch.rand(N, 1, max(2, H // 6), max(2, W // 6), generator=g)
    soft = F.interpolate(low, size=(H, W), mode="bilinear", align_corners=False)[:, 0]
    soft = torch.where(soft > 0.5, soft, torch.zeros_like(soft))
    m = {"f32": soft, "u8": (soft * 255).to(torch.uint8), "bool": soft > 0}[kind].to(dev)
    if layout == "perm":
        m = m.transpose(1, 2).contiguous().transpose(1, 2)
        assert not m.is_contiguous()
    elif layout == "n1hw":
        m = m[:, None]
    return m


def special_records(out, N, P0, S_mask, seed):
    """overwrite some (view, point) records with positions on pixel centres and edges of the mask, at and outside
    +-1, and non-finite ones (those points are made invisible in every view, as a render leaves them)"""
    H, W = S_mask
    g = torch.Generator().manual_seed(seed)
    rec = out.records.clone()
    vis = out.visible.clone()
    r = rec.view(N, P0, 8)
    v = vis.view(N, P0)
    k = max(1, P0 // 8)
    for n in range(N):
        rows = torch.randperm(P0, generator=g)[:k]
        kx = torch.randint(0, W + 1, (k,), generator=g).float()
        ky = torch.randint(0, H + 1, (k,), generator=g).float()
        centre = torch.rand(k, generator=g) < 0.5
        gx = torch.where(centre, (2 * kx + 1) / W - 1, 2 * kx / W - 1)
        gy = torch.where(torch.rand(k, generator=g) < 0.5, (2 * ky + 1) / H - 1, 2 * ky / H - 1)
        edge = torch.tensor([-1.0, 1.0, -1.5, 1.5, 3.0])
        pick = torch.rand(k, generator=g) < 0.2
        gx = torch.where(pick, edge[torch.randint(0, 5, (k,), generator=g)], gx)
        r[n, rows.to(r.device), 0] = (-gx).to(r.device)
        r[n, rows.to(r.device), 1] = (-gy).to(r.device)
        v[n, rows.to(r.device)] = (torch.rand(k, generator=g) < 0.7).to(torch.uint8).to(r.device)
    bad = torch.randperm(P0, generator=g)[: max(1, P0 // 50)].to(r.device)
    vals = torch.tensor([float("nan"), float("inf"), -float("inf")], device=r.device)
    r[:, bad, 0] = vals[torch.arange(bad.numel(), device=r.device) % 3]
    r[:, bad[::2], 1] = float("nan")
    v[:, bad] = 0
    return out._replace(records=rec, visible=vis), bad


def render_cloud(P0, N, S, dev, seed):
    """a sphere cloud with some points behind camera 0"""
    pts, nrm, col, proj, view, _ = scene(P0, N, seed=seed)
    pts, nrm, col, proj, view = (t.to(dev) for t in (pts, nrm, col, proj, view))
    if P0 >= 20:
        R, T = view[0, :3, :3], view[0, 3, :3]
        centre = -(T @ R.T)
        nb = P0 // 20
        pts[:nb] = centre + (-0.3 - 0.2 * torch.rand(nb, 1, device=dev)) * R[:, 2] + 0.05 * torch.randn(nb, 3, device=dev)
    prm = SplatParams(image_size=S, znear=0.1, clip_pts_grad=0.05)
    h = torch.full((N,), 3e-4, device=dev)
    with torch.no_grad():
        out = render_points(pts, nrm, col, proj, view, h, prm)
    return out, pts, proj


# ---- 1. the kernel against the reference's torch lines, bit for bit ------------------------------------------------
@pytest.mark.parametrize("N", [1, 3, 8, 256])
@pytest.mark.parametrize("P0", [1, 1000, 100003])
def test_point_filters_equal_the_torch_composition(cuda_device, N, P0):
    d = cuda_device
    S = 64
    out, pts, proj = render_cloud(P0, N, S, d, seed=N + P0)
    counts = []
    for msize in ((S, S), (48, 80)):
        special, bad = special_records(out, N, P0, msize, seed=P0 + msize[1])
        for kind, layout in (("f32", "contig"), ("u8", "perm"), ("bool", "n1hw"), ("f32", "perm"), ("u8", "n1hw"),
                             ("bool", "contig")):
            mask = make_mask(kind, layout, N, *msize, seed=N * 7 + msize[1], dev=d)
            for o in (out, special):
                vis, inm = point_filters(o, mask)
                want_vis, want_inm = torch_filters(o.records, o.visible, mask)
                assert vis.dtype == torch.bool and vis.shape == (P0,) and inm.shape == (P0,)
                assert torch.equal(vis, want_vis), (kind, layout, msize)
                assert torch.equal(inm, want_inm), (kind, layout, msize, int((inm != want_inm).sum()))
                counts.append((int(vis.sum()), int(inm.sum())))
            assert not inm[bad].any()     # non-finite positions
    if P0 >= 1000:   # points in the filter; and, with few views, visible points outside every mask
        assert any(c[1] > 0 for c in counts) and (N > 8 or any(c[0] > c[1] for c in counts))
    print("N=%d P0=%d (visible, inmask) counts: %s" % (N, P0, counts[:4]))


def test_point_filters_refuse_packed_clouds_and_bad_masks(cuda_device):
    d = cuda_device
    out, _, _ = render_cloud(1000, 3, 32, d, seed=1)
    mask = torch.ones(3, 32, 32, device=d)
    vis, inm = (torch.empty(1000, dtype=torch.uint8, device=d) for _ in range(2))
    strides = (C.c_int64 * 3)(*mask.stride())
    rc = _lib.load().dss_point_filters(_lib.ctx(d), _lib.ptr(out.records), _lib.ptr(out.visible), 0, 3, 1000,
                                       _lib.ptr(mask), 0, strides, 32, 32, _lib.ptr(vis), _lib.ptr(inm),
                                       _lib.stream_ptr(d))
    assert rc == -1 and "shared cloud" in _lib.last_error()
    with pytest.raises(RuntimeError, match="mask_img must have shape"):
        point_filters(out, torch.ones(2, 32, 32, device=d))
    with pytest.raises(TypeError, match="float32, uint8 or bool"):
        point_filters(out, torch.ones(3, 32, 32, device=d, dtype=torch.float64))
    f = set_point_filters(PointCloudsFilters(d), out, mask)
    assert f.visibility.shape == (1, 1000) and f.inmask.shape == (1, 1000) and f.inmask.dtype == torch.bool


# ---- 2. against a float64 projection of the world points -----------------------------------------------------------
def test_point_filters_match_a_float64_projection(cuda_device):
    d = cuda_device
    N, P0, S = 8, 100003, 128
    out, pts, proj = render_cloud(P0, N, S, d, seed=5)
    H, W = 96, 160
    mask = make_mask("f32", "contig", N, H, W, seed=3, dev=d)
    vis, inm = point_filters(out, mask)
    ph = torch.cat([pts.double(), torch.ones(P0, 1, dtype=torch.float64, device=d)], 1)
    clip = torch.einsum("pi,nij->npj", ph, proj.double())
    xy = clip[..., :2] / clip[..., 3:]
    g64 = (-xy).clamp(-1, 1)
    vals = F.grid_sample(mask.double()[:, None], g64[:, None], mode="bilinear", padding_mode="reflection",
                         align_corners=False)[:, 0, 0]
    want = (vals != 0).any(0) & vis
    differ = (want != inm).nonzero().flatten()
    # a disagreement needs, in some view, a float64 sample coordinate within 1e-4 px of a tap boundary
    ix = ((g64[..., 0] + 1) * W - 1) / 2
    iy = ((g64[..., 1] + 1) * H - 1) / 2
    near = torch.minimum((ix - ix.round()).abs(), (iy - iy.round()).abs()) < 1e-4
    assert near[:, differ].any(0).all(), differ[~near[:, differ].any(0)][:10]
    print("float64 projection: %d of %d points disagree, all within 1e-4 px of a tap boundary"
          % (differ.numel(), P0))
    assert differ.numel() <= P0 // 1000


# ---- 3. TrainStep against the composition of the public pieces -----------------------------------------------------
def batch(N, S, dev, seed):
    _, _, _, proj, view, _ = scene(10, N, seed=seed)
    g = torch.Generator().manual_seed(seed)
    img = torch.rand(N, S, S, 3, generator=g).to(dev)
    mask = make_mask("f32", "contig", N, S, S, seed=seed, dev=dev)
    lights = DirectionalLights(ambient_color=0.2 * torch.rand(N, 1, 3, generator=g),
                               diffuse_color=0.5 * torch.rand(N, 1, 3, generator=g),
                               specular_color=0.1 * torch.rand(N, 1, 3, generator=g),
                               direction=torch.randn(N, 1, 3, generator=g), device=dev)
    return img, mask, proj.to(dev), view.to(dev), lights


def composition(pts, nrm, col, prm, img, mask, proj, view, lights, lam_proj, lam_repel, radius=0.2):
    p = pts.detach().clone().requires_grad_(True)
    n = nrm.detach().clone().requires_grad_(True)
    normals = F.normalize(n, dim=-1)
    N = proj.shape[0]
    h0 = 0.5 * knn_sq_dists(p.detach(), K=7, radius=radius)[:, 1:].max(dim=-1)[0]
    h = h0.mean().clamp(5e-5, 1e-3).repeat(N)
    out = render_points(p, normals, col, proj, view, h, prm, shading=make_shading(lights, view))
    img_l = image_loss_torch(out.image, img, mask, 1.0, 1.0)
    vis, inm = torch_filters(out.records, out.visible, mask)
    cloud = PointClouds3D([p], [normals])
    filt = PointCloudsFilters(p.device, visibility=vis[None], inmask=inm[None])
    zero = torch.zeros((), device=p.device)
    lp = ProjectionLoss(knn_k=12, filter_scale=2.0).torch_body(cloud, filt, rebuild_knn=True).mean() * lam_proj \
        if lam_proj > 0 else zero
    lr = RepulsionLoss(knn_k=12, filter_scale=2.0).torch_body(cloud, filt, rebuild_knn=True).mean() * lam_repel \
        if lam_repel > 0 else zero
    total = lp + lr + img_l["loss"]
    total.backward()
    loss = {"loss": total, "loss_dr_rgb": img_l["loss_dr_rgb"], "loss_dr_silhouette": img_l["loss_dr_silhouette"],
            "loss_dr_proj": lp, "loss_dr_repel": lr}
    return loss, p.grad, n.grad, out.image.detach(), vis, inm


@pytest.mark.parametrize("lam_repel", [0.0, 0.05])
def test_train_step_equals_the_composition_of_the_public_pieces(cuda_device, lam_repel):
    d = cuda_device
    P0, N, S = 20000, 4, 128
    pts, nrm, col, _, _, _ = scene(P0, N, seed=41)
    pts, nrm, col = pts.to(d), nrm.to(d) * 1.7, col.to(d)        # normals of another length: the step normalises
    prm = SplatParams(image_size=S, points_per_pixel=5, znear=0.1, clip_pts_grad=0.05, radii_backward_scaler=5.0)
    img, mask, proj, view, lights = batch(N, S, d, seed=42)
    step = TrainStep(pts, nrm, col, prm, lambda_dr_proj=0.01, lambda_dr_repel=lam_repel)
    loss = step(img, mask, proj, view, lights)
    want, gp, gn, image, vis, inm = composition(pts, nrm, col, prm, img, mask, proj, view, lights, 0.01, lam_repel)
    assert torch.equal(step.image, image) and torch.equal(step.visibility, vis) and torch.equal(step.inmask, inm)
    assert inm.any() and (vis & ~inm).any()
    for k in want:
        w = float(want[k].detach())
        assert abs(float(loss[k]) - w) <= 1e-5 * abs(w) + 1e-12, (k, float(loss[k]), w)
    assert (float(loss["loss_dr_repel"]) > 0) == (lam_repel > 0) and float(loss["loss_dr_proj"]) > 0
    assert step.colours.grad is None
    for got, w in ((step.points.grad, gp), (step.normals.grad, gn)):
        scale = float(w.abs().max())
        assert scale > 0 and float((got - w).abs().max()) <= 1e-4 * scale


# ---- 4 + 5. GraphedTrainStep replays the eager step --------------------------------------------------------------
def test_graphed_train_step_replays_the_eager_step(cuda_device):
    d = cuda_device
    P0, N, S = 20000, 4, 128
    pts, nrm, col, _, _, _ = scene(P0, N, seed=51)
    pts, nrm, col = pts.to(d), nrm.to(d), col.to(d)
    prm = SplatParams(image_size=S, points_per_pixel=5, znear=0.1, clip_pts_grad=0.05, radii_backward_scaler=5.0)
    a, b = batch(N, S, d, seed=52), batch(N, S, d, seed=53)

    # the eager results first: eager calls between replays may need more library scratch than the capture held
    eager = TrainStep(pts, nrm, col, prm, lambda_dr_repel=0.05)
    keep = lambda s: ({k: v.clone() for k, v in s.loss.items()}, s.image.clone(), s.visibility.clone(),
                      s.inmask.clone(), s.points.grad.clone(), s.normals.grad.clone())
    eager(*a)
    want_a = keep(eager)
    eager(*b)
    want_b = keep(eager)
    eager.params = prm._replace(radii_backward_scaler=4.5)
    eager.lambda_dr_proj = 0.02
    eager(*b)
    want_c = keep(eager)

    step = GraphedTrainStep(pts, nrm, col, prm, *a, lambda_dr_repel=0.05)
    launches = _lib.launch_count()

    def check(want):
        step.replay()
        torch.cuda.synchronize()
        loss, image, vis, inm, gp, gn = want
        assert torch.equal(step.image, image) and torch.equal(step.visibility, vis) and torch.equal(step.inmask, inm)
        for k in loss:
            assert torch.equal(step.loss[k], loss[k]), k
        # float atomics in the colour scatter feed the shading's position and normal gradients
        torch.testing.assert_close(step.points.grad, gp, rtol=1e-4, atol=1e-9)
        torch.testing.assert_close(step.normals.grad, gn, rtol=1e-4, atol=1e-9)

    check(want_a)
    check(want_a)
    step.load(*b)
    check(want_b)
    nodes = step.kernel_nodes()
    assert _lib.launch_count() == launches            # replays launch nothing from the host
    step.params = prm._replace(radii_backward_scaler=4.5)
    step.lambda_dr_proj = 0.02
    check(want_c)                                     # captured again with the new settings
    assert step.kernel_nodes() == nodes
    scratch, launches = _lib.scratch_bytes(), _lib.launch_count()
    for _ in range(20):
        step.replay()
    torch.cuda.synchronize()
    assert _lib.scratch_bytes() == scratch and _lib.launch_count() == launches and step.kernel_nodes() == nodes
    assert not step.stale()
    print("graphed train step: %d kernel nodes per replay" % nodes)
