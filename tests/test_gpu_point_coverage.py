"""GPU: the view coverage (csrc/prune.cu; ops.accumulate_coverage and ops.point_coverage) against the float32 oracle of
tests/test_point_coverage_oracle.py, on renders of a seeded sphere cloud with planted points: behind every camera, far
outside the sphere but in a view's frame, and buried inside it.

What must hold:
  - the counts equal the oracle's exactly, for float32, uint8 and bool masks of any strides and size, and they add up:
    a second call doubles them, and calls over split views give the call over all of them;
  - the renders fill ``visible`` (the views whose K-lists hold the point) without a backward in sight;
  - the call replays from a CUDA graph to the same bits;
  - point_coverage gives the same counts for any batch, and equals the oracle on the data's renders and masks;
  - point_filters, whose mask sampling the coverage now shares, still equals its own oracle bit for bit."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from dss_b200 import _lib
from dss_b200.ops import (Coverage, SplatParams, _data_view_renderer, accumulate_coverage, point_coverage,
                          point_filters, render_points)
from tests.test_gpu_train_loop import data_dir, write_config  # noqa: F401  (data_dir: a fixture)
from tests.test_point_coverage_oracle import coverage_np
from tests.test_point_filter import filters_np
from tests.util import scene

pytestmark = pytest.mark.gpu

TAN_HALF_FOV = float(np.tan(np.radians(30.0)))   # the scene's cameras have a 60 degree field of view
CLUSTER = 12                                     # planted points along each corner ray


def planted_scene(P0, N, S, dev, seed):
    """a sphere cloud (radius 0.5) seen by N cameras, its silhouettes as (N,S,S) bool masks, and the cloud with its
    first rows replaced by planted points: one behind each camera, a cluster of CLUSTER along a ray through a corner of
    each view's frame (outside the sphere's silhouette, from 0.6 of the camera's distance on: the far ones hidden by
    the near ones in that view) and 2N buried within 0.1 of the centre.  Returns the planted cloud (points, normals,
    colours), proj, view, h, the masks and {kind: rows}."""
    pts, nrm, col, proj, view, _ = scene(P0, N, seed=seed)
    pts, nrm, col, proj, view = (t.to(dev) for t in (pts, nrm, col, proj, view))
    prm = SplatParams(image_size=S, znear=0.1)
    h = torch.full((N,), 3e-4, device=dev)
    with torch.no_grad():
        masks = render_points(pts, nrm, col, proj, view, h, prm).image[..., 3] > 0
    g = torch.Generator().manual_seed(seed)
    R, T = view[:, :3, :3], view[:, 3, :3]                     # p_view = p_world R + T (row vectors)
    centres = -torch.einsum("nj,nij->ni", T, R)                 # -T R^T
    behind = centres - 0.3 * R[:, :, 2]
    depth = (0.6 * centres.norm(dim=1))[:, None] + 0.05 * torch.rand(N, CLUSTER, generator=g).to(dev)
    sign = (torch.randint(0, 2, (N, 1, 2), generator=g) * 2 - 1).float().to(dev)
    corner_view = torch.cat([0.7 * TAN_HALF_FOV * depth[..., None] * sign, depth[..., None]], 2)
    corner = torch.einsum("nci,nji->ncj", corner_view - T[:, None], R).reshape(-1, 3)     # (p_view - T) R^T
    buried = F.normalize(torch.randn(2 * N, 3, generator=g), dim=1) * torch.rand(2 * N, 1, generator=g) * 0.1
    plants = torch.cat([behind, corner, buried.to(dev)])
    pts = pts.clone()
    pts[:plants.shape[0]] = plants
    C0 = N + N * CLUSTER
    rows = {"behind": np.arange(N), "corner": np.arange(N, C0), "buried": np.arange(C0, C0 + 2 * N)}
    return (pts, nrm, col), proj, view, h, prm, masks, rows


def render(cloud, proj, view, h, prm, sel=slice(None)):
    with torch.no_grad():
        return render_points(*cloud, proj[sel], view[sel], h[sel], prm)


def mask_variants(masks):
    """the silhouettes as float32 (contiguous), uint8 (column-major strides), bool (N,1,H,W) and a float32 mask of
    another size"""
    u8 = (masks.to(torch.uint8) * 255).transpose(1, 2).contiguous().transpose(1, 2)
    assert not u8.is_contiguous()
    other = F.interpolate(masks[:, None].float(), size=(48, 80), mode="nearest")[:, 0]
    return {"f32": masks.float(), "u8": u8, "bool": masks[:, None], "f32_48x80": other}


def oracle(out, mask, N):
    P0 = out.records.shape[0] // N
    m = mask[:, 0] if mask.dim() == 4 else mask
    return coverage_np(out.records[:, :3].reshape(N, P0, 3).cpu().numpy(), out.visible.reshape(N, P0).cpu().numpy(),
                       m.cpu().numpy())


def zeros(P0, dev):
    return Coverage(*(torch.zeros((P0,), dtype=torch.int32, device=dev) for _ in range(2)))


def visible_from_idx(out, N):
    """the (N*P0,) bytes of the points in some pixel's K-list, from idx (packed slots, -1 padded)"""
    v = torch.zeros(out.visible.shape, dtype=torch.uint8, device=out.idx.device)
    ids = out.idx[out.idx[..., :1].expand_as(out.idx) >= 0]
    v[ids[ids >= 0].long()] = 1
    return v


@pytest.mark.parametrize("N", [1, 5, 16])
def test_coverage_equals_the_oracle(cuda_device, N):
    d = cuda_device
    P0, S = 3000, 64
    cloud, proj, view, h, prm, masks, rows = planted_scene(P0, N, S, d, seed=N)
    out = render(cloud, proj, view, h, prm)
    assert torch.equal(out.visible, visible_from_idx(out, N))
    z = out.records[:, 2].reshape(N, P0)
    # each point behind its camera gives that view no evidence
    assert (z[torch.arange(N), torch.as_tensor(rows["behind"])] == -1).all()
    for name, mask in mask_variants(masks).items():
        cov = accumulate_coverage(out, mask, *zeros(P0, d))
        seen, outside = oracle(out, mask, N)
        got_seen, got_outside = cov.seen.cpu().numpy(), cov.outside.cpu().numpy()
        assert np.array_equal(got_seen, seen), name
        assert np.array_equal(got_outside, outside), (name, int((got_outside != outside).sum()))
        accumulate_coverage(out, mask, *cov)                       # the counters are added to
        assert np.array_equal(cov.seen.cpu().numpy(), 2 * seen)
        assert np.array_equal(cov.outside.cpu().numpy(), 2 * outside)
        if name == "f32_48x80":
            continue
        assert (outside[rows["corner"]] >= 1).all(), name           # over background in its own view at least
        assert (outside[rows["buried"]] == 0).all(), name           # inside every silhouette
        assert (seen > 0).sum() > P0 // 4
        if N == 1:                # the far corner points, hidden by the near ones, count over background
            assert ((seen == 0) & (outside > 0))[rows["corner"]].any(), name
        print("N=%d %s: seen in no view %d, outside in some view %d, hidden but outside %d" % (
            N, name, int((seen == 0).sum()), int((outside > 0).sum()), int(((seen == 0) & (outside > 0)).sum())))
    # calls over split views add up to the call over all of them (each view's records depend on that view alone)
    if N > 1:
        mask = mask_variants(masks)["u8"]
        k = N // 2
        split = zeros(P0, d)
        accumulate_coverage(render(cloud, proj, view, h, prm, slice(0, k)), mask[:k], *split)
        accumulate_coverage(render(cloud, proj, view, h, prm, slice(k, N)), mask[k:], *split)
        whole = accumulate_coverage(out, mask, *zeros(P0, d))
        assert torch.equal(split.seen, whole.seen) and torch.equal(split.outside, whole.outside)


def test_point_filters_keep_their_bits(cuda_device):
    d = cuda_device
    N, P0 = 8, 3000
    cloud, proj, view, h, prm, masks, _ = planted_scene(P0, N, 64, d, seed=3)
    out = render(cloud, proj, view, h, prm)
    xy = out.records[:, :2].reshape(N, P0, 2).cpu().numpy()
    for name, mask in mask_variants(masks).items():
        vis, inm = point_filters(out, mask)
        m = (mask[:, 0] if mask.dim() == 4 else mask).cpu().numpy()
        want_vis, want_inm, _ = filters_np(xy, out.visible.reshape(N, P0).cpu().numpy() != 0, m)
        assert np.array_equal(vis.cpu().numpy(), want_vis) and np.array_equal(inm.cpu().numpy(), want_inm), name


def test_coverage_replays_from_a_cuda_graph(cuda_device):
    d = cuda_device
    N, P0 = 6, 20000
    cloud, proj, view, h, prm, masks, _ = planted_scene(P0, N, 96, d, seed=11)
    out = render(cloud, proj, view, h, prm)
    mask = mask_variants(masks)["u8"]
    want = accumulate_coverage(out, mask, *zeros(P0, d))
    cov = zeros(P0, d)
    side = torch.cuda.Stream(d)
    side.wait_stream(torch.cuda.current_stream(d))
    with torch.cuda.stream(side):
        accumulate_coverage(out, mask, *cov)                       # warm-up outside the capture
    torch.cuda.current_stream(d).wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        cov.seen.zero_()
        cov.outside.zero_()
        accumulate_coverage(out, mask, *cov)
    for _ in range(2):
        cov.seen.fill_(-7)
        graph.replay()
        torch.cuda.synchronize(d)
        assert torch.equal(cov.seen, want.seen) and torch.equal(cov.outside, want.outside)


def test_coverage_refusals(cuda_device):
    d = cuda_device
    N, P0 = 3, 500
    cloud, proj, view, h, prm, masks, _ = planted_scene(P0, N, 32, d, seed=5)
    out = render(cloud, proj, view, h, prm)
    mask = masks.float()
    seen, outside = zeros(P0, d)
    strides = (C.c_int64 * 3)(*mask.stride())
    rc = _lib.load().dss_point_coverage(_lib.ctx(d), _lib.ptr(out.records), _lib.ptr(out.visible), 0, N, P0,
                                        _lib.ptr(mask), 0, strides, 32, 32, _lib.ptr(seen), _lib.ptr(outside),
                                        _lib.stream_ptr(d))
    assert rc == -1 and "shared cloud" in _lib.last_error()
    for bad in (torch.zeros(P0, dtype=torch.int64, device=d), torch.zeros(P0 + 1, dtype=torch.int32, device=d),
                torch.zeros(P0, dtype=torch.int32), torch.zeros(2 * P0, dtype=torch.int32, device=d)[::2], None):
        with pytest.raises(RuntimeError, match="must be a contiguous int32 tensor of shape"):
            accumulate_coverage(out, mask, bad, outside)
        with pytest.raises(RuntimeError, match="must be a contiguous int32 tensor of shape"):
            accumulate_coverage(out, mask, seen, bad)
    with pytest.raises(RuntimeError, match="mask_img must have shape"):
        accumulate_coverage(out, mask[:2], seen, outside)
    with pytest.raises(TypeError, match="float32, uint8 or bool"):
        accumulate_coverage(out, mask.double(), seen, outside)
    with pytest.raises(RuntimeError, match="RenderOutput of a shared cloud"):
        accumulate_coverage(out._replace(records=out.records[:-1]), mask, seen, outside)
    assert int(seen.abs().sum()) == 0 and int(outside.abs().sum()) == 0


def test_point_coverage_on_data(data_dir, tmp_path):  # noqa: F811
    from dss_b200.training.config import load_config, splat_params
    from dss_b200.utils.dataset import MVRData
    d = torch.device("cuda:0")
    data = MVRData(data_dir)
    cams = data.get_cameras()
    cfg = load_config(write_config(tmp_path / "c.yml", data_dir, tmp_path / "out"))
    params = splat_params(cfg, cams.znear, cams.zfar)
    gt = data.get_pointclouds()
    g = torch.Generator().manual_seed(0)
    idx = torch.randperm(gt.points_packed().shape[0], generator=g)[:3000]
    points = gt.points_packed()[idx].float().to(d)
    normals = gt.normals_packed()[idx].float().to(d)
    strays = torch.tensor([[0, 0.8, 0], [0, -0.8, 0], [0, 0.55, 0], [0.2, 0.7, -0.2], [1e3, 0, 0]], device=d)
    points[:strays.shape[0]] = strays
    views = data.device_views(d)
    V = len(views)
    covs = {B: point_coverage(points, normals, views, params, batch=B, Vrk_invariant=True, Vrk_isotropic=False)
            for B in (1, 3, V)}
    for B in (3, V):
        assert torch.equal(covs[B].seen, covs[1].seen) and torch.equal(covs[B].outside, covs[1].outside), B
    # an MVRData gives the same counts; views split over two calls add up
    from_data = point_coverage(points, normals, data, params, batch=4, Vrk_invariant=True, Vrk_isotropic=False)
    assert torch.equal(from_data.seen, covs[1].seen) and torch.equal(from_data.outside, covs[1].outside)
    a = point_coverage(points, normals, views, params, 2, range(0, V, 2), True, False)
    b = point_coverage(points, normals, views, params, 2, range(1, V, 2), True, False)
    assert torch.equal(a.seen + b.seen, covs[1].seen) and torch.equal(a.outside + b.outside, covs[1].outside)
    # the oracle on the same no-grad renders and the views' masks
    render = _data_view_renderer(points, normals, torch.ones_like(points), views, True, False, 0.2, 64.0)
    seen, outside = np.zeros(3000, np.int64), np.zeros(3000, np.int64)
    for v in range(V):
        out = render(params, [v])
        _, mask = views.gather(views.upload([v]))
        s, o = oracle(out, mask, 1)
        seen, outside = seen + s, outside + o
    assert np.array_equal(covs[1].seen.cpu().numpy(), seen) and np.array_equal(covs[1].outside.cpu().numpy(), outside)
    # the strays: over background somewhere, and the one past zfar nowhere at all
    assert (outside[:4] > 0).all() and seen[4] == 0 and outside[4] == 0
    assert (seen[5:] > 0).mean() > 0.8 and (outside[5:] == 0).mean() > 0.9
    print("torus sample: seen in no view %d, outside in some view %d of %d" % (
        int((seen == 0).sum()), int((outside > 0).sum()), seen.size))
    assert covs[1].seen.dtype == torch.int32 and int(covs[1].seen.max()) <= V
    empty = point_coverage(points, normals, views, params, views=[])
    assert int(empty.seen.abs().sum()) == 0 and int(empty.outside.abs().sum()) == 0
