"""GPU tests of the fused forward binning of dss_render_forward: the depth ranges come from a pre-pass over the world
points, the preprocess counts the tile lists as it writes the records, and the scatter reuses the preprocess's blocks.
Everything it produces must equal the separate count and scatter passes over the records (the DSS_BIN_NORECTS route,
switched on here with dss_debug_bin_no_rects): the depth ranges and tile offsets bit for bit, every (view, tile, slice)
list as a set (list order is set by atomics on both routes), and every render output bit for bit."""
import os

import numpy as np
import pytest
import torch

from dss_b200 import _lib
from dss_b200.core.lighting import DirectionalLights
from dss_b200.ops import SplatParams, local_frames, make_shading, render_points
from tests.test_gpu_raster_edges import _near_plane_cloud
from tests.util import scene

pytestmark = pytest.mark.gpu

OUTPUTS = ("image", "idx", "zbuf", "weights", "visible")


def _plan(N, S, K):
    """tile grid, depth slices and number of bins of the forward lists (raster_fwd.cu: plan_tiles)"""
    B = (S + 15) // 16
    NS = 1
    if K <= 8:
        NS = 8
        while NS > 1 and B * B * NS > 8 * 1024:
            NS >>= 1
    return B, NS, N * B * B * NS


def _bits(t):
    return t.contiguous().view(torch.int32) if t.dtype == torch.float32 else t


def _render(d, no_rects, args, kw, K, whole_lists=True):
    """(render output, zrange, offsets, ids) of one forward on the fused route or on the separate passes"""
    _lib.bin_no_rects(no_rects, d)
    try:
        out = render_points(*args, return_fragments=True, **kw)
    finally:
        _lib.bin_no_rects(os.environ.get("DSS_BIN_NORECTS", "") == "1", d)
    N, S = out.image.shape[0], out.image.shape[1]
    _, _, nb = _plan(N, S, K)
    _, off, _ = _lib.tile_lists(N, nb + 1, 0, d)
    n_ids = int(off[-1]) if whole_lists else 0
    zr, off, ids = _lib.tile_lists(N, nb + 1, n_ids, d)
    torch.cuda.synchronize(d)
    return out, zr, off, ids


def _sorted_lists(off, ids, P):
    """every entry keyed by (bin, id) and sorted: equal for two sets of lists that hold the same ids per bin"""
    counts = (off[1:] - off[:-1]).long()
    bins = torch.repeat_interleave(torch.arange(counts.numel(), device=off.device), counts)
    return torch.sort(bins * (P + 1) + ids[:bins.numel()].long()).values


def _check(d, args, kw, K, whole_lists=True):
    if whole_lists:   # the id buffer is sized from what an earlier call published: let it grow to these lists first
        for _ in range(2):
            render_points(*args, **kw)
            torch.cuda.synchronize(d)
    fused = _render(d, False, args, kw, K, whole_lists)
    ref = _render(d, True, args, kw, K, whole_lists)
    (out, zr, off, ids), (rout, rzr, roff, rids) = fused, ref
    assert torch.equal(_bits(zr), _bits(rzr))
    assert torch.equal(off, roff)
    if whole_lists:
        P = out.records.shape[0]
        assert torch.equal(_sorted_lists(off, ids, P), _sorted_lists(roff, rids, P))
    for name in OUTPUTS:
        assert torch.equal(_bits(getattr(out, name)), _bits(getattr(rout, name))), name
    assert int(off[-1]) > 0
    return out, zr


def _shared(d, P0, N, S, K, seed, h_scale=1.0, **prm_kw):
    pts, nrm, col, proj, view, _ = scene(P0, N, seed=seed)
    prm = SplatParams(image_size=S, points_per_pixel=K, znear=0.1, **prm_kw)
    h = torch.full((N,), h_scale * 3e-4 * (100.0 / S) ** 2 * (6000.0 / P0), device=d)
    colours = (col.repeat(N, 1) * torch.linspace(0.5, 1.0, N).repeat_interleave(P0)[:, None]).to(d)
    return (pts.to(d), nrm.to(d), colours, proj.to(d), view.to(d), h, prm), {}


def test_bench_scene(cuda_device):
    """bench.py's workload: a 1M-point sphere, 8 views of 512^2, K = 5"""
    d = cuda_device
    pts, nrm, col, proj, view, _ = scene(1_000_000, 8, seed=0)
    prm = SplatParams(image_size=512, points_per_pixel=5, clip_pts_grad=0.05, znear=0.1)
    h = torch.full((8,), 5e-5, device=d)
    out, zr = _check(d, (pts.to(d), nrm.to(d), col.to(d), proj.to(d), view.to(d), h, prm), {}, 5)
    assert (zr[:, 1] > zr[:, 0]).all() and out.visible.sum() > 0


@pytest.mark.parametrize("S,K,P0,N", [(17, 5, 2000, 2), (336, 5, 30000, 1), (368, 5, 30000, 2), (1000, 8, 60000, 1),
                                      (2048, 4, 60000, 1), (2080, 5, 20000, 1), (256, 8, 40000, 3),
                                      (256, 12, 40000, 3)])
def test_image_sizes_and_k(cuda_device, S, K, P0, N):
    """power-of-two and other sizes, 1 to 8 slices (S = 2048: 128 tiles per side, one slice, a 64 KB histogram), the
    global-atomic binning (S = 2080: 130 tiles per side, both runs take it) and K > 8 (one slice, pixel-parallel raster)"""
    args, kw = _shared(cuda_device, P0, N, S, K, seed=S + K)
    _check(cuda_device, args, kw, K)


@pytest.mark.parametrize("K", [5, 8, 12])
def test_packed_ragged_and_empty_views(cuda_device, K):
    d = cuda_device
    P0, N, S = 20000, 4, 256
    pts, nrm, col, proj, view, _ = scene(P0, N, seed=60 + K)
    num = torch.tensor([P0, P0 - 7001, 0, 1], dtype=torch.int64)
    first = torch.tensor([0, P0, 2 * P0 - 7001, 2 * P0 - 7001], dtype=torch.int64)
    sel = torch.cat([torch.arange(P0), torch.arange(P0 - 7001), torch.arange(1)])
    prm = SplatParams(image_size=S, points_per_pixel=K, znear=0.1)
    h = torch.full((sel.numel(),), 4e-4, device=d)
    args = (pts[sel].to(d), nrm[sel].to(d), col[sel].to(d), proj.to(d), view.to(d), h, prm)
    _check(d, args, dict(first_idx=first.to(d), num_points=num.to(d), shared_cloud=False), K)


@pytest.mark.parametrize("layout", ["shared", "packed"])
def test_nan_and_inf_rows(cuda_device, layout):
    """NaN / inf coordinates, normals and h: the depth pre-pass must skip exactly the depths the preprocess skips"""
    d = cuda_device
    P0, N, S, K = 30000, 3, 256, 5
    pts, nrm, col, proj, view, _ = scene(P0, N, seed=71)
    rng = np.random.default_rng(7)
    rows = torch.from_numpy(rng.choice(P0, 80, replace=False))
    pts[rows[:10], 0] = float("nan")
    pts[rows[10:20], 2] = float("inf")
    pts[rows[20:30]] = -float("inf")
    nrm[rows[30:40]] = float("nan")
    prm = SplatParams(image_size=S, points_per_pixel=K, znear=0.1)
    if layout == "shared":
        h = torch.full((N * P0,), 3e-4)
        h[rows[40:60]] = float("nan")
        h[rows[60:]] = float("inf")
        args = (pts.to(d), nrm.to(d), col.repeat(N, 1).to(d), proj.to(d), view.to(d), h.to(d), prm)
        kw = {}
    else:
        h = torch.full((N * P0,), 3e-4)
        h[rows[40:60] + P0] = float("nan")
        h[rows[60:]] = float("inf")
        first = torch.arange(N, dtype=torch.int64) * P0
        num = torch.full((N,), P0, dtype=torch.int64)
        args = (pts.repeat(N, 1).to(d), nrm.repeat(N, 1).to(d), col.repeat(N, 1).to(d), proj.to(d), view.to(d),
                h.to(d), prm)
        kw = dict(first_idx=first.to(d), num_points=num.to(d), shared_cloud=False)
    _check(d, args, kw, K)


def test_backface_culling(cuda_device):
    args, kw = _shared(cuda_device, 40000, 3, 256, 5, seed=21, backface_culling=True)
    out, _ = _check(cuda_device, args, kw, 5)
    kept = (out.records[:, 2] >= 0).float().mean().item()
    assert 0.3 < kept < 0.7


@pytest.mark.parametrize("K", [5, 12])
def test_near_plane_cloud(cuda_device, K):
    """points just past znear with huge splats far off the view axis, an ordinary cloud behind them"""
    d = cuda_device
    pts, nrm, col, proj, view = _near_plane_cloud(3000, seed=K)
    near = (pts[:, 2] < 0.16).float()
    N = proj.shape[0]
    h = (1e-5 + 4e-2 * near).repeat(N)
    prm = SplatParams(image_size=128, points_per_pixel=K, znear=0.1)
    _check(d, (pts.to(d), nrm.to(d), col.repeat(N, 1).to(d), proj.to(d), view.to(d), h.to(d), prm), {}, K)


@pytest.mark.parametrize("layout", ["shared", "packed"])
def test_anisotropic_frames(cuda_device, layout):
    d = cuda_device
    P0, N, S, K = 30000, 3, 256, 5
    pts, nrm, col, proj, view, _ = scene(P0, N, seed=81)
    prm = SplatParams(image_size=S, points_per_pixel=K, znear=0.1)
    if layout == "shared":
        fr = local_frames(pts.to(d))
        args = (pts.to(d), nrm.to(d), col.repeat(N, 1).to(d), proj.to(d), view.to(d), None, prm)
        kw = dict(frames=fr)
    else:
        first = torch.arange(N, dtype=torch.int64).to(d) * P0
        num = torch.full((N,), P0, dtype=torch.int64).to(d)
        pp = pts.repeat(N, 1).to(d)
        fr = local_frames(pp, first, num)
        args = (pp, nrm.repeat(N, 1).to(d), col.repeat(N, 1).to(d), proj.to(d), view.to(d), None, prm)
        kw = dict(frames=fr, first_idx=first, num_points=num, shared_cloud=False)
    _check(d, args, kw, K)


@pytest.mark.parametrize("K", [5, 12])
def test_fused_shading(cuda_device, K):
    d = cuda_device
    P0, N, S = 30000, 3, 256
    pts, nrm, col, proj, view, _ = scene(P0, N, seed=91)
    prm = SplatParams(image_size=S, points_per_pixel=K, znear=0.1)
    lights = DirectionalLights(direction=torch.tensor([[0.3, -0.5, 1.0]]), device=d)
    sh = make_shading(lights, view.to(d))
    args = (pts.to(d), nrm.to(d), col.to(d), proj.to(d), view.to(d), torch.full((N,), 3e-4, device=d), prm)
    _check(d, args, dict(shading=sh), K)


@pytest.mark.parametrize("K", [5, 8])
def test_tile_capacity_overflow(cuda_device, K):
    """lists that do not fit the id buffer: the scatter drops what lies past the capacity on both routes (which entries
    depends on the atomics' order), the rasterizer walks those tiles' records -- the outputs stay bit-identical"""
    d = cuda_device
    args, kw = _shared(d, 60000, 2, 128, K, seed=31)
    try:
        for cap in (50000, 2000, 1):
            _lib.limit_tile_capacity(cap, d)
            _check(d, args, kw, K, whole_lists=False)
    finally:
        _lib.limit_tile_capacity(0, d)
