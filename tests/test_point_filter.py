"""CPU tests of the point filters' specification (csrc/point_filter.cu, dss_b200.ops.point_filters).

The reference's inmask filter (DSS/models/point_modeling.py:188-212) samples the ground-truth masks with
``grid_sample(mask, clamp(-xy, -1, 1), bilinear, padding_mode='reflection', align_corners=False)``.  ``filters_np`` restates
what the kernel computes, step by step in float32: the clamp, the align_corners=False unnormalisation, the reflection
(the identity on the clamped range, but evaluated as ATen evaluates it), the clip to [0, size - 1], the four
bounds-checked taps summed in ATen's order nw, ne, sw, se, ``!= 0``, the OR over the views and ``& visibility``.  It is
checked against torch on the CPU: the sampled values bit for bit against ATen's scalar grid sampler (the CPU fallback
kernel, which shares the CUDA kernel's formulas), the booleans bit for bit against ``F.grid_sample`` itself (whose
vectorised CPU kernel unnormalises in another order, so its values may differ in the last bit, never its zeros)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

f32 = np.float32


def source_index_np(coord, size):
    """grid_sampler_compute_source_index, align_corners=False, reflection padding, for finite coord in [-1, 1]"""
    coord = ((coord + f32(1)) * f32(size) - f32(1)) / f32(2)
    lo, span = f32(-0.5), f32(size)
    mag = np.abs(coord - lo)
    extra = np.fmod(mag, span)
    flips = np.floor(mag / span).astype(np.int64)
    coord = np.where(flips % 2 == 0, extra + lo, (span - extra) + lo).astype(f32)
    return np.minimum(f32(size - 1), np.maximum(coord, f32(0)))


def sample_np(mask, gx, gy):
    """bilinear sample of one (H, W) mask at grid coordinates gx (indexes W), gy (indexes H), float32 throughout"""
    H, W = mask.shape
    mask = mask.astype(f32)
    ix, iy = source_index_np(gx, W), source_index_np(gy, H)
    x0, y0 = np.floor(ix).astype(np.int64), np.floor(iy).astype(np.int64)
    x1, y1 = x0 + 1, y0 + 1
    taps = ((y0, x0, (x1 - ix) * (y1 - iy)), (y0, x1, (ix - x0) * (y1 - iy)),   # nw, ne
            (y1, x0, (x1 - ix) * (iy - y0)), (y1, x1, (ix - x0) * (iy - y0)))   # sw, se
    acc = np.zeros(ix.shape, f32)
    for yy, xx, w in taps:
        inside = (yy >= 0) & (yy < H) & (xx >= 0) & (xx < W)
        v = mask[np.clip(yy, 0, H - 1), np.clip(xx, 0, W - 1)]
        acc = np.where(inside, acc + v * w.astype(f32), acc).astype(f32)
    return acc


def filters_np(xy, visible, masks):
    """xy (N, P0, 2) the projected NDC positions, visible (N, P0) bool, masks (N, H, W) -> (visibility, inmask, samples
    (N, P0) with NaN where the position is not finite)"""
    finite = np.isfinite(xy).all(-1)
    g = np.clip(-np.where(finite[..., None], xy, f32(0)), f32(-1), f32(1)).astype(f32)
    samples = np.stack([sample_np(m, g[n, :, 0], g[n, :, 1]) for n, m in enumerate(masks)])
    in_view = (samples != 0) & finite
    visibility = visible.any(0)
    return visibility, in_view.any(0) & visibility, np.where(finite, samples, f32(np.nan))


def torch_filters(xy, visible, masks, sampler=None):
    """the reference's lines on torch tensors: -xy, clamp, grid_sample, .bool(), any over views, & visibility"""
    p = (-torch.from_numpy(xy)).clamp(-1.0, 1.0)
    m = torch.from_numpy(masks).float()[:, None]
    if sampler is None:
        vals = F.grid_sample(m, p[:, None], mode="bilinear", padding_mode="reflection", align_corners=False)
    else:
        vals = sampler(m, p[:, None])
    vals = vals[:, 0, 0]
    vis = torch.from_numpy(visible).any(0, keepdim=True)
    return vis[0].numpy(), (vals.bool().any(0, keepdim=True) & vis)[0].numpy(), vals.numpy()


def aten_scalar_sampler(m, grid):
    # interpolation 0 = bilinear, padding 2 = reflection
    return torch._grid_sampler_2d_cpu_fallback(m, grid, 0, 2, False)


def make_masks(kind, N, H, W, seed):
    rng = np.random.default_rng(seed)
    if kind == "soft":
        m = rng.random((N, H, W)).astype(f32)
        m[m < 0.4] = 0
        return m
    if kind == "binary":
        return (rng.random((N, H, W)) < 0.5).astype(f32)
    if kind == "uint8":
        m = rng.integers(0, 256, (N, H, W)).astype(np.uint8)
        m[rng.random((N, H, W)) < 0.5] = 0
        return m
    return rng.random((N, H, W)) < 0.5


def special_coords(rng, P, H, W):
    """grid coordinates (gx, gy): on pixel centres, on pixel edges, at +-1, outside [-1, 1], random"""
    gx = rng.uniform(-1.3, 1.3, P).astype(f32)
    gy = rng.uniform(-1.3, 1.3, P).astype(f32)
    q = P // 6
    kx, ky = rng.integers(0, W, P), rng.integers(0, H, P)
    gx[:q] = ((2 * kx[:q] + 1) / W - 1).astype(f32)                 # x on centres
    gy[q:2 * q] = ((2 * ky[q:2 * q] + 1) / H - 1).astype(f32)       # y on centres
    gx[2 * q:3 * q] = (2 * rng.integers(0, W + 1, q) / W - 1).astype(f32)   # x on edges
    gy[2 * q:3 * q] = (2 * rng.integers(0, H + 1, q) / H - 1).astype(f32)   # and y on edges
    gx[3 * q:4 * q] = rng.choice(np.array([-1, 1, -1.0000001, 1.0000001, -7.5, 7.5], f32), q)
    gy[3 * q:4 * q] = rng.choice(np.array([-1, 1, -1.0000001, 1.0000001, -7.5, 7.5], f32), q)
    return gx, gy


@pytest.mark.parametrize("kind", ["soft", "binary", "uint8", "bool"])
@pytest.mark.parametrize("N,H,W", [(1, 16, 16), (3, 37, 20), (8, 64, 96)])
def test_restatement_matches_torch_grid_sample(kind, N, H, W):
    rng = np.random.default_rng(7 + N + H)
    P0 = 6000
    masks = make_masks(kind, N, H, W, seed=N * 100 + H)
    xy = np.stack([np.stack(special_coords(rng, P0, H, W), -1) for _ in range(N)])
    xy = (-xy).astype(f32)     # the records hold x, y; the reference samples at -xy
    visible = rng.random((N, P0)) < 0.3
    vis, inm, vals = filters_np(xy, visible, masks)
    t_vis, t_inm, t_vals = torch_filters(xy, visible, masks)
    a_vis, a_inm, a_vals = torch_filters(xy, visible, masks, aten_scalar_sampler)
    assert np.array_equal(vals.view(np.uint32), a_vals.view(np.uint32))      # bit for bit
    assert np.array_equal(vals != 0, t_vals != 0)
    assert np.array_equal(vis, t_vis) and np.array_equal(inm, t_inm) and np.array_equal(inm, a_inm)
    # samples inside and outside the masks, and points in the filter
    assert (vals == 0).any() and (vals != 0).any() and inm.any()


def test_or_over_views_not_per_view_and():
    """a point visible only in view 0 and inside the mask only in view 1 is in the mask"""
    H = W = 8
    masks = np.zeros((2, H, W), f32)
    masks[1] = 1.0
    xy = np.zeros((2, 3, 2), f32)
    visible = np.array([[True, False, False], [False, False, True]])
    vis, inm, _ = filters_np(xy, visible, masks)
    assert vis.tolist() == [True, False, True]
    assert inm.tolist() == [True, False, True]
    t_vis, t_inm, _ = torch_filters(xy, visible, masks)
    assert np.array_equal(vis, t_vis) and np.array_equal(inm, t_inm)


def test_pixel_centre_reads_one_column():
    """exactly on a pixel-centre column the other column's weight is exactly 0: a non-zero neighbour does not count"""
    H, W = 4, 6
    masks = np.zeros((1, H, W), f32)
    masks[0, :, 3] = 1.0
    gx = np.array([(2 * 2 + 1) / W - 1, (2 * 3 + 1) / W - 1, (2 * 2 + 1) / W - 1 + 1e-3], f32)   # centre of column 2,
    gy = np.zeros(3, f32)                                                                     # of 3, just right of 2
    xy = -np.stack([gx, gy], -1)[None]
    vis, inm, vals = filters_np(xy, np.ones((1, 3), bool), masks)
    assert inm.tolist() == [False, True, True]
    _, t_inm, _ = torch_filters(xy, np.ones((1, 3), bool), masks)
    assert np.array_equal(inm, t_inm)


def test_non_finite_positions_are_outside_the_mask():
    """NaN / inf projected positions (a point on the camera plane, a NaN input) never count as inside, while the OR over
    the views still takes the finite views of the same point"""
    masks = np.ones((2, 5, 5), f32)
    nan, inf = f32(np.nan), f32(np.inf)
    xy = np.array([[[nan, 0], [0, inf], [-inf, nan], [nan, 0]],
                   [[nan, 0], [0, -inf], [inf, 0], [0.1, 0.2]]], f32)
    vis, inm, vals = filters_np(xy, np.ones((2, 4), bool), masks)
    assert inm.tolist() == [False, False, False, True]
    assert np.isnan(vals[:, :3]).all()
