"""CPU tests of the view coverage's specification (csrc/prune.cu, dss_b200.ops.accumulate_coverage).

``coverage_np`` restates what the kernel counts for one shared cloud seen by N views, in float32: ``seen`` the views in
which the point is visible, ``outside`` the views in which its record has z > 0, finite x and y with |x|, |y| <= 1, and
the point filters' mask sample at -xy (``sample_np`` of tests/test_point_filter.py, checked there bit for bit against
ATen's grid sampler) is zero.  Here it is checked on hand-built cases and against torch's ``grid_sample``."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.test_point_filter import make_masks, sample_np

f32 = np.float32


def coverage_np(xyz, visible, masks):
    """xyz (N, P0, 3) the records' x, y, z, visible (N, P0), masks (N, H, W) float32 / uint8 / bool -> (seen, outside),
    (P0,) int32"""
    xyz = np.asarray(xyz, f32)
    x, y, z = xyz[..., 0], xyz[..., 1], xyz[..., 2]
    with np.errstate(invalid="ignore"):
        counted = (z > 0) & (np.abs(x) <= 1) & (np.abs(y) <= 1)
    gx, gy = np.where(counted, -x, f32(0)).astype(f32), np.where(counted, -y, f32(0)).astype(f32)
    samples = np.stack([sample_np(m, gx[n], gy[n]) for n, m in enumerate(masks)])
    seen = (np.asarray(visible) != 0).sum(0).astype(np.int32)
    outside = (counted & (samples == 0)).sum(0).astype(np.int32)
    return seen, outside


def torch_coverage(xyz, visible, masks):
    """the same counts through torch's grid_sample (bilinear, reflection padding, align_corners=False)"""
    t = torch.from_numpy(np.asarray(xyz, f32))
    counted = (t[..., 2] > 0) & (t[..., 0].abs() <= 1) & (t[..., 1].abs() <= 1)
    p = torch.where(counted[..., None], -t[..., :2], torch.zeros_like(t[..., :2]))
    m = torch.from_numpy(np.asarray(masks)).float()[:, None]
    vals = F.grid_sample(m, p[:, None], mode="bilinear", padding_mode="reflection", align_corners=False)[:, 0, 0]
    seen = torch.from_numpy(np.asarray(visible) != 0).sum(0)
    return seen.int().numpy(), (counted & (vals == 0)).sum(0).int().numpy()


def test_hand_built_cases():
    """one view whose mask is 1 on the left half of the image (x < 0 in grid coordinates, x > 0 in the records)"""
    H = W = 8
    masks = np.zeros((1, H, W), f32)
    masks[0, :, : W // 2] = 1
    nan, inf = f32(np.nan), f32(np.inf)
    rows = [  # x, y, z, visible -> counts as outside
        (0.5, 0.0, 2.0, 1, False),    # over the object, visible
        (-0.5, 0.0, 2.0, 1, True),    # over background, visible
        (-0.5, 0.0, 2.0, 0, True),    # over background, hidden: still counts
        (-1.0, 1.0, 2.0, 0, True),    # on the frame's corner: inside it
        (-1.5, 0.0, 2.0, 0, False),   # off the frame
        (-0.5, -1.01, 2.0, 0, False),  # off the frame
        (-0.5, 0.0, -1.0, 0, False),  # outside the depth range or behind the camera (the preprocess's z = -1)
        (-0.5, 0.0, 0.0, 0, False),   # z = 0 is not kept either
        (nan, 0.0, 2.0, 0, False),    # non-finite positions give no evidence
        (-0.5, inf, 2.0, 0, False),
        (-inf, 0.0, 2.0, 0, False),
    ]
    xyz = np.array([r[:3] for r in rows], f32)[None]
    vis = np.array([r[3] for r in rows], np.uint8)[None]
    seen, outside = coverage_np(xyz, vis, masks)
    assert seen.tolist() == vis[0].tolist()
    assert outside.tolist() == [int(r[4]) for r in rows]
    t_seen, t_outside = torch_coverage(np.nan_to_num(xyz, nan=9.0, posinf=9.0, neginf=9.0), vis, masks)
    assert np.array_equal(seen, t_seen) and np.array_equal(outside, t_outside)


def test_counts_sum_over_the_views():
    """a point over background in two views of three, hidden in all, behind the camera of the third"""
    masks = np.zeros((3, 4, 4), f32)
    xyz = np.array([[[0.1, 0.1, 3.0]], [[0.2, -0.3, 1.5]], [[0.1, 0.1, -1.0]]], f32)
    vis = np.array([[1], [0], [1]], np.uint8)
    seen, outside = coverage_np(xyz, vis, masks)
    assert seen.tolist() == [2] and outside.tolist() == [2]
    # split views add up to the whole
    s0, o0 = coverage_np(xyz[:1], vis[:1], masks[:1])
    s1, o1 = coverage_np(xyz[1:], vis[1:], masks[1:])
    assert (s0 + s1).tolist() == seen.tolist() and (o0 + o1).tolist() == outside.tolist()


@pytest.mark.parametrize("kind", ["soft", "binary", "uint8", "bool"])
@pytest.mark.parametrize("N,H,W", [(1, 16, 16), (5, 37, 20)])
def test_restatement_matches_torch_grid_sample(kind, N, H, W):
    rng = np.random.default_rng(11 + N + H)
    P0 = 5000
    masks = make_masks(kind, N, H, W, seed=N * 10 + W)
    xy = rng.uniform(-1.3, 1.3, (N, P0, 2)).astype(f32)
    xy[:, : P0 // 10] = rng.choice(np.array([-1, 1, -1.0000001, 1.0000001], f32), (N, P0 // 10, 2))
    z = np.where(rng.random((N, P0)) < 0.2, f32(-1), rng.uniform(0.1, 5, (N, P0))).astype(f32)
    xyz = np.concatenate([xy, z[..., None]], -1)
    vis = (rng.random((N, P0)) < 0.3).astype(np.uint8)
    seen, outside = coverage_np(xyz, vis, masks)
    t_seen, t_outside = torch_coverage(xyz, vis, masks)
    assert np.array_equal(seen, t_seen) and np.array_equal(outside, t_outside)
    assert outside.max() > 0 and (outside < N).any()
