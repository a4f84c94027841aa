"""Host tests of the upsampling and outlier oracle (tests/upsample_oracle.py): the round sizes, the new points and their
parents, where the first round inserts on a cloud of two densities, the outlier ratio against numpy.linalg.eigh, a plane
in volume noise, and the ValueError cases; and the library's host-side schedule against the oracle's."""
import numpy as np
import pytest

from dss_b200.ops import upsample_schedule
from tests import upsample_oracle as uo


def _patch(n, h, x0, rng):
    g = np.stack(np.meshgrid(np.arange(n), np.arange(n), indexing="ij"), -1).reshape(-1, 2) * h
    g = g + rng.uniform(-0.1 * h, 0.1 * h, g.shape)
    return np.concatenate([g + [x0, 0.0], rng.normal(scale=1e-3 * h, size=(len(g), 1))], 1).astype(np.float32)


def _sphere(n, seed=0):
    p = np.random.default_rng(seed).normal(size=(n, 3))
    return (p / np.linalg.norm(p, axis=1, keepdims=True)).astype(np.float32)


def test_round_sizes():
    sizes = uo.schedule([8000, 100, 50], [100_000, 100, 61], 16)
    assert len(sizes) == 28                       # 8 000 -> 100 000 takes 27 rounds
    for a, b in zip(sizes[:-1], sizes[1:]):
        for c, c1, n in zip(a, b, (100_000, 100, 61)):
            assert c1 - c == min(n - c, c // 10)
    assert sizes[-1] == [100_000, 100, 61]
    assert uo.schedule([20], [20], 16) == [[20]]
    for num, tgt in (([8000, 100, 50], [100_000, 100, 61]), ([100_000], [1_000_000]), ([17, 300], [40, 301])):
        assert upsample_schedule(num, tgt, 16) == uo.schedule(num, tgt, 16)


@pytest.mark.parametrize("num,target,k", [([100], [99], 16), ([16], [20], 16), ([9], [12], 3), ([12], [13], 12)])
def test_schedule_errors(num, target, k):
    with pytest.raises(ValueError):
        uo.schedule(num, target, k)
    with pytest.raises(ValueError):
        upsample_schedule(num, target, k)


def test_non_finite_raises():
    p = _sphere(200)
    p[7, 1] = np.inf
    with pytest.raises(ValueError):
        uo.upsample(p, 300, 8)


def test_neighbours_drop_own_index_or_last():
    rows = np.array([[0, 3, 5, 1], [2, 1, 4, 0], [0, 1, 3, 4]])
    assert uo.neighbours(rows).tolist() == [[3, 5, 1], [2, 4, 0], [0, 1, 3]]


@pytest.mark.parametrize("k", [8, 16])
def test_new_points_and_parents(k):
    rng = np.random.default_rng(1)
    p0 = _sphere(600)
    nrm = p0 * rng.uniform(0.5, 2.0, (600, 1)).astype(np.float32)          # not unit: normalised before use
    col = rng.uniform(0, 1, (600, 3)).astype(np.float32)
    p, n, f, par, sizes = uo.upsample(p0, 1500, k, nrm, col)
    assert len(p) == 1500 and sizes[0] == 600 and sizes[-1] == 1500
    assert np.array_equal(p[:600], p0) and np.array_equal(n[:600], nrm) and np.array_equal(f[:600], col)
    assert (par[:600] == -1).all()
    for c, c1 in zip(sizes[:-1], sizes[1:]):
        i, j = par[c:c1, 0], par[c:c1, 1]
        assert ((0 <= i) & (i < c) & (0 <= j) & (j < c) & (i != j)).all()
        assert (np.diff(i) > 0).all()                                     # in the order of the parents' indices
        assert np.array_equal(p[c:c1], (p[j] + np.float32(2) * p[i]) / np.float32(3))
        assert np.array_equal(f[c:c1], (f[j] + np.float32(2) * f[i]) / np.float32(3))
    assert np.allclose(np.linalg.norm(n, axis=1)[600:], 1.0, atol=1e-6)
    # a third of the way from p_i to q_j*, within float32 rounding
    i, j = par[600:, 0], par[600:, 1]
    third = p[i] + (p[j].astype(np.float64) - p[i]) / 3.0
    assert np.abs(p[600:] - third).max() < 1e-6
    assert (p[600:] >= p0.min(0)).all() and (p[600:] <= p0.max(0)).all()


def test_first_round_fills_the_sparse_patch():
    """A dense patch of spacing h next to a sparse one of spacing 3h: with m no larger than the sparse patch, every
    first-round parent lies in the sparse patch or within 3h of it."""
    rng = np.random.default_rng(2)
    h = 0.01
    dense, sparse = _patch(40, h, 0.0, rng), _patch(14, 3 * h, 40 * h + 3 * h, rng)
    p = np.concatenate([dense, sparse])
    m = min(len(sparse), len(p) // 10)
    _, _, _, par = uo.upsample_round(p, uo.knn_rows(p, 17), m)
    parents = p[par[:, 0]]
    assert (parents[:, 0] >= sparse[:, 0].min() - 3 * h).all()


def test_outlier_ratio_matches_eigh():
    rng = np.random.default_rng(3)
    p = (rng.normal(size=(500, 3)) * [1.0, 0.5, 0.2]).astype(np.float32)
    idx = uo.knn_rows(p, 16)
    ratio, keep = uo.outlier_ratio(p, idx, 0.05)
    q = p.astype(np.float64)[idx]
    d = q - q.mean(1, keepdims=True)
    lam = np.linalg.eigh(np.einsum("mki,mkj->mij", d, d) / 16)[0]
    ref = lam[:, 0] / lam.sum(1)
    assert np.allclose(ratio, ref, rtol=1e-9, atol=0)
    assert np.array_equal(keep, ratio < 0.05)
    idx[5, 3] = -1
    ratio, keep = uo.outlier_ratio(p, idx, 0.05)
    assert np.isnan(ratio[5]) and not keep[5]


def test_plane_in_volume_noise():
    """On a plane of noise 1e-3 with uniform noise in the surrounding cube, the plane is kept and most volume points go
    (the fractions are recorded in DESIGN.md)."""
    rng = np.random.default_rng(4)
    plane = np.concatenate([rng.uniform(-1, 1, (4000, 2)), rng.normal(scale=1e-3, size=(4000, 1))], 1)
    vol = rng.uniform(-1, 1, (400, 3))
    p = np.concatenate([plane, vol]).astype(np.float32)
    _, keep = uo.outlier_ratio(p, uo.knn_rows(p, 16), 0.05)
    kept_plane, kept_vol = keep[:4000].mean(), keep[4000:].mean()
    print("plane kept %.4f, volume kept %.4f" % (kept_plane, kept_vol))
    assert kept_plane > 0.9 and kept_vol < 0.5
