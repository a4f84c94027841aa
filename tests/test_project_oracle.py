"""CPU tests of the RIMLS projection and normal-denoising oracle (tests/project_oracle.py): fixed points, invariance,
a hand-computed case, both stops against a plain per-row restatement, and what the projection does to noise."""
import numpy as np

from tests import project_oracle as po
from tests import upsample_oracle as uo


def _sphere(n, sigma, seed):
    rng = np.random.default_rng(seed)
    u = rng.normal(size=(n, 3))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    return (0.5 + sigma * rng.normal(size=(n, 1))) * u, u


def _rows(p, k):
    return uo.knn_rows(p, k + 1)


def test_lane_sum_is_the_butterfly():
    v = np.random.default_rng(0).normal(size=(5, 32))
    ref = v.copy()
    for o in (16, 8, 4, 2, 1):
        ref = ref + ref[:, np.arange(32) ^ o]
    assert np.array_equal(po.lane_sum(v), ref[:, 0])
    assert np.all(ref == ref[:, :1])                     # every lane holds the same bits


def test_plane_is_a_fixed_point():
    rng = np.random.default_rng(1)
    p = np.concatenate([rng.uniform(-0.3, 0.3, (800, 2)), np.zeros((800, 1))], 1).astype(np.float32)
    n = np.tile(np.float32([0, 0, 1]), (800, 1))
    for k in (8, 31):
        out = po.project(p, n, _rows(p, k), k)
        assert np.array_equal(out.points, p.astype(np.float64))
        assert (out.iterations == 0).all() and out.inner_stops == 800
    assert np.array_equal(po.denoise_normals(p, n, _rows(p, 16)).normals, n.astype(np.float64))


def test_rotation_and_translation():
    p, n = _sphere(600, 0.01, 2)
    q, _ = np.linalg.qr(np.random.default_rng(3).normal(size=(3, 3)))
    t = np.array([0.3, -1.2, 0.7])
    rows = _rows(p, 31)
    a = po.project(p, n, rows)
    b = po.project(p @ q.T + t, n @ q.T, rows)
    assert a.margin > 1e-6 and b.margin > 1e-6 and (a.iterations > 0).all()
    assert np.array_equal(a.iterations, b.iterations)
    assert np.abs(a.points @ q.T + t - b.points).max() < 1e-12
    rows = _rows(p, 16)
    noisy = po.normalize(n + np.random.default_rng(4).normal(scale=0.1, size=n.shape))
    da, db = po.denoise_normals(p, noisy, rows), po.denoise_normals(p @ q.T + t, noisy @ q.T, rows)
    assert np.abs(da.normals @ q.T - db.normals).max() < 1e-12


def test_hand_computed_three_neighbours():
    p = np.array([[0.0, 0.0, 0.01], [0.1, 0.0, 0.0], [0.0, 0.1, 0.0], [-0.1, -0.1, 0.02]])
    n = po.normalize(np.array([[0.0, 0.0, 1.0], [0.1, 0.0, 1.0], [0.0, 0.1, 1.0], [0.0, 0.0, 1.0]]))
    out = po.project(p, n, _rows(p, 3), 3, max_proj_iters=1, max_est_iters=1)
    x = p[0]
    q, nq = p[1:], n[1:]
    d2 = ((x - q) ** 2).sum(1)
    inv = 1.0 / (16.0 * d2.min())
    phi = np.exp(-d2 * inv)
    fx = ((x - q) * nq).sum(1)
    w = phi                                               # alpha = 1 in the first estimate
    gw = 2.0 * (x - q) * (inv * phi * w)[:, None]
    f = (fx * w).sum() / w.sum()
    g = ((gw * fx[:, None]).sum(0) - f * gw.sum(0) + (w[:, None] * nq).sum(0)) / w.sum()
    assert np.allclose(out.points[0], x - f * g, rtol=0, atol=1e-15)
    assert out.iterations[0] == 1


def _naive_project(p, n, rows, k, T, S):
    """the rules once more, one row at a time, with plain sums"""
    r = po.cloud_radius(p, k, 16.0)
    out, its = p.copy(), np.zeros(len(p), np.int32)
    for i, nb in enumerate(uo.neighbours(rows)):
        q = np.array([p[j] for j in nb if j >= 0 and ((p[i] - p[j]) ** 2).sum() <= r * r]).reshape(-1, 3)
        nq = po.normalize(np.array([n[j] for j in nb if j >= 0 and ((p[i] - p[j]) ** 2).sum() <= r * r]).reshape(-1, 3))
        d2 = ((p[i] - q) ** 2).sum(1)
        if not (d2 > 0).any():
            continue
        inv = 1.0 / (16.0 * d2[d2 > 0].min())
        x = p[i].copy()
        for _ in range(T):
            fx = ((x - q) * nq).sum(1)
            alpha, f, g = np.ones(len(q)), 0.0, np.zeros(3)
            for s in range(S):
                if s > 0:
                    new = np.exp(-(np.linalg.norm(nq - g, axis=1) / 0.5) ** 2) * np.exp(-(fx - f) ** 2 * inv / 4)
                    if np.abs(new - alpha).max() < 1e-4:
                        break
                    alpha = new
                phi = np.exp(-((x - q) ** 2).sum(1) * inv)
                w = phi * alpha
                gw = 2 * (x - q) * (inv * phi * w)[:, None]
                f, g = (fx * w).sum() / w.sum(), ((gw * fx[:, None]).sum(0) - (fx * w).sum() / w.sum() * gw.sum(0)
                                                  + (w[:, None] * nq).sum(0)) / w.sum()
            x = x - f * g
            its[i] += bool((f * g != 0).any())
            if not np.linalg.norm(f * g) > 5e-4:
                break
        out[i] = x
    return out, its


def test_both_stops_against_a_plain_restatement():
    p, n = _sphere(400, 0.02, 5)
    for k, T, S in ((8, 10, 5), (31, 10, 5), (16, 3, 12)):
        rows = _rows(p, k)
        out = po.project(p, n, rows, k, T, S)
        assert out.margin > 1e-6 and out.inner_stops > 0 and out.outer_stops > 0
        ref, its = _naive_project(p, n, rows, k, T, S)
        assert np.array_equal(out.iterations, its)
        assert np.abs(out.points - ref).max() < 1e-12
    # a row that stopped after m < T moves made its last move at most 5e-4, every earlier one longer
    rows = _rows(p, 31)
    steps = [po.project(p, n, rows, 31, t).points for t in range(11)]
    its = po.project(p, n, rows, 31, 10).iterations
    moves = np.stack([np.linalg.norm(b - a, axis=1) for a, b in zip(steps[:-1], steps[1:])], 1)
    for i, m in enumerate(its):
        assert (moves[i, :m - 1] > 5e-4).all() and (m == 10 or moves[i, m - 1] <= 5e-4)
        assert (moves[i, m:] == 0).all()


def test_noisy_sphere_error_falls():
    p, n = _sphere(8000, 0.01, 6)
    out = po.project(p, n, _rows(p, 31))
    before = np.abs(np.linalg.norm(p, axis=1) - 0.5).mean()
    after = np.abs(np.linalg.norm(out.points, axis=1) - 0.5).mean()
    assert before / after >= 2.0, (before, after)


def test_denoise_lowers_angular_error_on_a_noisy_plane():
    rng = np.random.default_rng(7)
    p = np.concatenate([rng.uniform(-0.5, 0.5, (3000, 2)), 1e-3 * rng.normal(size=(3000, 1))], 1)
    n = po.normalize(np.array([0, 0, 1.0]) + rng.normal(scale=0.08, size=(3000, 3)))
    angle = lambda v: np.degrees(np.arccos(np.clip(v[:, 2], -1, 1))).mean()
    out = po.denoise_normals(p, n, _rows(p, 16))
    assert angle(out.normals) < 0.5 * angle(n), (angle(n), angle(out.normals))
    assert np.allclose(np.linalg.norm(out.normals, axis=1), 1.0)
