"""CPU: the Poisson-disk sampling rule as tests/poisson_disk_oracle.py states it -- the hash, the area-weighted draw,
the pool, the dart throw against a brute force, the geodesic distance and the radius search."""
import math

import numpy as np
import pytest

from tests import poisson_disk_oracle as pd
from tests.test_mesh_data import icosphere, torus


def test_splitmix64_matches_the_published_sequence():
    # SplitMix64 seeded with 0: its first two outputs
    out = pd.splitmix64(0, np.array([1, 2], dtype=np.uint64))
    assert [int(x) for x in out] == [0xE220A8397B1DCDAF, 0x6E789E6AA1B965F4]


def test_mulhi64_against_python_integers():
    rng = np.random.default_rng(0)
    a = rng.integers(0, 2 ** 63, 1000, dtype=np.uint64) * np.uint64(2) + np.uint64(1)
    for b in (1, 2 ** 32, 2 ** 63 - 25, 12345678901234567):
        got = pd.mulhi64(a, b)
        assert [int(x) for x in got] == [(int(x) * b) >> 64 for x in a]


def test_draw_frequencies_follow_the_area():
    # two faces of area 1 and 3
    verts = np.array([[0, 0, 0], [1, 0, 0], [0, 2, 0], [2, 0, 1], [5, 0, 1], [2, 2, 1]], np.float32)
    faces = np.array([[0, 1, 2], [3, 4, 5]])
    m = pd.faces_of(verts, faces)
    assert m["area"].tolist() == [1.0, 3.0]
    assert m["prefix"].tolist() == [0, math.ceil(2 ** 32 / 3), math.ceil(2 ** 32 / 3) + 2 ** 32]
    _, _, face = pd.pool(verts, faces, 5000, seed=7)
    frac = float((face == 1).mean())
    assert abs(frac - 0.75) < 6 * math.sqrt(0.75 * 0.25 / len(face)), frac


def test_unusable_faces_have_no_weight_and_change_nothing():
    v, f = icosphere(2)
    v, f = v.numpy(), f.numpy()
    junk_v = np.concatenate([v, [[np.nan, 0, 0], [1, 1, 1]]]).astype(np.float32)
    V = len(v)
    junk_f = np.concatenate([f[:7], [[0, 0, 1], [V, 1, 2], [0, 1, V + 5], [-1, 2, 3], [V + 1, V + 1, V + 1]],
                             f[7:]])
    m = pd.faces_of(junk_v, junk_f)
    assert m["usable"].sum() == len(f) and (m["prefix"][8:13] == m["prefix"][7]).all()
    a = pd.sample(v, f, 300, seed=3)
    b = pd.sample(junk_v, junk_f, 300, seed=3)
    assert np.array_equal(a["points"].view(np.int32), b["points"].view(np.int32))
    assert a["radius"] == b["radius"]


def test_pool_points_lie_in_their_faces():
    v, f = torus(nu=12, nv=8)
    v, f = v.numpy(), f.numpy()
    pts, nrm, face = pd.pool(v, f, 500, seed=1)
    a, b, c = (v[f[face, k]].astype(np.float64) for k in range(3))
    p = pts.astype(np.float64)
    n = np.cross(b - a, c - a)
    n /= np.linalg.norm(n, axis=1, keepdims=True)
    assert np.abs(((p - a) * n).sum(1)).max() < 1e-6
    assert np.abs(nrm - n).max() < 1e-6
    # barycentric coordinates of the projection
    e0, e1, q = b - a, c - a, p - a
    d00, d01, d11 = (e0 * e0).sum(1), (e0 * e1).sum(1), (e1 * e1).sum(1)
    d20, d21 = (q * e0).sum(1), (q * e1).sum(1)
    den = d00 * d11 - d01 * d01
    bv, bw = (d11 * d20 - d01 * d21) / den, (d00 * d21 - d01 * d20) / den
    assert bv.min() > -1e-6 and bw.min() > -1e-6 and (bv + bw).max() < 1 + 1e-6


@pytest.mark.parametrize("r", [0.05, 0.12, 0.4])
def test_selection_equals_brute_force_and_is_separated_and_maximal(r):
    v, f = icosphere(2)
    pts, nrm, _ = pd.pool(v.numpy(), f.numpy(), 150, seed=2)
    idx, _ = pd.select(pts, nrm, r)
    assert np.array_equal(idx, pd.brute_force_select(pts, r))
    p = pts.astype(np.float64)
    acc = p[idx]
    d = np.sqrt(((acc[:, None] - acc[None]) ** 2).sum(-1))
    assert d[~np.eye(len(acc), dtype=bool)].min() >= r * (1 - 1e-12)
    rejected = np.setdiff1d(np.arange(len(p)), idx)
    for i in rejected:
        earlier = idx[idx < i]
        assert (np.sqrt(((p[earlier] - p[i]) ** 2).sum(1)) < r).any()


def test_geodesic_distance_is_arc_over_chord_symmetric_and_at_least_euclidean():
    R = 0.7
    for theta in (1e-3, 0.2, 1.0, 2.5, 3.1):
        p0 = np.array([R, 0.0, 0.0])
        p1 = np.array([R * math.cos(theta), R * math.sin(theta), 0.0])
        d, g = pd.geodesic_distance(p0, p0 / R, p1, p1 / R)
        assert d == pytest.approx(R * theta, rel=1e-6)
        d2, _ = pd.geodesic_distance(p1, p1 / R, p0, p0 / R)
        assert d2 == pytest.approx(d, rel=1e-12)
        assert g >= 1.0 and d >= np.linalg.norm(p0 - p1) * (1 - 1e-15)
    rng = np.random.default_rng(0)
    for _ in range(200):
        p0, p1 = rng.normal(size=3), rng.normal(size=3)
        n0, n1 = (x / np.linalg.norm(x) for x in rng.normal(size=(2, 3)))
        d, g = pd.geodesic_distance(p0, n0, p1, n1)
        assert g >= 1.0 and d >= np.linalg.norm(p0 - p1) * (1 - 1e-15)
        assert pd.geodesic_distance(p1, n1, p0, n0)[0] == pytest.approx(d, rel=1e-9)


@pytest.mark.parametrize("geodesic", [False, True])
@pytest.mark.parametrize("N", [1, 60, 400])
def test_count_within_tolerance(N, geodesic):
    v, f = torus(nu=24, nv=12)
    out = pd.sample(v.numpy(), f.numpy(), N, geodesic=geodesic, seed=5)
    n = len(out["points"])
    assert abs(n - N) <= N // 200, (n, out["probes"])
    if N == 1:
        assert n == 1
    assert out["probes"][-1] == (out["radius"], n)
    # the returned samples are the pool's, in pool order
    assert (np.diff(out["indices"]) > 0).all()


def test_no_usable_face_gives_nothing():
    verts = np.array([[0, 0, 0], [1, 0, 0], [2, 0, 0]], np.float32)
    out = pd.sample(verts, np.array([[0, 1, 2], [0, 0, 1]]), 10)
    assert len(out["points"]) == 0 and out["radius"] == 0.0
