"""CPU: the float64 oracle of the screened Poisson reconstruction (tests/poisson_oracle.py) against the properties the
discretisation promises -- K 1 = 0, sum b = 0 and a zero mean of chi at the samples, the sphere's radius to a tenth of
a cell -- and its marching tetrahedra on analytic fields: closed, outward, of the right Euler characteristic; and
save_ply's face element read back by read_mesh."""
import numpy as np
import pytest

from dss_b200.utils.io import read_mesh, read_ply, save_ply
from tests import poisson_oracle as po


def sphere_samples(n=4000, radius=0.5, seed=0):
    """n Fibonacci points of a sphere about the origin plus its 6 axis points, so that its box is exactly
    [-radius, radius]^3; outward unit normals"""
    i = np.arange(n) + 0.5
    z = 1 - 2 * i / n
    phi = np.pi * (1 + 5 ** 0.5) * i
    r = np.sqrt(1 - z * z)
    d = np.stack([r * np.cos(phi), r * np.sin(phi), z], 1)
    d = np.concatenate([d, np.eye(3), -np.eye(3)])
    rng = np.random.default_rng(seed)
    d = d[rng.permutation(len(d))]
    return (radius * d).astype(np.float32), d.astype(np.float32)


def test_domain_rule():
    p, n = sphere_samples(500)
    p = np.concatenate([p, [[np.nan, 0, 0], [9, 9, 9], [1e9, 0, 0]]]).astype(np.float32)
    n = np.concatenate([n, [[1, 0, 0], [0, 0, 0], [np.inf, 0, 0]]]).astype(np.float32)
    ok, c, L = po.domain(p, n)
    assert ok.sum() == 506 and not ok[-3:].any()
    assert np.array_equal(c, np.zeros(3, np.float32)) and L == np.float32(1.1)
    u = (p[ok].astype(np.float64) - c) / np.float64(L) + 0.5
    assert u.min() >= 0.045 - 1e-7 and u.max() <= 0.955 + 1e-7


@pytest.mark.parametrize("R", [8, 16])
def test_operator_identities(R):
    p, n = sphere_samples(1500)
    s = po.assemble(p, n, R)
    ones = np.ones(s["K"].shape[0])
    assert np.abs(s["K"] @ ones).max() < 1e-12
    assert abs(s["b"].sum()) < 1e-12 * np.abs(s["b"]).sum()
    chi, _ = po.solve(p, n, R)
    at = s["Phi"] @ chi
    assert abs(at.sum()) < 1e-9 * np.abs(at).sum()
    # negative inside, positive outside
    N1 = R + 1
    g = chi.reshape(N1, N1, N1)
    assert g[R // 2, R // 2, R // 2] < 0 and g[0, 0, 0] > 0


def test_sphere_radius_within_a_tenth_of_a_cell():
    R = 24
    p, n = sphere_samples(4000)
    chi, s = po.solve(p, n, R)
    g = chi.reshape(R + 1, R + 1, R + 1)
    h, L = 1.0 / R, float(s["L"])
    r_u = 0.5 / L
    worst = 0.0
    for line in (g[:, R // 2, R // 2], g[R // 2, :, R // 2], g[R // 2, R // 2, :]):
        sign = line < 0
        cross = np.nonzero(sign[:-1] != sign[1:])[0]
        assert len(cross) == 2
        for i in cross:
            t = -line[i] / (line[i + 1] - line[i])
            x = (i + t) * h
            worst = max(worst, abs(abs(x - 0.5) - r_u) / h)
    assert worst < 0.1, worst


def analytic_grid(kind, R):
    x = np.arange(R + 1) / R - 0.5
    X, Y, Z = np.meshgrid(x, x, x, indexing="ij")
    if kind == "sphere":
        f = np.sqrt((X - 0.03) ** 2 + (Y + 0.02) ** 2 + Z ** 2) - 0.31
    else:
        f = (np.sqrt(X ** 2 + Y ** 2) - 0.25) ** 2 + Z ** 2 - 0.1 ** 2
    return f.astype(np.float32)


@pytest.mark.parametrize("kind,euler", [("sphere", 2), ("torus", 0)])
@pytest.mark.parametrize("R", [12, 31])
def test_marching_tetrahedra_closed_outward(kind, euler, R):
    chi = analytic_grid(kind, R)
    c, L = np.array([0.5, -1.0, 2.0], np.float32), np.float32(2.0)
    v, f = po.marching_tetrahedra(chi, c, L)
    assert len(f) > 0 and f.max() < len(v)
    assert (f[:, 0] != f[:, 1]).all() and (f[:, 1] != f[:, 2]).all() and (f[:, 0] != f[:, 2]).all()
    assert po.closed_manifold(f)
    assert po.euler_characteristic(v, f) == euler
    vol = po.signed_volume(v, f)
    exact = (4 / 3 * np.pi * 0.31 ** 3 if kind == "sphere" else 2 * np.pi ** 2 * 0.25 * 0.1 ** 2) * 8.0
    # the torus's tube is 1.2 cells thick at R = 12
    assert vol > 0 and abs(vol - exact) < (0.25 if R < 16 else 0.1) * exact
    # every vertex lies on its edge, inside the grid's box
    lo, hi = c - L / 2, c + L / 2
    assert (v >= lo - 1e-6).all() and (v <= hi + 1e-6).all()


def test_marching_tetrahedra_exact_zeros_are_outside():
    R = 6
    chi = np.ones((R + 1,) * 3, np.float32)
    chi[2:5, 2:5, 2:5] = 0.0
    chi[3, 3, 3] = -1.0
    v, f = po.marching_tetrahedra(chi, np.zeros(3, np.float32), 1.0)
    assert po.closed_manifold(f) and po.euler_characteristic(v, f) == 2 and po.signed_volume(v, f) > 0
    # the zero nodes are outside: every vertex sits on a node next to the one inside node (t = 1)
    assert np.allclose(np.abs(v).max(1), 1.0 / R, atol=1e-6)
    empty_v, empty_f = po.marching_tetrahedra(np.zeros((5, 5, 5), np.float32), np.zeros(3, np.float32), 1.0)
    assert len(empty_v) == 0 and len(empty_f) == 0


@pytest.mark.parametrize("binary", [True, False])
def test_save_ply_faces_round_trip(tmp_path, binary):
    v, f = po.marching_tetrahedra(analytic_grid("torus", 10), np.zeros(3, np.float32), 1.0)
    n = np.random.default_rng(0).normal(size=v.shape).astype(np.float32)
    path = str(tmp_path / "m.ply")
    save_ply(path, v, normals=n, faces=f, binary=binary)
    rv, rf = read_mesh(path)
    assert np.array_equal(rv, v) and np.array_equal(rf, f)
    cloud = read_ply(path)
    assert np.array_equal(cloud["points"], v) and np.array_equal(cloud["normals"], n)
    # without faces the file is what it was
    save_ply(str(tmp_path / "a.ply"), v, normals=n, binary=binary)
    save_ply(str(tmp_path / "b.ply"), v, normals=n, faces=None, binary=binary)
    assert open(tmp_path / "a.ply", "rb").read() == open(tmp_path / "b.ply", "rb").read()
    assert b"element face" not in open(tmp_path / "a.ply", "rb").read()[:300]
