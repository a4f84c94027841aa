"""GPU tests of normal estimation (ops.estimate_normals, csrc/normals.cu): the PCA against float64, its degenerate and
invalid rows, the forest, roots and oriented normals bit for bit against tests/normals_oracle.py from the device's own
unoriented normals, determinism and graph capture, orientation against true normals, Poisson reconstruction from
estimated normals, and the command line."""
import os

import numpy as np
import pytest
import torch

from dss_b200 import _lib
from dss_b200.core.cloud import PointClouds3D
from dss_b200.frnn_grid import knn_points_packed
from dss_b200.ops import estimate_normals, point_mesh_distance, poisson_reconstruction, sample_points_poisson_disk
from dss_b200.utils.create_mvr_data import ico_sphere
from dss_b200.utils.io import read_ply, save_ply
from tests import normals_oracle as no
from tests.test_mesh_data import torus

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "ply")
FIXTURES = ("sphere_2k", "bunny-8000", "teapot_normal_dense")


def _sphere(n, seed=0, centre=(0.0, 0.0, 0.0)):
    rng = np.random.default_rng(seed)
    p = rng.normal(size=(n, 3))
    return (p / np.linalg.norm(p, axis=1, keepdims=True) + np.asarray(centre)).astype(np.float32)


def _plane(n, seed=0, noise=1e-3):
    rng = np.random.default_rng(seed)
    p = np.concatenate([rng.uniform(-1, 1, (n, 2)), rng.normal(scale=noise, size=(n, 1))], 1)
    return (p @ np.linalg.qr(rng.normal(size=(3, 3)))[0]).astype(np.float32)    # a tilted plane


def _torus_mesh(dev):
    v, f = torus()
    return v.to(dev), f[:, [0, 2, 1]].to(dev)       # the helper's faces wind inwards


def _torus_samples(dev, n=3000):
    v, f = _torus_mesh(dev)
    s = sample_points_poisson_disk(v, f, n)
    return s.points, s.normals


CLOUDS = {
    "sphere": lambda dev: _sphere(2000),
    "torus": lambda dev: _torus_samples(dev)[0].cpu().numpy(),
    "plane": lambda dev: _plane(2000),
    "plane_1e-3": lambda dev: _plane(2000) * np.float32(1e-3),
    "plane_1e3": lambda dev: _plane(2000) * np.float32(1e3),
}


def _idx(pts, k):
    dev = pts.device
    first = torch.zeros(1, dtype=torch.int64, device=dev)
    num = torch.full((1,), pts.shape[0], dtype=torch.int64, device=dev)
    return knn_points_packed(pts, first, num, k, -1.0)[1].cpu().numpy()


# ---- PCA ------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("k", [3, 8, 20, 32])
@pytest.mark.parametrize("name", sorted(CLOUDS))
def test_pca_matches_float64(cuda_device, name, k):
    p = torch.from_numpy(CLOUDS[name](cuda_device)).to(cuda_device)
    est = estimate_normals(p, k=k, orient=False)
    n = est.normals.cpu().numpy()
    assert (est.root == -1).all() and (est.parent == -1).all()
    ref, lam = no.pca_normals(p.cpu().numpy(), _idx(p, k))
    gap = (lam[:, 1] - lam[:, 0]) > 1e-3 * lam[:, 2]
    assert gap.mean() > 0.5, name
    dots = np.abs(np.sum(n.astype(np.float64) * ref, 1))
    assert (dots[gap] >= 1 - 1e-6).all(), (name, k, dots[gap].min())
    assert np.array_equal(n, no.canonical(n))                       # the canonical sign, on the rounded values
    assert np.allclose(np.linalg.norm(n, axis=1), 1, atol=1e-6)


def test_packed_equals_alone(cuda_device):
    clouds = [_sphere(700, 1), _plane(1300, 2), _sphere(40, 3, (3, 0, 0))]
    pts = torch.from_numpy(np.concatenate(clouds)).to(cuda_device)
    num = torch.tensor([len(c) for c in clouds], dtype=torch.int64, device=cuda_device)
    first = torch.cumsum(num, 0) - num
    for orient in (False, True):
        packed = estimate_normals(pts, 20, orient, first, num)
        for c, f0 in zip(clouds, first.tolist()):
            alone = estimate_normals(torch.from_numpy(c).to(cuda_device), 20, orient)
            for a, b in zip(alone, packed):
                assert torch.equal(a, b[f0:f0 + len(c)])
    # the cloud object gives the same normals, padded, and can take them
    cloud = PointClouds3D([torch.from_numpy(c).to(cuda_device) for c in clouds])
    padded = cloud.estimate_normals(assign_to_self=True)
    assert padded.shape == (3, 1300, 3)
    assert torch.equal(cloud.normals_packed(), packed.normals)
    assert torch.equal(padded[1, :1300], packed.normals[700:2000])


# ---- edges ----------------------------------------------------------------------------------------------------------

def test_degenerate_rows(cuda_device):
    rng = np.random.default_rng(4)
    dup = np.tile(np.float32([[0.5, -1.0, 2.0]]), (30, 1))
    est = estimate_normals(torch.from_numpy(dup).to(cuda_device), k=8)
    assert (est.normals.cpu() == torch.tensor([0.0, 0.0, 1.0])).all()
    line = np.outer(rng.uniform(-1, 1, 50), [1.0, 2.0, -0.5]).astype(np.float32)
    est = estimate_normals(torch.from_numpy(line).to(cuda_device), k=8, orient=False)
    n = est.normals.cpu().numpy()
    d = np.float32([1.0, 2.0, -0.5]) / np.linalg.norm([1.0, 2.0, -0.5])
    assert np.isfinite(n).all() and np.abs(n @ d).max() < 1e-6
    # f2 x e_k with e_k the axis of the smallest |f2_k| (z here): the same normal on every row
    f = np.cross(d, [0.0, 0.0, 1.0])
    assert np.allclose(np.abs(n @ (f / np.linalg.norm(f))), 1, atol=1e-6)
    est2 = estimate_normals(torch.from_numpy(line).to(cuda_device), k=8, orient=False)
    assert torch.equal(est.normals, est2.normals)


def test_invalid_rows_small_clouds_and_arguments(cuda_device):
    p = _sphere(500, 5)
    p[[7, 300]] = np.nan
    p[100, 1] = np.inf
    est = estimate_normals(torch.from_numpy(p).to(cuda_device), k=20)
    bad = np.zeros(500, bool)
    bad[[7, 100, 300]] = True
    n, root, parent = (t.cpu().numpy() for t in est)
    assert np.isnan(n[bad]).all() and (root[bad] == -1).all() and (parent[bad] == -1).all()
    assert np.isfinite(n[~bad]).all() and (root[~bad] >= 0).all() and not np.isin(parent, np.nonzero(bad)[0]).any()
    assert (np.sum(n[~bad] * p[~bad], 1) > 0).all()
    # a cloud smaller than k, alone and packed next to a full one
    small = torch.from_numpy(_sphere(10, 6)).to(cuda_device)
    est = estimate_normals(small, k=20)
    assert torch.isnan(est.normals).all() and (est.root == -1).all() and (est.parent == -1).all()
    both = torch.cat([small, torch.from_numpy(_sphere(100, 7)).to(cuda_device)])
    num = torch.tensor([10, 100], dtype=torch.int64, device=cuda_device)
    est = estimate_normals(both, 20, True, torch.tensor([0, 10], device=cuda_device), num)
    assert torch.isnan(est.normals[:10]).all() and torch.isfinite(est.normals[10:]).all()
    assert int(est.root[10:].min()) >= 0 and int(est.root[10:].max()) < 100
    # empty
    est = estimate_normals(torch.zeros((0, 3), device=cuda_device))
    assert all(t.shape[0] == 0 for t in est)
    empty_packed = estimate_normals(both, 8, True, torch.tensor([0, 10], device=cuda_device),
                                    torch.tensor([0, 100], device=cuda_device))
    assert torch.isfinite(empty_packed.normals[10:]).all()
    for k in (2, 33, 0, 2.5, True):
        with pytest.raises(ValueError):
            estimate_normals(small, k=k)
    with pytest.raises(TypeError):
        estimate_normals(small.double())
    with pytest.raises(RuntimeError):
        estimate_normals(small.cpu())


# ---- exactness against the oracle -----------------------------------------------------------------------------------

def _exact_cases():
    out = {name: read_ply(os.path.join(GOLDEN, name + ".ply"))["points"] for name in FIXTURES}
    out["two_spheres"] = np.concatenate([_sphere(800, 8), _sphere(600, 9, (10.0, 0.0, -3.0))])
    return out


@pytest.mark.parametrize("name", list(FIXTURES) + ["two_spheres"])
@pytest.mark.parametrize("k", [8, 20])
def test_orientation_matches_oracle(cuda_device, name, k):
    p_np = _exact_cases()[name]
    p = torch.from_numpy(p_np).to(cuda_device)
    unoriented = estimate_normals(p, k=k, orient=False).normals.cpu().numpy()
    est = estimate_normals(p, k=k)
    ref = no.orient(p_np, unoriented, _idx(p, k))
    assert np.array_equal(est.normals.cpu().numpy(), ref["normals"])
    assert np.array_equal(est.root.cpu().numpy(), ref["root"])
    assert np.array_equal(est.parent.cpu().numpy(), ref["parent"])
    assert no.parent_edges(est.parent.cpu().numpy()) == {tuple(e) for e in ref["edges"].tolist()}
    if name == "two_spheres":
        assert len(np.unique(ref["root"])) == 2


def test_deterministic_and_capturable(cuda_device):
    p = torch.from_numpy(_sphere(50000, 10)).to(cuda_device)
    a, b = estimate_normals(p), estimate_normals(p)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    # the library call alone replays in a CUDA graph with the eager bits
    P, k = p.shape[0], 20
    first = torch.zeros(1, dtype=torch.int64, device=cuda_device)
    num = torch.full((1,), P, dtype=torch.int64, device=cuda_device)
    idx = knn_points_packed(p, first, num, k, -1.0)[1]
    out = (torch.empty((P, 3), device=cuda_device), torch.empty(P, dtype=torch.int32, device=cuda_device),
           torch.empty(P, dtype=torch.int32, device=cuda_device))
    call = lambda: _lib.call("dss_estimate_normals", cuda_device, p, first, num, 1, P, idx, k, 1, *out)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        call()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        call()
    for t in out:
        t.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(x, y) for x, y in zip(a, out))


def test_million_points(cuda_device):
    p = torch.from_numpy(_sphere(1_000_000, 11)).to(cuda_device)
    est = estimate_normals(p)
    assert (torch.sum(est.normals * p, 1) > 0).all()
    assert torch.unique(est.root).numel() == 1 and int((est.parent < 0).sum()) == 1


# ---- orientation quality --------------------------------------------------------------------------------------------

def test_outward_on_sphere_and_torus(cuda_device):
    for v, f in (ico_sphere(4), _torus_mesh(cuda_device)):
        s = sample_points_poisson_disk(v.to(cuda_device), f.to(cuda_device), 5000)
        n = estimate_normals(s.points).normals
        agree = torch.sum(n * s.normals, 1)
        assert (agree > 0).all(), float(agree.min())


# the share of normals agreeing in sign with the fixture's stored normals (k = 20) was first measured on an H100 80GB
# HBM3 as sphere 1.0000, bunny 0.9810, teapot 0.9301 (1001 points: the spout and handle are a few points thick); the
# thresholds sit a point below those first measurements
AGREE = {"sphere_2k": 1.0, "bunny-8000": 0.97, "teapot_normal_dense": 0.92}


@pytest.mark.parametrize("name", FIXTURES)
def test_agrees_with_fixture_normals(cuda_device, name):
    d = read_ply(os.path.join(GOLDEN, name + ".ply"))
    n = estimate_normals(torch.from_numpy(d["points"]).to(cuda_device)).normals.cpu().numpy()
    share = float(np.mean(np.sum(n * d["normals"], 1) > 0))
    print("%s: %.4f of the estimated normals agree in sign with the stored ones" % (name, share))
    assert share >= AGREE[name]


def test_poisson_from_estimated_normals(cuda_device):
    v, f = _torus_mesh(cuda_device)
    p, n_true = _torus_samples(cuda_device, 20000)
    n_est = estimate_normals(p).normals
    err = {}
    for key, n in (("true", n_true), ("estimated", n_est)):
        m = poisson_reconstruction(p, n, depth=7)
        err[key] = float(point_mesh_distance(m.verts, v, f).sq_dists.sqrt().mean())
    print("torus depth 7: mean vertex-to-torus distance %.3e with the true normals, %.3e with estimated ones"
          % (err["true"], err["estimated"]))
    # first measured on an H100: 4.88e-4 with the true normals, 5.92e-4 (1.21 x) with the estimated ones
    assert err["estimated"] <= 1.5 * err["true"]


# ---- command line ---------------------------------------------------------------------------------------------------

def test_cli(cuda_device, tmp_path):
    from dss_b200.utils.normals import main
    d = read_ply(os.path.join(GOLDEN, "bunny-8000.ply"))
    src = str(tmp_path / "bunny.xyz")
    np.savetxt(src, d["points"], fmt="%.9g")
    ply_src = str(tmp_path / "bunny_with_normals.ply")
    save_ply(ply_src, d["points"], normals=-d["normals"])          # normals in the input are ignored
    api = estimate_normals(torch.from_numpy(d["points"]).to(cuda_device), k=12).normals.cpu().numpy()
    for i, inp in enumerate((src, ply_src)):
        out, mesh = str(tmp_path / ("out%d.ply" % i)), str(tmp_path / ("mesh%d.obj" % i))
        assert main([inp, out, "--k", "12", "--mesh", mesh, "--depth", "6"]) == 0
        got = read_ply(out)
        assert np.array_equal(got["points"], d["points"]) and np.array_equal(got["normals"], api)
        assert os.path.getsize(mesh) > 0
    out = str(tmp_path / "plain.ply")
    assert main([src, out, "--no-orient"]) == 0
    plain = estimate_normals(torch.from_numpy(d["points"]).to(cuda_device), orient=False).normals.cpu().numpy()
    assert np.array_equal(read_ply(out)["normals"], plain)
