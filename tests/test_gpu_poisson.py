"""GPU: screened Poisson reconstruction (csrc/poisson.cu) against the float64 oracle of tests/poisson_oracle.py at
depths 3 to 5 on the golden clouds; marching tetrahedra bit for bit against the numpy oracle; closed, accurate meshes
at depth 8 from 200k samples of a sphere and a torus; determinism, input order, unusable rows and degenerate input;
and the generation export on a cloud from a short training run."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import yaml

from dss_b200.ops import marching_tetrahedra, point_mesh_distance, poisson_reconstruction
from dss_b200.utils.create_mvr_data import ico_sphere, sample_points_from_mesh
from dss_b200.utils.io import read_mesh, read_ply
from tests import poisson_oracle as po
from tests.test_mesh_data import torus

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = ["sphere_2k", "bunny-8000", "teapot_normal_dense"]


def golden(name):
    d = read_ply(os.path.join(ROOT, "tests", "golden", "ply", name + ".ply"))
    return d["points"], d["normals"]


def same(a, b):
    return a.shape == b.shape and torch.equal(a.cpu(), b.cpu() if torch.is_tensor(b) else torch.from_numpy(b))


@pytest.mark.parametrize("name", GOLDEN)
@pytest.mark.parametrize("depth", [3, 4, 5])
def test_solve_matches_oracle(cuda_device, name, depth):
    p, n = golden(name)
    m = poisson_reconstruction(torch.from_numpy(p).to(cuda_device), torch.from_numpy(n).to(cuda_device), depth=depth,
                               return_grid=True)
    ok, c, L = po.domain(p, n)
    assert np.array_equal(m.origin.numpy(), c) and np.float32(m.side) == L
    R = 1 << depth
    chi, _ = po.solve(p, n, R)
    g = m.grid.double().cpu().numpy().reshape(-1)
    err = np.abs(g - chi).max() / (chi.max() - chi.min())
    print("poisson %s depth %d: max |chi - oracle| / range = %.2e, %d iterations, residual %.2e"
          % (name, depth, err, m.iterations, m.residual))
    assert err < 1e-4
    assert m.residual <= 1e-6 and m.iterations > 0
    # and the extraction of the kernel's own chi, bit for bit
    v, f = po.marching_tetrahedra(m.grid.cpu().numpy(), m.origin.numpy(), m.side)
    assert same(m.verts, v) and same(m.faces, f)


def analytic(kind, R):
    x = np.arange(R + 1, dtype=np.float64) / R - 0.5
    X, Y, Z = np.meshgrid(x, x, x, indexing="ij")
    if kind == "sphere":
        return (np.sqrt((X - 0.03) ** 2 + (Y + 0.02) ** 2 + Z ** 2) - 0.31).astype(np.float32)
    if kind == "torus":
        return ((np.sqrt(X ** 2 + Y ** 2) - 0.25) ** 2 + Z ** 2 - 0.1 ** 2).astype(np.float32)
    # integer steps: exact zeros on many nodes and edges that end on them
    return np.round(8 * (np.abs(X) + np.abs(Y - 0.1) + np.abs(Z)) - 2.0).astype(np.float32)


@pytest.mark.parametrize("kind", ["sphere", "torus", "zeros"])
@pytest.mark.parametrize("R", [7, 32])
def test_extraction_matches_oracle(cuda_device, kind, R):
    chi = analytic(kind, R)
    c, L = np.array([0.25, -3.0, 1.5], np.float32), np.float32(1.7)
    v, f = marching_tetrahedra(torch.from_numpy(chi).to(cuda_device), c, L)
    ov, of = po.marching_tetrahedra(chi, c, L)
    assert len(of) > 0
    assert same(v, ov) and same(f, of)
    assert po.closed_manifold(of)


def test_extraction_empty_and_nan(cuda_device):
    v, f = marching_tetrahedra(torch.ones(9, 9, 9, device=cuda_device), (0, 0, 0), 1.0)
    assert v.shape == (0, 3) and f.shape == (0, 3)
    g = torch.from_numpy(analytic("sphere", 8)).to(cuda_device)
    g[0, 0, 0] = float("nan")             # NaN is outside, like the positive corner it replaces
    v, f = marching_tetrahedra(g, (0, 0, 0), 1.0)
    ov, of = po.marching_tetrahedra(g.cpu().numpy(), np.zeros(3, np.float32), 1.0)
    assert same(v, ov) and same(f, of)


def sphere_mesh():
    return ico_sphere(6)


def torus_mesh():
    v, f = torus()
    return v, f[:, [0, 2, 1]]       # the helper's faces wind inwards


@pytest.mark.parametrize("kind,euler", [("sphere", 2), ("torus", 0)])
def test_depth8_end_to_end(cuda_device, kind, euler):
    verts, faces = sphere_mesh() if kind == "sphere" else torus_mesh()
    verts, faces = verts.to(cuda_device), faces.to(cuda_device)
    gen = torch.Generator(device=cuda_device).manual_seed(0)
    p, n = sample_points_from_mesh(verts, faces, 200000, generator=gen)
    m = poisson_reconstruction(p, n, depth=8)
    f = m.faces.cpu().numpy()
    v = m.verts.cpu().numpy()
    assert po.closed_manifold(f)
    assert po.euler_characteristic(v, f) == euler
    vol, src = po.signed_volume(v, f), po.signed_volume(verts.cpu().numpy(), faces.cpu().numpy())
    h = m.side / 256
    d_out = point_mesh_distance(m.verts, verts, faces).sq_dists.sqrt()
    d_in = point_mesh_distance(p, m.verts, m.faces).sq_dists.sqrt()
    print("poisson depth 8 %s: %d verts %d faces, volume %.5f vs %.5f (%.3f%%), mesh->source max %.3f h mean %.4f h, "
          "samples->mesh max %.3f h mean %.4f h, %d iterations, residual %.2e"
          % (kind, len(v), len(f), vol, src, 100 * (vol - src) / src, float(d_out.max()) / h, float(d_out.mean()) / h,
             float(d_in.max()) / h, float(d_in.mean()) / h, m.iterations, m.residual))
    assert abs(vol - src) < 0.01 * src
    assert float(d_out.max()) < h and float(d_out.mean()) < 0.1 * h
    assert float(d_in.mean()) < 0.1 * h


def test_determinism_order_and_unusable_rows(cuda_device):
    verts, faces = sphere_mesh()
    gen = torch.Generator().manual_seed(1)
    p, n = sample_points_from_mesh(verts, faces, 20000, generator=gen)
    n = n * (0.5 + torch.rand(n.shape[0], 1, generator=gen))           # not unit
    p, n = p.to(cuda_device), n.to(cuda_device)
    a = poisson_reconstruction(p, n, depth=6, return_grid=True)
    b = poisson_reconstruction(p, n, depth=6, return_grid=True)
    assert torch.equal(a.grid, b.grid) and torch.equal(a.verts, b.verts) and torch.equal(a.faces, b.faces)
    assert a.iterations == b.iterations and a.residual == b.residual
    perm = torch.randperm(p.shape[0], generator=gen).to(cuda_device)
    c = poisson_reconstruction(p[perm], n[perm], depth=6, return_grid=True)
    assert torch.equal(a.grid, c.grid) and torch.equal(a.verts, c.verts) and torch.equal(a.faces, c.faces)
    nan, inf = float("nan"), float("inf")
    junk_p = torch.tensor([[nan, 0, 0], [inf, 0, 0], [5, 5, 5], [0, 0, 0], [-7, 2, 1], [0.1, 0.2, 0.3]])
    junk_n = torch.tensor([[1, 0, 0], [0, 1, 0], [0, 0, 0], [nan, 0, 0], [0, -inf, 0], [0, 0, 0]])
    pp = torch.cat([junk_p[:3].to(cuda_device), p, junk_p[3:].to(cuda_device)])
    nn = torch.cat([junk_n[:3].to(cuda_device), n, junk_n[3:].to(cuda_device)])
    d = poisson_reconstruction(pp, nn, depth=6, return_grid=True)
    assert torch.equal(a.grid, d.grid) and torch.equal(a.verts, d.verts) and torch.equal(a.faces, d.faces)
    assert torch.equal(a.origin, d.origin) and a.side == d.side


def test_degenerate_input(cuda_device):
    e = poisson_reconstruction(torch.zeros(0, 3, device=cuda_device), torch.zeros(0, 3, device=cuda_device), depth=5)
    assert e.verts.shape == (0, 3) and e.faces.shape == (0, 3) and e.iterations == 0
    one = torch.tensor([[0.3, -0.2, 1.0]], device=cuda_device).repeat(50, 1)
    nrm = torch.randn(50, 3, generator=torch.Generator().manual_seed(0)).to(cuda_device)
    e = poisson_reconstruction(one, nrm, depth=5, return_grid=True)
    assert e.verts.shape == (0, 3) and e.faces.shape == (0, 3) and e.side == 0.0
    assert (e.grid == 1).all()
    bad = torch.full((10, 3), float("nan"), device=cuda_device)
    e = poisson_reconstruction(bad, bad, depth=4)
    assert e.verts.shape == (0, 3) and e.faces.shape == (0, 3)
    with pytest.raises(RuntimeError, match="no backward"):
        poisson_reconstruction(one.clone().requires_grad_(True), nrm, depth=4)
    with pytest.raises(ValueError):
        poisson_reconstruction(one, nrm, depth=10)


@pytest.fixture(scope="module")
def data_dir(cuda_device, tmp_path_factory):
    from dss_b200.utils.create_mvr_data import main
    from dss_b200.utils.io import save_obj
    tmp = tmp_path_factory.mktemp("generate_data")
    verts, faces = torus()
    mesh = tmp / "torus.obj"
    save_obj(str(mesh), verts.numpy(), faces.numpy())
    return main(["--points", str(mesh), "--output", str(tmp / "data"), "--num_cameras", "16", "--image-size", "128",
                 "--tri_color_light", "--point_lights", "--seed", "3"])[0]


def run(module, *args):
    env = dict(os.environ)
    env["PYTHONPATH"] = ROOT + os.pathsep + env.get("PYTHONPATH", "")
    r = subprocess.run([sys.executable, "-m", module, *args], cwd=ROOT, env=env, stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=1200)
    return r.returncode, r.stdout


def test_generate_cli(data_dir, tmp_path):
    from dss_b200.utils.generate import load_cloud
    from tests.test_gpu_train_loop import write_config
    cfg_path = write_config(tmp_path / "c.yml", data_dir, tmp_path / "out")
    code, log = run("dss_b200.training.train", "--config", cfg_path, "--max-it", "101")
    assert code == 0, log
    out = tmp_path / "out" / "torus"
    assert (out / "model_best.pt").exists()
    points, normals, colours = load_cloud(str(out / "model_best.pt"), torch.device("cuda:0"))
    m = poisson_reconstruction(points, normals, depth=7)
    assert len(m.faces) > 0
    with open(cfg_path) as f:
        cfg = yaml.safe_load(f)
    for ext in ("ply", "obj"):
        cfg["generation"] = {"mesh_extension": ext, "generation_dir": "gen_" + ext, "with_colors": ext == "ply"}
        with open(cfg_path, "w") as f:
            yaml.safe_dump(cfg, f)
        code, log = run("dss_b200.utils.generate", "--config", cfg_path, "--depth", "7")
        assert code == 0, log
        cloud = read_ply(str(out / ("gen_" + ext) / "pointcloud.ply"))
        assert np.array_equal(cloud["points"], points.cpu().numpy())
        assert np.array_equal(cloud["normals"], normals.cpu().numpy())
        assert (cloud["colors"] is not None) == (ext == "ply")
        v, f = read_mesh(str(out / ("gen_" + ext) / ("mesh." + ext)))
        assert np.array_equal(v, m.verts.cpu().numpy()) and np.array_equal(f, m.faces.cpu().numpy())
