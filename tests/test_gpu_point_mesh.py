"""GPU: point_mesh_distance (csrc/mesh_distance.cu) against the float64 oracle of tests/point_mesh_oracle.py on several
meshes and query sets, its edges, determinism and face-order independence; evaluate_cloud and the evaluation CLI; the
exact p2f metric against the sampled chamfer proxy; and the training loop selecting by p2f_avg."""
import csv
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

from dss_b200.ops import chamfer_distance, point_mesh_distance
from dss_b200.utils.create_mvr_data import ico_sphere, sample_points_from_mesh
from dss_b200.utils.io import read_ply, save_obj, save_ply
from tests.point_mesh_oracle import point_mesh_distance as oracle
from tests.test_mesh_data import torus

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def ulps(a, b):
    """|a - b| in float32 units in the last place, for non-negative finite a, b"""
    return (a.view(torch.int32).long() - b.view(torch.int32).long()).abs()


def tmax(t):
    return float(t.max()) if t.numel() else 0.0


def check(q, verts, faces, dev, subset=None):
    """the kernel against the oracle on the device; returns the kernel's result"""
    r = point_mesh_distance(q, verts, faces, return_closest=True)
    qs = q if subset is None else q[subset]
    sq, fi, cl = (r.sq_dists, r.face_idx, r.closest) if subset is None else (
        r.sq_dists[subset], r.face_idx[subset], r.closest[subset])
    o_sq, o_face, o_cl, o_second = oracle(qs, verts, faces)
    nan = torch.isnan(o_sq)
    assert torch.equal(torch.isnan(sq), nan) and torch.equal(fi[nan], torch.full_like(fi[nan], -1))
    assert torch.isnan(cl[nan]).all()
    ok = ~nan
    assert tmax(ulps(sq[ok], o_sq[ok].float())) <= 2
    clear = ok & (torch.isinf(o_second) | (o_second - o_sq > 1e-9 * o_second))
    assert torch.equal(fi[clear], o_face[clear])
    v = verts.double()
    fin = torch.isfinite(v).all(1)
    diag = float((v[fin].max(0).values - v[fin].min(0).values).norm()) if fin.any() else 1.0
    same = ok & (fi == o_face)
    assert tmax((cl[same].double() - o_cl[same]).abs()) <= 1e-6 * diag
    return r


def soup(dev, n=600, seed=0):
    """random triangles in [-1, 1]^3 with slivers, huge and tiny faces"""
    g = torch.Generator().manual_seed(seed)
    c = torch.rand(n, 1, 3, generator=g) * 2 - 1
    tri = c + (torch.rand(n, 3, 3, generator=g) - 0.5) * 0.2
    tri[:50, 2] = tri[:50, 0] + (tri[:50, 1] - tri[:50, 0]) * 0.5 + 1e-5 * torch.randn(50, 3, generator=g)  # slivers
    tri[50:55] = c[50:55] + (torch.rand(5, 3, 3, generator=g) - 0.5) * 20                                    # huge
    tri[55:105] = c[55:105] + (torch.rand(50, 3, 3, generator=g) - 0.5) * 1e-5                              # tiny
    return tri.reshape(-1, 3).to(dev), torch.arange(3 * n).reshape(n, 3).to(dev)


def degenerate_mesh(dev):
    v, f = torus()
    f = f.clone()
    f[::7, 1] = f[::7, 0]                         # repeated vertices
    f[3::11] = f[3::11, :1].repeat(1, 3)          # points
    v = torch.cat([v, torch.tensor([[0.0, 0.0, 0.0], [0.5, 0.0, 0.0], [1.0, 0.0, 0.0]])])
    n = v.shape[0]
    f = torch.cat([f, torch.tensor([[n - 3, n - 2, n - 1], [n - 1, n - 3, n - 2]])])       # collinear
    return v.to(dev), f.to(dev)


MESHES = {
    "torus": lambda dev: tuple(t.to(dev) for t in torus()),
    "ico4": lambda dev: tuple(t.to(dev) for t in ico_sphere(4)),
    "soup": soup,
    "degenerate": degenerate_mesh,
}


def queries(kind, verts, faces, dev, n=3000, seed=1):
    g = torch.Generator(device=dev).manual_seed(seed)
    lo, hi = verts.min(0).values, verts.max(0).values
    diag = float((hi - lo).norm())
    if kind == "surface":
        return sample_points_from_mesh(verts, faces.long(), n, generator=g)[0]
    if kind == "vertices":
        return verts.clone()
    if kind == "box":
        return lo + (hi - lo) * torch.rand(n, 3, device=dev, generator=g)
    # far: random directions at 1 to 10^3 box diagonals from the box centre
    d = torch.randn(n, 3, device=dev, generator=g)
    r = diag * 10 ** (3 * torch.rand(n, 1, device=dev, generator=g))
    return ((lo + hi) / 2 + d / d.norm(dim=1, keepdim=True) * r).float()


@pytest.mark.parametrize("mesh", sorted(MESHES))
@pytest.mark.parametrize("kind", ["surface", "vertices", "box", "far"])
def test_against_oracle(cuda_device, mesh, kind):
    verts, faces = MESHES[mesh](cuda_device)
    q = queries(kind, verts, faces, cuda_device)
    r = check(q, verts, faces, cuda_device)
    if kind == "surface" or (kind == "vertices" and mesh != "degenerate"):
        assert float(r.sq_dists.max()) <= 1e-12          # d <= 1e-6


def test_edges(cuda_device):
    dev = cuda_device
    v, f = (t.to(dev) for t in torus())
    q = torch.randn(100, 3, device=dev)
    r = point_mesh_distance(q[:0], v, f, return_closest=True)
    assert r.sq_dists.shape == (0,) and r.face_idx.shape == (0,) and r.closest.shape == (0, 3)
    r = point_mesh_distance(q, v, f[:0])                                          # F = 0
    assert torch.isnan(r.sq_dists).all() and (r.face_idx == -1).all() and r.closest is None
    check(q, v, f[5:6], dev)                                                      # one face
    bad = q.clone()
    bad[::3, 0], bad[1::3, 2], bad[2::9, 1] = float("nan"), float("inf"), -float("inf")
    r = check(bad, v, f, dev)
    assert torch.isnan(r.sq_dists[::3]).all() and (r.face_idx[1::3] == -1).all()
    # faces on non-finite vertices are never nearest and do not shape the grid
    v2 = torch.cat([v, torch.tensor([[float("nan"), 0, 0], [1e30, float("inf"), 0]], device=dev)])
    n = v.shape[0]
    f2 = torch.cat([f, torch.tensor([[n, 0, 1], [2, n + 1, 3], [n, n + 1, 4]], device=dev)])
    r2 = check(q, v2, f2, dev)
    r1 = point_mesh_distance(q, v, f)
    assert torch.equal(r2.sq_dists, r1.sq_dists) and torch.equal(r2.face_idx, r1.face_idx)
    r = point_mesh_distance(q, v2, f2[-3:])                                       # no usable face at all
    assert torch.isnan(r.sq_dists).all() and (r.face_idx == -1).all()
    # int64 and int32 faces alike; an index out of range raises
    r3 = point_mesh_distance(q, v, f.int())
    assert torch.equal(r3.sq_dists, r1.sq_dists) and r3.face_idx.dtype == torch.int64
    for badf in (f.clone().index_fill_(0, torch.tensor([7], device=dev), n), f.clone().index_fill_(0, torch.tensor([7], device=dev), -1)):
        with pytest.raises(ValueError):
            point_mesh_distance(q, v, badf)
    with pytest.raises(RuntimeError):
        point_mesh_distance(q.requires_grad_(True), v, f)


def test_at_scale(cuda_device):
    sys.path.insert(0, os.path.join(ROOT, "scripts"))
    from mesh_raster_time import displaced_sphere
    dev = cuda_device
    v, f = (t.to(dev) for t in displaced_sphere())
    assert f.shape[0] > 600_000
    g = torch.Generator(device=dev).manual_seed(5)
    surf = sample_points_from_mesh(v, f, 100_000, generator=g)[0]
    box = (torch.rand(100_000, 3, device=dev, generator=g) * 2.2 - 1.1)
    q = torch.cat([surf, box])
    sub = torch.randperm(q.shape[0], generator=torch.Generator().manual_seed(6))[:2000].to(dev)
    r = check(q, v, f, dev, subset=sub)
    assert float(r.sq_dists[:100_000].max()) <= 1e-12


def test_deterministic_and_face_order(cuda_device):
    dev = cuda_device
    v, f = (t.to(dev) for t in ico_sphere(4))
    g = torch.Generator(device=dev).manual_seed(2)
    q = torch.cat([queries("box", v, f, dev, 5000), queries("surface", v, f, dev, 5000), v])
    a = point_mesh_distance(q, v, f, return_closest=True)
    b = point_mesh_distance(q, v, f, return_closest=True)
    assert torch.equal(a.sq_dists, b.sq_dists) and torch.equal(a.face_idx, b.face_idx)
    assert torch.equal(a.closest, b.closest)
    perm = torch.randperm(f.shape[0], device=dev, generator=g)
    c = point_mesh_distance(q, v, f[perm])
    assert torch.equal(c.sq_dists, a.sq_dists)
    o_sq, _, _, second = oracle(q, v, f)
    clear = second > o_sq
    assert torch.equal(perm[c.face_idx][clear], a.face_idx[clear])
    assert (~clear).any()              # the vertices are exact ties between their faces


def test_evaluate_cloud(cuda_device):
    from dss_b200.utils.evaluate import evaluate_cloud
    dev = cuda_device
    v, f = (t.to(dev) for t in torus())
    g = torch.Generator(device=dev).manual_seed(3)
    gt = sample_points_from_mesh(v, f, 3000, generator=g)[0]
    pred = sample_points_from_mesh(v, f, 2000, generator=g)[0] + 0.01 * torch.randn(2000, 3, device=dev, generator=g)
    s = evaluate_cloud(pred, gt, (v, f))
    d = torch.cdist(pred.double(), gt.double()) ** 2
    fwd, bwd = d.min(1).values, d.min(0).values
    assert torch.allclose(s.cd_forward.double(), fwd, rtol=1e-5, atol=1e-12)
    assert torch.allclose(s.cd_backward.double(), bwd, rtol=1e-5, atol=1e-12)
    assert s.CD == pytest.approx(float(fwd.mean() + bwd.mean()), rel=1e-5)
    assert s.hausdorff == pytest.approx(float(fwd.max() + bwd.max()), rel=1e-5)
    p2f = oracle(pred, v, f)[0].float().double().sqrt()
    assert torch.equal(s.p2f, p2f)
    assert s.p2f_avg == pytest.approx(float(p2f.mean()), rel=1e-12)
    assert s.p2f_std == pytest.approx(float(p2f.std(unbiased=False)), rel=1e-12)
    assert s.cd_forward_mean + s.cd_backward_mean == pytest.approx(s.CD, rel=1e-15)


def test_cli_end_to_end(cuda_device, tmp_path):
    from dss_b200.utils.evaluate import evaluate_cloud
    dev = cuda_device
    v, f = torus()
    save_obj(str(tmp_path / "mesh.obj"), v.numpy(), f.numpy())
    vd, fd = v.to(dev), f.to(dev)
    g = torch.Generator(device=dev).manual_seed(4)
    gt = sample_points_from_mesh(vd, fd, 4000, generator=g)[0]
    save_ply(str(tmp_path / "gt.ply"), gt.cpu().numpy())
    preds = {}
    for i, noise in enumerate((0.0, 0.003, 0.01)):
        p = sample_points_from_mesh(vd, fd, 1500, generator=g)[0] + noise * torch.randn(1500, 3, device=dev, generator=g)
        preds["p%d" % i] = p
        save_ply(str(tmp_path / "pred" / ("p%d.ply" % i)), p.cpu().numpy())
    env = dict(os.environ)
    env["PYTHONPATH"] = ROOT + os.pathsep + env.get("PYTHONPATH", "")
    r = subprocess.run([sys.executable, "-m", "dss_b200.utils.evaluate", "--gt", str(tmp_path / "gt.ply"), "--pred",
                        str(tmp_path / "pred"), "--name", "*.ply", "--mesh", str(tmp_path / "mesh.obj")], cwd=ROOT,
                       env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0, r.stdout
    with open(tmp_path / "pred" / "evaluation.csv") as fh:
        rows = list(csv.DictReader(fh))
    assert [row["name"] for row in rows] == ["p0.ply", "p1.ply", "p2.ply", "-"]
    all_p2f = []
    for row in rows[:3]:
        name = row["name"][:-4]
        p = torch.from_numpy(read_ply(str(tmp_path / "pred" / row["name"]))["points"]).to(dev)
        s = evaluate_cloud(p, gt, (vd, fd))
        assert float(row["CD"]) == s.CD and float(row["hausdorff"]) == s.hausdorff
        assert float(row["p2f avg"]) == pytest.approx(s.p2f_avg, rel=1e-12)
        assert float(row["p2f std"]) == pytest.approx(s.p2f_std, rel=1e-12)
        xyz = np.loadtxt(str(tmp_path / "pred" / (name + "_point2mesh_distance.xyz")), ndmin=2)
        d = point_mesh_distance(p, vd, fd).sq_dists.double().sqrt().cpu().numpy()
        assert np.array_equal(xyz[:, 3], d) and np.array_equal(xyz[:, :3].astype(np.float32), p.cpu().numpy())
        all_p2f.append(d)
        for suffix in ("_cdF.ply", "_cdB.ply"):
            assert read_ply(str(tmp_path / "pred" / (name + suffix)))["colors"] is not None
    assert float(rows[3]["p2f avg"]) == pytest.approx(float(np.nanmean(np.concatenate(all_p2f))), rel=1e-12)
    assert "pred" in r.stdout


@pytest.fixture(scope="module")
def data_dir(cuda_device, tmp_path_factory):
    from dss_b200.utils.create_mvr_data import main
    tmp = tmp_path_factory.mktemp("p2f_data")
    verts, faces = torus()
    mesh = tmp / "torus.obj"
    save_obj(str(mesh), verts.numpy(), faces.numpy())
    return main(["--points", str(mesh), "--output", str(tmp / "data"), "--num_cameras", "16", "--image-size", "128",
                 "--tri_color_light", "--point_lights", "--seed", "3"])[0]


def test_exact_metric_versus_sampled_proxy(data_dir, cuda_device):
    """a cloud ON the mesh: exact p2f ~ 0, while the loop's chamfer proxy against 8000 samples stays well above 0"""
    from dss_b200.training.train import ground_truth_cloud
    from dss_b200.utils.dataset import MVRData
    from dss_b200.utils.evaluate import p2f_stats
    from dss_b200.utils.io import read_mesh
    dev = cuda_device
    v, f = read_mesh(os.path.join(data_dir, "mesh.obj"))
    v, f = torch.from_numpy(v).float().to(dev), torch.from_numpy(f).to(dev)
    cloud, nrm = sample_points_from_mesh(v, f.long(), 2000, generator=torch.Generator(device=dev).manual_seed(9))
    _, avg, _ = p2f_stats(cloud, (v, f))
    gt = ground_truth_cloud(MVRData(data_dir), data_dir, 8000, dev)
    cd, _ = chamfer_distance(gt[0][None], cloud[None])
    print("cloud on the mesh: p2f avg %.3g, chamfer_point %.3g" % (avg, float(cd)))
    assert avg <= 1e-6
    assert float(cd) > 1e3 * max(avg, 1e-9) and float(cd) > 1e-5


def test_loop_selects_by_p2f(data_dir, cuda_device, tmp_path):
    from tests.test_gpu_train_loop import run_cli, write_config
    from dss_b200.training.config import load_config
    from dss_b200.training.train import Trainer, initial_cloud
    from dss_b200.utils.evaluate import p2f_stats
    from dss_b200.utils.io import read_mesh
    dev = cuda_device
    cfg = write_config(tmp_path / "c.yml", data_dir, tmp_path / "out", model_selection_metric="p2f_avg")
    code, log = run_cli(cfg, "--max-it", "1000")
    assert code == 0, log
    assert '"p2f_avg"' in log and '"p2f_std"' in log
    out = tmp_path / "out" / "torus"
    best = torch.load(out / "model_best.pt", map_location="cpu", weights_only=False)
    v, f = read_mesh(os.path.join(data_dir, "mesh.obj"))
    mesh = (torch.from_numpy(v).float().to(dev), torch.from_numpy(f).to(dev))
    ply = torch.from_numpy(read_ply(str(out / "val" / "best.ply"))["points"]).to(dev)
    _, again, _ = p2f_stats(ply, mesh)
    assert again == best["loss_val_best"]
    _, init, _ = p2f_stats(initial_cloud(2000, 0, dev)[0], mesh)
    print("p2f_avg: initial %.5f, best %.5f (%.3fx) at it %d" % (init, again, again / init, best["it"]))
    # the mean is held up by a tail of points the image losses do not move (p2f_std stays ~0.13): 0.60x at it 800
    assert again <= 0.7 * init
    # a data directory without mesh.obj fails at start-up
    bare = tmp_path / "bare"
    shutil.copytree(data_dir, bare)
    os.remove(bare / "mesh.obj")
    with pytest.raises(ValueError, match="mesh.obj"):
        Trainer(load_config(write_config(tmp_path / "b.yml", str(bare), tmp_path / "out_b",
                                         model_selection_metric="p2f_avg")))
