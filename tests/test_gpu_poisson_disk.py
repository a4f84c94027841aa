"""GPU: sample_points_poisson_disk (csrc/mesh_sample.cu) against the numpy rule of tests/poisson_disk_oracle.py -- bit
for bit with the Euclidean distance, as sets with the geodesic one -- its edges, its determinism and its counts; then
its callers: MVRData.get_pointclouds(num_points), the training loop's eval_sampling and evaluate --gt-samples."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from dss_b200 import _lib
from dss_b200.ops import point_mesh_distance, poisson_disk_stats, sample_points_poisson_disk
from dss_b200.utils.io import read_ply, save_obj
from tests import poisson_disk_oracle as pd
from tests.test_mesh_data import icosphere, torus

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def bits(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float32)).view(np.int32)


def raw(verts, faces, N, geodesic=False, seed=0, max_out=None, fill=0.0):
    """the C entry point without the Python checks (faces may hold any index): (rc, points, normals, n, radius)"""
    dev = torch.device("cuda", torch.cuda.current_device())
    v = torch.as_tensor(np.asarray(verts, np.float32)).reshape(-1, 3).to(dev).contiguous()
    f = torch.as_tensor(np.asarray(faces, np.int64)).reshape(-1, 3).to(torch.int32).to(dev).contiguous()
    cap = 20 * N if max_out is None else max_out
    pts = torch.full((max(cap, 1), 3), fill, dtype=torch.float32, device=dev)
    nrm = torch.full((max(cap, 1), 3), fill, dtype=torch.float32, device=dev)
    n, r = C.c_int64(-1), C.c_double(-1.0)
    rc = _lib.load().dss_sample_mesh_poisson_disk(_lib.ctx(dev), _lib.ptr(v), v.shape[0], _lib.ptr(f), f.shape[0], N,
                                                  int(geodesic), seed, _lib.ptr(pts), _lib.ptr(nrm), cap,
                                                  C.byref(n), C.byref(r), _lib.stream_ptr(dev))
    torch.cuda.synchronize()
    k = max(n.value, 0) if rc == 0 else 0
    return rc, pts[:k].cpu().numpy(), nrm[:k].cpu().numpy(), n.value, r.value, pts.cpu().numpy()


def op(verts, faces, N, geodesic=False, seed=0):
    dev = torch.device("cuda", torch.cuda.current_device())
    s = sample_points_poisson_disk(torch.as_tensor(np.asarray(verts, np.float32)).to(dev),
                                   torch.as_tensor(np.asarray(faces, np.int64)).to(dev), N, geodesic=geodesic,
                                   seed=seed)
    return s.points.cpu().numpy(), s.normals.cpu().numpy(), s.radius


def np_mesh(m):
    return m[0].numpy(), m[1].numpy()


def soup():
    """icosphere(2) with zero-area, NaN-vertex and out-of-range faces spread through its faces"""
    v, f = np_mesh(icosphere(2))
    V = len(v)
    v = np.concatenate([v, [[np.nan, 0.0, 0.0], [0.5, 0.5, np.inf], [2.0, 2.0, 2.0]]]).astype(np.float32)
    junk = np.array([[0, 0, 1], [3, 3, 3], [V, 1, 2], [4, V + 1, 5], [V + 2, V + 2, 7], [0, 1, V + 3],
                     [-1, 2, 3], [6, 7, 2 ** 31 - 1]])
    out = []
    for i, face in enumerate(f):
        out.append(face)
        if i % 97 == 0:
            out.append(junk[(i // 97) % len(junk)])
    return v, np.asarray(out), (v[:V], f)


CASES = {
    "ico3": (lambda: np_mesh(icosphere(3)), 500),
    "torus": (lambda: np_mesh(torus()), 1000),
    "single_face": (lambda: (np.array([[0, 0, 0], [1, 0, 0], [0.3, 0.8, 0]], np.float32), np.array([[0, 1, 2]])), 200),
    "n1": (lambda: np_mesh(torus()), 1),
    "offset": (lambda: (np_mesh(icosphere(3))[0] + np.float32(1e4), np_mesh(icosphere(3))[1]), 400),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_euclidean_equals_the_oracle_bit_for_bit(case, cuda_device):
    make, N = CASES[case]
    v, f = make()
    want = pd.sample(v, f, N, seed=11)
    p, n, r = op(v, f, N, seed=11)
    assert r == want["radius"], (r, want["probes"])
    assert np.array_equal(bits(p), bits(want["points"])) and np.array_equal(bits(n), bits(want["normals"]))
    assert abs(len(p) - N) <= N // 200
    if N == 1:
        assert len(p) == 1
    stats = poisson_disk_stats()
    assert [(a, b) for a, b in zip(stats["radii"], stats["counts"])] == want["probes"]


def test_unusable_faces_change_no_bit(cuda_device):
    v, f, (v0, f0) = soup()
    want = pd.sample(v, f, 300, seed=4)
    clean = op(v0, f0, 300, seed=4)
    rc, p, n, count, r, _ = raw(v, f, 300, seed=4)
    assert rc == 0 and count == len(p)
    assert np.array_equal(bits(p), bits(want["points"])) and np.array_equal(bits(n), bits(want["normals"]))
    assert r == want["radius"] == clean[2]
    assert np.array_equal(bits(p), bits(clean[0])) and np.array_equal(bits(n), bits(clean[1]))


def test_repeatable_and_seeded(cuda_device):
    v, f = np_mesh(torus())
    a, b, c = op(v, f, 2000, seed=1), op(v, f, 2000, seed=1), op(v, f, 2000, seed=2)
    assert np.array_equal(bits(a[0]), bits(b[0])) and np.array_equal(bits(a[1]), bits(b[1])) and a[2] == b[2]
    common = set(map(tuple, bits(a[0]).tolist())) & set(map(tuple, bits(c[0]).tolist()))
    assert len(common) < len(a[0]) // 10


def test_samples_lie_on_the_surface(cuda_device):
    dev = cuda_device
    for v, f in (np_mesh(torus()), np_mesh(icosphere(4)), (np_mesh(icosphere(3))[0] + np.float32(1e4),
                                                          np_mesh(icosphere(3))[1])):
        s = sample_points_poisson_disk(torch.from_numpy(v).to(dev), torch.from_numpy(f).to(dev), 3000)
        d = point_mesh_distance(s.points, torch.from_numpy(v).to(dev), torch.from_numpy(f).to(dev)).sq_dists
        extent = float((v.max(0) - v.min(0)).max())
        assert float(d.double().sqrt().max()) <= 1e-6 * max(extent, float(np.abs(v).max()))
        assert torch.allclose(s.normals.norm(dim=1), torch.ones(len(s.normals), device=dev), atol=1e-6)


@pytest.mark.parametrize("N", [100, 1000, 8000, 20000])
def test_count_within_half_a_percent(N, cuda_device):
    v, f = np_mesh(torus(nu=96, nv=48))
    for geodesic in (False, True):
        p, n, r = op(v, f, N, geodesic=geodesic)
        assert abs(len(p) - N) <= N // 200, (N, geodesic, len(p))
        assert r > 0


def test_degenerate_inputs_and_capacity(cuda_device):
    # no usable face
    verts = np.array([[0, 0, 0], [1, 0, 0], [2, 0, 0], [np.nan, 1, 0]], np.float32)
    rc, p, n, count, r, _ = raw(verts, [[0, 1, 2], [0, 0, 1], [0, 1, 3], [0, 1, 9]], 50)
    assert rc == 0 and count == 0 and r == 0.0 and len(p) == 0
    p, n, r = op(verts, np.array([[0, 1, 2]]), 50)
    assert p.shape == (0, 3) and n.shape == (0, 3) and r == 0.0
    rc, *_ = raw(np.zeros((0, 3)), np.zeros((0, 3)), 10)
    assert rc == 0
    # too small an output: DSS_E_CAPACITY, the count, nothing written
    v, f = np_mesh(icosphere(2))
    rc, _, _, count, r, buf = raw(v, f, 300, max_out=100, fill=7.0)
    assert rc == _lib.DSS_E_CAPACITY and abs(count - 300) <= 1 and r > 0
    assert (buf == 7.0).all()
    # invalid counts
    assert raw(v, f, 0)[0] == -1
    with pytest.raises(ValueError):
        op(v, f, 0)
    dev = cuda_device
    n_big = (2 ** 31 - 1) // 20 + 1
    rc = _lib.load().dss_sample_mesh_poisson_disk(_lib.ctx(dev), None, 0, None, 0, n_big, 0, 0, None, None, 0,
                                                  C.byref(C.c_int64()), C.byref(C.c_double()), _lib.stream_ptr(dev))
    assert rc == -1


def geodesic_checks(v, f, N, seed):
    p, n, r = op(v, f, N, geodesic=True, seed=seed)
    assert abs(len(p) - N) <= N // 200
    pool_p, pool_n, _ = pd.pool(v, f, N, seed)
    # the device's pool is the oracle's: every sample is a pool sample, in pool order
    key = {tuple(row): i for i, row in enumerate(bits(pool_p).tolist())}
    idx = np.array([key[tuple(row)] for row in bits(p).tolist()])
    assert (np.diff(idx) > 0).all() and np.array_equal(bits(n), bits(pool_n[idx]))
    want, margin = pd.select(pool_p, pool_n, r, geodesic=True)
    if margin > 1e-12:
        assert np.array_equal(idx, want)
    # separated and maximal, with a relative slack of 1e-12 for the device's asin
    P = pool_p.astype(np.float64)
    acc = set(idx.tolist())
    for i in range(len(P)):
        near = np.nonzero(((P[idx] - P[i]) ** 2).sum(1) < r * r * (1 + 1e-9))[0]
        ds = [(int(idx[k]), pd.geodesic_distance(P[max(i, idx[k])], pool_n[max(i, idx[k])], P[min(i, idx[k])],
                                                 pool_n[min(i, idx[k])])[0]) for k in near if idx[k] != i]
        if i in acc:
            assert all(d >= r * (1 - 1e-12) for _, d in ds), i
        else:
            assert any(k < i and d < r * (1 + 1e-12) for k, d in ds), i
    return margin


@pytest.mark.parametrize("case", ["ico3", "torus"])
def test_geodesic_selection_is_the_sequential_one(case, cuda_device):
    make, N = CASES[case]
    v, f = make()
    geodesic_checks(v, f, N, seed=5)


# ---- callers -------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def data_dir(cuda_device, tmp_path_factory):
    from dss_b200.utils.create_mvr_data import main
    tmp = tmp_path_factory.mktemp("pd_data")
    verts, faces = torus()
    mesh = tmp / "torus.obj"
    save_obj(str(mesh), verts.numpy(), faces.numpy())
    return main(["--points", str(mesh), "--output", str(tmp / "data"), "--num_cameras", "16", "--image-size", "128",
                 "--tri_color_light", "--point_lights", "--seed", "3"])[0]


def test_mvr_data_get_pointclouds(data_dir, cuda_device, tmp_path):
    import shutil

    from dss_b200.utils.dataset import MVRData
    from dss_b200.utils.io import read_mesh
    data = MVRData(data_dir)
    stored = data.get_pointclouds()
    assert torch.equal(stored.points_packed(), torch.tensor(np.asarray(data.data_dict["points"]), dtype=torch.float32))
    same = data.get_pointclouds(num_points=stored.points_packed().shape[0])
    assert torch.equal(same.points_packed(), stored.points_packed())
    pc = data.get_pointclouds(8000)
    v, f = read_mesh(os.path.join(data_dir, "mesh.obj"))
    p, n, _ = op(v, f, 8000, geodesic=True, seed=0)
    assert np.array_equal(bits(pc.points_packed().numpy()), bits(p))
    assert np.array_equal(bits(pc.normals_packed().numpy()), bits(n))
    assert data.get_pointclouds(8000).points_packed().data_ptr() != pc.points_packed().data_ptr()   # a copy
    bare = tmp_path / "bare"
    shutil.copytree(data_dir, bare)
    os.remove(bare / "mesh.obj")
    with pytest.raises(ValueError, match="mesh.obj"):
        MVRData(str(bare)).get_pointclouds(8000)


def test_loop_validates_against_poisson_disk_samples(data_dir, cuda_device, tmp_path):
    from dss_b200.ops import chamfer_distance
    from dss_b200.core.cloud import PointClouds3D
    from dss_b200.training.train import EVAL_SEED, ground_truth_cloud
    from dss_b200.utils.create_mvr_data import sample_points_from_mesh
    from dss_b200.utils.dataset import MVRData
    from dss_b200.utils.io import read_mesh
    from tests.test_gpu_train_loop import run_cli, write_config
    dev = cuda_device
    # the default keeps today's uniform samples, bit for bit
    v, f = read_mesh(os.path.join(data_dir, "mesh.obj"))
    g = torch.Generator(device=dev).manual_seed(EVAL_SEED)
    old = sample_points_from_mesh(torch.from_numpy(v).float().to(dev), torch.from_numpy(f).long().to(dev), 8000,
                                  generator=g)
    now = ground_truth_cloud(MVRData(data_dir), data_dir, 8000, dev)
    assert torch.equal(old[0], now[0]) and torch.equal(old[1], now[1])
    with pytest.raises(ValueError, match="eval_sampling"):
        ground_truth_cloud(MVRData(data_dir), data_dir, 8000, dev, "meshlab")
    # poisson_disk: the loop's chamfer is measured against get_pointclouds(8000)
    cfg = write_config(tmp_path / "c.yml", data_dir, tmp_path / "out", validate_every=10, eval_sampling="poisson_disk")
    code, log = run_cli(cfg, "--max-it", "20")
    assert code == 0, log
    assert "eval_sampling" not in log          # a known key: no warning
    vals = [json.loads(line.split("  (", 1)[1].rstrip(")")) for line in log.splitlines() if "Validation metric" in line]
    assert len(vals) == 1                      # iterations 0-19: validated at it 10
    best = torch.load(tmp_path / "out" / "torus" / "model_best.pt", map_location="cpu", weights_only=False)
    gt = MVRData(data_dir).get_pointclouds(8000)
    pts = best["model"]["points"][0].to(dev)
    nrm = torch.nn.functional.normalize(best["model"]["normals"][0].to(dev), dim=-1)
    cd, _ = chamfer_distance(PointClouds3D([gt.points_packed().to(dev)], [gt.normals_packed().to(dev)]),
                             PointClouds3D([pts], [nrm]))
    assert float(cd) == best["loss_val_best"] == min(v_["chamfer_point"] for v_ in vals)


def test_evaluate_against_mesh_samples(cuda_device, tmp_path):
    from dss_b200.utils.io import save_ply
    v, f = np_mesh(torus())
    save_obj(str(tmp_path / "mesh.obj"), v, f)
    (tmp_path / "pred").mkdir()
    rng = np.random.default_rng(0)
    save_ply(str(tmp_path / "pred" / "a.ply"), (v[rng.integers(0, len(v), 500)] + 0.01).astype(np.float32))
    env = dict(os.environ)
    env["PYTHONPATH"] = ROOT + os.pathsep + env.get("PYTHONPATH", "")
    cmd = [sys.executable, "-m", "dss_b200.utils.evaluate", "--gt", str(tmp_path / "mesh.obj"), "--pred",
           str(tmp_path / "pred"), "--name", "*.ply", "--gt-samples", "2000"]
    r = subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0, r.stdout
    got = read_ply(str(tmp_path / "pred" / "a_cdB.ply"))["points"]
    p, _, _ = op(v, f, 2000)
    assert np.array_equal(bits(got), bits(p))
    assert (tmp_path / "pred" / "evaluation.csv").exists()
    # a directory of ground truths cannot be sampled
    bad = subprocess.run(cmd[:4] + [str(tmp_path / "pred")] + cmd[5:], cwd=ROOT, env=env, stdout=subprocess.PIPE,
                         stderr=subprocess.STDOUT, text=True, timeout=600)
    assert bad.returncode == 2 and "--gt-samples" in bad.stdout
