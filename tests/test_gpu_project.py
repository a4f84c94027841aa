"""GPU tests of the RIMLS projection and normal denoising (ops.project_to_surface, ops.denoise_normals,
csrc/rimls.cu): parity with tests/project_oracle.py from the device's own K-NN rows, packed clouds with gaps,
determinism, duplicates and isolated rows, the ValueError cases, the reference-shaped twins, the command line, and
the quality on a noisy torus."""
import os

import numpy as np
import pytest
import torch

from dss_b200.core.cloud import PointClouds3D, denoise_normals as denoise_twin, project_to_latent_surface
from dss_b200.frnn_grid import knn_points_packed
from dss_b200.ops import (denoise_normals, point_mesh_distance, project_to_surface, sample_points_poisson_disk,
                          upsample_points)
from dss_b200.utils.io import read_ply, save_ply
from tests import project_oracle as po
from tests.test_mesh_data import torus

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "ply")
FIXTURES = ("sphere_2k", "bunny-8000", "teapot_normal_dense")


def _noisy_torus(dev, n, sigma, seed=0):
    """Poisson-disk samples of the torus mesh moved along their normals by N(0, sigma^2)"""
    v, f = torus()
    s = sample_points_poisson_disk(v.to(dev), f[:, [0, 2, 1]].to(dev), n)
    g = torch.Generator().manual_seed(seed)
    noise = (sigma * torch.randn((s.points.shape[0], 1), generator=g)).to(dev)
    return (s.points + noise * s.normals).contiguous(), s.normals.contiguous()


def _cloud(name, dev):
    if name == "torus":
        return _noisy_torus(dev, 3000, 0.005)
    if name == "upsampled":
        p, n = _noisy_torus(dev, 2000, 0.0)
        up = upsample_points(p, 10_000, 16, n)
        return up.points, up.normals
    d = read_ply(os.path.join(GOLDEN, name + ".ply"))
    return torch.from_numpy(d["points"]).to(dev), torch.from_numpy(d["normals"]).to(dev)


def _rows(points, k):
    dev = points.device
    first = torch.zeros(1, dtype=torch.int64, device=dev)
    num = torch.full((1,), points.shape[0], dtype=torch.int64, device=dev)
    return knn_points_packed(points, first, num, k + 1, -1.0)[1].cpu().numpy()


def _within_ulp(got, ref, floor=1e-6):
    """every float32 value of got within one float32 ulp of the float64 ref (ulps of |ref| below floor: at floor)"""
    r32 = ref.astype(np.float32)
    tol = np.spacing(np.maximum(np.abs(r32), np.float32(floor))).astype(np.float64)
    err = np.abs(got.astype(np.float64) - r32.astype(np.float64))
    return bool((err <= tol).all()), float((err / tol).max())


@pytest.mark.parametrize("name", FIXTURES + ("torus", "upsampled"))
@pytest.mark.parametrize("k", [8, 31])
def test_parity_with_oracle(cuda_device, name, k):
    p, n = _cloud(name, cuda_device)
    rows = _rows(p, k)
    pn, nn = p.cpu().numpy(), n.cpu().numpy()
    got = project_to_surface(p, n, k)
    ref = po.project(pn, nn, rows, k)
    assert ref.margin > 1e-9, ref.margin                     # no decision close enough to flip
    assert np.array_equal(got.iterations.cpu().numpy(), ref.iterations)
    ok, worst = _within_ulp(got.points.cpu().numpy(), ref.points)
    assert ok, worst
    assert (ref.iterations > 0).mean() > 0.5
    dn = denoise_normals(p, n, k)
    dref = po.denoise_normals(pn, nn, rows, k)
    assert dref.margin > 1e-9, dref.margin
    ok, worst = _within_ulp(dn.cpu().numpy(), dref.normals)
    assert ok, worst
    assert torch.equal(p.cpu(), torch.from_numpy(pn))          # the inputs are not modified


def test_packed_with_gaps_and_deterministic(cuda_device):
    a, na = _cloud("sphere_2k", cuda_device)
    b, nb = _noisy_torus(cuda_device, 1500, 0.005, 1)
    P = a.shape[0] + 100 + b.shape[0] + 50
    buf = torch.full((P, 3), float("nan"), device=cuda_device)          # the gaps are never read
    nbuf = torch.full((P, 3), float("nan"), device=cuda_device)
    f1 = a.shape[0] + 100
    buf[:a.shape[0]], buf[f1:f1 + b.shape[0]] = a, b
    nbuf[:a.shape[0]], nbuf[f1:f1 + b.shape[0]] = na, nb
    first = torch.tensor([0, f1], device=cuda_device)
    num = torch.tensor([a.shape[0], b.shape[0]], device=cuda_device)
    out = project_to_surface(buf, nbuf, 16, first_idx=first, num_points=num)
    den = denoise_normals(buf, nbuf, 12, first_idx=first, num_points=num)
    for (x, nx), f0 in (((a, na), 0), ((b, nb), f1)):
        one = project_to_surface(x, nx, 16)
        assert torch.equal(out.points[f0:f0 + x.shape[0]], one.points)
        assert torch.equal(out.iterations[f0:f0 + x.shape[0]], one.iterations)
        assert torch.equal(den[f0:f0 + x.shape[0]], denoise_normals(x, nx, 12))
    assert bool(out.points[a.shape[0]:f1].isnan().all()) and bool((out.iterations[a.shape[0]:f1] == 0).all())
    rows = torch.zeros(P, dtype=torch.bool, device=cuda_device)
    rows[:a.shape[0]], rows[f1:f1 + b.shape[0]] = True, True
    again = project_to_surface(buf, nbuf, 16, first_idx=first, num_points=num)
    assert torch.equal(again.points[rows], out.points[rows]) and torch.equal(again.iterations, out.iterations)
    assert torch.equal(denoise_normals(buf, nbuf, 12, first_idx=first, num_points=num)[rows], den[rows])


def test_duplicates_and_isolated_rows(cuda_device):
    p, n = _cloud("sphere_2k", cuda_device)
    p, n = p.clone(), n.clone()
    p[1] = p[0]                                                  # a pair
    p[10:50] = p[10]                                              # 40 copies: no neighbour at a positive distance
    p[60] = torch.tensor([5.0, 5.0, 5.0])                         # no neighbour within the radius
    n[70] = 0.0                                                   # a zero normal stays zero and contributes nothing
    k = 8
    got = project_to_surface(p, n, k)
    ref = po.project(p.cpu().numpy(), n.cpu().numpy(), _rows(p, k), k)
    assert np.array_equal(got.iterations.cpu().numpy(), ref.iterations)
    assert _within_ulp(got.points.cpu().numpy(), ref.points)[0]
    assert bool(torch.isfinite(got.points).all())
    assert torch.equal(got.points[10:50], p[10:50]) and bool((got.iterations[10:50] == 0).all())
    assert torch.equal(got.points[60], p[60]) and int(got.iterations[60]) == 0
    assert int(got.iterations[0]) > 0 and int(got.iterations[1]) > 0
    dn = denoise_normals(p, n, k)
    assert torch.allclose(dn[60], n[60] / n[60].norm(), rtol=0, atol=1e-7)    # all weights zero: its own normal
    assert bool(torch.isfinite(dn).all())
    assert _within_ulp(dn.cpu().numpy(), po.denoise_normals(p.cpu().numpy(), n.cpu().numpy(), _rows(p, k), k).normals)[0]


def test_value_errors(cuda_device):
    p, n = _cloud("sphere_2k", cuda_device)
    for k in (2, 32):
        with pytest.raises(ValueError):
            project_to_surface(p, n, k)
        with pytest.raises(ValueError):
            denoise_normals(p, n, k)
    q = p.clone()
    q[5, 1] = float("nan")
    with pytest.raises(ValueError):
        project_to_surface(q, n)
    m = n.clone()
    m[7, 0] = float("inf")
    with pytest.raises(ValueError):
        denoise_normals(p, m)
    with pytest.raises(ValueError):
        project_to_surface(p, n, 8, max_proj_iters=-1)
    first, num = torch.tensor([0, 100], device=cuda_device), torch.tensor([200, 200], device=cuda_device)
    with pytest.raises(ValueError):
        project_to_surface(p, n, 8, first_idx=first, num_points=num)          # overlapping clouds
    with pytest.raises(ValueError):
        denoise_twin(p[None], n[None], knn_result=object())


def test_reference_twins(cuda_device):
    a, na = _cloud("sphere_2k", cuda_device)
    b, nb = _noisy_torus(cuda_device, a.shape[0], 0.005, 2)
    P = min(a.shape[0], b.shape[0])
    pts, nrm = torch.stack([a[:P], b[:P]]), torch.stack([na[:P], nb[:P]])
    before = pts.clone()
    out = project_to_latent_surface(pts, nrm, neighborhood_size=20, max_proj_iters=4, max_est_iter=3)
    assert out.shape == pts.shape and torch.equal(pts, before)
    assert torch.equal(out[1], project_to_surface(b[:P], nb[:P], 20, 4, 3).points)
    num = torch.tensor([P, P - 300], device=cuda_device)
    dn = denoise_twin(pts, nrm, num, sharpness_sigma=20, neighborhood_size=12)
    assert torch.equal(dn[1, :P - 300], denoise_normals(b[:P - 300], nb[:P - 300], 12, 20.0))
    assert torch.equal(dn[1, P - 300:], nrm[1, P - 300:])
    col = torch.rand((P, 3), device=cuda_device)
    clouds = PointClouds3D([a[:P], b[:P - 300]], normals=[na[:P], nb[:P - 300]], features=[col, col[:P - 300]])
    moved = clouds.project_to_latent_surface(12)
    assert torch.equal(moved.points_list()[1], project_to_surface(b[:P - 300], nb[:P - 300], 12).points)
    assert torch.equal(moved.normals_list()[0], na[:P]) and torch.equal(moved.features_list()[1], col[:P - 300])
    with pytest.raises(ValueError):
        PointClouds3D([a]).project_to_latent_surface()


def test_cli(cuda_device, tmp_path):
    from dss_b200.utils.resample import main
    p, n = _noisy_torus(cuda_device, 2000, 0.005, 3)
    pts, nrm = p.cpu().numpy(), n.cpu().numpy()
    col = np.random.default_rng(4).uniform(0, 1, (len(pts), 3)).astype(np.float32)
    src = str(tmp_path / "in.ply")
    save_ply(src, pts, colors=col, normals=nrm)
    out = str(tmp_path / "out.ply")
    assert main([src, out, "--project", "--project-k", "20"]) == 0
    got = read_ply(out)
    assert np.array_equal(got["points"], project_to_surface(p, n, 20).points.cpu().numpy())
    assert np.array_equal(got["normals"], nrm) and got["colors"].shape == col.shape
    out2 = str(tmp_path / "out2.ply")
    assert main([src, out2, "--upsample", "5000", "--denoise-normals", "--project"]) == 0
    got2 = read_ply(out2)
    up = upsample_points(p, 5000, 16, n)
    dn = denoise_normals(up.points, up.normals)
    assert np.array_equal(got2["normals"], dn.cpu().numpy())
    assert np.array_equal(got2["points"], project_to_surface(up.points, dn).points.cpu().numpy())
    xyz = str(tmp_path / "in.xyz")
    np.savetxt(xyz, pts, fmt="%.9g")
    with pytest.raises(ValueError, match="dss_b200.utils.normals"):
        main([xyz, str(tmp_path / "out3.ply"), "--project"])


def test_quality_on_noisy_torus(cuda_device):
    """20 000 torus samples moved along their normals by noise of half their spacing: the mean distance to the torus
    mesh falls more than 2x, by the factor the oracle gives on the same input."""
    v, f = (t.to(cuda_device) for t in torus())
    f = f[:, [0, 2, 1]].contiguous()
    p, _ = _noisy_torus(cuda_device, 20_000, 0.0)
    first = torch.zeros(1, dtype=torch.int64, device=cuda_device)
    num = torch.full((1,), p.shape[0], dtype=torch.int64, device=cuda_device)
    spacing = float(knn_points_packed(p, first, num, 2, -1.0)[0][:, 1].sqrt().mean())
    p, n = _noisy_torus(cuda_device, 20_000, 0.5 * spacing, 5)
    got = project_to_surface(p, n)
    ref = po.project(p.cpu().numpy(), n.cpu().numpy(), _rows(p, 31), 31)
    mean = lambda x: float(point_mesh_distance(x, v, f).sq_dists.double().sqrt().mean())
    before, after = mean(p), mean(got.points)
    after_ref = mean(torch.from_numpy(ref.points.astype(np.float32)).to(cuda_device))
    assert before / after > 2.0, (before, after)
    assert abs(before / after - before / after_ref) <= 1e-4 * (before / after), (after, after_ref)
