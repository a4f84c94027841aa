"""GPU tests of upsampling and outlier removal (ops.upsample_points, csrc/upsample.cu; ops.outlier_ratio,
csrc/normals.cu): every round bit for bit against tests/upsample_oracle.py from the device's own K-NN rows, packed
batches with gaps, determinism, the ValueError cases, what holds by construction on a torus, the outlier ratio against
float64 eigh with its invalid rows and graph capture, the reference-shaped twins and the command line."""
import os

import numpy as np
import pytest
import torch

from dss_b200.core.cloud import PointClouds3D, remove_outliers, upsample
from dss_b200.frnn_grid import knn_points_packed
from dss_b200.ops import outlier_ratio, sample_points_poisson_disk, upsample_points
from dss_b200.utils.io import read_ply, save_ply
from tests import upsample_oracle as uo
from tests.test_mesh_data import torus

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "ply")
FIXTURES = ("sphere_2k", "bunny-8000", "teapot_normal_dense")


def _sphere(n, seed=0):
    p = np.random.default_rng(seed).normal(size=(n, 3))
    return (p / np.linalg.norm(p, axis=1, keepdims=True)).astype(np.float32)


def _torus_samples(dev, n):
    v, f = torus()
    s = sample_points_poisson_disk(v.to(dev), f[:, [0, 2, 1]].to(dev), n)
    return s.points.contiguous(), s.normals.contiguous()


def _cloud(name, dev):
    """points, normals, colours (P,3) on the device"""
    if name == "torus":
        p, n = _torus_samples(dev, 2000)
    else:
        d = read_ply(os.path.join(GOLDEN, name + ".ply"))
        p, n = torch.from_numpy(d["points"]).to(dev), torch.from_numpy(d["normals"]).to(dev)
    col = torch.from_numpy(np.random.default_rng(5).uniform(0, 1, (p.shape[0], 3)).astype(np.float32)).to(dev)
    return p, n, col


def _rows(points, c, K):
    dev = points.device
    first = torch.zeros(1, dtype=torch.int64, device=dev)
    num = torch.full((1,), c, dtype=torch.int64, device=dev)
    return knn_points_packed(points, first, num, K, -1.0)[1][:c].cpu().numpy()


@pytest.mark.parametrize("name", FIXTURES + ("torus",))
@pytest.mark.parametrize("k", [8, 16])
@pytest.mark.parametrize("factor", [2, 5])
def test_round_parity(cuda_device, name, k, factor):
    """Every round's points, normals, features and parents equal the oracle's from the device's K-NN rows of the
    cloud as it stood before the round (a prefix of the output: rows never move)."""
    p, n, col = _cloud(name, cuda_device)
    P = p.shape[0]
    up = upsample_points(p, factor * P, k, n, col)
    pts, nrm, ftr, par = (t.cpu().numpy() for t in (up.points, up.normals, up.features, up.parents))
    assert pts.shape == (factor * P, 3) and up.num_points.tolist() == [factor * P] and up.first_idx.tolist() == [0]
    assert np.array_equal(pts[:P], p.cpu().numpy()) and np.array_equal(nrm[:P], n.cpu().numpy())
    assert np.array_equal(ftr[:P], col.cpu().numpy()) and (par[:P] == -1).all()
    sizes = [s[0] for s in uo.schedule([P], [factor * P], k)]
    for c, c1 in zip(sizes[:-1], sizes[1:]):
        new_p, new_n, new_f, new_par = uo.upsample_round(pts[:c], _rows(up.points, c, k + 1), c1 - c, nrm[:c], ftr[:c])
        assert np.array_equal(par[c:c1], new_par), (c, c1)
        assert np.array_equal(pts[c:c1], new_p), (c, c1)
        assert np.array_equal(nrm[c:c1], new_n), (c, c1)
        assert np.array_equal(ftr[c:c1], new_f), (c, c1)


def test_packed_batch_with_gaps(cuda_device):
    a = torch.from_numpy(_sphere(1500, 1)).to(cuda_device)
    b, nb = _torus_samples(cuda_device, 900)
    na = a.clone()
    buf = torch.full((2700, 3), float("nan"), device=cuda_device)         # the gaps are never read
    nbuf = torch.full((2700, 3), float("nan"), device=cuda_device)
    buf[:1500], buf[1600:1600 + b.shape[0]] = a, b
    nbuf[:1500], nbuf[1600:1600 + b.shape[0]] = na, nb
    first = torch.tensor([0, 1600], device=cuda_device)
    num = torch.tensor([1500, b.shape[0]], device=cuda_device)
    up = upsample_points(buf, [4000, 2100], 12, nbuf, first_idx=first, num_points=num)
    assert up.first_idx.tolist() == [0, 4000] and up.num_points.tolist() == [4000, 2100]
    for (p, n), f0, tgt in (((a, na), 0, 4000), ((b, nb), 4000, 2100)):
        one = upsample_points(p, tgt, 12, n)
        assert torch.equal(up.points[f0:f0 + tgt], one.points)
        assert torch.equal(up.normals[f0:f0 + tgt], one.normals)
        assert torch.equal(up.parents[f0:f0 + tgt], one.parents)
    # a cloud already at its target is left as it is
    same = upsample_points(buf, [1500, 2100], 12, first_idx=first, num_points=num)
    assert torch.equal(same.points[:1500], a)


def test_deterministic(cuda_device):
    p = torch.from_numpy(_sphere(50_000, 2)).to(cuda_device)
    col = torch.rand((50_000, 4), generator=torch.Generator().manual_seed(0)).to(cuda_device)
    x, y = upsample_points(p, 200_000, 16, features=col), upsample_points(p, 200_000, 16, features=col)
    assert torch.equal(x.points, y.points) and torch.equal(x.features, y.features)
    assert torch.equal(x.parents, y.parents)


def test_value_errors(cuda_device):
    p = torch.from_numpy(_sphere(300, 3)).to(cuda_device)
    with pytest.raises(ValueError):
        upsample_points(p, 299)                                             # below the cloud's size
    with pytest.raises(ValueError):
        upsample_points(p[:16], 20, 16)                                     # at most k points
    with pytest.raises(ValueError):
        upsample_points(p[:9], 12, 3)                                       # fewer than 10 points
    with pytest.raises(ValueError):
        upsample_points(p, 400, 32)                                         # k above 31
    q = p.clone()
    q[11, 2] = float("nan")
    with pytest.raises(ValueError):
        upsample_points(q, 400)
    with pytest.raises(ValueError):
        upsample(p[None], 400, knn_result=object())
    assert torch.equal(upsample_points(p, 300).points, p)


def test_torus_by_construction(cuda_device):
    """2 000 Poisson-disk samples of a torus grown to 20 000: every new point lies inside the input's bounding box, a
    third of the way from its parent to the chosen neighbour, within float32 rounding."""
    p, n = _torus_samples(cuda_device, 2000)
    P = p.shape[0]
    up = upsample_points(p, 20_000, 16, n)
    pts, par = up.points.double(), up.parents.long()
    new = pts[P:]
    lo, hi = p.min(0).values.double(), p.max(0).values.double()
    ulp = 2.0 ** -23 * torch.maximum(lo.abs(), hi.abs())                    # one rounding of the division
    assert bool(((new >= lo - ulp) & (new <= hi + ulp)).all())
    i, j = par[P:, 0], par[P:, 1]
    third = pts[i] + (pts[j] - pts[i]) / 3.0
    scale = pts.abs().max()
    assert float((new - third).abs().max()) <= 4 * 2.0 ** -24 * float(scale)
    assert bool((i < torch.arange(P, 20_000, device=cuda_device)).all())
    assert torch.allclose(up.normals.norm(dim=1)[P:], torch.ones(20_000 - P, device=cuda_device), atol=1e-6)


def _plane_and_noise(dev, seed=6):
    rng = np.random.default_rng(seed)
    plane = np.concatenate([rng.uniform(-1, 1, (20_000, 2)), rng.normal(scale=1e-3, size=(20_000, 1))], 1)
    vol = rng.uniform(-1, 1, (2_000, 3))
    return torch.from_numpy(np.concatenate([plane, vol]).astype(np.float32)).to(dev)


def test_outlier_ratio_against_eigh(cuda_device):
    p = _plane_and_noise(cuda_device)
    p[:50] = p[50]                                                          # a cluster of 51 duplicates: 0 / 0
    p[100, 0] = float("inf")                                                # invalid: no neighbours
    tol = 0.05
    out = outlier_ratio(p, 16, tol)
    ratio, keep = out.ratio.cpu().numpy(), out.keep.cpu().numpy()
    idx = _rows(p, p.shape[0], 16)
    ok = (idx >= 0).all(1)
    q = p.double().cpu().numpy()[idx[ok]]
    d = q - q.mean(1, keepdims=True)
    lam = np.linalg.eigh(np.einsum("mki,mkj->mij", d, d) / 16)[0]
    ref = np.full(len(idx), np.nan)
    with np.errstate(invalid="ignore", divide="ignore"):
        ref[ok] = lam[:, 0] / lam.sum(1)
    gap = np.zeros(len(idx), bool)
    gap[ok] = (lam[:, 1] - lam[:, 0]) > 1e-6 * lam[:, 2]
    assert gap.sum() > 15_000
    assert np.allclose(ratio[gap], ref[gap], rtol=1e-9, atol=0)
    clear = np.isfinite(ratio) & (np.abs(ratio - tol) > 1e-9)
    assert np.array_equal(keep[clear], ref[clear] < tol)
    assert np.isnan(ratio[:51]).all() and not keep[:51].any()
    assert np.isnan(ratio[100]) and not keep[100] and (idx[100] == -1).all()
    assert np.array_equal(keep, ratio < tol)
    # the plane stays and most of the volume goes
    assert keep[51:20_000].mean() > 0.9 and keep[20_000:].mean() < 0.5
    # the oracle's closed-form ratio marks the same invalid rows
    oratio, _ = uo.outlier_ratio(p.cpu().numpy(), idx, tol)
    assert np.array_equal(np.isnan(oratio), np.isnan(ratio))


def test_outlier_ratio_packed_and_capturable(cuda_device):
    a = _plane_and_noise(cuda_device, 7)
    b = torch.from_numpy(_sphere(5000, 8)).to(cuda_device)
    buf = torch.cat([a, torch.zeros((100, 3), device=cuda_device), b])
    first = torch.tensor([0, a.shape[0] + 100], device=cuda_device)
    num = torch.tensor([a.shape[0], b.shape[0]], device=cuda_device)
    out = outlier_ratio(buf, 16, 0.05, first, num)
    for x, f0 in ((a, 0), (b, a.shape[0] + 100)):
        one = outlier_ratio(x, 16, 0.05)
        assert torch.equal(out.ratio[f0:f0 + x.shape[0]], one.ratio)
    assert bool(out.ratio[a.shape[0]:a.shape[0] + 100].isnan().all())
    # the whole op replays in a CUDA graph with the eager bits
    P = a.shape[0]
    eager = outlier_ratio(a, 16, 0.05)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        outlier_ratio(a, 16, 0.05)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        cap = outlier_ratio(a, 16, 0.05)
    cap.ratio.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(cap.ratio, eager.ratio) and torch.equal(cap.keep, eager.keep) and cap.ratio.shape == (P,)


def test_reference_twins(cuda_device):
    p = torch.from_numpy(np.stack([_sphere(600, 9), _sphere(600, 10)])).to(cuda_device)
    num = torch.tensor([600, 450], device=cuda_device)
    padded, n_out = upsample(p, torch.tensor([1500, 900]), num, neighborhood_size=10)
    assert n_out.tolist() == [1500, 900] and padded.shape == (2, 1500, 3)
    one = upsample_points(p[1, :450], 900, 10).points
    assert torch.equal(padded[1, :900], one) and bool((padded[1, 900:] == 0).all())
    clouds = PointClouds3D([torch.cat([p[0], torch.rand((60, 3), device=cuda_device) * 2 - 1])],
                           normals=[torch.cat([p[0], p[0][:60]])], features=[torch.rand((660, 3), device=cuda_device)])
    kept = remove_outliers(clouds, 16, 0.05)
    mask = outlier_ratio(clouds.points_packed(), 16, 0.05).keep
    assert torch.equal(kept.points_list()[0], clouds.points_list()[0][mask])
    assert torch.equal(kept.features_list()[0], clouds.features_list()[0][mask])
    with pytest.raises(ValueError):
        remove_outliers(PointClouds3D([p[0, :16]]), 16)
    grown = clouds.upsample(1000, 12)
    assert grown.points_list()[0].shape == (1000, 3) and grown.normals_list()[0].shape == (1000, 3)
    assert grown.features_list()[0].shape == (1000, 3)


def test_cli(cuda_device, tmp_path):
    from dss_b200.utils.resample import main
    d = read_ply(os.path.join(GOLDEN, "sphere_2k.ply"))
    rng = np.random.default_rng(11)
    noise = rng.uniform(-1.2, 1.2, (40, 3)).astype(np.float32)
    pts = np.concatenate([d["points"], noise])
    nrm = np.concatenate([d["normals"], np.tile([[0, 0, 1]], (40, 1))]).astype(np.float32)
    col = rng.integers(0, 256, (len(pts), 3)).astype(np.float32) / 255.0
    src = str(tmp_path / "in.ply")
    save_ply(src, pts, colors=col, normals=nrm)
    out = str(tmp_path / "out.ply")
    assert main([src, out, "--upsample", "3000", "--k", "12"]) == 0
    got = read_ply(out)
    assert got["points"].shape == (3000, 3) and got["normals"].shape == (3000, 3) and got["colors"].shape == (3000, 3)
    assert np.array_equal(got["points"][:len(pts)], pts) and np.array_equal(got["normals"][:len(pts)], nrm)
    up = upsample_points(torch.from_numpy(pts).to(cuda_device), 3000, 12).points.cpu().numpy()
    assert np.array_equal(got["points"], up)
    out2 = str(tmp_path / "out2.ply")
    assert main([src, out2, "--remove-outliers", "--upsample", "2500"]) == 0
    got2 = read_ply(out2)
    keep = outlier_ratio(torch.from_numpy(pts).to(cuda_device), 16, 0.05).keep.cpu().numpy()
    assert got2["points"].shape == (2500, 3) and np.array_equal(got2["points"][:keep.sum()], pts[keep])
    xyz = str(tmp_path / "in.xyz")
    np.savetxt(xyz, pts, fmt="%.9g")
    out3 = str(tmp_path / "out3.ply")
    assert main([xyz, out3, "--upsample", "2000"]) == 0
    assert read_ply(out3)["points"].shape == (2000, 3)
