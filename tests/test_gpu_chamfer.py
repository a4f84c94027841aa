"""GPU: ops.chamfer_distance (csrc/chamfer.cu) against a float64 brute force on the CPU (torch.cdist in float64, the
smallest index on ties), its sums against the float64 sum of the K = 1 rows knn_points_packed returns, determinism and
a CUDA-graph replay."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from dss_b200.core.cloud import PointClouds3D
from dss_b200.frnn_grid import knn_points_packed
from dss_b200.ops import _chamfer_sums, chamfer_distance

pytestmark = pytest.mark.gpu


# ---- the float64 oracle ------------------------------------------------------------------------------------------------

def nearest64(q, p):
    """(Q,3), (P,3) float64 -> (min squared distance (Q,), argmin (Q,)): NaN distances never win, the smallest index wins
    a tie, a row without a finite distance gets NaN / -1"""
    Q = q.shape[0]
    best = torch.full((Q,), float("nan"), dtype=torch.float64)
    arg = torch.full((Q,), -1, dtype=torch.int64)
    if Q == 0 or p.shape[0] == 0:
        return best, arg
    chunk = max(1, (1 << 25) // p.shape[0])       # 256 MB of distances at a time
    for s in range(0, Q, chunk):
        d = torch.cdist(q[s:s + chunk], p) ** 2
        d = torch.where(torch.isfinite(d), d, torch.full_like(d, float("inf")))
        m, a = d.min(1)                       # first occurrence of the minimum
        ok = torch.isfinite(m)
        # the exact float64 distance of the chosen row (cdist's mm path rounds |q|^2 + |p|^2 - 2 q.p)
        exact = ((q[s:s + chunk] - p[a]) ** 2).sum(1)
        best[s:s + chunk] = torch.where(ok, exact, torch.full_like(exact, float("nan")))
        arg[s:s + chunk] = torch.where(ok, a, torch.full_like(a, -1))
    return best, arg


def cosine_term(a, b):
    """1 - |cosine_similarity(eps=1e-6)| in float64, NaN where b is missing"""
    return 1.0 - F.cosine_similarity(a.double(), b.double(), dim=1, eps=1e-6).abs()


def oracle(x, y, xl, yl, xn=None, yn=None):
    """per cloud n: float64 {sum_x d, sum_y d, sum_x c, sum_y c} at the oracle's neighbours, and those neighbours"""
    N = x.shape[0]
    out = torch.zeros((N, 4), dtype=torch.float64)
    args = []
    for n in range(N):
        X, Y = x[n, :xl[n]].double().cpu(), y[n, :yl[n]].double().cpu()
        dx, ax = nearest64(X, Y)
        dy, ay = nearest64(Y, X)
        out[n, 0], out[n, 1] = dx.sum(), dy.sum()
        if xn is not None:
            XN, YN = xn[n, :xl[n]].cpu(), yn[n, :yl[n]].cpu()
            nan3 = lambda k: torch.full((k, 3), float("nan"), dtype=torch.float64)
            gx = torch.where((ax >= 0)[:, None], YN[ax.clamp(min=0)].double(), nan3(len(ax))) if len(YN) else nan3(len(ax))
            gy = torch.where((ay >= 0)[:, None], XN[ay.clamp(min=0)].double(), nan3(len(ay))) if len(XN) else nan3(len(ay))
            out[n, 2], out[n, 3] = cosine_term(XN, gx).sum(), cosine_term(YN, gy).sum()
        args.append((ax, ay))
    return out, args


def kernel_rows(x, y, xl, yl):
    """the K = 1 rows the kernel's searches produce: knn_points_packed on the padded storage passed as packed"""
    N, P1, P2 = x.shape[0], x.shape[1], y.shape[1]
    dev = x.device
    xf = torch.arange(N, device=dev, dtype=torch.int64) * P1
    yf = torch.arange(N, device=dev, dtype=torch.int64) * P2
    xr, yr = x.reshape(-1, 3).contiguous(), y.reshape(-1, 3).contiguous()
    dx, ix = knn_points_packed(yr, yf, yl, 1, -1.0, queries=xr, query_first_idx=xf, query_num=xl)
    dy, iy = knn_points_packed(xr, xf, xl, 1, -1.0, queries=yr, query_first_idx=yf, query_num=yl)
    return dx.view(N, P1).cpu(), ix.view(N, P1).long().cpu(), dy.view(N, P2).cpu(), iy.view(N, P2).long().cpu()


def padded(N, P, lengths, gen, scale=1.0, normals=True):
    """(N,P,3) points on a noisy unit sphere and unit-ish normals, the padding rows NaN"""
    p = F.normalize(torch.randn(N, P, 3, generator=gen), dim=-1) * scale + 0.01 * torch.randn(N, P, 3, generator=gen)
    n = torch.randn(N, P, 3, generator=gen) if normals else None
    for i, l in enumerate(lengths):
        p[i, l:] = float("nan")
        if normals:
            n[i, l:] = float("nan")
    return p, n


def check_case(x, y, xl, yl, xn=None, yn=None, rel=1e-6):
    d = torch.device("cuda:0")
    xd, yd = x.to(d), y.to(d)
    xld, yld = torch.as_tensor(xl, device=d), torch.as_tensor(yl, device=d)
    xnd, ynd = (None, None) if xn is None else (xn.to(d), yn.to(d))
    sums, _, _, _ = _chamfer_sums(xd, yd, xld, yld, xnd, ynd)
    sums = sums.cpu()
    want, args = oracle(x, y, xl, yl, xn, yn)
    dx, ix, dy, iy = kernel_rows(xd, yd, xld, yld)
    N = x.shape[0]
    for n in range(N):
        kx, ky = ix[n, :xl[n]], iy[n, :yl[n]]
        ox, oy = args[n]
        # same rows without a neighbour
        assert torch.equal(kx < 0, ox < 0) and torch.equal(ky < 0, oy < 0)
        # each chosen neighbour within 1e-6 of the float64 minimum
        for q, p, k, o in ((x[n, :xl[n]], y[n, :yl[n]], kx, ox), (y[n, :yl[n]], x[n, :xl[n]], ky, oy)):
            ok = k >= 0
            if ok.any():
                q64, p64 = q.double()[ok], p.double()
                dk = ((q64 - p64[k[ok]]) ** 2).sum(1)
                do = ((q64 - p64[o[ok]]) ** 2).sum(1)
                assert ((dk - do).abs() <= rel * do + 1e-300).all()
        # reduction exactness: the kernel's sums are the float64 sums of those rows
        for col, rows in ((0, dx[n, :xl[n]]), (1, dy[n, :yl[n]])):
            r = torch.where(rows >= 0, rows.double(), torch.full_like(rows.double(), float("nan"))).sum()
            if torch.isnan(r):
                assert torch.isnan(sums[n, col])
            else:
                assert abs(float(sums[n, col]) - float(r)) <= 1e-14 * abs(float(r)) + 1e-300
        # distance term within 1e-6 of float64
        for col in (0, 1):
            a, b = float(sums[n, col]), float(want[n, col])
            assert np.isnan(a) == np.isnan(b)
            if not np.isnan(b):
                assert abs(a - b) <= rel * abs(b) + 1e-300, (n, col, a, b)
        # normal term: float64 cosine at the kernel's own neighbours
        if xn is not None:
            for col, qn, pn, k in ((2, xn[n, :xl[n]], yn[n, :yl[n]], kx), (3, yn[n, :yl[n]], xn[n, :xl[n]], ky)):
                nan3 = torch.full((len(k), 3), float("nan"), dtype=torch.float64)
                g = torch.where((k >= 0)[:, None], pn[k.clamp(min=0)].double(), nan3) if len(pn) else nan3
                ref = float(cosine_term(qn, g).sum())
                a = float(sums[n, col])
                assert np.isnan(a) == np.isnan(ref)
                if not np.isnan(ref):
                    assert abs(a - ref) <= 1e-6 * max(1.0, abs(ref)), (n, col, a, ref)
        else:
            assert (sums[n, 2:] == 0).all()
    # every reduction, from the oracle's float64 sums at the kernel's neighbours for the normal term
    lens = torch.tensor([xl, yl, xl, yl], dtype=torch.float64).T
    expect = sums.clone()
    expect[:, :2] = want[:, :2]
    for pr in ("mean", "sum"):
        t = expect / lens if pr == "mean" else expect
        for br in ("mean", "sum", None):
            got = chamfer_distance(xd, yd, xld, yld, xnd, ynd, batch_reduction=br, point_reduction=pr)
            e = t if br is None else (t.sum(0) if br == "sum" else t.sum(0) / N)
            ed = (e[..., 0] + e[..., 1]).float()
            assert got[0].dtype == torch.float32 and got[0].is_cuda and got[0].shape == ed.shape
            assert torch.allclose(got[0].cpu(), ed, rtol=2e-6, atol=0, equal_nan=True), (pr, br, got[0], ed)
            if xn is None:
                assert got[1] is None
            else:
                en = (e[..., 2] + e[..., 3]).float()
                assert torch.allclose(got[1].cpu(), en, rtol=2e-6, atol=1e-6, equal_nan=True)
    return sums


# ---- cases -------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("P1,P2", [(1, 1), (1, 7), (5, 1), (64, 300), (3000, 2000)])
@pytest.mark.parametrize("normals", [False, True])
def test_single_cloud(cuda_device, P1, P2, normals):
    g = torch.Generator().manual_seed(P1 * 1000 + P2)
    x, xn = padded(1, P1, [P1], g, normals=normals)
    y, yn = padded(1, P2, [P2], g, scale=0.9, normals=normals)
    check_case(x, y, [P1], [P2], xn, yn)


@pytest.mark.parametrize("normals", [False, True])
def test_ragged_batch_nan_padding(cuda_device, normals):
    g = torch.Generator().manual_seed(7)
    xl, yl = [500, 1, 1200], [900, 333, 40]
    x, xn = padded(3, 1200, xl, g, normals=normals)
    y, yn = padded(3, 900, yl, g, scale=1.1, normals=normals)
    sums = check_case(x, y, xl, yl, xn, yn)
    assert torch.isfinite(sums).all()            # the NaN padding was never read


def test_large(cuda_device):
    g = torch.Generator().manual_seed(11)
    x, xn = padded(1, 8000, [8000], g)
    y, yn = padded(1, 200000, [200000], g, scale=0.95)
    check_case(x, y, [8000], [200000], xn, yn)


def test_point_clouds_input_matches_padded(cuda_device):
    d = cuda_device
    g = torch.Generator().manual_seed(3)
    xl, yl = [300, 41], [128, 500]
    x, xn = padded(2, 300, xl, g)
    y, yn = padded(2, 500, yl, g)
    cx = PointClouds3D([x[i, :xl[i]].to(d) for i in range(2)], [xn[i, :xl[i]].to(d) for i in range(2)])
    cy = PointClouds3D([y[i, :yl[i]].to(d) for i in range(2)], [yn[i, :yl[i]].to(d) for i in range(2)])
    for br in ("mean", "sum", None):
        a = chamfer_distance(cx, cy, batch_reduction=br)
        b = chamfer_distance(x.to(d), y.to(d), torch.tensor(xl, device=d), torch.tensor(yl, device=d), xn.to(d),
                             yn.to(d), batch_reduction=br)
        # the same rows; the per-block sums may split differently between the two layouts
        assert torch.allclose(a[0], b[0], rtol=1e-6, atol=0) and torch.allclose(a[1], b[1], rtol=1e-6, atol=0)
    # clouds without normals: no normal term
    assert chamfer_distance(PointClouds3D([x[i, :xl[i]].to(d) for i in range(2)]), cy)[1] is None


def test_duplicates_smallest_index_wins(cuda_device):
    g = torch.Generator().manual_seed(5)
    base, bn = padded(1, 200, [200], g)
    # y: every point three times at indices i, 200 + i, 400 + i, each copy with its own normal
    y = base.repeat(1, 3, 1)
    yn = torch.randn(1, 600, 3, generator=g)
    x = base[:, :150] + 0.003 * torch.randn(1, 150, 3, generator=g)
    xn = torch.randn(1, 150, 3, generator=g)
    check_case(x, y, [150], [600], xn, yn)
    d = cuda_device
    _, ix, _, _ = kernel_rows(x.to(d), y.to(d), torch.tensor([150], device=d), torch.tensor([600], device=d))
    _, args = oracle(x, y, [150], [600], xn, yn)
    assert torch.equal(ix[0], args[0][0]) and (ix[0] < 200).all()
    # the normal term has the oracle's choice: the same value as at the oracle's neighbours
    sums = _chamfer_sums(x.to(d), y.to(d), x_normals=xn.to(d), y_normals=yn.to(d))[0].cpu()
    want, _ = oracle(x, y, [150], [600], xn, yn)
    assert abs(float(sums[0, 2]) - float(want[0, 2])) <= 1e-12 * abs(float(want[0, 2]))


def test_nan_point_and_empty_cloud(cuda_device):
    g = torch.Generator().manual_seed(9)
    xl, yl = [100, 100, 0, 80], [120, 0, 50, 120]
    x, xn = padded(4, 100, xl, g)
    y, yn = padded(4, 120, yl, g)
    x[0, 17, 1] = float("nan")                   # cloud 0: a NaN query
    y[3, 5, 0] = float("inf")                    # cloud 3: an infinite point (a query without neighbour itself)
    d = cuda_device
    sums = check_case(x, y, xl, yl, xn, yn)
    want, _ = oracle(x, y, xl, yl, xn, yn)
    assert torch.equal(torch.isnan(sums), torch.isnan(want))
    assert torch.isnan(sums[0, [0, 2]]).all() and torch.isfinite(sums[0, [1, 3]]).all()
    assert torch.isnan(sums[1, [0, 2]]).all() and (sums[1, [1, 3]] == 0).all()   # y empty: x has no neighbour
    assert (sums[2, [0, 2]] == 0).all() and torch.isnan(sums[2, [1, 3]]).all()
    per = chamfer_distance(x.to(d), y.to(d), torch.tensor(xl, device=d), torch.tensor(yl, device=d), xn.to(d),
                           yn.to(d), batch_reduction=None)[0].cpu()
    assert torch.isnan(per).tolist() == [True, True, True, True]
    # x empty with the mean reduction is 0/0 even against an empty y
    e = chamfer_distance(torch.zeros(1, 4, 3, device=d), torch.zeros(1, 4, 3, device=d),
                         torch.zeros(1, dtype=torch.int64, device=d), torch.zeros(1, dtype=torch.int64, device=d))[0]
    assert torch.isnan(e)


def test_refusals(cuda_device):
    d = cuda_device
    x = torch.rand(1, 10, 3, device=d)
    with pytest.raises(RuntimeError, match="backward"):
        chamfer_distance(x.clone().requires_grad_(True), x)
    with pytest.raises(RuntimeError, match="backward"):
        chamfer_distance(x, x, x_normals=x.clone().requires_grad_(True), y_normals=x)
    with pytest.raises(RuntimeError, match="CUDA"):
        chamfer_distance(x.cpu(), x.cpu())
    x3 = torch.rand(3, 10, 3, device=d)
    with pytest.raises(ValueError, match="shape"):            # fewer lengths than clouds: never reaches the kernel
        chamfer_distance(x3, x3, x_lengths=torch.tensor([10], device=d))
    with pytest.raises(ValueError, match="shape"):
        chamfer_distance(x3, x3, y_lengths=torch.full((3, 1), 10, device=d))
    with pytest.raises(ValueError):
        chamfer_distance(x, x, batch_reduction="max")
    with pytest.raises(ValueError):
        chamfer_distance(x, x, point_reduction=None)


def test_deterministic_and_graph_replay(cuda_device):
    d = cuda_device
    g = torch.Generator().manual_seed(21)
    x, xn = padded(2, 8000, [8000, 6000], g)
    y, yn = padded(2, 50000, [50000, 31111], g)
    args = (x.to(d), y.to(d), torch.tensor([8000, 6000], device=d), torch.tensor([50000, 31111], device=d), xn.to(d),
            yn.to(d))
    a = _chamfer_sums(*args)[0].clone()
    b = _chamfer_sums(*args)[0].clone()
    assert torch.equal(a, b)
    s = torch.cuda.Stream(device=d)
    s.wait_stream(torch.cuda.current_stream(d))
    with torch.cuda.stream(s):
        _chamfer_sums(*args)
    torch.cuda.current_stream(d).wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = _chamfer_sums(*args)[0]
    graph.replay()
    torch.cuda.synchronize(d)
    assert torch.equal(out, a)


def test_same_cloud_as_x_and_y_follows_the_tie_rule(cuda_device):
    """one cloud object as both x and y (the same rows and offsets): every row's nearest is the smallest index among its
    exact duplicates, itself or an earlier copy, so the normal term uses that copy's normal"""
    d = cuda_device
    g = torch.Generator().manual_seed(13)
    base, _ = padded(1, 150, [150], g)
    pts = torch.cat([base[0], base[0, :100]])                 # rows 150.. duplicate rows 0..99
    nrm = torch.randn(250, 3, generator=g)
    c = PointClouds3D([pts.to(d)], [nrm.to(d)])
    sums = _chamfer_sums(c, c)[0].cpu()
    want, args = oracle(pts[None], pts[None], [250], [250], nrm[None], nrm[None])
    assert args[0][0][150:].tolist() == list(range(100))      # the oracle picks the earlier copy
    assert (sums[0, :2] == 0).all()
    assert abs(float(sums[0, 2]) - float(want[0, 2])) <= 1e-12 * abs(float(want[0, 2]))
    assert abs(float(sums[0, 3]) - float(want[0, 3])) <= 1e-12 * abs(float(want[0, 3]))
    assert float(sums[0, 2]) > 0                               # the duplicates' own normals would give 0 there
