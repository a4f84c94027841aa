"""The K-NN grid search (dss_knn_points, dss_b200/csrc/knn.cu) against the brute force (oracle.knn_brute, the
restatement of the reference's FRNNBruteForceCPU) bit for bit -- distances and indices, self mode and general mode --
at the places where a grid search goes wrong: the K boundaries of the knn_search_kernel<8/16/32> instantiations,
d == r^2, ties on cell faces and across the K-th slot, every branch of the grid parameters, the ring bound at the
largest grid, queries outside the box, gapped and padded layouts, and non-finite or far-flung coordinates (their rows
have no neighbours; every other row equals the brute force on the same cloud).  Every family is seeded."""
import numpy as np
import pytest
import torch

import oracle
from tests.util import knn_long_line

pytestmark = pytest.mark.gpu

F32 = np.float32


def _t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _covered(first, num, rows):
    m = np.zeros(rows, bool)
    for f, n in zip(first, num):
        m[int(f):int(f) + int(n)] = True
    return m


def run_knn(dev, x, first, num, K, r, q=None, qfirst=None, qnum=None):
    """kernel through knn_points_packed -> (dists, idxs) as numpy; rows no query range covers are dropped to -1"""
    from dss_b200.frnn_grid import knn_points_packed
    first, num = np.asarray(first, np.int64), np.asarray(num, np.int64)
    if q is None:
        d, i = knn_points_packed(_t(x, dev), _t(first, dev), _t(num, dev), K, r)
        cover = _covered(first, num, len(x))
    else:
        qfirst, qnum = np.asarray(qfirst, np.int64), np.asarray(qnum, np.int64)
        d, i = knn_points_packed(_t(x, dev), _t(first, dev), _t(num, dev), K, r, _t(q, dev), _t(qfirst, dev),
                                 _t(qnum, dev))
        cover = _covered(qfirst, qnum, len(q))
    d, i = d.cpu().numpy(), i.cpu().numpy()
    d[~cover], i[~cover] = -1, -1
    return d, i


def want_knn(x, first, num, K, r, q=None, qfirst=None, qnum=None):
    if q is None:
        q, qfirst, qnum = x, first, num
    return oracle.knn_brute(q, qfirst, qnum, x, first, num, K, r)


def check(dev, x, first, num, K, r, q=None, qfirst=None, qnum=None):
    """kernel == brute force bit for bit on every covered row -> the brute force's (dists, idxs)"""
    got_d, got_i = run_knn(dev, x, first, num, K, r, q, qfirst, qnum)
    want_d, want_i = want_knn(x, first, num, K, r, q, qfirst, qnum)
    cover = _covered(first if q is None else qfirst, num if q is None else qnum, len(x) if q is None else len(q))
    want_d[~cover], want_i[~cover] = -1, -1
    bad = ~((got_d.view(np.uint32) == want_d.view(np.uint32)).all(1) & (got_i == want_i).all(1))
    assert not bad.any(), "%d rows differ, first %d: got %s / %s, want %s / %s" % (
        bad.sum(), np.argmax(bad), got_d[bad][0], got_i[bad][0], want_d[bad][0], want_i[bad][0])
    return want_d, want_i


def check_both(dev, x, first, num, K, r, seed=0):
    """self mode, then general mode with a separate seeded query set near the same clouds"""
    out = check(dev, x, first, num, K, r)
    rng = np.random.default_rng(seed)
    qnum = np.array([min(int(n), 50) + (i % 3) for i, n in enumerate(num)], np.int64)
    qfirst = (np.cumsum(qnum) - qnum).astype(np.int64)
    qs = []
    for f, n, m in zip(first, num, qnum):
        if n > 0:
            src = x[int(f) + rng.integers(0, int(n), int(m))]
            qs.append((src + rng.standard_normal(src.shape).astype(F32) * F32(0.02)).astype(F32))
        else:
            qs.append(rng.uniform(-1, 1, (int(m), 3)).astype(F32))
    q = np.concatenate(qs) if qs else np.zeros((0, 3), F32)
    check(dev, x, first, num, K, r, q, qfirst, qnum)
    return out


def packed(*clouds):
    x = np.ascontiguousarray(np.concatenate(clouds).astype(F32)) if clouds else np.zeros((0, 3), F32)
    num = np.array([len(c) for c in clouds], np.int64)
    return x, (np.cumsum(num) - num).astype(np.int64), num


# ---------------------------------------------------------------------------------------------------------------------
KS = [1, 2, 7, 8, 9, 16, 17, 31, 32]


@pytest.mark.parametrize("K", KS)
@pytest.mark.parametrize("r", [-1.0, 0.15])
def test_k_across_dispatch(cuda_device, K, r):
    """every K on both sides of the 8 / 16 / 32 instantiations; clouds of 1, K-1, K and K+1 points (short lists,
    -1 padding) and a ragged batch with empty clouds"""
    rng = np.random.default_rng(100 + K)
    sizes = [1, K - 1, K, K + 1, 0, 300, 0, 2000]
    clouds = [rng.uniform(-0.3, 0.3, (n, 3)).astype(F32) for n in sizes]
    x, first, num = packed(*clouds)
    d, i = check_both(cuda_device, x, first, num, K, r, seed=K)
    # the small clouds: every point of the cloud is listed when there is no radius, the rest is -1
    if r < 0:
        for c in range(4):
            f, n = int(first[c]), int(num[c])
            assert ((i[f:f + n] >= 0).sum(1) == min(n, K)).all()


def test_radius_boundary(cuda_device):
    """d == r^2 exactly (dyadic coordinates, exact sums: excluded), one ulp inside (included), r <= 0, r at and
    above the extent, and r below the smallest spacing (self only)"""
    rng = np.random.default_rng(7)
    r = F32(5 / 16)
    r2 = F32(r * r)
    offs = np.array([[3, 4, 0], [4, 0, 3], [0, 3, 4], [5, 0, 0], [0, -5, 0], [0, 0, 5], [-3, -4, 0], [4, 3, 0]],
                    F32) / F32(16)
    # integer centres, 1 apart at least, so only the designed pairs are within r; offsets are multiples of 1/16
    centres = rng.permutation(np.stack(np.meshgrid(*[np.arange(-4, 5)] * 3, indexing="ij"), -1).reshape(-1, 3))[:40]
    centres = centres.astype(F32)
    pts = [centres]
    on = centres[:, None, :] + offs[rng.integers(0, len(offs), len(centres))][:, None, :]
    pts.append(on[:, 0])
    # the squared distance in the kernel's order of operations
    d = lambda p, c: F32(F32(F32(F32(p[0] - c[0]) ** 2) + F32(F32(p[1] - c[1]) ** 2)) + F32(F32(p[2] - c[2]) ** 2))
    assert all(d(on[j, 0], centres[j]) == r2 for j in range(len(centres)))
    # just inside: step one non-zero coordinate towards the centre, ulp by ulp, until d < r^2 (one step where the
    # coordinate is large, a few where it is small and one ulp of it moves d by less than an ulp of r^2)
    inside = on[:, 0].copy()
    ax = rng.integers(0, 3, len(centres))
    for j, a in enumerate(ax):
        nz = np.nonzero(inside[j] != centres[j])[0]
        a = nz[a % len(nz)]
        while not d(inside[j], centres[j]) < r2:
            inside[j, a] = np.nextafter(inside[j, a], centres[j, a])
    assert all(F32(r2 - d(inside[j], centres[j])) < 1e-6 for j in range(len(centres)))
    x, first, num = packed(np.concatenate([centres, on[:, 0]]))
    wd, wi = check_both(cuda_device, x, first, num, 8, float(r))
    n = len(centres)
    assert (wi[:n, 1] == -1).all()                              # the r^2 pairs are not neighbours
    x, first, num = packed(np.concatenate([centres, inside]))
    wd, wi = check_both(cuda_device, x, first, num, 8, float(r))
    assert (wi[:n, 1] == np.arange(n) + n).all()                # one ulp inside: neighbours
    # r <= 0, r at the extent, r above it, r below the smallest spacing (self only)
    x, first, num = packed(np.concatenate([centres, on[:, 0], inside]))
    ext = float((x.max(0) - x.min(0)).max())
    for rr in (-1.0, 0.0, ext, 2 * ext):
        check_both(cuda_device, x, first, num, 16, rr)
    wd, wi = check(cuda_device, x, first, num, 4, 1e-9)
    assert (wi[:, 0] == np.arange(len(x))).all() and (wi[:, 1:] == -1).all()


@pytest.mark.parametrize("K", [1, 4, 7, 19, 20, 32])
def test_ties(cuda_device, K):
    """more than K exact duplicates (the smallest indices win), integer lattices whose points sit on cell faces (the
    radius 1 + 2^-20 sets the cell to it, so every coordinate lands just below a face) with equal distances, and
    ties that straddle the K-th slot"""
    rng = np.random.default_rng(30 + K)
    base = rng.uniform(-1, 1, (300, 3)).astype(F32)
    dup = np.repeat(base[:3], 40, axis=0)
    x = np.concatenate([base, dup]).astype(F32)
    x = x[rng.permutation(len(x))]
    first, num = np.zeros(1, np.int64), np.array([len(x)], np.int64)
    for r in (-1.0, 0.2):
        check_both(cuda_device, x, first, num, K, r, seed=K)
    g = np.stack(np.meshgrid(*[np.arange(12)] * 3, indexing="ij"), -1).reshape(-1, 3).astype(F32)
    g = g[rng.permutation(len(g))]
    gp = g[g[:, 2] == 5]                                        # a planar lattice
    x, first, num = packed(g, gp, g * F32(0.125))
    for r in (-1.0, 1.0 + 2.0 ** -20, 1.5, 0.125 * (1 + 2.0 ** -20)):
        check_both(cuda_device, x, first, num, K, r, seed=K + 1)


def test_grid_parameter_branches(cuda_device):
    """every branch of knn_params_kernel: the density cell, the emax/1024 floor, the radius clamp, the degenerate
    cloud (cell = 1), the growth loop, planar and line clouds, two clusters far apart"""
    dev = cuda_device
    rng = np.random.default_rng(11)
    sph = rng.standard_normal((8000, 3)); sph = (0.5 * sph / np.linalg.norm(sph, axis=1, keepdims=True)).astype(F32)
    needle = (rng.uniform(0, 1, (8000, 3)) * [1, 1e-3, 1e-3]).astype(F32)          # area tiny: the 1/1024 floor wins
    cube = rng.uniform(-0.5, 0.5, (12000, 3)).astype(F32)                        # r = 0.006: (1/0.006)^3 > 2^21 cells
    plane = np.concatenate([rng.uniform(-1, 1, (5000, 2)), np.zeros((5000, 1))], 1).astype(F32)
    line = np.concatenate([rng.uniform(-1, 1, (3000, 1)), np.zeros((3000, 2))], 1).astype(F32)
    clusters = np.concatenate([rng.standard_normal((1500, 3)) * 0.05 - 1000, rng.standard_normal((1500, 3)) * 0.05 + 1000]
                              ).astype(F32)
    one = np.array([[0.25, -0.5, 3.0]], F32)
    same = np.tile(np.array([[1.5, 2.5, -0.5]], F32), (50, 1))
    for cloud, rs in ((sph, (0.2, -1.0, 0.01)), (needle, (-1.0, 0.002)), (cube, (0.006, 0.05)),
                      (plane, (0.05, -1.0)), (line, (0.01, -1.0)), (clusters, (0.2, -1.0)), (one, (0.2, -1.0)),
                      (same, (0.2, -1.0))):
        x, first, num = packed(cloud)
        for r in rs:
            for K in (7, 32):
                check_both(dev, x, first, num, K, r, seed=len(cloud))
    # all of them in one call
    x, first, num = packed(sph, needle, one, same, line, clusters)
    check_both(dev, x, first, num, 9, 0.2)


def test_ring_bound_long_line(cuda_device):
    """The line of tests.util.knn_long_line: 2095001 cells along x (the most the radius clamp allows at r = 0.2), and
    triples A, B, C where B is two computed cells right of A at less than a cell, and C in A's cell a little farther.
    A's nearest other point is B; a search that stopped after ring 1 would return C.  Queries: the points
    themselves, and general-mode queries on and a few ulps off the A's."""
    dev = cuda_device
    pts, A, B, C = knn_long_line()
    first, num = np.zeros(1, np.int64), np.array([len(pts)], np.int64)
    for K in (2, 3, 7):
        wd, wi = check(dev, pts, first, num, K, 0.2)
        if K == 2:
            assert (wi[A, 1] == B).all()
    qs = [pts[A]]
    for s in (-np.inf, np.inf):
        qa = pts[A].copy()
        for _ in range(3):                                      # 1, 2 and 3 ulps off A along x, on both sides
            qa[:, 0] = np.nextafter(qa[:, 0], F32(s))
            qs.append(qa.copy())
    q = np.concatenate(qs).astype(F32)
    for K in (1, 2):
        check(dev, pts, first, num, K, 0.2, q, np.zeros(1, np.int64), np.array([len(q)], np.int64))


def test_general_mode_queries(cuda_device):
    """queries far outside the box (clamped to a border cell) with r > 0 (no neighbours) and r <= 0 (K neighbours),
    queries identical to data points, empty query clouds against points and queries against empty clouds"""
    dev = cuda_device
    rng = np.random.default_rng(21)
    a = rng.uniform(-0.5, 0.5, (3000, 3)).astype(F32)
    b = rng.uniform(-0.5, 0.5, (40, 3)).astype(F32)
    x, first, num = packed(a, np.zeros((0, 3), F32), b, rng.uniform(0, 1, (500, 3)).astype(F32))
    far = np.concatenate([rng.uniform(-1, 1, (20, 3)) * 1e3, rng.uniform(-1, 1, (10, 3)) * 1e30,
                          np.array([[0.6, 0, 0], [0, -0.6, 0], [0.5, 0.5, 0.5]])]).astype(F32)
    same = a[rng.integers(0, len(a), 30)]
    q, qfirst, qnum = packed(np.concatenate([far, same]), rng.uniform(-1, 1, (7, 3)).astype(F32), np.zeros((0, 3), F32),
                             far)
    for K in (1, 7, 17, 32):
        for r in (-1.0, 0.2):
            wd, wi = check(dev, x, first, num, K, r, q, qfirst, qnum)
            if r > 0:
                assert (wi[:30] == -1).all()
            else:                                   # at 1e30 the squared distance overflows: no neighbour there
                assert (wi[:20] >= 0).all() and (wi[20:30] == -1).all()
            assert (wi[33:63, 0] >= 0).all() and (wd[33:63, 0] == 0).all()
            assert (wi[63:70] == -1).all()                                  # against the empty cloud


def test_layouts(cuda_device):
    """gapped first_idx (self and general mode), padded storage passed as packed (first = n Pmax, num = lengths;
    padding rows are never written), and 64 clouds of 0, 1, 2, ... points in one call"""
    dev = cuda_device
    rng = np.random.default_rng(41)
    lens = [700, 0, 1, 33, 1200]
    gaps = [5, 3, 0, 17, 2, 9]
    x = rng.uniform(-0.4, 0.4, (sum(lens) + sum(gaps), 3)).astype(F32)
    first = np.array([sum(lens[:n]) + sum(gaps[:n + 1]) for n in range(len(lens))], np.int64)
    num = np.array(lens, np.int64)
    for K, r in ((7, 0.2), (16, -1.0), (32, 0.1)):
        check_both(dev, x, first, num, K, r)
    Pmax = 900
    lengths = np.array([900, 0, 450, 1, 899], np.int64)
    pad = np.full((len(lengths), Pmax, 3), F32(7), F32)
    for n, L in enumerate(lengths):
        pad[n, :L] = rng.uniform(-0.5, 0.5, (L, 3))
    xp = pad.reshape(-1, 3)
    fp = np.arange(len(lengths), dtype=np.int64) * Pmax
    for K, r in ((7, 0.2), (9, -1.0)):
        check_both(dev, xp, fp, lengths, K, r)
    x64, f64, n64 = packed(*[rng.uniform(-0.5, 0.5, (n, 3)).astype(F32) for n in range(64)])
    for K, r in ((1, -1.0), (8, 0.3), (32, -1.0)):
        check_both(dev, x64, f64, n64, K, r)


def test_nonfinite_and_extreme_coordinates(cuda_device):
    """NaN, +inf or -inf in one axis (for a data point and for a query), +-3e38 in one cloud (the extent overflows),
    three outliers at 1e8 on three axes with r = 0.2, -0.0 next to +0.0: rows with a non-finite coordinate are all -1,
    every other row equals the brute force on the same cloud"""
    dev = cuda_device
    rng = np.random.default_rng(51)

    def body(n):
        return rng.uniform(-0.5, 0.5, (n, 3)).astype(F32)

    bad = []
    for v in (np.nan, np.inf, -np.inf):
        for ax in range(3):
            p = np.zeros(3, F32)
            p[ax] = v
            bad.append(p)
    bad = np.array(bad, F32)
    c0 = np.concatenate([body(1000), bad, body(200)])                       # non-finite data points
    c1 = np.concatenate([body(500), [[3e38, 0, 0], [-3e38, 0.1, 0], [3e38, 3e38, -3e38]]]).astype(F32)
    c2 = np.concatenate([body(800), [[1e8, 0, 0], [0, 1e8, 0], [0, 0, 1e8]]]).astype(F32)
    c3 = np.array([[-0.0, 0, 0], [0.0, 0, 0], [0, -0.0, 0.25], [0, 0.0, 0.25], [-0.0, -0.0, -0.0], [0.5, 0, 0]], F32)
    c4 = np.concatenate([bad, bad]).astype(F32)                             # nothing finite at all
    for clouds in ((c0,), (c1,), (c2,), (c3,), (c4,), (c0, c1, c2, c3, c4)):
        x, first, num = packed(*clouds)
        nonfinite = ~np.isfinite(x).all(1)
        for K in (1, 7, 16, 32):
            for r in (0.2, -1.0):
                wd, wi = check_both(dev, x, first, num, K, r, seed=K)
                assert (wi[nonfinite] == -1).all() and (wd[nonfinite] == -1).all()
    # queries with a non-finite coordinate against a finite cloud
    q = np.concatenate([bad, body(20)]).astype(F32)
    xq, fq, nq = packed(body(400))
    for r in (0.2, -1.0):
        wd, wi = check(dev, xq, fq, nq, 8, r, q, np.zeros(1, np.int64), np.array([len(q)], np.int64))
        assert (wi[:len(bad)] == -1).all() and (wi[len(bad):, 0] >= 0).all()


def test_compute_h_consumers(cuda_device):
    """SurfaceSplatting._compute_h (isotropic and invariant) bit for bit against the same rule on the brute force's
    distances: clouds below 7 points, rows with fewer than 6 neighbours inside r"""
    from dss_b200.core.cloud import PointClouds3D
    from dss_b200.core.rasterizer import PointsRasterizationSettings, SurfaceSplatting
    dev = cuda_device
    rng = np.random.default_rng(61)
    sph = rng.standard_normal((3000, 3)); sph = (0.5 * sph / np.linalg.norm(sph, axis=1, keepdims=True)).astype(F32)
    sparse = rng.uniform(-2, 2, (400, 3)).astype(F32)                       # most rows: fewer than 6 within 0.2
    tiny = rng.uniform(-0.1, 0.1, (5, 3)).astype(F32)
    clouds = [sph, sparse, tiny, sph[:7]]
    for iso in (True, False):
        settings = PointsRasterizationSettings(Vrk_isotropic=iso, Vrk_invariant=not iso)
        rast = SurfaceSplatting(raster_settings=settings)
        pc = PointClouds3D([_t(c, dev) for c in clouds])
        h = rast._compute_h(pc).cpu()
        want = []
        for c in clouds:
            if len(c) < 7:
                want.append(torch.full((len(c),), 0.5e-3, device=dev))
                continue
            n1 = np.array([len(c)], np.int64)
            d, _ = oracle.knn_brute(c, np.zeros(1, np.int64), n1, c, np.zeros(1, np.int64), n1, 7, 0.2)
            want.append(0.5 * _t(d, dev)[:, 1:].max(dim=-1)[0])
        if iso:
            w = torch.cat(want).clamp(5e-5, 0.01).float()
        else:
            w = torch.stack([v.mean().clamp(5e-5, 1e-3) for v in want]).float()
        assert torch.equal(h, w.cpu())


def test_padded_wrappers_ragged(cuda_device):
    """frnn_grid_points (-1 padding) and knn_points (zero padding) on ragged padded batches, self and cross"""
    from dss_b200.frnn_grid import frnn_grid_points, knn_points
    dev = cuda_device
    rng = np.random.default_rng(71)
    N, P1, P2 = 4, 600, 900
    p1 = rng.uniform(-0.5, 0.5, (N, P1, 3)).astype(F32)
    p2 = rng.uniform(-0.5, 0.5, (N, P2, 3)).astype(F32)
    l1 = np.array([600, 0, 3, 250], np.int64)
    l2 = np.array([900, 17, 0, 40], np.int64)
    z = np.zeros(1, np.int64)
    for K, r in ((7, 0.2), (12, -1.0)):
        a, la = _t(p2, dev), _t(l2, dev)
        d, i, _, _ = frnn_grid_points(a, a, la, la, K=K, r=r)
        d2, i2, _, _ = frnn_grid_points(_t(p1, dev), a, _t(l1, dev), la, K=K, r=r)
        kd, ki, _ = knn_points(_t(p1, dev), a, _t(l1, dev), la, K=K)
        for n in range(N):
            L1, L2 = int(l1[n]), int(l2[n])
            wd, wi = oracle.knn_brute(p2[n, :L2], z, [L2], p2[n, :L2], z, [L2], K, r)
            assert np.array_equal(d[n, :L2].cpu().numpy(), wd) and np.array_equal(i[n, :L2].cpu().numpy(), wi)
            assert (d[n, L2:] == -1).all() and (i[n, L2:] == -1).all()
            wd, wi = oracle.knn_brute(p1[n, :L1], z, [L1], p2[n, :L2], z, [L2], K, r)
            assert np.array_equal(d2[n, :L1].cpu().numpy(), wd) and np.array_equal(i2[n, :L1].cpu().numpy(), wi)
            assert (d2[n, L1:] == -1).all() and (i2[n, L1:] == -1).all()
            wd, wi = oracle.knn_brute(p1[n, :L1], z, [L1], p2[n, :L2], z, [L2], K, -1.0)
            assert np.array_equal(kd[n, :L1].cpu().numpy(), np.where(wi < 0, 0, wd))
            assert np.array_equal(ki[n, :L1].cpu().numpy(), np.maximum(wi, 0))


def test_input_checks_raise_before_any_launch(cuda_device):
    """K = 0 and 33 and N = 1024 (N * 2^21 cells) raise, in the wrapper and in the C ABI, and launch nothing"""
    from dss_b200 import _lib
    from dss_b200.frnn_grid import knn_points_packed
    dev = cuda_device
    x = _t(np.zeros((4, 3), F32), dev)
    f, n = _t(np.zeros(1, np.int64), dev), _t(np.array([4], np.int64), dev)
    torch.cuda.synchronize()
    before = _lib.launch_count(dev)
    for K in (0, 33):
        with pytest.raises(RuntimeError):
            knn_points_packed(x, f, n, K, 0.2)
        d = torch.empty((4, max(K, 1)), device=dev)
        with torch.cuda.device(dev):
            rc = _lib.load().dss_knn_points(_lib.ctx(dev), None, None, None, _lib.ptr(x), _lib.ptr(f), _lib.ptr(n), 1,
                                            4, 4, K, 0.2, _lib.ptr(d), None, _lib.stream_ptr(dev))
        assert rc != 0
    f1024 = _t(np.zeros(1024, np.int64), dev)
    n1024 = _t(np.zeros(1024, np.int64), dev)
    n1024[0] = 4
    with pytest.raises(RuntimeError, match="too many clouds"):
        knn_points_packed(x, f1024, n1024, 7, 0.2)
    assert _lib.launch_count(dev) == before


def test_two_calls_identical_bits(cuda_device):
    dev = cuda_device
    rng = np.random.default_rng(81)
    x, first, num = packed(rng.uniform(-0.5, 0.5, (20000, 3)).astype(F32), np.repeat(rng.uniform(-1, 1, (10, 3)), 50, 0),
                           rng.uniform(-0.5, 0.5, (3000, 3)).astype(F32))
    for K, r in ((7, 0.2), (32, -1.0)):
        a = run_knn(dev, x, first, num, K, r)
        b = run_knn(dev, x, first, num, K, r)
        assert np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32)) and np.array_equal(a[1], b[1])


@pytest.mark.parametrize("P,K,r", [(1_000_000, 7, 0.2), (1_000_000, 32, -1.0), (300_000, 17, 0.05)])
def test_large_clouds_sampled_rows(cuda_device, P, K, r):
    """up to 1M points: a seeded sample of self-mode rows equals the brute force run with those rows as queries,
    distances and indices"""
    from dss_b200.frnn_grid import knn_points_packed
    from tests.util import sample_rows, sphere_cloud
    dev = cuda_device
    x = sphere_cloud(P, seed=P % 7)[0].numpy()
    f, n = np.zeros(1, np.int64), np.array([P], np.int64)
    d, i = knn_points_packed(_t(x, dev), _t(f, dev), _t(n, dev), K, r)
    rows = sample_rows(P, 256, seed=K)
    wd, wi = oracle.knn_brute(x[rows], f, np.array([len(rows)], np.int64), x, f, n, K, r)
    assert np.array_equal(d.cpu().numpy()[rows].view(np.uint32), wd.view(np.uint32))
    assert np.array_equal(i.cpu().numpy()[rows], wi)


def test_kernel_reproduces_reference_bruteforce_edge_vectors(cuda_device):
    """the edge families minted from the reference's own FRNNBruteForceCPU (tests/golden/make_golden_knn.py), on the
    kernel through the padded wrapper"""
    from dss_b200.frnn_grid import frnn_grid_points
    from tests.test_knn import GOLD, edge_cases
    d = np.load(GOLD)
    for name, pts, lens, K, r in edge_cases(d):
        p, l = _t(pts, cuda_device), _t(lens, cuda_device)
        dist, idx, _, _ = frnn_grid_points(p, p, l, l, K=K, r=r)
        assert np.array_equal(dist.cpu().numpy().view(np.uint32), d[name + "__dists"].view(np.uint32)), name
        assert np.array_equal(idx.cpu().numpy(), d[name + "__idxs"].astype(np.int64)), name
