"""The fused projection / repulsion regularisers (`dss_surface_regulariser`, csrc/regularisers.cu) against the torch
body of `ProjectionLoss` / `RepulsionLoss` run in float64 on the same K-NN rows, point by point, at their corners.

Both sides get one K-NN computed by the CUDA kernel: the fused route as packed rows, the torch body as a padded
`knn_tree` with the float32 distances promoted to float64 (and the -1 padding turned into pytorch3d's 0 / 0, which the
fused kernel does itself).  Only rounding differs, and `bound` limits that difference per point and component.
"""
import pytest
import torch

from dss_b200 import _lib
from dss_b200.core.cloud import PointClouds3D, PointCloudsFilters
from dss_b200.frnn_grid import knn_points_packed
from dss_b200.training.losses import ProjectionLoss, RepulsionLoss, surface_regulariser
from tests.util import sphere_cloud

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
LOSSES = {"projection": ProjectionLoss, "repulsion": RepulsionLoss}


@pytest.fixture(autouse=True)
def _cuda(cuda_device):
    return cuda_device


def noisy_sphere(P, seed):
    pts, nrm, _ = sphere_cloud(P, seed=seed)
    g = torch.Generator().manual_seed(seed)
    pts = pts + 0.002 * torch.randn(P, 3, generator=g)
    nrm = torch.nn.functional.normalize(nrm + 0.2 * torch.randn(P, 3, generator=g), dim=1)
    return pts, nrm


def make_clouds(sizes, seed, dev):
    pts, nrm = [], []
    for k, P in enumerate(sizes):
        p, n = noisy_sphere(max(P, 1), seed + k)
        pts.append(p[:P].to(dev))
        nrm.append(n[:P].to(dev))
    return pts, nrm


def padded_tree(d, i, sizes, dtype):
    """packed (P,K) CUDA K-NN rows -> the padded (N, P_max, K) tree of the torch body, -1 -> pytorch3d's 0 / 0"""
    N, Pm, K = len(sizes), max(sizes), d.shape[1]
    dd = torch.zeros(N, Pm, K, dtype=dtype, device=d.device)
    ii = torch.zeros(N, Pm, K, dtype=torch.int64, device=d.device)
    o = 0
    for n, P in enumerate(sizes):
        miss = i[o:o + P] < 0
        dd[n, :P] = torch.where(miss, 0.0, d[o:o + P].to(dtype))
        ii[n, :P] = torch.where(miss, 0, i[o:o + P].long())
        o += P
    return dd, ii


def pack(x, sizes):
    return torch.cat([x[n, :P] for n, P in enumerate(sizes)])


def make_filter(kind, sizes, batch, seed, dev):
    if kind is None:
        return None
    g = torch.Generator().manual_seed(seed)
    Pm = max(sizes)
    vis = (torch.rand(batch, Pm, generator=g) < 0.6).to(dev)
    inm = (torch.rand(batch, Pm, generator=g) < 0.8).to(dev) if kind == "vis&inmask" else None
    return PointCloudsFilters(device=dev, visibility=vis, inmask=inm)


def run_fused(kind, pts, nrm, K, filt, kw, grad_seed, reduction="none", tree=None, loss=None, rebuild_knn=True):
    ps = [p.clone().requires_grad_(True) for p in pts]
    cloud = PointClouds3D(ps, normals=nrm)
    if tree is not None:
        kw = dict(kw, knn_tree=tree)
    loss = loss or LOSSES[kind](reduction=reduction, knn_k=K)
    out = loss(cloud, points_filter=filt, rebuild_knn=rebuild_knn, **kw)
    g = torch.randn(out.shape, generator=torch.Generator().manual_seed(grad_seed)).double()     # float32-exact
    (out * g.to(out.device, out.dtype)).sum().backward()
    return out.detach(), torch.cat([p.grad for p in ps]), g


def twin_f64(kind, pts, nrm, K, filt, kw, tree, g, loss=None):
    """the torch body in float64 -> (loss, grad, magnitudes used by the bound) on the packed rows; tree None: the
    tree `loss` stored in an earlier call (rebuild_knn=False)"""
    sizes = [p.shape[0] for p in pts]
    ps = [p.double().clone().requires_grad_(True) for p in pts]
    cloud = PointClouds3D(ps, normals=[n.double() for n in nrm])
    loss = loss or LOSSES[kind](reduction="none", knn_k=K)
    if tree is not None:
        kw = dict(kw, knn_tree=tree)
    out = loss(cloud, points_filter=filt, rebuild_knn=False, **kw)
    (out * g.to(out.device)).sum().backward()
    grad = torch.cat([p.grad for p in ps])
    with torch.no_grad():
        mag = magnitudes(kind, loss, cloud, filt, out, g.to(out.device), kw, sizes)
    return out.detach(), grad, mag


def magnitudes(kind, loss, cloud, filt, out, g, kw, sizes):
    """Float64 magnitudes of each row's terms, with every factor replaced by a bound on its size (see `bound`)."""
    tree = loss.knn_tree
    dist, h = tree.dists, tree.dists.mean(dim=-1, keepdim=True) * 4
    t = (1 - dist / h).clamp(min=0)
    phib = t ** 4 + 4 * t ** 3                                        # |phi| + |d phi / d t|
    den = loss._denoise_normals(cloud, loss.get_phi(cloud), filt)
    nw = loss.get_normal_w(den, **kw)
    lengths = cloud.num_points_per_cloud()
    from dss_b200.training.losses import knn_gather
    nz = knn_gather(den, tree.idx, lengths).abs()
    pts = cloud.points_padded()
    u = (tree.knn - pts[:, :, None, :]).abs()
    sbar = (u * nz).sum(-1)                                          # magnitude of sdf = (q - p) . n^
    if kind == "projection":
        vis = getattr(filt, "visibility", None) if filt is not None else None
        if vis is not None and vis.shape[0] != len(sizes) and len(sizes) == 1:
            vis = vis.any(dim=0, keepdim=True)
        vw = 1.0 if vis is None else torch.where(knn_gather(vis[..., None], tree.idx, lengths)[..., 0], 1.0, 0.1)
        wb = phib * nw * vw
        E = (loss.get_phi(cloud) * nw * vw).sum(-1).abs().clamp(min=1e-17)
        lmag = (wb * sbar ** 2).sum(-1) / E
        gmag = 2 * (wb[..., None] * sbar[..., None] * nz).sum(-2) / E[..., None]
        return pack(lmag, sizes), pack(gmag, sizes)
    sp = loss.get_spatial_w(cloud, **kw)
    arg = -torch.log(sp.clamp(min=1e-300))
    wb = sp * nw * (1 + arg)
    w = sp * nw
    E = w.sum(-1).abs().clamp(min=1e-17)
    dens = sp.sum(-1) + 1
    R = dens[..., None] / E[..., None] * (wb[..., None] * (u + sbar[..., None] * nz)).sum(-2)
    J = dens[..., None, None] / E[..., None, None] * (
        wb.sum(-1)[..., None, None] * torch.eye(3, dtype=wb.dtype, device=wb.device)
        + (wb[..., None, None] * nz[..., :, None] * nz[..., None, :]).sum(-3))
    return pack(R, sizes), pack(J, sizes)


def bound(kind, K, sigma, out64, mag, g):
    """|fused - f64| <= c * 2^-24 * S per point and component.

    Error model: every float32 operation rounds with relative error <= u = 2^-24; a sum of m terms adds m - 1
    roundings, each bounded by u times the running sum of magnitudes.  Along the kernel's sequence (neighbour j):
      h = 4 * sum(d) / (K-1): K + 1 roundings; t = 1 - d/h: absolute error <= (K + 3) u (d/h <= 1 where t > 0);
      phi = (t^2)^2: |d phi| <= 4 t^3 (K + 3) u + 2 u phi  -> (K + 5) u * (phi + 4 t^3) = (K + 5) u * phib;
      n^ (denoise): K - 1 products and sums and one division: (K + 2) u on a unit-sized vector; normalize: 4 u more;
      normal_w = exp(-|m - n|^2 / sigma^2): the argument's absolute error <= (2 (K + 6) + 4) u * 4 / sigma^2
        (|m - n|^2 <= 4), exp adds 2 u: c_nw = 4 (2K + 16) / sigma^2 + 2;
      projection: sdf = sum (q - p) n^: 1 (subtraction) + (K + 2) (n^) + 3 (products, sums) u on sbar;
        w sdf^2 / E: c = (K + 5) + c_nw + 2 (visibility, products) + 2 (K + 6) (sdf^2) + (K - 1) (sum) + (K - 1) (E)
        + 1 (division); the gradient -2 sum w sdf n^ / E carries the same count plus (K + 2) for n^: S = gmag |g|.
      repulsion: spatial_w = exp(-a), a = |q - p|^2 P / diag^2 * fs: relative error of a <= 10 u (diag, products),
        so that of spatial_w <= 10 u a + 2 u, in wb = sp nw (1 + a); r = dens / E * sum w proj, proj = u - (u.n^) n^
        with magnitude |u| + sbar |n^|: c = c_nw + 12 + 2 (K + 6) + 3 (K - 1) (w, dens, E sums) + 3; the loss
        exp(-|r|) has |d loss| <= loss (|d r| + 2 u): S = loss (R + 1); the gradient J (g * s), s = -sign(r) loss:
        S = sum_b |g_b| J_ab loss_b (R_b + 1) with J's own error inside the same count.
    A factor 1.25 covers the second-order terms; the float64 side's own error is below 2^-40 relative."""
    c_nw = 4 * (2 * K + 16) / sigma ** 2 + 2
    if kind == "projection":
        lmag, gmag = mag
        c = 1.25 * ((K + 5) + c_nw + 2 + 2 * (K + 6) + 2 * (K - 1) + 1)
        gc = c + 1.25 * (K + 2)
        return c * U * lmag, gc * U * gmag * g.abs()[:, None]
    R, J = mag
    c = 1.25 * (c_nw + 12 + 2 * (K + 6) + 3 * (K - 1) + 3)
    l64 = out64.abs()
    lb = c * U * l64 * (R + 1)
    gb = c * U * (J * (g.abs() * l64 * (R + 1))[:, None, :]).sum(-1)
    return lb, gb


def check(kind, sizes, K, filt_kind="vis", batch=None, kw=None, seed=0, tree_layout="self", ratios=None):
    dev = torch.device("cuda:0")
    pts, nrm = make_clouds(sizes, seed, dev)
    kw = dict(kw or {})
    N = len(sizes)
    filt = make_filter(filt_kind, sizes, batch or N, seed + 100, dev)
    P = sum(sizes)
    first = torch.tensor([sum(sizes[:n]) for n in range(N)], dtype=torch.int64, device=dev)
    num = torch.tensor(sizes, dtype=torch.int64, device=dev)
    d, i = knn_points_packed(torch.cat(pts), first, num, K)
    tree32, tree64 = padded_tree(d, i, sizes, torch.float32), padded_tree(d, i, sizes, torch.float64)
    if tree_layout == "noself":
        tree32, tree64 = (tuple(t[..., 1:].contiguous() for t in tr) for tr in (tree32, tree64))
    fused_tree = None if tree_layout == "search" else (*tree32, None)      # "search": the module's own K-NN
    out, grad, g = run_fused(kind, pts, nrm, K, filt, kw, seed + 7, tree=fused_tree)
    out64, grad64, mag = twin_f64(kind, pts, nrm, K, filt, kw, (*tree64, None), g)
    compare(kind, K, kw, out, grad, out64, grad64, mag, g, ratios)
    return out, grad


def compare(kind, K, kw, out, grad, out64, grad64, mag, g, ratios):
    """same NaN entries, and every other entry within the bound"""
    lb, gb = bound(kind, K, kw.get("sharpness_sigma", 0.75), out64, mag, g.to(out64.device))
    for a, b, B, what in ((out, out64, lb, "loss"), (grad, grad64, gb, "grad")):
        a, b = a.double(), b
        nan = torch.isnan(b)
        assert torch.equal(torch.isnan(a), nan), "%s: NaN rows differ" % what
        err = (a - b).abs()[~nan]
        Bv = B.reshape(b.shape)[~nan]
        ok = err <= Bv
        assert bool(ok.all()), "%s: %d of %d beyond the bound, worst err %.3g at bound %.3g" % (
            what, int((~ok).sum()), ok.numel(), float(err[~ok].max()), float(Bv[~ok][err[~ok].argmax()]))
        if ratios is not None:
            pos = Bv > 0
            ratios.append(float((err[pos] / Bv[pos]).max()) if bool(pos.any()) else 0.0)


@pytest.fixture(scope="module")
def worst():
    """each check's worst |fused - f64| / bound, printed when the module ends (a report: every check asserts its own
    bound)"""
    ratios = []
    yield ratios
    if ratios:
        print("\nworst ratio to the bound: %.3g over %d checks" % (max(ratios), len(ratios)))


@pytest.mark.parametrize("kind", ["projection", "repulsion"])
@pytest.mark.parametrize("P", [400, 5000, 200000])
def test_noisy_spheres_against_float64(kind, P, worst):
    check(kind, [P], 12, "vis&inmask", seed=P, ratios=worst)


@pytest.mark.parametrize("kind", ["projection", "repulsion"])
@pytest.mark.parametrize("K", [2, 12, 32])
@pytest.mark.parametrize("filt", [None, "vis", "vis&inmask"])
def test_ragged_clouds_against_float64(kind, K, filt, worst):
    """three ragged packed clouds with 1, 2, 11, 12 and 13 points among them: fewer points than knn_k included, given
    as a tree in pytorch3d's 0 / 0 padding and through the module's own K-NN, whose -1 padding the kernel maps"""
    for sizes in ([1, 12, 300], [2, 11, 13], [13, 1, 2]):
        for layout in ("self", "search"):
            check(kind, sizes, K, filt, seed=K + len(sizes), tree_layout=layout, ratios=worst)


@pytest.mark.parametrize("kind", ["projection", "repulsion"])
def test_filter_over_a_single_cloud_is_or_ed(kind, worst):
    """a filter of batch 3 over one cloud: the torch body ors it over the batch"""
    check(kind, [500], 12, "vis&inmask", batch=3, seed=5, ratios=worst)


def test_batch_one_filter_over_several_clouds(worst):
    """repulsion broadcasts a batch-1 filter over N > 1 clouds; the projection's per-neighbour gather raises, as the
    torch body's knn_gather does"""
    check("repulsion", [40, 300, 13], 12, "vis&inmask", batch=1, seed=6, ratios=worst)
    dev = torch.device("cuda:0")
    pts, nrm = make_clouds([40, 300], 1, dev)
    filt = make_filter("vis", [40, 300], 1, 3, dev)
    for d in (dev, "cpu"):
        cloud = PointClouds3D([p.to(d) for p in pts], normals=[n.to(d) for n in nrm])
        f = PointCloudsFilters(device=d, visibility=filt.visibility.to(d))
        kw = {}
        if d == "cpu":
            P = torch.cat(pts)
            first = torch.tensor([0, 40], device=dev)
            dd, ii = knn_points_packed(P, first, torch.tensor([40, 300], device=dev), 12)
            kw["knn_tree"] = tuple(t.cpu() for t in padded_tree(dd, ii, [40, 300], torch.float32)) + (None,)
        with pytest.raises(RuntimeError):
            ProjectionLoss(knn_k=12)(cloud, points_filter=f, **kw)


@pytest.mark.parametrize("kind", ["projection", "repulsion"])
def test_overrides_reductions_and_tree_layouts(kind, worst):
    kw = {"sharpness_sigma": 0.4, "filter_scale": 3.0}
    check(kind, [700, 13], 12, "vis", kw=kw, seed=11, ratios=worst)
    check(kind, [700, 13], 12, "vis", seed=12, tree_layout="noself", ratios=worst)
    check(kind, [700, 13], 12, "vis&inmask", seed=13, tree_layout="search", ratios=worst)
    # the three reductions of one call agree with the reduced per-point loss
    dev = torch.device("cuda:0")
    pts, nrm = make_clouds([900], 3, dev)
    cloud = PointClouds3D(pts, normals=nrm)
    per = LOSSES[kind](reduction="none", knn_k=12)(cloud)
    for red, f in (("sum", torch.sum), ("mean", torch.mean)):
        v = LOSSES[kind](reduction=red, knn_k=12)(cloud)
        torch.testing.assert_close(v, f(per), rtol=1e-6, atol=0)
    # a tree without the query column sets the width itself, as in the torch body: the constructor's knn_k = 33 is
    # then no error
    first, num = torch.zeros(1, dtype=torch.int64, device=dev), torch.full((1,), 900, dtype=torch.int64, device=dev)
    d, i = knn_points_packed(pts[0], first, num, 12)
    tree = tuple(t[..., 1:].contiguous() for t in padded_tree(d, i, [900], torch.float32)) + (None,)
    assert torch.equal(LOSSES[kind](reduction="none")(cloud, knn_tree=tree),
                       LOSSES[kind](reduction="none", knn_k=12)(cloud, knn_tree=tree))


@pytest.mark.parametrize("kind", ["projection", "repulsion"])
@pytest.mark.parametrize("source", ["rebuild_false", "tree_knn_self", "tree_knn_noself"])
def test_kept_neighbour_positions_against_float64(kind, source, worst):
    """The torch body keeps the neighbour positions of its tree.  With rebuild_knn=False after the points moved, they
    are the positions the rows were built on; a tree that carries `knn` brings its own.  The fused route uses the same
    positions."""
    dev = torch.device("cuda:0")
    sizes, K = [2000, 13], 12
    pts, nrm = make_clouds(sizes, 31, dev)
    gen = torch.Generator().manual_seed(5)
    moved = [p + (0.01 * torch.randn(p.shape, generator=gen)).to(dev) for p in pts]
    filt = make_filter("vis", sizes, 2, 32, dev)
    first = torch.tensor([0, sizes[0]], dtype=torch.int64, device=dev)
    d, i = knn_points_packed(torch.cat(pts), first, torch.tensor(sizes, dtype=torch.int64, device=dev), K)
    dd32, ii = padded_tree(d, i, sizes, torch.float32)
    dd64, _ = padded_tree(d, i, sizes, torch.float64)
    if source == "rebuild_false":
        f_loss, t_loss = LOSSES[kind](reduction="none", knn_k=K), LOSSES[kind](reduction="none", knn_k=K)
        run_fused(kind, pts, nrm, K, filt, {}, 1, loss=f_loss)                        # own search at `pts`
        twin_f64(kind, pts, nrm, K, filt, {}, (dd64, ii, None), torch.zeros(()), loss=t_loss)
        rows = f_loss.knn_rows
        out, grad, g = run_fused(kind, moved, nrm, K, filt, {}, 2, loss=f_loss, rebuild_knn=False)
        assert f_loss.knn_rows is rows
        out64, grad64, mag = twin_f64(kind, moved, nrm, K, filt, {}, None, g, loss=t_loss)
    else:
        # positions of the unmoved cloud at the tree's indices, jittered so that they are nobody's current position
        pp = torch.zeros(2, max(sizes), 3, device=dev)
        for n, P in enumerate(sizes):
            pp[n, :P] = pts[n]
        knn = torch.gather(pp[:, None].expand(-1, pp.shape[1], -1, -1), 2, ii[..., None].expand(-1, -1, -1, 3))
        knn = knn + (1e-3 * torch.randn(knn.shape, generator=gen)).to(dev)
        t32, t64 = (dd32, ii, knn), (dd64, ii, knn.double())
        if source == "tree_knn_noself":
            t32, t64 = (tuple(t[:, :, 1:].contiguous() for t in tr) for tr in (t32, t64))
        out, grad, g = run_fused(kind, moved, nrm, K, filt, {}, 3, tree=t32)
        out64, grad64, mag = twin_f64(kind, moved, nrm, K, filt, {}, t64, g)
    compare(kind, K, {}, out, grad, out64, grad64, mag, g, worst)


@pytest.mark.parametrize("kind", ["projection", "repulsion"])
def test_duplicates_give_the_twin_nan_rows(kind):
    """a point whose K-1 neighbours all lie at distance 0 has h = 0: its row is NaN, and the NaN reaches the rows that
    see its denoised normal, exactly as in the torch body"""
    dev = torch.device("cuda:0")
    p, n = noisy_sphere(600, 21)
    p[100:112] = p[100]                                      # 12 copies: with knn_k = 12 each has 11 at distance 0
    p[300:305] = p[300]                                      # 5 copies: not enough for h = 0
    pts, nrm = [p.to(dev)], [n.to(dev)]
    filt = make_filter("vis", [600], 1, 22, dev)
    first, num = torch.zeros(1, dtype=torch.int64, device=dev), torch.full((1,), 600, dtype=torch.int64, device=dev)
    d, i = knn_points_packed(pts[0], first, num, 12)
    o, gr, g = run_fused(kind, pts, nrm, 12, filt, {}, 9, tree=(*padded_tree(d, i, [600], torch.float32), None))
    o64, gr64, mag = twin_f64(kind, pts, nrm, 12, filt, {}, (*padded_tree(d, i, [600], torch.float64), None), g)
    nan_rows = torch.isnan(o64).reshape(600, -1).any(1)
    assert bool(nan_rows[100:112].all()) and int(nan_rows.sum()) > 12
    assert torch.equal(torch.isnan(o), torch.isnan(o64)) and torch.equal(torch.isnan(gr), torch.isnan(gr64))
    lb, gb = bound(kind, 12, 0.75, o64, mag, g.to(dev))
    ok = ~torch.isnan(o64)
    assert bool(((o.double() - o64).abs()[ok] <= lb.reshape(o64.shape)[ok]).all())
    okg = ~torch.isnan(gr64)
    assert bool(((gr.double() - gr64).abs()[okg] <= gb.reshape(gr64.shape)[okg]).all())


@pytest.mark.parametrize("kind", ["projection", "repulsion"])
def test_flat_lattice_interior_is_exactly_zero(kind):
    """a flat square lattice with float32-exact coordinates and knn_k = 9: every interior neighbourhood is two whole
    shells (4 at distance 1, 4 at distance 2), so no tie is split, r == 0 exactly and the gradient is exactly 0"""
    dev = torch.device("cuda:0")
    s = 24
    y, x = torch.meshgrid(torch.arange(s, dtype=torch.float32), torch.arange(s, dtype=torch.float32), indexing="ij")
    pts = torch.stack([x.reshape(-1) * 0.125, y.reshape(-1) * 0.125, torch.zeros(s * s)], 1).to(dev)
    nrm = torch.zeros_like(pts)
    nrm[:, 2] = 1
    ps = pts.clone().requires_grad_(True)
    out = LOSSES[kind](reduction="none", knn_k=9)(PointClouds3D([ps], normals=[nrm]))
    out.sum().backward()
    interior = ((x > 1) & (x < s - 2) & (y > 1) & (y < s - 2)).reshape(-1).to(dev)
    if kind == "projection":
        assert bool((out[interior] == 0).all())
    else:
        assert bool((out[interior] == 1).all())                # exp(-|0|)
    assert bool((ps.grad[interior] == 0).all())


@pytest.mark.parametrize("kind", ["projection", "repulsion"])
def test_two_calls_give_identical_bits(kind):
    dev = torch.device("cuda:0")
    pts, nrm = make_clouds([20000, 777], 8, dev)
    filt = make_filter("vis&inmask", [20000, 777], 2, 8, dev)
    a = run_fused(kind, pts, nrm, 12, filt, {}, 1)
    b = run_fused(kind, pts, nrm, 12, filt, {}, 1)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


@pytest.mark.parametrize("kind", ["projection", "repulsion"])
def test_no_host_sync_and_fixed_launch_count(kind):
    """after one warm-up call, the K-NN and the fused forward and backward on packed inputs do not synchronise the
    host, and neither does the loss module on a warmed cloud with a filter; the library's launch count per step does
    not depend on P or N"""
    dev = torch.device("cuda:0")
    counts = []
    for sizes in ([5000], [30000, 100, 7000]):
        pts, nrm = make_clouds(sizes, 2, dev)
        P, N = sum(sizes), len(sizes)
        p, n = torch.cat(pts).requires_grad_(True), torch.cat(nrm)
        first = torch.tensor([sum(sizes[:k]) for k in range(N)], dtype=torch.int64, device=dev)
        num = torch.tensor(sizes, dtype=torch.int64, device=dev)
        rel = torch.rand(P, device=dev) < 0.5
        vis = torch.rand(P, device=dev) < 0.5

        def step():
            d, i = knn_points_packed(p, first, num, 12)
            surface_regulariser(kind, p, n, first, num, d, i, reliable=rel, visible=vis).mean().backward()

        step()
        torch.cuda.synchronize()
        before = _lib.launch_count(dev)
        torch.cuda.set_sync_debug_mode("error")
        try:
            step()
        finally:
            torch.cuda.set_sync_debug_mode("default")
        counts.append(_lib.launch_count(dev) - before)
    # K-NN: bbox init, bbox, grid parameters, bin count, scan, bin scatter, search; regulariser: 2 / 3
    assert counts[0] == counts[1] == 7 + (2 if kind == "projection" else 3)
    # the module on a warmed single cloud, filter included
    cloud = PointClouds3D([pts[0].clone().requires_grad_(True)], normals=[nrm[0]])
    filt = make_filter("vis&inmask", [30000], 1, 2, dev)
    loss = LOSSES[kind](reduction="mean", knn_k=12)
    loss(cloud, points_filter=filt, rebuild_knn=True).backward()
    torch.cuda.set_sync_debug_mode("error")
    try:
        loss(cloud, points_filter=filt, rebuild_knn=True).backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")


def test_input_checks_raise_before_any_launch():
    dev = torch.device("cuda:0")
    pts, nrm = make_clouds([100], 0, dev)
    p, n = pts[0], nrm[0]
    first, num = torch.zeros(1, dtype=torch.int64, device=dev), torch.full((1,), 100, dtype=torch.int64, device=dev)
    d, i = knn_points_packed(p, first, num, 12)
    wide = (torch.rand(1, 100, 33, device=dev), torch.zeros(1, 100, 33, dtype=torch.int64, device=dev), None)
    torch.cuda.synchronize()
    before = _lib.launch_count(dev)
    bad = [
        lambda: ProjectionLoss(knn_k=33)(PointClouds3D([p], normals=[n]), knn_tree=wide),    # 33 columns
        lambda: ProjectionLoss(knn_k=33)(PointClouds3D([p], normals=[n])),
        lambda: RepulsionLoss(knn_k=1)(PointClouds3D([p], normals=[n])),
        lambda: surface_regulariser("projection", p, n, first, num, d[:, :1].contiguous(), i[:, :1].contiguous()),
        lambda: surface_regulariser("projection", p, n[:50], first, num, d, i),
        lambda: surface_regulariser("repulsion", p, n, first, num, d[:50], i[:50]),
        lambda: surface_regulariser("repulsion", p, n, first, num, d, i.long()),
        lambda: surface_regulariser("repulsion", p, n, first, num, d.t().contiguous().t(), i),
        lambda: surface_regulariser("repulsion", p, n, first, num, d, i[:, ::1].t().contiguous().t()),
        lambda: surface_regulariser("projection", p, n, first, num, d, i, reliable=torch.ones(99, dtype=torch.bool,
                                                                                              device=dev)),
    ]
    for f in bad:
        with pytest.raises(RuntimeError):
            f()
    assert _lib.launch_count(dev) == before
