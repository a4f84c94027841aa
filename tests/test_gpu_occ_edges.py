"""The occupancy gather (`occ_backward`) against the float64 oracle, point by point, on every dispatch path and at its
edges.

Which kernel serves a view is decided on the host from the PREVIOUS call's search radii (the staged-window hint): the
halo `R_box` of the staged box is `(occ_hh(1.15 * max rs) + 2 + 3) & ~3`, clamped to [8, 40], over the first
min(N, 96) views.  A view whose window half-width `hh = occ_hh(r)` fits (`hh + 1 <= R_box`, r < 4) takes
`occ_tile_kernel`, in the lane mapping chosen by `need = 2 * hh + 2` (`MAPPINGS`), with exact row steps for a
power-of-two S or a row table otherwise; every other view takes `occ_generic_kernel`.  At the operator level
(`_C.occ_backward`) the search radii are an input, so every case primes the hint with a call at chosen radii, then
makes the measured call, and asserts in Python which path each view takes.

The oracle is `oracle.occ_backward_fast(..., fma_mode=1)`: its disc test rounds d2 as `fmaf(dx, dx, dy*dy)` like
both kernels, and dx, dy, r*r and the box test are the same fp32 expressions on both sides, so the kernels must find
exactly the oracle's pairs.  Only the summation differs, and `bound_c` bounds that difference per point.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import oracle
from dss_b200 import _C, _lib, ops
from dss_b200.ops import SplatParams
from tests.util import occ_edge_splats, scene

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
RBOX_MAX = 40
# need <= bound -> (lanes per splat, column pairs per lane), occ_tile_kernel's consumer dispatch
MAPPINGS = [(8, 4, 1), (16, 4, 2), (24, 4, 3), (32, 4, 4), (40, 4, 5), (48, 8, 3), (64, 8, 4), (96, 16, 3)]
F = np.float32


def _t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


# ---------------------------------------------------------------------------------------------------------------------
# the host's and the device's view of the dispatch
# ---------------------------------------------------------------------------------------------------------------------
def hh_host(r, S):
    """occ_hh on the host (no contraction): floor(((r * 0.5) * S + 0.5) + 1e-3) in fp32"""
    return int(np.floor(F(F(F(F(r) * F(0.5)) * F(S)) + F(0.5)) + F(1e-3)))


def hh_device(r, S):
    """occ_hh on the device, where nvcc contracts (r * 0.5) * S + 0.5 into one FMA ((r * 0.5) * S is exact in
    float64, so the float64 sum rounded once to fp32 is that FMA)"""
    a = float(F(r) * F(0.5))
    return int(np.floor(F(F(a * S + 0.5) + F(1e-3))))


def r_box(prime_rs, S):
    """the staged halo of a call that follows one with search radii `prime_rs` (occ_backward's host code)"""
    hint = 0.0
    for v in np.asarray(prime_rs, F)[:96]:
        hint = max(hint, float(v))
    R = 20
    if 0.0 < hint < 4.0:
        R = (hh_host(F(F(hint) * F(1.15)), S) + 2 + 3) & ~3
    return min(max(R, 8), RBOX_MAX)


def view_path(r, S, R):
    """("tile", LPS, PPL) or ("generic",) for a view of search radius r under halo R"""
    r = F(r)
    if not (r >= 0 and r < 4) or hh_device(r, S) + 1 > R:
        return ("generic",)
    need = 2 * hh_device(r, S) + 2
    for bound, lps, ppl in MAPPINGS:
        if need <= bound:
            return ("tile", lps, ppl)
    raise AssertionError(need)


def path_name(p):
    return "g" if p[0] == "generic" else "%dx%d" % p[1:]


def bound_c(path, r, S):
    """c of the per-point bound |ours - f64| <= c * 2^-24 * sum|t| (sum over the point's terms t = d/den * g, for the
    x and the y component separately).  Both sides find the same terms; dx, dy are the same exact fp32 values.

    tile kernel, per term: d2 = fma(dx, dx, dy*dy) (2 roundings, <= 2u relative, both summands positive), the
    product of the pair's two d2 (1), rcp.approx (<= 1 ulp = 2u), times the other d2 (1), times g (1): 7u.  Then a
    row sum of at most 2*hh + 1 terms per column (sw += w, swy = fma(w, dy, swy): 2*hh roundings after the first),
    the 2*PPL column sums of the lane (dx * sw folded into an FMA each; dy-part one addition per column), and
    log2(LPS) shuffle additions: c = 7 + 2*hh + 2*PPL + log2(LPS).
    generic kernel, per term: d2 (2u), the IEEE division (u), times g (u): 4u; then each lane sums its share of
    the W x H window (W, H <= 2 r S / 2 + 5 pixels), ceil(W*H / 32) terms, and 5 shuffle additions.
    The 1.05 covers the second-order terms, 2^-45 the float64 oracle's own sum."""
    if path[0] == "tile":
        _, lps, ppl = path
        return 1.05 * (7 + 2 * hh_device(r, S) + 2 * ppl + math.log2(lps))
    W = min(S, int(math.ceil(float(r) * S)) + 6)
    return 1.05 * (4 + math.ceil(W * W / 32) + 5)


def occ_run(dev, d, rs, prime_rs):
    """prime the hint with a call at `prime_rs`, then the measured call at `rs` -> (P,2) numpy"""
    args = [_t(d[k], dev) for k in ("pts", "rad", "vis")]
    g, first, num = _t(d["g"], dev), _t(d["first"], dev), _t(d["num"], dev)
    _C.occ_backward(*args, _t(np.asarray(prime_rs, F), dev), g, first, num)
    torch.cuda.synchronize(dev)
    out = _C.occ_backward(*args, _t(np.asarray(rs, F), dev), g, first, num).cpu().numpy()
    torch.cuda.synchronize(dev)
    return out


def check_against_f64(out, d, rs, paths, S):
    """every point within its bound of the float64 sums; invisible, off-image and behind-camera points exactly 0.
    -> worst |ours - f64| / bound"""
    pts, vis, first, num = d["pts"], d["vis"], d["first"], d["num"]
    _, g64, st = oracle.occ_backward_fast(pts, d["rad"], vis, rs, d["g"], first, num, fma_mode=1, stats=True)
    c = np.zeros(len(pts))
    for n, (f, m) in enumerate(zip(first, num)):
        c[f:f + m] = bound_c(paths[n], rs[n], S)
    bound = c[:, None] * U * st["abs"] + 2.0 ** -45 * st["abs"]
    err = np.abs(out.astype(np.float64) - g64)
    bad = ~(err <= bound)
    assert not bad.any(), "%d points outside their bound; worst err %.3e at bound %.3e" % (
        int(bad.any(1).sum()), float(err[bad].max()), float(bound[bad][np.argmax(err[bad])]))
    dead = (vis == 0) | (pts[:, 2] < 0) | (np.abs(pts[:, 0]) > 1) | (np.abs(pts[:, 1]) > 1)
    assert (out[dead] == 0).all()
    live = st["abs"] > 0
    assert live.any()
    return float((err[live] / (c[:, None] * U * st["abs"])[live]).max())


def random_occ_inputs(S, r_list, seed, P=150):
    """one view per entry of r_list (radius in pixels; 0 -> rs = 0; "big" -> rs = 4 NDC; "none" -> rs = 0 and nothing
    visible): random splats, some invisible, behind the camera or outside the image, random alpha gradient"""
    rng = np.random.default_rng(5000 + seed)
    pix = 2.0 / S
    xs, rads, viss, num, rs = [], [], [], [], []
    for r in r_list:
        n = 8 if r == "big" else P
        x = np.stack([rng.uniform(-1.05, 1.05, n), rng.uniform(-1.05, 1.05, n), rng.uniform(0.5, 3, n)], 1)
        x[rng.random(n) < 0.05, 2] *= -1
        vis = (rng.random(n) < 0.9).astype(np.uint8)
        if r == "none":
            vis[:] = 0
        xs.append(x)
        rads.append(rng.uniform(0.5, 6, (n, 2)) * pix)
        viss.append(vis)
        num.append(n)
        rs.append(F(4.0) if r == "big" else F(0) if r in (0, "none") else F(r * pix))
    num = np.array(num, np.int64)
    g = (rng.standard_normal((len(r_list), S, S)) * 1e-3).astype(F)
    g[rng.random(g.shape) < 0.5] = 0
    return dict(pts=np.concatenate(xs).astype(F), rad=np.concatenate(rads).astype(F),
                vis=np.concatenate(viss), first=(np.cumsum(num) - num).astype(np.int64), num=num, g=g,
                rs=np.array(rs, F), flips=[])


# ---------------------------------------------------------------------------------------------------------------------
# the cases: (id, inputs, S, priming radius in pixels (0: rs = 0, hint 0, R_box 20), claimed path of every view)
# ---------------------------------------------------------------------------------------------------------------------
BRACKET_HH = [3, 4, 7, 8, 11, 12, 15, 16, 19, 20, 23, 24, 31, 32, 39, 40]
BRACKET_CLAIM = "4x1 4x2 4x2 4x3 4x3 4x4 4x4 4x5 4x5 8x3 8x3 8x4 8x4 16x3 16x3 g"

CASES = [
    ("brackets_pow2", ("random", BRACKET_HH, 1), 256, 31, BRACKET_CLAIM),
    ("brackets_other", ("random", BRACKET_HH, 2), 200, 31, BRACKET_CLAIM),
    ("small_box", ("random", [0, "none", 7, 8, "big"], 3), 128, 1, "4x1 4x1 4x2 g g"),
    ("default_box", ("random", [19, 20, 0], 4), 96, 0, "4x5 g 4x1"),
    ("tile_binning", ("random", [3] * 33, 5), 1024, 3, "4x1"),
    ("s8192", ("random", [3], 6), 8192, 3, "4x1"),
    ("disc_edge_r5", ("disc_edge", 128, None), 128, 5, "4x2"),
    ("disc_edge_r10_tile", ("disc_edge", 256, 10), 256, 10, "4x3"),
    ("disc_edge_r10_generic", ("disc_edge", 256, 10), 256, 1, "g"),
    ("disc_edge_r13", ("disc_edge", 512, 13), 512, 13, "4x4"),
    ("disc_near_pow2", ("disc_near", 128, None), 128, 4.6, "4x2"),
    ("disc_near_other", ("disc_near", 200, None), 200, 4.6, "4x2"),
    ("disc_near_generic", ("disc_near", 256, 9.6), 256, 1, "g"),
    ("box_edge", ("box_edge", 128, None), 128, 6, "4x2"),
    ("box_edge_generic", ("box_edge", 256, 10), 256, 1, "g"),
    ("centre", ("centre", 64, None), 64, 3.4, "4x1"),
    ("border_17", ("border", 17, None), 17, 3.7, "4x2"),
    ("border_100", ("border", 100, None), 100, 3.7, "4x2"),
    ("border_200", ("border", 200, None), 200, 3.7, "4x2"),
    ("dense", ("dense", 64, None), 64, 3.3, "4x1"),
    ("many_tiles", ("many_tiles", 1024, None), 1024, 3.2, "4x1"),
    ("ragged", ("ragged", 64, None), 64, 4.2, "4x2"),
]


def case_inputs(spec, S):
    if spec[0] == "random":
        return random_occ_inputs(S, spec[1], spec[2])
    return occ_edge_splats(spec[0], spec[1], seed=7, r_px=spec[2])


def case_plan(case):
    """-> (inputs, measured rs, priming rs, R_box, path of every view), with the claims checked against the model"""
    cid, spec, S, prime_px, claim = case
    d = case_inputs(spec, S)
    rs = d["rs"]
    N = len(rs)
    prime = np.full(N, F(prime_px * 2.0 / S), F)
    R = r_box(prime, S)
    paths = [view_path(r, S, R) for r in rs]
    claims = claim.split()
    claims = claims * N if len(claims) == 1 else claims
    assert [path_name(p) for p in paths] == claims, (cid, R, [path_name(p) for p in paths])
    return d, rs, prime, R, paths


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_occ_gather_per_point_bound(cuda_device, case):
    S = case[2]
    d, rs, prime, R, paths = case_plan(case)
    out = occ_run(cuda_device, d, rs, prime)
    worst = check_against_f64(out, d, rs, paths, S)
    print("%s: R_box %d, paths %s, worst |ours - f64| / bound %.4f" % (case[0], R, " ".join(path_name(p) for p in paths),
                                                                      worst))


def test_occ_dispatch_coverage():
    """the cases above reach every path: all 8 lane mappings with and without a power-of-two S, both sides of every
    `need` bracket edge and the largest need at R_box = 40, hh = 0 (rs = 0, and nothing visible), the last window that
    fits and the first that does not, rs >= 4, one launch that mixes mappings and the generic kernel, one that bins
    more than 2^25 cells (the large scan and the scratch it needs), and one view of 256 x 256 tiles (S = 8192)"""
    maps, needs, seen = set(), set(), set()
    for case in CASES:
        cid, spec, S, _, _ = case
        d, rs, prime, R, paths = case_plan(case)
        pow2 = S & (S - 1) == 0
        kinds = set()
        for n, (r, p) in enumerate(zip(rs, paths)):
            hh = hh_device(r, S)
            kinds.add(p[0])
            if p[0] == "tile":
                maps.add((p[1], p[2], pow2))
                needs.add(2 * hh + 2)
                if hh + 1 == R:
                    seen.add("last_fit")
                if hh == 0 and r == 0:
                    seen.add("rs0")
                if hh == 0 and d["vis"][d["first"][n]:d["first"][n] + d["num"][n]].sum() == 0:
                    seen.add("none_visible")
                if R == RBOX_MAX and 2 * hh + 2 == 2 * (RBOX_MAX - 1) + 2:
                    seen.add("largest_need")
            else:
                if hh + 1 == R + 1 and r < 4:
                    seen.add("first_no_fit")
                if r >= 4:
                    seen.add("rs_ge_4")
        if len(kinds) == 2 and len({p for p in paths if p[0] == "tile"}) > 1:
            seen.add("mixed")
        if len(rs) * ((S + 31) // 32) ** 2 * 1024 > (32 << 20):
            seen.add("over_2p25_cells")
        if "tile" in kinds and S >= 8192:
            seen.add("s8192_tiles")
        # work items of <= 128 splats per tile, handed out in groups of 4 to at most 2 persistent CTAs per SM
        live = d["vis"] > 0
        view = np.repeat(np.arange(len(rs)), d["num"])[live]
        cell = np.clip(np.floor((d["pts"][live, :2] + F(1)) * F(0.5 * S)), 0, S - 1).astype(np.int64) // 32
        _, per_tile = np.unique((view * 4096 + cell[:, 1]) * 4096 + cell[:, 0], return_counts=True)
        items = int(((per_tile + 127) // 128).sum())
        if per_tile.max() > 128:
            seen.add("items_per_tile")
        if (items + 3) // 4 > 2 * 132:
            seen.add("groups_over_ctas")
    assert maps == {(lps, ppl, p2) for _, lps, ppl in MAPPINGS for p2 in (True, False)}, maps
    for lo, hi in ((8, 10), (16, 18), (24, 26), (32, 34), (40, 42), (48, 50), (64, 66)):
        assert lo in needs and hi in needs, (lo, hi)
    want = {"last_fit", "first_no_fit", "rs0", "none_visible", "largest_need", "rs_ge_4", "mixed", "over_2p25_cells",
            "s8192_tiles", "items_per_tile", "groups_over_ctas"}
    assert want <= seen, want - seen
    print("mappings (lanes, pairs, pow2): %s; needs: %s; %s" % (sorted(maps), sorted(needs), sorted(seen)))


# ---------------------------------------------------------------------------------------------------------------------
# search radius: the lower median, bit for bit, through both record sources of the radix select
# ---------------------------------------------------------------------------------------------------------------------
def radius_views(seed=0):
    """per view: (radii (n,2), visible (n,)) -- 1..4 visible splats, all radii equal, radii equal in their top 24 /
    16 / 8 key bits (each radix pass decides), radii over many binades, nothing visible"""
    rng = np.random.default_rng(700 + seed)

    def bits(top, n):
        base = np.float32(0.0173).view(np.uint32)
        low = rng.integers(0, 1 << (32 - top), (n, 2), dtype=np.uint64).astype(np.uint32)
        return ((base & np.uint32((0xFFFFFFFF << (32 - top)) & 0xFFFFFFFF)) | low).view(F)

    views = []
    for k in (1, 2, 3, 4):
        vis = np.zeros(9, np.uint8)
        vis[rng.choice(9, k, replace=False)] = 1
        views.append((rng.uniform(0.001, 0.1, (9, 2)).astype(F), vis))
    views.append((np.full((300, 2), F(0.0123)), np.ones(300, np.uint8)))
    for top in (24, 16, 8):
        views.append((bits(top, 501), (rng.random(501) < 0.8).astype(np.uint8)))
    views.append(((10.0 ** rng.uniform(-6, 1, (800, 2))).astype(F), (rng.random(800) < 0.7).astype(np.uint8)))
    views.append((rng.uniform(0.001, 0.1, (50, 2)).astype(F), np.zeros(50, np.uint8)))
    rad = np.concatenate([v[0] for v in views]).astype(F)
    vis = np.concatenate([v[1] for v in views])
    num = np.array([len(v[1]) for v in views], np.int64)
    return rad, vis, (np.cumsum(num) - num).astype(np.int64), num


@pytest.mark.parametrize("radii_s", [5.0, 1.0])
def test_search_radius_packed_records_bit_exact(cuda_device, radii_s):
    rad, vis, first, num = radius_views()
    got = _C.search_radius(_t(rad, cuda_device), _t(vis, cuda_device), _t(first, cuda_device), _t(num, cuda_device),
                           radii_s).cpu().numpy()
    want = oracle.search_radius(rad, vis, first, num, radii_s)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (got, want)
    assert want[-1] == 0 and (want[:-1] > 0).all()


def test_search_radius_compact_records_bit_exact(cuda_device):
    """the fused backward's median runs over the compact records of its binning; dss_render_backward returns it
    (dss_render_args.search_radius).  Fed these radii, visibility and screen positions instead of a forward's records
    (records = NULL: the backward packs them from ndc and radii), it must return the oracle's median"""
    dev = cuda_device
    rad, vis, first, num = radius_views(seed=1)
    N, P, S, K = len(num), len(rad), 64, 5
    rng = np.random.default_rng(9)
    ndc = np.stack([rng.uniform(-0.95, 0.95, P), rng.uniform(-0.95, 0.95, P), rng.uniform(0.5, 3, P)], 1).astype(F)
    pts = torch.from_numpy(rng.uniform(-0.5, 0.5, (P, 3)).astype(F)).to(dev)
    _, _, _, proj, view, _ = scene(16, N, seed=3)
    proj, view = proj.to(dev).contiguous(), view.to(dev).contiguous()
    prm = SplatParams(image_size=S, points_per_pixel=K, znear=0.1)
    first_t, num_t = _t(first, dev), _t(num, dev)
    ndc_t, rad_t, vis_t = _t(ndc, dev), _t(rad, dev), _t(vis, dev)
    h = torch.ones(N, device=dev)
    a = _lib.RenderArgs()
    ops._fill_common(a, pts, None, None, proj, view, h, first_t, num_t, False, N, P, P, prm)
    a.records = None
    a.ndc, a.radii, a.visible = _lib.ptr(ndc_t), _lib.ptr(rad_t), _lib.ptr(vis_t)
    idx = torch.full((N, S, S, K), -1, dtype=torch.int32, device=dev)
    weights = torch.zeros((N, S, S, K), device=dev)
    grad_image = torch.zeros((N, S, S, 4), device=dev)
    grad_image[..., 3] = torch.randn(N, S, S, device=dev) * 1e-3
    a.idx, a.weights, a.grad_image = _lib.ptr(idx), _lib.ptr(weights), _lib.ptr(grad_image)
    grad_points = torch.zeros_like(pts)
    grad_ndc = torch.zeros((P, 3), device=dev)
    rs = torch.full((N,), float("nan"), device=dev)
    a.grad_points_world, a.grad_ndc, a.search_radius = _lib.ptr(grad_points), _lib.ptr(grad_ndc), _lib.ptr(rs)
    lib, ctx, st = _lib.load(), _lib.ctx(dev), _lib.stream_ptr(dev)
    _lib.check(lib.dss_render_backward(ctx, C.byref(a), st), "dss_render_backward")
    torch.cuda.synchronize(dev)
    got = rs.cpu().numpy()
    want = oracle.search_radius(rad, vis, first, num, prm.radii_backward_scaler)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (got, want)


# ---------------------------------------------------------------------------------------------------------------------
# non-finite alpha gradients
# ---------------------------------------------------------------------------------------------------------------------
BAD_PIXELS = [(30, 40), (90, 64), (64, 100)]       # NDC-index (xi, yi)


def nonfinite_inputs(S=128, r_px=9):
    rng = np.random.default_rng(77)
    pix = 2.0 / S
    d = random_occ_inputs(S, [r_px], seed=77, P=600)
    # splats around every bad pixel, their boxes holding it
    extra = []
    for xi, yi in BAD_PIXELS:
        c = np.array([-1 + (2 * xi + 1) / S, -1 + (2 * yi + 1) / S])
        extra.append(c + rng.uniform(-2, 2, (6, 2)) * pix)
    extra = np.concatenate(extra)
    m = len(extra)
    d["pts"] = np.concatenate([d["pts"], np.concatenate([extra, np.ones((m, 1))], 1)]).astype(F)
    d["rad"] = np.concatenate([d["rad"], np.full((m, 2), 4 * pix)]).astype(F)
    d["vis"] = np.concatenate([d["vis"], np.ones(m, np.uint8)])
    d["num"] = d["num"] + m
    return d


@pytest.mark.parametrize("kernel", ["tile", "generic"])
@pytest.mark.parametrize("value", [float("nan"), float("inf"), float("-inf")], ids=["nan", "+inf", "-inf"])
def test_occ_nonfinite_alpha_gradient(cuda_device, kernel, value):
    """a non-finite alpha gradient reaches every point whose reference term set holds the pixel (the disc; for +inf
    the part inside the point's box) on both kernels; points whose window cannot reach it are bit-identical to a run
    without it"""
    S, r_px = 128, 9
    d = nonfinite_inputs(S, r_px)
    rs = d["rs"]
    prime = np.full(1, F((r_px if kernel == "tile" else 1) * 2.0 / S), F)
    assert view_path(rs[0], S, r_box(prime, S))[0] == kernel
    bad = np.zeros_like(d["g"])
    for xi, yi in BAD_PIXELS:
        bad[0, S - 1 - yi, S - 1 - xi] = value
    # the reference's term sets: the oracle on the non-finite pixels alone
    _, ref = oracle.occ_backward_fast(d["pts"], d["rad"], d["vis"], rs, bad, d["first"], d["num"], fma_mode=1)
    hit = ~np.isfinite(ref).all(1)
    clean = dict(d)
    g = d["g"].copy()
    for xi, yi in BAD_PIXELS:
        g[0, S - 1 - yi, S - 1 - xi] = 0
    clean["g"] = g
    dirty = dict(clean)
    dirty["g"] = np.where(np.isnan(bad) | np.isinf(bad), bad, g).astype(F)
    out = occ_run(cuda_device, dirty, rs, prime)
    want = occ_run(cuda_device, clean, rs, prime)
    assert hit.sum() >= 6
    assert (~np.isfinite(out[hit])).all(), "%d of %d points lost the non-finite term" % (
        int(np.isfinite(out[hit]).any(1).sum()), int(hit.sum()))
    hh = hh_device(rs[0], S)
    cy = np.clip(np.floor((d["pts"][:, 1] + F(1)) * F(0.5 * S)), 0, S - 1)
    far = np.ones(len(cy), bool)
    for _, yi in BAD_PIXELS:
        far &= np.abs(cy - yi) > hh + 4
    assert far.sum() > 100
    assert np.array_equal(out[far].view(np.uint32), want[far].view(np.uint32))
    print("non-finite points: %d (reference term sets: %d)" % (int((~np.isfinite(out)).any(1).sum()), int(hit.sum())))
