"""The shading-gradient kernels against float64 at their edges, output by output, within the bound of
tests/shading_grad_oracle.py (c·u·Σ|terms| counted along the kernels' expression tree, plus half an ulp):
dss_light_backward (light_partials_kernel + grad_finish_kernel: every light row and the ambient), dss_camera_backward
with shading (camera_partials_kernel<true>: the camera centres, next to synthetic grad_ndc for the proj / view sums)
and dss_colour_backward (shade_backward_kernel for shared clouds, shade_backward_packed_kernel for packed ones: albedo,
normal, position per point or row).

d L / d shaded reaches the kernels through an idx that gives every (view, point) slot exactly one pixel, so it is known
exactly and no atomics reorder it.  The edge slots (n·d = 0 and ±2^-40, v·r = 0 and 2^-30, zero normals, |n| =
float32(1e-6) and one ulp either side, a point at and 1e-6f from the camera and the point light, light and camera 1e4
from the origin next to the point, zero light colours) each sit alone in a view of their own with per-view lights, so
every camera and light output holds one slot only; a NaN in d L / d shaded poisons exactly the outputs float64 poisons,
and slots whose d L / d shaded is 0 contribute nothing, NaN rows included.  Layouts: shared clouds with shared and
per-view lights (1, 2, 8), packed clouds that are ragged, have an empty view, overlapping ranges and rows no range
covers, N = 1 / P0 = 1, N·L slices above twice the SM count, a partial CAM_BATCH tail, only the ambient or only the
lights requiring grad.  Shininess 1, 13.5 and 64 (below 1 the reference's pow backward is NaN at alpha = 0).  Every
case runs twice and must give the same bits."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from dss_b200 import _lib, ops
from dss_b200.ops import Shading, SplatParams
from tests.shading_grad_oracle import Bounded, U, edge_slots, ordinary_slots, slot_outputs, within

pytestmark = pytest.mark.gpu

SHINS = (1.0, 13.5, 64.0)
_WORST = {}


def _library(dev, sh, pts, nrm, alb, first, num, gc, gndc, lights=True, ambient=True, cam=True):
    """dss_colour_backward over an idx that gives every slot of view n's range (shared: the P0 points) one pixel of
    view n, then dss_camera_backward and dss_light_backward.  gc: (P,3) d L / d shaded per packed row (shared: per
    slot n*P0 + i).  -> dict of the outputs (None where not asked for)"""
    N = sh.cam_centres.shape[0]
    shared = first is None
    P0 = pts.shape[0]
    P = P0 * N if shared else P0
    fr = [n * P0 for n in range(N)] if shared else first.tolist()
    nr = [P0] * N if shared else num.tolist()
    S = max(1, math.ceil(math.sqrt(max(nr + [1]))))
    idx = torch.full((N, S * S), -1, dtype=torch.int32)
    gi = torch.zeros(N, S * S, 4)
    gcc = torch.as_tensor(gc, dtype=torch.float32)
    for n, (f, k) in enumerate(zip(fr, nr)):
        idx[n, :k] = torch.arange(f, f + k, dtype=torch.int32)
        gi[n, :k, :3] = gcc[f:f + k]
    idx, gi = idx.view(N, S, S, 1).to(dev), gi.view(N, S, S, 4).to(dev)
    weights = torch.ones((N, S, S, 1), device=dev)
    proj = torch.eye(4, device=dev).repeat(N, 1, 1)
    proj[:, 3, 3] = 2.0
    a = _lib.RenderArgs()
    ops._fill_common(a, pts, nrm, None, proj, proj, None, None if shared else first, None if shared else num, shared,
                     N, P0, P, SplatParams(image_size=S, points_per_pixel=1))
    ops._fill_shading(a, sh, alb)
    grad_colours = torch.empty((P, 3), device=dev)
    out = {k: torch.zeros_like(pts) for k in ("alb", "nrm", "pos")}
    out.update(proj=torch.empty(N, 4, 4, device=dev), view=torch.empty(N, 4, 4, device=dev),
               cam=torch.full((N, 3), float("nan"), device=dev) if cam else None,
               lights=torch.full_like(sh.lights, float("nan")) if lights else None,
               ambient=torch.full_like(sh.ambient, float("nan")) if ambient else None)
    a.idx, a.weights, a.grad_image, a.grad_colours = (_lib.ptr(t) for t in (idx, weights, gi, grad_colours))
    a.grad_ndc = _lib.ptr(gndc)
    a.grad_albedo, a.grad_normals_world, a.grad_points_shading = (_lib.ptr(out[k]) for k in ("alb", "nrm", "pos"))
    lib, ctx, st = _lib.load(), _lib.ctx(dev), _lib.stream_ptr(dev)
    _lib.check(lib.dss_colour_backward(ctx, C.byref(a), st), "dss_colour_backward")
    _lib.check(lib.dss_camera_backward(ctx, C.byref(a), _lib.ptr(out["proj"]), _lib.ptr(out["view"]),
                                       _lib.ptr(out["cam"]), st), "dss_camera_backward")
    if lights or ambient:
        _lib.check(lib.dss_light_backward(ctx, C.byref(a), _lib.ptr(out["lights"]), _lib.ptr(out["ambient"]), st),
                   "dss_light_backward")
    # the proj / view sums of the camera kernel without shading: the same launches' other outputs
    pv = (torch.empty(N, 4, 4, device=dev), torch.empty(N, 4, 4, device=dev))
    _lib.check(lib.dss_camera_backward(ctx, C.byref(a), _lib.ptr(pv[0]), _lib.ptr(pv[1]), None, st),
               "dss_camera_backward")
    torch.cuda.synchronize(dev)
    out["proj_plain"], out["view_plain"] = pv
    return {k: (None if v is None else v.cpu()) for k, v in out.items()}


def _run_twice(*args, rows_once=None, **kw):
    """two runs, the same bits; rows_once: the packed rows one view covers (a row of two views' ranges is written by
    each of them, in either order)"""
    r1, r2 = _library(*args, **kw), _library(*args, **kw)
    for k, v in r1.items():
        if v is not None:
            if rows_once is not None and k in ("alb", "nrm", "pos"):
                v, r2[k] = v[rows_once], r2[k][rows_once]
            assert torch.equal(v.nan_to_num(7.0), r2[k].nan_to_num(7.0)) and \
                torch.equal(v.isnan(), r2[k].isnan()), ("run to run", k)
    # the shading launch leaves the projection / view sums as the plain camera kernel gives them
    for k in ("proj", "view"):
        assert torch.equal(r1[k].nan_to_num(7.0), r1[k + "_plain"].nan_to_num(7.0)), k
    return r1


def _want(views, rows_of_view, s_world, cams, lights, amb, gc_row, lt, shin, P_rows, shared):
    """float64 outputs and bounds of the layout.  views: view per slot; rows_of_view: the slot's row (packed row, or
    world point of a shared cloud); s_world: dict p / n / alb per row; lights (N,L,9) and amb (N,3) per view;
    gc_row: d L / d shaded per slot"""
    s = dict(p=s_world["p"][rows_of_view], n=s_world["n"][rows_of_view], alb=s_world["alb"][rows_of_view],
             cam=cams[views], lights=lights[views], amb=amb[views], gc=gc_row, light_type=lt, shin=shin)
    o = slot_outputs(Bounded, s)
    N, L = lights.shape[0], lights.shape[1]
    res = {}

    def scatter(idx, n_out, v, e, f32_terms):
        val = np.zeros((n_out,) + v.shape[1:])
        bnd = np.zeros_like(val)
        mag = np.zeros_like(val)
        np.add.at(val, idx, v)
        np.add.at(bnd, idx, e)
        np.add.at(mag, idx, np.abs(v) + e)
        cnt = np.bincount(idx, minlength=n_out).reshape((-1,) + (1,) * (v.ndim - 1))
        # float32 sums over f32_terms terms (shared cloud: the views) or float64 ones (partials)
        acc = (np.maximum(cnt - 1, 0) * U) if f32_terms else 2.0 ** -50 * cnt
        return val, bnd + acc * mag

    res["cam"] = scatter(views, N, *o["cam"], False)
    res["lights_vec"] = scatter(views, N, *o["vec"], False)
    res["lights_cd"] = scatter(views, N, *o["cd"], False)
    res["lights_cs"] = scatter(views, N, *o["cs"], False)
    res["ambient"] = scatter(views, N, *o["amb"], False)
    for k in ("alb", "nrm", "pos"):
        res[k] = scatter(rows_of_view, P_rows, *o[k], shared)
    return res


def _compare(label, got, want, rows_mask=None, per_view_lights=True, check_lights=True, check_amb=True):
    """every output within its bound, NaN where float64 is NaN; -> worst ratio per output"""
    worst = {}

    def one(name, g, w):
        val, bnd = w
        r, same = within(g.numpy().astype(np.float64), val, bnd)
        assert same.all(), (label, name, "NaN pattern", np.argwhere(~same)[:5])
        worst[name] = float(r.max()) if r.size else 0.0
        assert worst[name] <= 1, (label, name, worst[name], np.unravel_index(np.argmax(r), r.shape))

    one("cam", got["cam"], want["cam"])
    fold = (lambda v, b: (v, b)) if per_view_lights else (lambda v, b: (v.sum(0, keepdims=True), b.sum(0, keepdims=True)))
    if check_lights:
        gl = got["lights"].reshape(-1, got["lights"].shape[-2], 9)
        for j, k in enumerate(("vec", "cd", "cs")):
            one("lights_" + k, gl[..., 3 * j:3 * j + 3], fold(*want["lights_" + k]))
    if check_amb:
        one("ambient", got["ambient"].reshape(-1, 3), fold(*want["ambient"]))
    m = slice(None) if rows_mask is None else rows_mask
    for k in ("alb", "nrm", "pos"):
        one(k, got[k][m], (want[k][0][m], want[k][1][m]))
    fam = label.split(" ")[0]
    for k, v in worst.items():
        _WORST.setdefault(fam, {})
        _WORST[fam][k] = max(_WORST[fam].get(k, 0.0), v)
    print("%s: worst ratio %s" % (label, {k: "%.3g" % v for k, v in worst.items()}))
    return worst


def _t(x, dev):
    return torch.as_tensor(np.ascontiguousarray(x), dtype=torch.float32).to(dev)


# ---- 1. the edge slots, one per view ---------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["sun", "point"])
@pytest.mark.parametrize("L", [1, 2, 8])
@pytest.mark.parametrize("shin", SHINS)
def test_edge_slots_one_per_view_within_the_bound(cuda_device, kind, L, shin):
    d = cuda_device
    s, labels = edge_slots(kind, L, shin, seed=L)
    o = ordinary_slots(3, kind, L, shin, seed=100 + L)
    # a NaN in d L / d shaded (one channel), and zero d L / d shaded on rows of NaN geometry
    o["gc"][0] = [np.nan, 0.5, -0.25]                     # lit, camera in the mirror direction: specular live
    o["p"][0], o["n"][0], o["cam"][0] = [0.5, 0.25, -0.125], [0.0, 0.0, 1.0], [0.25, 0.25, 0.875]
    o["lights"][0, 0, :3] = [0.75, 0.25, 0.875] if s["light_type"] else [0.25, 0.0, 1.0]
    o["gc"][1] = 0.0
    o["p"][1], o["n"][1], o["alb"][1] = np.nan, np.nan, np.nan
    o["gc"][2] = 0.0                                      # a view whose d L / d shaded is all zero
    labels = labels + ["NaN in dL/dshaded", "zero dL/dshaded, NaN row", "zero dL/dshaded"]
    cat = {k: np.concatenate([s[k], o[k]]) for k in ("p", "n", "alb", "cam", "lights", "amb", "gc")}
    M = len(labels)
    first = torch.arange(M, dtype=torch.int64)
    num = torch.ones(M, dtype=torch.int64)
    sh = Shading(_t(cat["lights"], d), _t(cat["amb"], d), _t(cat["cam"], d), s["light_type"], shin)
    gndc = torch.randn(M, 3, generator=torch.Generator().manual_seed(L)).to(d)
    got = _run_twice(d, sh, _t(cat["p"], d), _t(cat["n"], d), _t(cat["alb"], d), first.to(d), num.to(d), cat["gc"],
                     gndc)
    views = np.arange(M)
    want = _want(views, views, cat, cat["cam"], cat["lights"], cat["amb"], cat["gc"], s["light_type"], shin, M, False)
    _compare("edges %s L=%d shin=%g" % (kind, L, shin), got, want)
    # the NaN slot poisons its view's camera row and light rows; the zero slots leave exact zeros
    nan_v, zero_v = M - 3, [M - 2, M - 1]
    assert torch.isnan(got["cam"][nan_v]).any() and torch.isnan(got["lights"][nan_v]).any()
    for v in zero_v:
        for k in ("cam", "lights", "ambient", "alb", "nrm", "pos"):
            assert (got[k][v] == 0).all(), (labels[v], k)
    # the eps branches give the float64 values (g / eps below eps, the projection at and above it), and n.d = 0 exactly
    # gives no diffuse or specular light gradient through the normal's direction
    i = labels.index("|n|=eps")
    assert abs(float(got["nrm"][i, 2])) < 1e-3 * float(got["nrm"][i].abs().max())


# ---- 2. shared clouds -----------------------------------------------------------------------------------------------
def _shared_case(kind, L, shin, N, P0, per_view, seed):
    """a sphere cloud with camera-independent edge points in front (zero normal, |n| = eps and one ulp either side,
    zero d L / d shaded with NaN geometry), N cameras, lights shared or per view"""
    o = ordinary_slots(P0, kind, L, shin, seed=seed)
    rng = np.random.default_rng(seed)
    world = dict(p=o["p"], n=o["n"], alb=o["alb"])
    eps = float(np.float32(1e-6))
    if P0 >= 6:
        world["n"][0] = 0.0
        world["n"][1] = [0.0, 0.0, eps]
        world["n"][2] = [0.0, 0.0, float(np.nextafter(np.float32(eps), np.float32(0)))]
        world["n"][3] = [0.0, 0.0, float(np.nextafter(np.float32(eps), np.float32(1)))]
        world["p"][4] = np.nan
    nl = N if per_view else 1
    lights = o["lights"][:nl] if nl <= P0 else np.concatenate([o["lights"]] * (nl // P0 + 1))[:nl]
    if kind == "point" and P0 >= 6:
        world["p"][5] = lights[0, 0, :3]                   # a point at the point light (view 0's)
    amb = np.asarray(0.2 * rng.random((nl, 3)), np.float32).astype(np.float64)
    cam = rng.normal(size=(N, 3))
    cams = np.asarray(2.0 * cam / np.linalg.norm(cam, axis=1, keepdims=True), np.float32).astype(np.float64)
    gc = np.asarray(rng.normal(size=(N * P0, 3)), np.float32).astype(np.float64)
    if P0 >= 6:
        gc[4::P0] = 0.0                                    # NaN geometry, zero d L / d shaded in every view
    if N > 1:
        gc[(N - 1) * P0:] = 0.0                            # the last view's d L / d shaded is all zero
    return world, lights, amb, cams, gc


def _check_shared(d, label, kind, L, shin, N, P0, per_view, seed, lights_grad=True, amb_grad=True):
    world, lights, amb, cams, gc = _shared_case(kind, L, shin, N, P0, per_view, seed)
    lt = 1 if kind == "point" else 0
    sh = Shading(_t(lights if per_view else lights[0], d), _t(amb if per_view else amb[0], d), _t(cams, d), lt, shin)
    gndc = torch.randn(N * P0, 3, generator=torch.Generator().manual_seed(seed)).to(d)
    got = _run_twice(d, sh, _t(world["p"], d), _t(world["n"], d), _t(world["alb"], d), None, None, gc, gndc,
                     lights=lights_grad, ambient=amb_grad)
    views = np.repeat(np.arange(N), P0)
    pts = np.tile(np.arange(P0), N)
    lv = lights if per_view else np.broadcast_to(lights[0], (N,) + lights.shape[1:])
    av = amb if per_view else np.broadcast_to(amb[0], (N, 3))
    want = _want(views, pts, world, cams, lv, av, gc, lt, shin, P0, True)
    _compare(label, got, want, per_view_lights=per_view, check_lights=lights_grad, check_amb=amb_grad)
    if N > 1:
        assert (got["cam"][N - 1] == 0).all()
        for k, on in (("lights", lights_grad), ("ambient", amb_grad)):
            if per_view and on:
                assert (got[k][N - 1] == 0).all(), k
    return got


@pytest.mark.parametrize("kind", ["sun", "point"])
@pytest.mark.parametrize("per_view", [False, True])
@pytest.mark.parametrize("L,shin", [(1, 1.0), (2, 13.5), (8, 64.0)])
def test_shared_cloud_within_the_bound(cuda_device, kind, per_view, L, shin):
    _check_shared(cuda_device, "shared %s per_view=%s L=%d shin=%g" % (kind, per_view, L, shin), kind, L, shin, 3,
                  3000, per_view, seed=L)


@pytest.mark.parametrize("kind", ["sun", "point"])
def test_launch_shapes(cuda_device, kind):
    d = cuda_device
    # N = 1 and P0 = 1
    _check_shared(d, "shapes N=1,P0=1 %s" % kind, kind, 2, 13.5, 1, 1, True, seed=1)
    _check_shared(d, "shapes N=1,P0=1 %s" % kind, kind, 2, 13.5, 1, 1, False, seed=2)
    _check_shared(d, "shapes N=4,P0=1 %s" % kind, kind, 1, 64.0, 4, 1, True, seed=3)
    # 40 views x 8 lights = 320 slices, above twice the SM count: one block per slice, every thread loops
    _check_shared(d, "shapes N=40,L=8 %s" % kind, kind, 8, 13.5, 40, 700, True, seed=4)
    # 33 views x 4 lights = 132 slices: two blocks per slice, and 3001 points leave a partial CAM_BATCH tail
    _check_shared(d, "shapes N=33,L=4,P0=3001 %s" % kind, kind, 4, 64.0, 33, 3001, True, seed=5)


@pytest.mark.parametrize("kind", ["sun", "point"])
def test_only_the_ambient_or_only_the_lights(cuda_device, kind):
    """the ambient sums live in the l = 0 slice: with only the ambient requiring grad that slice alone runs (nl = 1),
    and gives the bits of the full launch; with only the lights, the same light rows"""
    d = cuda_device
    full = _check_shared(d, "grad-subsets %s" % kind, kind, 8, 13.5, 3, 2000, True, seed=7)
    amb = _check_shared(d, "grad-subsets %s ambient only" % kind, kind, 8, 13.5, 3, 2000, True, seed=7,
                        lights_grad=False)
    lig = _check_shared(d, "grad-subsets %s lights only" % kind, kind, 8, 13.5, 3, 2000, True, seed=7, amb_grad=False)
    assert torch.equal(amb["ambient"], full["ambient"]) and torch.equal(lig["lights"], full["lights"])


# ---- 3. packed clouds -----------------------------------------------------------------------------------------------
def _packed_layout(P0):
    """five views over packed rows: ragged, an empty view, two views whose ranges overlap, and rows no range
    covers -> (first, num, rows covered exactly once)"""
    first = np.array([0, P0 // 3, P0 // 2, P0 // 2, 2 * P0 // 3 + 7], np.int64)
    num = np.array([P0 // 3 - 5, P0 // 4, 0, P0 // 6 + 11, P0 - (2 * P0 // 3 + 7) - 20], np.int64)
    cover = np.zeros(P0, int)
    for f, k in zip(first, num):
        cover[f:f + k] += 1
    assert (cover == 0).any() and (cover > 1).any()
    return first, num, cover == 1


@pytest.mark.parametrize("kind", ["sun", "point"])
@pytest.mark.parametrize("per_view", [False, True])
@pytest.mark.parametrize("L,shin", [(1, 64.0), (2, 1.0), (8, 13.5)])
def test_packed_cloud_within_the_bound(cuda_device, kind, per_view, L, shin):
    d = cuda_device
    P0 = 4000
    first, num, once = _packed_layout(P0)
    N = len(first)
    o = ordinary_slots(P0, kind, L, shin, seed=20 + L)
    rng = np.random.default_rng(L)
    world = dict(p=o["p"], n=o["n"], alb=o["alb"])
    world["n"][first[0]] = 0.0
    world["n"][first[1]] = [0.0, float(np.float32(1e-6)), 0.0]
    nl = N if per_view else 1
    lights, amb = o["lights"][:nl], o["amb"][:nl]
    cam = rng.normal(size=(N, 3))
    cams = np.asarray(2.0 * cam / np.linalg.norm(cam, axis=1, keepdims=True), np.float32).astype(np.float64)
    lt = 1 if kind == "point" else 0
    gc_rows = o["gc"].copy()
    gc_rows[first[3]:first[3] + 10] = 0.0
    sh = Shading(_t(lights if per_view else lights[0], d), _t(amb if per_view else amb[0], d), _t(cams, d), lt, shin)
    gndc = torch.randn(P0, 3, generator=torch.Generator().manual_seed(L)).to(d)
    got = _run_twice(d, sh, _t(world["p"], d), _t(world["n"], d), _t(world["alb"], d), torch.as_tensor(first).to(d),
                     torch.as_tensor(num).to(d), gc_rows, gndc, rows_once=torch.as_tensor(once))
    views = np.concatenate([np.full(k, n) for n, k in enumerate(num)])
    rows = np.concatenate([np.arange(f, f + k) for f, k in zip(first, num)])
    # d L / d shaded of a row two views cover is the float32 sum of both views' pixels
    gsum = np.zeros((P0, 3), np.float32)
    for r_ in rows:
        gsum[r_] += np.float32(gc_rows[r_])
    lv = lights if per_view else np.broadcast_to(lights[0], (N,) + lights.shape[1:])
    av = amb if per_view else np.broadcast_to(amb[0], (N, 3))
    want = _want(views, rows, world, cams, lv, av, gsum[rows].astype(np.float64), lt, shin, P0, False)
    # rows two views cover are written by each of them (the caller's layouts do not overlap): checked through the
    # camera and light sums only; rows no view covers stay as the caller left them
    _compare("packed %s per_view=%s L=%d shin=%g" % (kind, per_view, L, shin), got, want, rows_mask=once,
             per_view_lights=per_view)
    cover0 = np.ones(P0, bool)
    cover0[rows] = False
    for k in ("alb", "nrm", "pos"):
        assert (got[k][cover0] == 0).all(), k
    assert (got["cam"][2] == 0).all()
    if per_view:
        assert (got["lights"][2] == 0).all() and (got["ambient"][2] == 0).all()


def test_zz_print_worst_ratios_per_family():
    """the worst ratio to the bound of every family this session ran"""
    for fam, r in sorted(_WORST.items()):
        print("worst ratio %-8s %s" % (fam, {k: "%.3g" % v for k, v in sorted(r.items())}))
        assert max(r.values()) <= 1
