"""Seeded synthetic scenes shared by tests, smoke() and bench.py (SURVEY.md section 8d), the helpers that store
and read what the reference's own kernels computed on them (tests/golden/), and the float64 reference of the fused
backward (render_backward_f64)."""
import ctypes as C
import os

import numpy as np
import torch

from dss_b200 import _lib, ops
from dss_b200.core.camera import FoVPerspectiveCameras, look_at_view_transform, camera_matrices

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
# outputs of the reference's CUDA kernels (oracle/_ref/dss_ref_cuda on an H100), minted by tests/golden/make_golden_ref_cuda.py
REF_CUDA_GOLDEN = os.path.join(GOLDEN_DIR, "ref_cuda_witness.npz")


def golden_case(path, case):
    """The arrays stored for `case` in a golden file (keys "<case>__<name>")."""
    d = np.load(path)
    out = {k[len(case) + 2:]: d[k] for k in d.files if k.startswith(case + "__")}
    assert out, "no golden data for %s in %s" % (case, path)
    return out


def sample_rows(n, k, seed):
    """A fixed, sorted sample of min(k, n) of the indices 0..n-1."""
    return np.sort(np.random.default_rng(seed).choice(n, min(k, n), replace=False))


def row_hash(a):
    """(M, ...) -> (M,) uint64: an exact hash of the bit patterns of each row (32-bit elements)."""
    b = np.ascontiguousarray(a).reshape(a.shape[0], -1).view(np.uint32).astype(np.uint64)
    h = np.full(b.shape[0], 14695981039346656037, np.uint64)
    for k in range(b.shape[1]):
        h = (h ^ b[:, k]) * np.uint64(1099511628211)
    return h


def digest(a):
    """One exact, position-sensitive uint64 digest of the bit patterns of a whole 32-bit array."""
    b = np.ascontiguousarray(a).reshape(-1).view(np.uint32).astype(np.uint64)
    w = np.arange(b.size, dtype=np.uint64) * np.uint64(2654435761) + np.uint64(97)
    return np.uint64((b * w + b).sum(dtype=np.uint64))


def sphere_cloud(P0, seed=0, radius=0.5):
    """P0 points uniform on a sphere of radius 0.5 (the training init, config.py:177-182),
    outward normals, random colours."""
    g = torch.Generator().manual_seed(1234 + seed)
    p = torch.nn.functional.normalize(torch.randn(P0, 3, generator=g), dim=1)
    colours = torch.rand(P0, 3, generator=g)
    return (radius * p).contiguous(), p.clone().contiguous(), colours.contiguous()


def random_cameras(N, seed=0, dist=(1.2, 2.2), znear=0.1, zfar=100.0):
    """Look-at cameras as DSS/core/camera.py:42-51 samples them (fov 60, znear 0.1, zfar 100)."""
    g = torch.Generator().manual_seed(4321 + seed)
    d = torch.rand(N, generator=g) * (dist[1] - dist[0]) + dist[0]
    azim = torch.rand(N, generator=g) * 360 - 180
    elev = torch.rand(N, generator=g) * 180 - 90
    at = torch.rand(N, 3, generator=g) * 0.1 - 0.05
    R, T = look_at_view_transform(d, elev, azim, at=at)
    return FoVPerspectiveCameras(znear=znear, zfar=zfar, R=R, T=T)


def scene(P0, N, seed=0):
    pts, nrm, col = sphere_cloud(P0, seed)
    cams = random_cameras(N, seed)
    proj, view = camera_matrices(cams)
    return pts, nrm, col, proj, view, cams


def packed_offsets(N, P0):
    first = torch.arange(N, dtype=torch.int64) * P0
    num = torch.full((N,), P0, dtype=torch.int64)
    return first, num


def random_screen_splats(P, N, S, seed=0, rad_px=(0.8, 4.0), z=(0.5, 3.0), behind_frac=0.05, ragged=True):
    """Random packed screen-space splats for the _C-level operators: points (P,3), ellipse (P,3),
    cutoff (P,), radii (P,2), first_idx, num_points.  Radii are the exact bbox of the conic at cutoff."""
    rng = np.random.default_rng(100 + seed)
    pts = np.concatenate([rng.uniform(-1.05, 1.05, (P, 2)), rng.uniform(z[0], z[1], (P, 1))], 1).astype(np.float32)
    behind = rng.random(P) < behind_frac
    pts[behind, 2] = -pts[behind, 2]
    pix = 2.0 / S
    # random SPD 2x2 variance -> conic = inverse
    s1 = rng.uniform(rad_px[0] * pix, rad_px[1] * pix, P)
    s2 = rng.uniform(rad_px[0] * pix, rad_px[1] * pix, P)
    th = rng.uniform(0, np.pi, P)
    c, s = np.cos(th), np.sin(th)
    G00 = (c * s1) ** 2 + (s * s2) ** 2
    G11 = (s * s1) ** 2 + (c * s2) ** 2
    G01 = c * s * (s1 ** 2 - s2 ** 2)
    det = G00 * G11 - G01 ** 2
    cutoff = rng.uniform(0.5, 2.0, P).astype(np.float32)
    ell = np.stack([G11 / det, -2 * G01 / det, G00 / det], 1).astype(np.float32)
    rad = np.stack([np.sqrt(cutoff * G00), np.sqrt(cutoff * G11)], 1).astype(np.float32)
    if ragged and N > 1:
        cuts = np.sort(rng.choice(np.arange(1, P), N - 1, replace=False))
        bounds = np.concatenate([[0], cuts, [P]])
    else:
        bounds = np.linspace(0, P, N + 1).astype(np.int64)
    first = bounds[:-1].astype(np.int64)
    num = (bounds[1:] - bounds[:-1]).astype(np.int64)
    return pts, ell, cutoff, rad, first, num


def _conic_splats(rng, cx, cy, z, s1, s2, cutoff, aligned=False):
    """packed screen splats (points, ellipse, cutoff, radii) with principal std devs s1, s2 (NDC) at random angles
    (along x and y when `aligned`); radii are the exact bbox of the conic at the cutoff, as in random_screen_splats"""
    th = np.zeros(len(cx)) if aligned else rng.uniform(0, np.pi, len(cx))
    c, s = np.cos(th), np.sin(th)
    G00 = (c * s1) ** 2 + (s * s2) ** 2
    G11 = (s * s1) ** 2 + (c * s2) ** 2
    G01 = c * s * (s1 ** 2 - s2 ** 2)
    det = G00 * G11 - G01 ** 2
    pts = np.stack([cx, cy, z], 1).astype(np.float32)
    ell = np.stack([G11 / det, -2 * G01 / det, G00 / det], 1).astype(np.float32)
    rad = np.stack([np.sqrt(cutoff * G00), np.sqrt(cutoff * G11)], 1).astype(np.float32)
    return pts, ell, np.asarray(cutoff, np.float32), rad


EDGE_FAMILIES = ("ties", "merge", "dense", "huge", "ragged")


def edge_screen_splats(family, S, seed=0, P=1200):
    """Seeded packed screen splats for the _C-level operators at the places where a rasterizer goes wrong.  Same
    outputs as random_screen_splats: points (P,3), ellipse (P,3), cutoff (P,), radii (P,2), first_idx, num_points.

    ties   : view 0 draws z from four values only, plus z = +0.0, -0.0 and +inf; view 1 gives every splat the same z
             (a degenerate depth range: every splat in one depth slice)
    merge  : z in {0.5, 0.5625, 0.625, 0.75}, exact in fp32, so z_k - z_0 hits a merge threshold of 0.0625 exactly
    dense  : ~2000 splats over one tile and ~1000 over another, next to empty tiles, in ascending (view 0), descending
             (view 1) and random (view 2) depth order by index; long tile lists, several list chunks per tile; and
             ~13 * P splats of one depth over one tile (view 3)
    huge   : radii >= 2 NDC, centres at |c| >= 4 (up to 1e6) whose boxes reach into the image (boxes tighter than
             the ellipses), centres on tile edges and on pixel centres, box edges exactly on pixel centres
    ragged : views with no splat, one splat, only splats behind the camera, and an ordinary one
    """
    rng = np.random.default_rng(1000 + seed + 7 * EDGE_FAMILIES.index(family))
    pix = 2.0 / S
    ndc = lambda i: np.float32(-1) + np.float32(2 * np.asarray(i) + 1) / np.float32(S)   # pixel centre, fp32

    def small(n, lo=0.8, hi=4.0):
        return rng.uniform(lo * pix, hi * pix, n), rng.uniform(lo * pix, hi * pix, n)

    def cut(n):
        return rng.uniform(0.5, 2.0, n).astype(np.float32)

    views = []
    if family == "ties":
        n = P
        z = rng.choice(np.float32([0.5, 0.75, 1.0, 1.25]), n)
        z[rng.random(n) < 0.08] = 0.0
        z[rng.random(n) < 0.08] = -0.0
        z[rng.random(n) < 0.04] = np.inf
        views.append(_conic_splats(rng, rng.uniform(-1, 1, n), rng.uniform(-1, 1, n), z, *small(n, 1.5, 6.0), cut(n)))
        n = P // 2
        views.append(_conic_splats(rng, rng.uniform(-1, 1, n), rng.uniform(-1, 1, n), np.full(n, 0.875),
                                   *small(n, 1.5, 6.0), cut(n)))
    elif family == "merge":
        n = P
        z = rng.choice(np.float32([0.5, 0.5625, 0.625, 0.75]), n)
        views.append(_conic_splats(rng, rng.uniform(-1, 1, n), rng.uniform(-1, 1, n), z, *small(n, 1.5, 6.0), cut(n)))
    elif family == "dense":
        B = (S + 15) // 16
        t0 = (min(1, B - 1), min(1, B - 1))            # (ty, tx) of the dense tiles
        t1 = (min(1, B - 1), min(3, B - 1))
        for order in ("asc", "desc", "rand"):
            cs = []
            for (ty, tx), m in ((t0, 2 * P), (t1, P)):
                lo_x, hi_x = ndc(16 * tx), ndc(min(16 * tx + 15, S - 1))
                lo_y, hi_y = ndc(16 * ty), ndc(min(16 * ty + 15, S - 1))
                cs.append((rng.uniform(lo_x, hi_x, m), rng.uniform(lo_y, hi_y, m)))
            cx = np.concatenate([c[0] for c in cs])
            cy = np.concatenate([c[1] for c in cs])
            n = len(cx)
            z = np.sort(rng.uniform(0.5, 3.0, n)).astype(np.float32)
            if order == "desc":
                z = z[::-1].copy()
            elif order == "rand":
                z = rng.permutation(z)
            views.append(_conic_splats(rng, cx, cy, z, *small(n, 0.8, 5.0), cut(n)))
        # one depth for all: more than three binning blocks of splats over one tile, so that the list arrives in no
        # particular id order and equal-depth splats meet a block threshold equal to their own depth
        n = 13 * P
        ty, tx = t0
        cx = rng.uniform(ndc(16 * tx), ndc(min(16 * tx + 15, S - 1)), n)
        cy = rng.uniform(ndc(16 * ty), ndc(min(16 * ty + 15, S - 1)), n)
        views.append(_conic_splats(rng, cx, cy, np.ones(n), *small(n, 0.8, 5.0), cut(n)))
    elif family == "huge":
        parts = []
        n = 40                                          # radius >= 2 NDC, centres inside or near the image
        s = rng.uniform(2.0, 6.0, n)
        parts.append(_conic_splats(rng, rng.uniform(-1.5, 1.5, n), rng.uniform(-1.5, 1.5, n),
                                   rng.uniform(0.5, 3.0, n), s, s * rng.uniform(0.5, 1.0, n), np.ones(n)))
        n = 60                                          # far-off centres (|c| from 4 to 1e6) reaching into the image
        far = np.exp(rng.uniform(np.log(4.0), np.log(1e6), n)) * rng.choice([-1.0, 1.0], n)
        reach = rng.uniform(0.2, 1.9, n)               # how far the box reaches past the near image edge
        r = np.abs(far) - 1.0 + reach
        other = rng.uniform(-0.9, 0.9, n)
        swap = rng.random(n) < 0.5
        cx, cy = np.where(swap, other, far), np.where(swap, far, other)
        q = rng.uniform(0.3, 1.0, n)
        sx, sy = np.where(swap, q * 0.2, r), np.where(swap, r, q * 0.2)
        parts.append(_conic_splats(rng, cx, cy, rng.uniform(0.1, 0.4, n), sx, sy, np.ones(n), aligned=True))
        # boxes tighter than the ellipses (q <= 1/4 on the box edge), so that the box edge decides whole pixel columns
        for pp in parts:
            pp[1][:] = pp[1] * np.float32(0.25)
        n = P                                           # ordinary splats centred on tile edges and pixel centres
        i = rng.integers(0, S, (n, 2))
        on_edge = rng.random((n, 2)) < 0.5
        cx = np.where(on_edge[:, 0], ndc(16 * (i[:, 0] // 16)) - np.float32(1.0 / S), ndc(i[:, 0]))
        cy = np.where(on_edge[:, 1], ndc(16 * (i[:, 1] // 16)) - np.float32(1.0 / S), ndc(i[:, 1]))
        parts.append(_conic_splats(rng, cx, cy, rng.uniform(0.5, 3.0, n), *small(n, 1.0, 5.0), cut(n)))
        # boxes whose edges fall exactly on pixel centres: centre on a pixel centre, radius a whole number of pixels
        pts_, ell_, cut_, rad_ = parts[-1]
        k = rng.integers(1, 6, (n, 2)).astype(np.float32) * np.float32(pix)
        exact = rng.random(n) < 0.5
        rad_[exact] = k[exact]
        pts_[exact, :2] = np.stack([ndc(i[exact, 0]), ndc(i[exact, 1])], 1)
        views.append(tuple(np.concatenate(a) for a in zip(*parts)))
    elif family == "ragged":
        empty = (np.zeros((0, 3), np.float32), np.zeros((0, 3), np.float32), np.zeros(0, np.float32),
                 np.zeros((0, 2), np.float32))
        views.append(empty)
        views.append(_conic_splats(rng, np.zeros(1), np.zeros(1), np.ones(1), np.full(1, 6 * pix), np.full(1, 4 * pix),
                                   np.ones(1)))
        n = P // 4
        views.append(_conic_splats(rng, rng.uniform(-1, 1, n), rng.uniform(-1, 1, n), -rng.uniform(0.5, 3.0, n),
                                   *small(n), cut(n)))
        n = P
        views.append(_conic_splats(rng, rng.uniform(-1.05, 1.05, n), rng.uniform(-1.05, 1.05, n),
                                   rng.uniform(0.5, 3.0, n), *small(n), cut(n)))
        views.append(empty)
    else:
        raise ValueError(family)
    pts, ell, cutoff, rad = (np.ascontiguousarray(np.concatenate(a)) for a in zip(*views))
    num = np.array([len(v[0]) for v in views], np.int64)
    first = (np.cumsum(num) - num).astype(np.int64)
    return pts, ell, cutoff, rad, first, num


def pix_ndc(i, S):
    """fp32 NDC centre of pixel index i (NDC-index orientation), as pix_to_ndc computes it: -1 + (2i + 1) / S"""
    return np.float32(-1) + np.float32(2 * np.asarray(i) + 1) / np.float32(S)


def occ_d2_modes(dx, dy):
    """fp32 d2 of the occupancy gather's disc test in both roundings -> (dx*dx + dy*dy, fmaf(dx, dx, dy*dy)), exact.
    dx*dx is exact in float64 and, while dx*dx and dy*dy lie within a factor 16 of each other, so is its sum with the
    rounded dy*dy; the caller keeps only such pairs (`ok`).  -> (d2_mode0, d2_mode1, ok)"""
    dx, dy = np.asarray(dx, np.float32), np.asarray(dy, np.float32)
    xx, yy = dx.astype(np.float64) ** 2, dy.astype(np.float64) ** 2
    yyf = yy.astype(np.float32)
    d0 = (xx.astype(np.float32) + yyf).astype(np.float32)
    d1 = (xx + yyf.astype(np.float64)).astype(np.float32)
    ok = (xx <= 16 * yy) & (yy <= 16 * xx)
    return d0, d1, ok


OCC_FAMILIES = ("disc_edge", "disc_near", "box_edge", "centre", "border", "dense", "many_tiles", "ragged")


def occ_edge_splats(family, S, seed=0, r_px=None):
    """Seeded inputs of the occupancy gather (_C.occ_backward) at the places where it goes wrong -> dict of
    pts (P,3), rad (P,2), vis (P,) uint8, first, num (N,), g (N,S,S) alpha gradient in image orientation (row r, col c
    is NDC-index pixel (S-1-c, S-1-r)), rs (N,) search radii, and `flips` (disc_near: the (view, point, xi, yi) pairs
    whose disc membership differs between fma_mode 0 and 1).  Radii in pixels below are multiples of 2/S in NDC.

    disc_edge : S a power of two, centres on pixel centres, r = 5 px, g != 0 at the (3,4,5) offsets, where
                d2 == r^2 exactly (view 0: included); view 1 is the same with r one ulp smaller (excluded)
    disc_near : sub-pixel centres placed so that d2 lies within an ulp of r^2 at one pixel each, kept where the two
                roundings of d2 decide the pair differently (at least 20 such pairs)
    box_edge  : positive gradients at |dx| == rx and |dy| == ry exactly (and the same box one ulp smaller), ry > r
                (the centre-row band capped at the window), ry below half a pixel, rx >> r
    centre    : points on pixel centres with g != 0 there (d2 = 0), and a few ulp off them (d2 < 1e-10)
    border    : |x| or |y| exactly 1 (gradient), nextafter(1, 2) (none), centres within a window of the edges and
                corners
    dense     : 129 and ~5000 splats over one tile, 257 in one pixel: several work items per tile
    many_tiles: S = 1024, two views, a few splats in nearly every tile: more item groups than persistent CTAs
    ragged    : views with 0, 1 and 2 visible splats (and invisible ones), an empty range, and visible splats behind
                the camera or outside the image
    """
    rng = np.random.default_rng(3000 + seed + 13 * OCC_FAMILIES.index(family))
    pix = 2.0 / S
    f32 = np.float32
    views = []            # per view: (x, y, z, rx, ry, vis, g, rs)

    def grad(lo=0.5, hi=1.5, zero=0.5, neg=0.5):
        g = rng.uniform(lo, hi, (S, S)) * 1e-3
        g[rng.random((S, S)) < neg] *= -1
        g[rng.random((S, S)) < zero] = 0
        return g.astype(f32)

    def put(g, xi, yi, v):
        g[S - 1 - np.asarray(yi), S - 1 - np.asarray(xi)] = v

    def view(x, y, rx, ry, g, rs, z=None, vis=None):
        n = len(x)
        views.append((np.asarray(x, f32), np.asarray(y, f32), f32(1) if z is None else np.asarray(z, f32),
                      np.asarray(rx, f32) * np.ones(n, f32), np.asarray(ry, f32) * np.ones(n, f32),
                      np.ones(n, np.uint8) if vis is None else np.asarray(vis, np.uint8), g, f32(rs)))

    flips = []
    if family == "disc_edge":
        assert S & (S - 1) == 0
        r_px = r_px or 5
        a_, b_ = {5: (3, 4), 10: (6, 8), 13: (5, 12)}[r_px]           # a^2 + b^2 = r^2
        r = f32(r_px * pix)
        c = np.arange(r_px + 1, S - r_px - 1, 2 * r_px + 3)
        xi, yi = (a.ravel() for a in np.meshgrid(c, c))
        g = grad(zero=0.3)
        for kx, ky in ((a_, b_), (b_, a_), (r_px, 0), (0, r_px)):
            for sx in (-1, 1):
                for sy in (-1, 1):
                    put(g, xi + sx * kx, yi + sy * ky, (rng.uniform(0.5, 1.5, len(xi)) * 1e-3 *
                                                        rng.choice([-1, 1], len(xi))).astype(f32))
        for rv in (r, np.nextafter(r, f32(0))):
            view(pix_ndc(xi, S), pix_ndc(yi, S), (r_px + 1) * pix, (r_px + 1) * pix, g, rv)
    elif family == "disc_near":
        r_px = r_px or 4.6
        r = f32(r_px * pix)
        r2 = f32(r * r)
        g = grad(zero=0.5)
        xs, ys, used = [], [], set()
        for _ in range(200):
            m = 4096
            e = int(r_px) + 2
            xi = rng.integers(e, S - e, m)
            yi = rng.integers(e, S - e, m)
            kx = np.rint(r_px * rng.choice([0.5, 0.6, 0.7, 0.8], m)).astype(np.int64)
            ky = np.rint(np.sqrt(r_px ** 2 - kx ** 2)).astype(np.int64) * rng.choice([-1, 1], m)
            kx = kx * rng.choice([-1, 1], m)
            px = (pix_ndc(xi, S) + f32(pix) * rng.uniform(-0.45, 0.45, m).astype(f32)).astype(f32)
            dx = (pix_ndc(xi + kx, S) - px).astype(f32)
            dyt = np.sqrt(np.maximum(float(r2) - dx.astype(np.float64) ** 2, 0.0))
            py = (pix_ndc(yi + ky, S).astype(np.float64) - np.sign(ky) * dyt).astype(f32)
            dy = (pix_ndc(yi + ky, S) - py).astype(f32)
            d0, d1, ok = occ_d2_modes(dx, dy)
            sel = np.nonzero(ok & ((d0 <= r2) != (d1 <= r2)) & (np.abs(py) < 1) & (np.abs(px) < 1))[0]
            for i in sel:
                key = (int(xi[i] + kx[i]), int(yi[i] + ky[i]))
                if key in used:
                    continue
                used.add(key)
                xs.append(px[i])
                ys.append(py[i])
                flips.append((0, len(xs) - 1, key[0], key[1]))
            if len(flips) >= 40:
                break
        assert len(flips) >= 20, len(flips)
        for _, _, fx, fy in flips:    # a negative gradient acts on the whole disc
            put(g, fx, fy, f32(-rng.uniform(0.5, 1.5) * 1e-3))
        m = 100
        xs += list(rng.uniform(-1, 1, m).astype(f32))
        ys += list(rng.uniform(-1, 1, m).astype(f32))
        view(xs, ys, (r_px + 1) * pix, (r_px + 1) * pix, g, r)
    elif family == "box_edge":
        assert S & (S - 1) == 0
        r_px = r_px or 6
        c = np.arange(r_px + 2, S - r_px - 2, 2 * r_px + 3)
        xi, yi = (a.ravel() for a in np.meshgrid(c, c))
        n = len(xi)
        kind = np.arange(n) % 6
        kx = rng.integers(2, 5, n).astype(f32)
        ky = rng.integers(2, 5, n).astype(f32)
        rx = np.select([kind == 0, kind == 1, kind == 2, kind == 3, kind == 4],
                       [kx * f32(pix), np.nextafter(kx * f32(pix), f32(0)), f32(1.5 * r_px * pix), f32(3 * pix),
                        f32(3 * r_px * pix)], f32(4 * pix)).astype(f32)
        ry = np.select([kind == 0, kind == 1, kind == 2, kind == 3, kind == 4],
                       [ky * f32(pix), np.nextafter(ky * f32(pix), f32(0)), f32(1.5 * r_px * pix), f32(0.3 * pix),
                        f32(2 * pix)], f32(4 * pix)).astype(f32)
        x = pix_ndc(xi, S)
        y = pix_ndc(yi, S)
        y = np.where(kind == 3, y + f32(0.2 * pix), y).astype(f32)    # off the row centre, within ry of it
        g = grad(zero=0.1, neg=0.2)
        view(x, y, rx, ry, g, f32(r_px * pix))
    elif family == "centre":
        assert S & (S - 1) == 0
        c = np.arange(4, S - 4, 9)
        xi, yi = (a.ravel() for a in np.meshgrid(c, c))
        x, y = pix_ndc(xi, S), pix_ndc(yi, S)
        n = len(x)
        k = np.arange(n) % 4            # 0: on the centre; 1..3: that many ulp off it (x, y or both)
        for _ in range(3):
            step = k > _
            x = np.where(step & (np.arange(n) % 3 != 1), np.nextafter(x, f32(2)), x).astype(f32)
            y = np.where(step & (np.arange(n) % 3 != 0), np.nextafter(y, f32(-2)), y).astype(f32)
        g = grad(zero=0.2)
        put(g, xi, yi, (rng.uniform(0.5, 1.5, n) * 1e-3 * rng.choice([-1, 1], n)).astype(f32))
        view(x, y, 3 * pix, 3 * pix, g, f32(3.4 * pix))
    elif family == "border":
        m = 60
        one, past = f32(1), np.nextafter(f32(1), f32(2))
        side = rng.choice([-1, 1], (m, 2)).astype(f32)
        t = rng.uniform(-1, 1, m).astype(f32)
        axis = np.arange(m) % 2
        edge = np.where(np.arange(m) % 3 == 2, past, one)
        x = np.where(axis == 0, side[:, 0] * edge, t).astype(f32)
        y = np.where(axis == 1, side[:, 1] * edge, t).astype(f32)
        corners = np.array([[a * b, c * d] for a in (1, -1) for c in (1, -1) for b, d in ((one, one), (past, one))],
                           f32)
        near = rng.uniform(-1, 1, (200, 2)).astype(f32)
        near = np.sign(near) * (1 - np.abs(near) * f32(6 * pix))          # within 6 px of an edge or a corner
        pts = np.concatenate([np.stack([x, y], 1), corners, near.astype(f32)])
        view(pts[:, 0], pts[:, 1], 2 * pix, 2 * pix, grad(zero=0.2), f32(3.7 * pix))
    elif family == "dense":
        def in_tile(tx, ty, n):
            lo = lambda t: pix_ndc(32 * t, S) - f32(0.5 * pix)
            hi = lambda t: pix_ndc(min(32 * t + 31, S - 1), S) + f32(0.45 * pix)
            return rng.uniform(lo(tx), hi(tx), n), rng.uniform(lo(ty), hi(ty), n)
        parts = [in_tile(0, 0, 129), in_tile(1, 1, 5000)]
        px_, py_ = pix_ndc(45, S), pix_ndc(12, S)
        parts.append((px_ + rng.uniform(-0.45, 0.45, 257) * pix, py_ + rng.uniform(-0.45, 0.45, 257) * pix))
        x = np.concatenate([p[0] for p in parts])
        y = np.concatenate([p[1] for p in parts])
        n = len(x)
        view(x, y, rng.uniform(0.5, 4, n) * pix, rng.uniform(0.5, 4, n) * pix, grad(zero=0.3), f32(3.3 * pix))
    elif family == "many_tiles":
        for _ in range(2):
            n = 3000
            view(rng.uniform(-1, 1, n), rng.uniform(-1, 1, n), rng.uniform(0.5, 4, n) * pix,
                 rng.uniform(0.5, 4, n) * pix, grad(zero=0.9), f32(3.2 * pix))
    elif family == "ragged":
        def some(n, nvis):
            vis = np.zeros(n, np.uint8)
            vis[rng.choice(n, nvis, replace=False)] = 1
            return rng.uniform(-0.9, 0.9, n), rng.uniform(-0.9, 0.9, n), vis
        for n, nvis in ((3, 0), (3, 1), (4, 2), (0, 0)):
            x, y, vis = some(n, nvis)
            view(x, y, 3 * pix, 3 * pix, grad(zero=0.2), f32(4.2 * pix), vis=vis)
        n = 30       # visible, but behind the camera / outside the image / ordinary
        x, y = rng.uniform(-0.9, 0.9, n), rng.uniform(-0.9, 0.9, n)
        z = np.where(np.arange(n) % 3 == 0, -rng.uniform(0.5, 2, n), rng.uniform(0.5, 2, n))
        x = np.where(np.arange(n) % 3 == 1, rng.choice([-1.01, 1.01], n), x)
        view(x, y, 3 * pix, 3 * pix, grad(zero=0.2), f32(4.2 * pix), z=z)
    else:
        raise ValueError(family)
    num = np.array([len(v[0]) for v in views], np.int64)
    first = (np.cumsum(num) - num).astype(np.int64)
    P = int(num.sum())
    pts = np.zeros((P, 3), np.float32)
    rad = np.zeros((P, 2), np.float32)
    vis = np.zeros(P, np.uint8)
    for (x, y, z, rx, ry, v, _, _), f, m in zip(views, first, num):
        pts[f:f + m] = np.stack([x, y, np.broadcast_to(z, x.shape)], 1)
        rad[f:f + m] = np.stack([rx, ry], 1)
        vis[f:f + m] = v
    g = np.ascontiguousarray(np.stack([v[6] for v in views]))
    rs = np.array([v[7] for v in views], np.float32)
    return dict(pts=pts, rad=rad, vis=vis, first=first, num=num, g=g, rs=rs, flips=flips)


def rim_mask(q, cutoff_at_idx):
    """pixels whose fragments sit within a few ulp of the cutoff (FMA contraction can flip them)."""
    return np.abs(q - cutoff_at_idx) <= 8 * np.spacing(np.abs(cutoff_at_idx).astype(np.float32))


def assert_fragments_exact(got, want, cutoff):
    """got / want = (idx, zbuf, qvalue, occ) of a forward and of the oracle (fma_mode=1) on the same records.  idx, q
    and occupancy must be equal bit for bit and zbuf too, up to the sign of zero (the kernels canonicalise -0 to +0, the
    oracle stores the input).  The one admissible difference is a rim pixel: a fragment within a few ulp of its
    cutoff in either output.  Returns (number of rim pixels, mask of the pixels whose idx agree)."""
    idx, z, q, occ = (_npy(a) for a in got)
    widx, wz, wq, wocc = want
    same = (idx == widx).all(-1)
    rim = 0
    if not same.all():
        bad = ~same
        ok = np.zeros_like(bad)
        for a, b in ((idx, q), (widx, wq)):
            c = np.where(a >= 0, cutoff[np.maximum(a, 0)], np.inf)
            ok |= (rim_mask(b, c) & (a >= 0)).any(-1)
        assert (ok | ~bad).all(), "idx differs at %d non-rim pixels" % int((bad & ~ok).sum())
        rim = int(bad.sum())
    assert np.array_equal(z[same].view(np.uint32), (wz[same] + np.float32(0)).view(np.uint32))
    assert np.array_equal(q[same].view(np.uint32), wq[same].view(np.uint32))
    assert np.array_equal(occ[same].view(np.uint32), wocc[same].view(np.uint32))
    return rim, same


def assert_fragments_accepted(idx, q, points, radii, cutoff):
    """Without an oracle: every emitted fragment passes the acceptance test in fp32 at its own emitted q
    (q <= cutoff, |dx| <= rx, |dy| <= ry at the pixel centre), and the lists are -1 padded after the first gap."""
    idx, q = _npy(idx), _npy(q)
    S = idx.shape[1]
    c = np.float32(-1) + (2 * np.arange(S) + 1).astype(np.float32) / np.float32(S)   # pix_to_ndc, fp32
    c = c[::-1]                                      # output row r / column c is NDC index S-1-r / S-1-c
    live = idx >= 0
    assert not (live[..., 1:] & ~live[..., :-1]).any()
    i = np.maximum(idx, 0)
    dx = (c[None, None, :, None] - points[i, 0]).astype(np.float32)
    dy = (c[None, :, None, None] - points[i, 1]).astype(np.float32)
    ok = (np.abs(dx) <= radii[i, 0]) & (np.abs(dy) <= radii[i, 1]) & (q <= cutoff[i])
    assert ok[live].all(), "%d emitted fragments fail the acceptance test" % int((~ok & live).sum())


def assert_blend_matches(image, weights, widx, wq, wocc, scaler, colours, same):
    """Fused image (N,S,S,4) and normalised weights against oracle.blend_forward on the oracle's fragments, on the
    pixels whose idx agree.  The kernel's error bound, relative to each (non-negative) value: w_k = expf(-q/2) * scaler
    is within 3 ulp (expf 2 ulp, one product), a sum of at most K positive terms adds K ulp of the sum, then one IEEE
    reciprocal and one product: weights within (K + 5) ulp, colours (a ratio of two such sums) within (2K + 8) ulp.  The
    oracle's own rounding (float w, double sums, one final rounding) adds a few ulp: the test allows 8 more.
    Returns the largest error of each, in units of K ulp."""
    import oracle
    K = widx.shape[-1]
    u = 2.0 ** -24
    wimg = oracle.blend_forward(widx, wq, wocc, scaler, colours).astype(np.float64)
    img = _npy(image).astype(np.float64)
    err = np.abs(img - wimg)[same]
    assert (err <= (2 * K + 16) * u * np.abs(wimg[same])).all(), float((err / np.maximum(np.abs(wimg[same]), 1e-30)).max())
    live = widx >= 0
    w = np.where(live, np.exp(-0.5 * wq.astype(np.float64)) * scaler[np.maximum(widx, 0)].astype(np.float64), 0.0)
    wn = w / np.maximum(w.sum(-1, keepdims=True), 1e-4)
    werr = np.abs(_npy(weights).astype(np.float64) - wn)[same]
    assert (werr <= (K + 13) * u * wn[same]).all(), float((werr / np.maximum(wn[same], 1e-30)).max())
    rel = lambda e, v: float((e / np.maximum(np.abs(v), 1e-30)).max()) / (K * u) if e.size else 0.0
    return rel(err, wimg[same]), rel(werr, wn[same])


def backward_via_lib(out, pts, proj, view, first, num, shared, prm, grad_image, grad_zbuf, repeat_camera=1):
    """dss_render_backward with grad_ndc set, then `repeat_camera` calls of dss_camera_backward (as ops.py does) ->
    (grad_ndc (P,3), grad_points (P0,3) / (P,3), [(grad_proj, grad_view)] of every repetition).  No forward cell counts
    are passed, so the backward runs its own count pass."""
    dev = pts.device
    N = proj.shape[0]
    P0 = pts.shape[0]
    P = N * P0 if shared else P0
    a = _lib.RenderArgs()
    ops._fill_common(a, pts, None, None, proj, view, None, first, num, shared, N, P0, P, prm)
    a.records, a.idx, a.weights, a.visible = (_lib.ptr(t) for t in (out.records, out.idx, out.weights, out.visible))
    a.grad_image, a.grad_zbuf = _lib.ptr(grad_image), _lib.ptr(grad_zbuf)
    # rows that no view range covers are never written (ops.py zero-fills them the same way)
    grad_points = torch.zeros_like(pts)
    grad_ndc = torch.zeros((P, 3), dtype=torch.float32, device=dev)
    a.grad_points_world, a.grad_ndc = _lib.ptr(grad_points), _lib.ptr(grad_ndc)
    lib, ctx, st = _lib.load(), _lib.ctx(dev), _lib.stream_ptr(dev)
    _lib.check(lib.dss_render_backward(ctx, C.byref(a), st), "dss_render_backward")
    res = []
    for _ in range(repeat_camera):
        gP, gV = (torch.full((N, 4, 4), float("nan"), device=dev) for _ in range(2))
        _lib.check(lib.dss_camera_backward(ctx, C.byref(a), _lib.ptr(gP), _lib.ptr(gV), None, st), "dss_camera_backward")
        res.append((gP, gV))
    torch.cuda.synchronize(dev)
    return grad_ndc, grad_points, res


def _npy(t):
    return t.detach().cpu().numpy() if torch.is_tensor(t) else np.asarray(t)


def view_ranges(N, P0, first, num):
    """(first, num) as int64 numpy arrays; a shared cloud (first = None) of P0 points is N ranges of P0 slots"""
    if first is None:
        return np.arange(N, dtype=np.int64) * P0, np.full(N, P0, np.int64)
    return _npy(first).astype(np.int64), _npy(num).astype(np.int64)


def preprocess_f64_slots(pts, nrm, proj, view, h, prm, first=None, num=None):
    """oracle.preprocess_f64 for every slot of a shared (first = None) or packed cloud: one call per view on that view's
    slice of the points, the normals and h (per view (N,), or per splat (P,) -- the slice then sets its per_splat mode)
    -> dict of (P, .) float64 arrays ndc, radii, scaler, jac; rows outside every view range are NaN."""
    import oracle
    pts, nrm, projn, viewn, h = _npy(pts), _npy(nrm), _npy(proj), _npy(view), _npy(h).reshape(-1)
    N, shared = projn.shape[0], first is None
    first, num = view_ranges(N, pts.shape[0], first, num)
    P = N * pts.shape[0] if shared else pts.shape[0]
    per_splat = h.size == P and h.size != N
    out = dict(ndc=np.full((P, 3), np.nan), radii=np.full((P, 2), np.nan), scaler=np.full(P, np.nan),
               jac=np.full((P, 3, 2), np.nan))
    for n in range(N):
        f, m = int(first[n]), int(num[n])
        if m == 0:
            continue
        src = slice(0, m) if shared else slice(f, f + m)
        pre = oracle.preprocess_f64(projn[n:n + 1], viewn[n:n + 1], pts[src], nrm[src],
                                    h[f:f + m] if per_splat else h[n:n + 1], prm.cutoff_threshold,
                                    prm.antialiasing_sigma, prm.image_size)
        for k in out:
            out[k][f:f + m] = pre[k]
    return out


def render_backward_f64(ndc, radii, idx, qvalue, scaler, pts, proj, view, prm, grad_image, grad_zbuf=None,
                        first=None, num=None):
    """Float64 reference of the whole fused backward (dss_render_backward) on a forward's own fragments.

    ndc (P,3), radii (P,2)     : the per-slot screen records the forward rasterized (records[:, :3], records[:, 3:5])
    idx, qvalue (N,S,S,K)       : its fragments;  scaler (P,): its per-slot scaler
    pts (P0,3) / (P,3)          : world points of a shared cloud (first = num = None) or of the packed slots
    proj, view (N,4,4)          : the cameras; prm: the SplatParams of the call
    grad_image (N,S,S,4), grad_zbuf (N,S,S,K) or None

    Composes the oracle: visibility -> exact lower median per (ragged) view -> occupancy gather (its float64 sums) ->
    z-buffer scatter (float64) -> clip of the 3-vector (rasterizer.py:667-673) in float64 -> chain through the float64
    Jacobian of oracle.preprocess_f64 and V[:3, 2] (the view depth) -> world gradient; and the colour gradient.
    Returns a dict of float64 arrays:
      ndc (P,3)       clipped NDC gradient per slot;   ndc_raw (P,3): the same before the clip
      ndc_err32 (P,)  per slot, |fp32 oracle - float64| of the pre-clip vector (fp32 sums in pixel order)
      world           (P0,3) summed over the views (shared) or (P,3) per packed row (rows no range covers: 0)
      colours (P,3)   colour gradient per slot
      vis (P,) uint8, rs (N,): the visibility and search radius it used
    """
    import oracle
    ndc = np.ascontiguousarray(_npy(ndc), np.float32)
    radii = np.ascontiguousarray(_npy(radii), np.float32)
    idx = np.ascontiguousarray(_npy(idx), np.int32)
    qvalue, scaler = _npy(qvalue), _npy(scaler)
    pts, viewn = _npy(pts), _npy(view)
    gi = np.ascontiguousarray(_npy(grad_image), np.float32)
    N, P = viewn.shape[0], ndc.shape[0]
    shared = first is None
    first, num = view_ranges(N, pts.shape[0], first, num)
    vis = oracle.visibility(idx, P)
    rs = oracle.search_radius(radii, vis, first, num, prm.radii_backward_scaler)
    g32, g64 = oracle.occ_backward_fast(ndc, radii, vis, rs, np.ascontiguousarray(gi[..., 3]), first, num, fma_mode=1)
    raw = np.concatenate([g64, np.zeros((P, 1))], 1)
    raw32 = np.concatenate([g32.astype(np.float64), np.zeros((P, 1))], 1)
    if grad_zbuf is not None:
        gz = np.ascontiguousarray(_npy(grad_zbuf), np.float32)
        # rasterize_points.cu:823-846: every fragment up to the first empty one
        live = np.cumprod(idx >= 0, axis=-1).astype(bool)
        np.add.at(raw[:, 2], idx[live], gz[live].astype(np.float64))
        raw32[:, 2] = oracle.zbuf_backward(idx, gz, P)
    err32 = np.linalg.norm(raw32 - raw, axis=1)
    g = raw.copy()
    if prm.clip_pts_grad > 0:
        nrm = np.linalg.norm(g, axis=1, keepdims=True)
        g = g / np.maximum(nrm, 1e-12) * np.minimum(nrm, prm.clip_pts_grad)
    # chain: d ndc_xy / d world = J (float64, from the world points; the normals and h do not enter it),
    # d z_view / d world = V[:3, 2]
    jac = preprocess_f64_slots(pts, np.zeros_like(pts), proj, view, np.ones(N, np.float32), prm,
                               None if shared else first, None if shared else num)["jac"]
    world = np.zeros((pts.shape[0], 3))
    for n in range(N):
        f, m = int(first[n]), int(num[n])
        gs = g[f:f + m]
        w = np.einsum("pkj,pj->pk", jac[f:f + m], gs[:, :2]) + gs[:, 2:3] * viewn[n, :3, 2].astype(np.float64)[None]
        if shared:
            world[:m] += w
        else:
            world[f:f + m] += w
    colours = oracle.blend_backward_colours(idx, qvalue, scaler, gi, P).astype(np.float64)
    return dict(ndc=g, ndc_raw=raw, ndc_err32=err32, world=world, colours=colours, vis=vis, rs=rs)


def render_backward_f64_of(out, pts, proj, view, prm, grad_image, grad_zbuf=None, first=None, num=None):
    """render_backward_f64 on the fragments of render_points(..., return_fragments=True)"""
    return render_backward_f64(out.records[:, :3], out.records[:, 3:5], out.idx, out.qvalue, out.scaler, pts, proj,
                               view, prm, grad_image, grad_zbuf, first, num)
