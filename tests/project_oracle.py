"""Host oracle of dss_denoise_normals and dss_project_to_surface (csrc/rimls.cu; the rules are in include/dss_b200.h
and DESIGN.md), restated from those rules in numpy float64.

* ``cloud_radius``: a cloud's neighbourhood radius min(scale avg k, 0.2), avg = sqrt(diag / c).
* ``neighbourhood``: the K-NN rows at K = k + 1 less each row's own index (the rule of ``upsample_oracle.neighbours``),
  less the entries beyond the radius, laid out as the device's 32 lanes.
* ``lane_sum``: the xor-butterfly sum over the 32 lanes, in the device's order.
* ``denoise_normals`` and ``project``: one cloud from its K-NN rows.  Both also return the smallest relative distance
  of any decision to its threshold (the radius, the 32 / c cutoff, the weight and move stops, zero-weight rows), so a
  test can assert that no decision is close enough to flip between two float64 implementations.
"""
from typing import NamedTuple

import numpy as np

from tests.upsample_oracle import neighbours as _own_excluded

LANES = 32
ALPHA_TOL, MOVE_TOL = 1e-4, 5e-4


def dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def normalize(v):
    """F.normalize in float64: v / max(|v|, 1e-12)"""
    v = np.asarray(v, np.float64)
    return v / np.maximum(np.sqrt(dot(v, v)), 1e-12)[..., None]


def eps_denom(s):
    m = np.where(np.abs(s) < 1e-17, 1e-17, np.abs(s))
    return np.where(s < 0, -m, m)


def lane_sum(v):
    """sum over axis 1 (32 lanes) by the butterfly 16, 8, 4, 2, 1: v_l + v_{l+h} for l < h"""
    h = v.shape[1]
    while h > 1:
        h //= 2
        v = v[:, :h] + v[:, h:2 * h]
    return v[:, 0]


def cloud_radius(points, k, scale):
    p = np.asarray(points, np.float64)
    if len(p) == 0:
        return 0.0
    d = p.max(0) - p.min(0)
    diag = np.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2])
    return min(scale * np.sqrt(diag / len(p)) * k, 0.2)


class Hood(NamedTuple):
    q: np.ndarray         # (c, 32, 3) neighbour positions, 0 where not ok
    n: np.ndarray         # (c, 32, 3) unit normals, 0 where not ok
    d2: np.ndarray        # (c, 32) squared distances, 0 where not ok
    ok: np.ndarray        # (c, 32) bool
    margin: float         # smallest |d2 - r^2| / r^2 over the present entries


def neighbourhood(points, normals, rows, r):
    p = np.asarray(points, np.float64)
    nb = _own_excluded(np.asarray(rows))
    c, k = nb.shape
    idx = np.full((c, LANES), -1, np.int64)
    idx[:, :k] = nb
    present = idx >= 0
    safe = np.where(present, idx, 0)
    q = p[safe]
    dd = p[:, None, :] - q
    d2 = dot(dd, dd)
    r2 = r * r
    margin = float(np.min(np.abs(d2[present] - r2)) / r2) if present.any() and r2 > 0 else np.inf
    ok = present & (d2 <= r2)
    n = normalize(np.asarray(normals, np.float64)[safe])
    z = ~ok
    q[z], n[z], d2[z] = 0.0, 0.0, 0.0
    return Hood(q, n, d2, ok, margin)


class Denoised(NamedTuple):
    normals: np.ndarray   # (c, 3) float64
    margin: float


def denoise_normals(points, normals, rows, k=16, sigma=30.0):
    """denoise_normals of one cloud from its K-NN rows (c, k + 1)"""
    p = np.asarray(points, np.float64)
    c = len(p)
    h = neighbourhood(p, normals, rows, cloud_radius(p, k, 4.0))
    ni = normalize(normals)
    inv = c / 2.0
    cut = 16.0 / inv
    margin = h.margin
    if h.ok.any():
        margin = min(margin, float(np.min(np.abs(h.d2[h.ok] - cut)) / cut))
    use = h.ok & ~(h.d2 > cut)
    t = (1.0 - dot(ni[:, None, :], h.n)) / sigma
    w = np.where(use, np.exp(-h.d2 * inv) * np.exp(-(t * t)), 0.0)
    if use.any() and np.min(w[use]) < 1e-290:          # an underflowing weight could decide a zero-weight row
        margin = 0.0
    sw = lane_sum(w)
    sn = np.stack([lane_sum(h.n[..., a] * w) for a in range(3)], 1)
    with np.errstate(invalid="ignore", divide="ignore"):
        out = np.where((sw != 0)[:, None], normalize(sn / eps_denom(sw)[:, None]), ni)
    return Denoised(out, margin)


class Projection(NamedTuple):
    points: np.ndarray        # (c, 3) float64
    iterations: np.ndarray    # (c,) int32
    margin: float
    inner_stops: int          # inner loops that stopped on the weight test
    outer_stops: int          # rows that stopped on the move test before max_proj_iters


def project(points, normals, rows, k=31, max_proj_iters=10, max_est_iters=5):
    """project_to_surface of one cloud from its K-NN rows (c, k + 1), the samples fixed at the input"""
    p = np.asarray(points, np.float64)
    c = len(p)
    h = neighbourhood(p, normals, rows, cloud_radius(p, k, 16.0))
    margin = h.margin
    d2min = np.where(h.ok & (h.d2 > 0), h.d2, np.inf).min(1)
    has = d2min < np.inf
    with np.errstate(divide="ignore"):
        inv = 1.0 / (16.0 * d2min)
    x = p.copy()
    iters = np.zeros(c, np.int32)
    active = has.copy()
    inner_stops = outer_stops = 0
    for _ in range(max_proj_iters):
        rws = np.flatnonzero(active)
        if len(rws) == 0:
            break
        X, Q, N, OK, INV = x[rws], h.q[rws], h.n[rws], h.ok[rws], inv[rws][:, None]
        m = len(rws)
        dx = X[:, None, :] - Q
        fx = np.where(OK, dot(dx, N), 0.0)
        alpha = np.ones_like(fx)
        f, g = np.zeros(m), np.zeros((m, 3))
        run = np.ones(m, bool)
        for s in range(max_est_iters):
            if s > 0:
                dn = N - g[:, None, :]
                u = np.sqrt(dot(dn, dn)) / 0.5
                v = fx - f[:, None]
                nxt = np.exp(-(u * u)) * np.exp(-(v * v * INV / 4.0))
                diff = np.where(OK, np.abs(nxt - alpha), 0.0).max(1)
                margin = min(margin, float(np.min(np.abs(diff[run] - ALPHA_TOL))) / ALPHA_TOL)
                stop = run & (diff < ALPHA_TOL)
                inner_stops += int(stop.sum())
                run &= ~stop
                alpha = np.where(run[:, None], nxt, alpha)
                if not run.any():
                    break
            phi = np.exp(-dot(dx, dx) * INV)
            w = np.where(OK, phi * alpha, 0.0)
            gs = np.where(OK, (INV * phi) * w, 0.0)
            gw = 2.0 * dx * gs[..., None]
            sw, sf = lane_sum(w), lane_sum(fx * w)
            sgw = np.stack([lane_sum(gw[..., a]) for a in range(3)], 1)
            sgf = np.stack([lane_sum(gw[..., a] * fx) for a in range(3)], 1)
            sn = np.stack([lane_sum(w * N[..., a]) for a in range(3)], 1)
            e = eps_denom(sw)
            fn = sf / e
            gn = ((sgf - fn[:, None] * sgw) + sn) / e[:, None]
            f = np.where(run, fn, f)
            g = np.where(run[:, None], gn, g)
        mv = f[:, None] * g
        x[rws] = X - mv
        iters[rws] += (mv != 0).any(1)
        nm = np.sqrt(dot(mv, mv))
        margin = min(margin, float(np.min(np.abs(nm - MOVE_TOL))) / MOVE_TOL)
        active[rws] = nm > MOVE_TOL
        outer_stops += int((~active[rws]).sum())
    return Projection(x, iters, margin, inner_stops, outer_stops)
