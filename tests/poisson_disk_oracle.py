"""numpy restatement of dss_sample_mesh_poisson_disk (csrc/mesh_sample.cu; the rule is in include/dss_b200.h).

Steps 1-4 of the rule: the usable faces and their integer weights, the SplitMix64 draws and the Monte Carlo pool, the
sequential dart throw over a hash grid of the accepted samples, and the radius search.  Every float64 operation is
the kernel's, in the kernel's order (numpy and Python floats round each operation on its own), so the pool, the
Euclidean selection and the radius equal the device's bit for bit.  The geodesic distance calls Python's asin, which
may differ from the device's in the last bit: :func:`select` reports the smallest relative gap |d - r| / r over the
pairs whose geodesic distance decided something, so a test knows when the two must agree."""
import math

import numpy as np

MONTECARLO_RATE = 20
MAX_PROBES = 64

_GOLDEN, _MIX1, _MIX2 = np.uint64(0x9E3779B97F4A7C15), np.uint64(0xBF58476D1CE4E5B9), np.uint64(0x94D049BB133111EB)
_LO32 = np.uint64(0xFFFFFFFF)


def splitmix64(seed, j):
    """the j-th output (j a uint64 array, from 1) of SplitMix64 seeded with ``seed``"""
    with np.errstate(over="ignore"):
        z = np.uint64(int(seed) & (2 ** 64 - 1)) + np.asarray(j, dtype=np.uint64) * _GOLDEN
        z = (z ^ (z >> np.uint64(30))) * _MIX1
        z = (z ^ (z >> np.uint64(27))) * _MIX2
        return z ^ (z >> np.uint64(31))


def mulhi64(a, b):
    """the high 64 bits of the 128-bit products a * b (uint64 arrays or scalars)"""
    a, b = np.asarray(a, dtype=np.uint64), np.uint64(b)
    s32 = np.uint64(32)
    with np.errstate(over="ignore"):
        a_lo, a_hi, b_lo, b_hi = a & _LO32, a >> s32, b & _LO32, b >> s32
        ll, hl, lh, hh = a_lo * b_lo, a_hi * b_lo, a_lo * b_hi, a_hi * b_hi
        cross = (ll >> s32) + (hl & _LO32) + lh
        return hh + (hl >> s32) + (cross >> s32)


def faces_of(verts, faces):
    """Step 1: {usable (F,) bool, area (F,) f64, cross (F,3) f64, length (F,) f64, prefix (F+1,) int64, W, amax, A}"""
    v = np.asarray(verts, dtype=np.float32).astype(np.float64)
    f = np.asarray(faces, dtype=np.int64).reshape(-1, 3)
    V, F = len(v), len(f)
    in_range = ((f >= 0) & (f < V)).all(1) if F else np.zeros(0, bool)
    fi = np.where(in_range[:, None], f, 0)
    if V == 0:
        fi, v = np.zeros_like(f), np.zeros((1, 3))
    a, b, c = v[fi[:, 0]], v[fi[:, 1]], v[fi[:, 2]]
    with np.errstate(invalid="ignore", over="ignore"):
        finite = np.isfinite(a).all(1) & np.isfinite(b).all(1) & np.isfinite(c).all(1)
        ab, ac = b - a, c - a
        cross = np.stack([ab[:, 1] * ac[:, 2] - ab[:, 2] * ac[:, 1], ab[:, 2] * ac[:, 0] - ab[:, 0] * ac[:, 2],
                          ab[:, 0] * ac[:, 1] - ab[:, 1] * ac[:, 0]], 1)
        length = np.sqrt((cross[:, 0] * cross[:, 0] + cross[:, 1] * cross[:, 1]) + cross[:, 2] * cross[:, 2])
        area = 0.5 * length
        usable = in_range & finite & (area > 0)
    area = np.where(usable, area, 0.0)
    amax = float(area.max()) if usable.any() else 0.0
    w = np.zeros(F, dtype=np.int64)
    if usable.any():
        w[usable] = np.maximum(1, np.ceil(area[usable] * 2.0 ** 32 / amax)).astype(np.int64)
    prefix = np.concatenate([[0], np.cumsum(w)]).astype(np.int64)
    W = int(prefix[-1])
    return {"usable": usable, "area": area, "cross": cross, "length": length, "prefix": prefix, "W": W,
            "amax": amax, "A": float(W) * amax * 2.0 ** -32, "v": v, "f": fi}


def pool(verts, faces, num_samples, seed=0, mesh=None):
    """Step 2: (points (M,3) f32, normals (M,3) f32, face (M,) int64) of the M = 20 N pool samples"""
    m = faces_of(verts, faces) if mesh is None else mesh
    M = MONTECARLO_RATE * int(num_samples)
    if m["W"] == 0:
        return np.zeros((0, 3), np.float32), np.zeros((0, 3), np.float32), np.zeros(0, np.int64)
    j = np.arange(M, dtype=np.uint64) * np.uint64(3) + np.uint64(1)
    x0, x1, x2 = splitmix64(seed, j), splitmix64(seed, j + np.uint64(1)), splitmix64(seed, j + np.uint64(2))
    t = mulhi64(x0, m["W"]).astype(np.int64)
    face = np.searchsorted(m["prefix"], t, side="right") - 1
    u = (x1 >> np.uint64(11)).astype(np.float64) * 2.0 ** -53
    v = (x2 >> np.uint64(11)).astype(np.float64) * 2.0 ** -53
    su = np.sqrt(u)
    w0, w1, w2 = (1.0 - su)[:, None], (su * (1.0 - v))[:, None], (su * v)[:, None]
    fi = m["f"][face]
    a, b, c = m["v"][fi[:, 0]], m["v"][fi[:, 1]], m["v"][fi[:, 2]]
    points = ((w0 * a + w1 * b) + w2 * c).astype(np.float32)
    normals = (m["cross"][face] / m["length"][face][:, None]).astype(np.float32)
    return points, normals, face


def geodesic_distance(p0, n0, p1, n1):
    """the approximate geodesic distance of the rule (p0 the later sample), Python floats; (distance, factor)"""
    dx, dy, dz = float(p0[0]) - float(p1[0]), float(p0[1]) - float(p1[1]), float(p0[2]) - float(p1[2])
    d2 = (dx * dx + dy * dy) + dz * dz
    if d2 == 0.0:
        return 0.0, 1.0
    de = math.sqrt(d2)
    vx, vy, vz = dx / de, dy / de, dz / de
    c0 = min(max((vx * float(n0[0]) + vy * float(n0[1])) + vz * float(n0[2]), -1.0), 1.0)
    c1 = min(max((vx * float(n1[0]) + vy * float(n1[1])) + vz * float(n1[2]), -1.0), 1.0)
    dc = c0 - c1
    if abs(dc) < 1e-4:
        q = 1.0 - c0 * c1
        g = 1.0 / math.sqrt(q) if q > 0.0 else math.inf
    else:
        g = (math.asin(c0) - math.asin(c1)) / dc
    g = max(g, 1.0)
    return de * g, g


def select(points, normals, r, geodesic=False):
    """Step 3, the sequential dart throw at radius r: (accepted pool indices (n,) int64 in pool order, smallest
    |d - r| / r over the geodesic distances that were computed (inf when none or Euclidean))"""
    P = [tuple(map(float, p)) for p in np.asarray(points, dtype=np.float32)]
    Nm = np.asarray(normals, dtype=np.float32)
    r = float(r)
    r2 = r * r
    cell = r * 1.001
    grid, accepted = {}, []
    margin = math.inf
    for i, (x, y, z) in enumerate(P):
        cx, cy, cz = math.floor(x / cell), math.floor(y / cell), math.floor(z / cell)
        hit = False
        for kx in (cx - 1, cx, cx + 1):
            for ky in (cy - 1, cy, cy + 1):
                for kz in (cz - 1, cz, cz + 1):
                    for k in grid.get((kx, ky, kz), ()):
                        qx, qy, qz = P[k]
                        dx, dy, dz = x - qx, y - qy, z - qz
                        d2 = (dx * dx + dy * dy) + dz * dz
                        if not geodesic:
                            hit = d2 < r2
                        elif d2 == 0.0:
                            hit = True
                        elif not math.sqrt(d2) < r:
                            hit = False
                        else:
                            d, _ = geodesic_distance(P[i], Nm[i], P[k], Nm[k])
                            margin = min(margin, abs(d - r) / r)
                            hit = d < r
                        if hit:
                            break
                    if hit:
                        break
                if hit:
                    break
            if hit:
                break
        if not hit:
            accepted.append(i)
            grid.setdefault((cx, cy, cz), []).append(i)
    return np.asarray(accepted, dtype=np.int64), margin


def sample(verts, faces, num_samples, geodesic=False, seed=0):
    """Step 4, the whole rule: {points, normals, radius, indices, probes [(r, n)], pool (points, normals)}"""
    N = int(num_samples)
    m = faces_of(verts, faces)
    pts, nrm, _ = pool(verts, faces, N, seed, mesh=m)
    empty = np.zeros((0, 3), np.float32)
    if m["W"] == 0:
        return {"points": empty, "normals": empty, "radius": 0.0, "indices": np.zeros(0, np.int64), "probes": [],
                "pool": (pts, nrm)}
    tol = N // 200
    r = math.sqrt(m["A"] / (0.7 * math.pi * N))
    lo = hi = -1.0
    best = None
    probes = []
    while len(probes) < MAX_PROBES:
        idx, _ = select(pts, nrm, r, geodesic)
        n = len(idx)
        probes.append((r, n))
        d = abs(n - N)
        if best is None or d < best[0]:
            best = (d, r, idx)
        if d <= tol:
            break
        if n > N:
            lo = r
        else:
            hi = r
        r = 2.0 * r if hi < 0.0 else 0.5 * r if lo < 0.0 else 0.5 * (lo + hi)
    _, radius, idx = best
    return {"points": pts[idx], "normals": nrm[idx], "radius": radius, "indices": idx, "probes": probes,
            "pool": (pts, nrm)}


def brute_force_select(points, r):
    """the Euclidean dart throw without a grid (every accepted sample tested), for checking :func:`select`"""
    p = np.asarray(points, dtype=np.float32).astype(np.float64)
    r2 = float(r) * float(r)
    acc = []
    for i in range(len(p)):
        if acc:
            d = p[i] - p[acc]
            d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
            if (d2 < r2).any():
                continue
        acc.append(i)
    return np.asarray(acc, dtype=np.int64)
