"""Float64 oracle of dss_point_mesh_distance (csrc/mesh_distance.cu): the closest point of every face to every query by
the Voronoi regions of a closed triangle, with the closest of the three edges for faces whose edge vectors have an
exactly zero cross product (segments and points).  Written in torch float64 with the kernel's operations in the
kernel's order, one rounding each, so that it runs on the CPU for the closed-form tests and on the GPU at scale, and
gives the kernel's bits."""
import torch


def _dot(u, v):
    return (u[..., 0] * v[..., 0] + u[..., 1] * v[..., 1]) + u[..., 2] * v[..., 2]


def _axpy(a, t, u):
    """a + t u, t (...) broadcast over the last axis"""
    return a + t[..., None] * u


def _seg_closest(p, a, b):
    ab, ap = b - a, p - a
    ln = _dot(ab, ab)
    t = torch.where(ln > 0, (_dot(ap, ab) / ln).clamp(0.0, 1.0), torch.zeros_like(ln))
    return _axpy(a, t, ab)


def _ratio(num, den):
    return torch.where(den > 0, num / den, torch.zeros_like(num))


def closest_points(p, a, b, c):
    """closest point of the closed triangle (a, b, c) to p; float64 tensors (..., 3) broadcast together"""
    p, a, b, c = torch.broadcast_tensors(p, a, b, c)
    ab, ac, ap, bp, cp = b - a, c - a, p - a, p - b, p - c
    flat = ((ab[..., 1] * ac[..., 2] - ab[..., 2] * ac[..., 1] == 0) & (ab[..., 2] * ac[..., 0] - ab[..., 0] * ac[..., 2] == 0)
            & (ab[..., 0] * ac[..., 1] - ab[..., 1] * ac[..., 0] == 0))
    d1, d2, d3, d4, d5, d6 = _dot(ab, ap), _dot(ac, ap), _dot(ab, bp), _dot(ac, bp), _dot(ab, cp), _dot(ac, cp)
    vc = d1 * d4 - d3 * d2
    vb = d5 * d2 - d1 * d6
    va = d3 * d6 - d5 * d4
    e43, e56 = d4 - d3, d5 - d6
    denom = (va + vb) + vc
    # the closest of the three edges, the first of ab, bc, ca on a tie
    xs = [_seg_closest(p, a, b), _seg_closest(p, b, c), _seg_closest(p, c, a)]
    ss = [_dot(p - x, p - x) for x in xs]
    x, s = xs[0], ss[0]
    for xi, si in zip(xs[1:], ss[1:]):
        better = si < s
        x, s = torch.where(better[..., None], xi, x), torch.where(better, si, s)
    # the regions in reverse order of the kernel's tests: a later assignment is an earlier test
    cases = [
        (denom > 0, _axpy(_axpy(a, _ratio(vb, denom), ab), _ratio(vc, denom), ac)),                 # interior
        ((va <= 0) & (e43 >= 0) & (e56 >= 0), _axpy(b, _ratio(e43, e43 + e56), c - b)),             # edge bc
        ((vb <= 0) & (d2 >= 0) & (d6 <= 0), _axpy(a, _ratio(d2, d2 - d6), ac)),                     # edge ac
        ((d6 >= 0) & (d5 <= d6), c),                                                                  # vertex c
        ((vc <= 0) & (d1 >= 0) & (d3 <= 0), _axpy(a, _ratio(d1, d1 - d3), ab)),                     # edge ab
        ((d3 >= 0) & (d4 <= d3), b),                                                                  # vertex b
        ((d1 <= 0) & (d2 <= 0), a),                                                                   # vertex a
    ]
    for cond, xc in cases:
        x = torch.where((cond & ~flat)[..., None], xc, x)
    return x


def usable_faces(verts, faces):
    """bool (F,): every index in [0, V) and every coordinate finite"""
    V = verts.shape[0]
    ok = ((faces >= 0) & (faces < V)).all(1)
    safe = torch.where(ok[:, None], faces, torch.zeros_like(faces))
    if V == 0:
        return torch.zeros(faces.shape[0], dtype=torch.bool, device=faces.device)
    return ok & torch.isfinite(verts[safe]).all(2).all(1)


def point_mesh_distance(points, verts, faces, chunk_elems=1 << 22):
    """Brute force over all faces -> (sq (P,) float64, face (P,) int64, closest (P,3) float64, second (P,) float64): the
    smallest squared distance and its face (ties to the smaller index), the closest point, and the second smallest
    distance over the other faces (inf with one face).  NaN / -1 / NaN / inf where a query is not finite or no face is
    usable.  points, verts float (any), faces integer (F,3); on the device of points."""
    dev = points.device
    p = points.to(torch.float64)
    v = verts.to(device=dev, dtype=torch.float64)
    f = faces.to(device=dev, dtype=torch.int64)
    P = p.shape[0]
    ok = usable_faces(v, f)
    fid = torch.nonzero(ok).flatten()
    best = torch.full((P,), float("inf"), dtype=torch.float64, device=dev)
    second = torch.full((P,), float("inf"), dtype=torch.float64, device=dev)
    bi = torch.full((P,), -1, dtype=torch.int64, device=dev)
    cl = torch.full((P, 3), float("nan"), dtype=torch.float64, device=dev)
    fin = torch.isfinite(p).all(1)
    if P and fid.numel():
        tri = v[f[fid]]                                            # (Fu, 3, 3)
        step = max(1, chunk_elems // max(P, 1))
        for s in range(0, fid.numel(), step):
            t = tri[s:s + step]
            x = closest_points(p[:, None, :], t[None, :, 0], t[None, :, 1], t[None, :, 2])     # (P, C, 3)
            r = p[:, None, :] - x
            d = _dot(r, r)
            k = min(2, d.shape[1])
            two = torch.topk(d, k, dim=1, largest=False).values
            dmin = two[:, 0]
            # the smallest face index among exact ties
            ar = torch.arange(d.shape[1], device=dev).expand_as(d)
            j = torch.where(d == dmin[:, None], ar, d.shape[1]).min(1).values
            jc = j.clamp(max=d.shape[1] - 1)
            xmin = x[torch.arange(P, device=dev), jc]
            nd2 = two[:, 1] if k > 1 else torch.full_like(dmin, float("inf"))
            better = dmin < best
            second = torch.where(better, torch.minimum(best, nd2), torch.minimum(second, dmin))
            best = torch.where(better, dmin, best)
            bi = torch.where(better, fid[s + jc], bi)
            cl = torch.where(better[:, None], xmin, cl)
    hit = fin & (bi >= 0)
    nan = torch.tensor(float("nan"), dtype=torch.float64, device=dev)
    return (torch.where(hit, best, nan), torch.where(hit, bi, -1), torch.where(hit[:, None], cl, nan),
            torch.where(hit, second, float("inf")))
