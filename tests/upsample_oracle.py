"""Host oracle of dss_upsample_points and dss_outlier_ratio (csrc/upsample.cu, csrc/normals.cu; the rules are in
include/dss_b200.h and DESIGN.md), restated from those rules in numpy.

* ``schedule``: the sizes before every round and after the last.
* ``neighbours``: a K-NN row at K = k + 1 less the point's own index (less its last entry when the index is absent).
* ``upsample_round``: one round from given neighbour rows, in float32 with every operation rounded as the device does,
  so that from the device's own K-NN rows it gives the device's new points, normals, features and parents bit for bit.
* ``upsample``: every round of one cloud from ``knn_rows`` (a brute-force search ordered by (distance, index)).
* ``outlier_ratio``: l0 / (l0 + l1 + l2) of the population covariance of each neighbour row, with the eigenvalues from
  the closed-form (trigonometric) solution of the characteristic cubic in float64.
"""
import numpy as np

F2, F3 = np.float32(2.0), np.float32(3.0)


def schedule(num_points, targets, k):
    """list of R + 1 lists of sizes: each round adds min(n - c, c // 10) to every cloud below its target"""
    c, n = [int(x) for x in num_points], [int(x) for x in targets]
    for ci, ni in zip(c, n):
        if ni < ci:
            raise ValueError("target below the cloud's size")
        if ni > ci and (ci <= k or ci < 10):
            raise ValueError("a cloud that grows needs more than k and at least 10 points")
    out = [c]
    while any(ci < ni for ci, ni in zip(c, n)):
        c = [ci + min(ni - ci, ci // 10) for ci, ni in zip(c, n)]
        out.append(c)
    return out


def knn_rows(points, K, chunk=2048):
    """(P,K) int32: every point's K nearest points of the cloud (itself included), ascending by (squared distance in
    float64, index)"""
    p = np.asarray(points, np.float64)
    P = p.shape[0]
    out = np.empty((P, K), np.int32)
    for a in range(0, P, chunk):
        d2 = ((p[a:a + chunk, None, :] - p[None, :, :]) ** 2).sum(-1)
        part = np.argpartition(d2, K, axis=1)[:, :K + 1] if P > K + 1 else np.tile(np.arange(P), (d2.shape[0], 1))
        dd = np.take_along_axis(d2, part, 1)
        order = np.lexsort((part, dd), axis=1)[:, :K]
        out[a:a + chunk] = np.take_along_axis(part, order, 1)
    return out


def neighbours(rows):
    """(c, k) from K-NN rows (c, k + 1): the row less its own index, or less its last entry"""
    rows = np.asarray(rows)
    c, K = rows.shape
    own = rows == np.arange(c)[:, None]
    drop = np.where(own.any(1), own.argmax(1), K - 1)
    keep = np.ones_like(own)
    keep[np.arange(c), drop] = False
    return rows[keep].reshape(c, K - 1)


def normalize(v):
    v = np.asarray(v, np.float32)
    ln = np.sqrt((v[..., 0] * v[..., 0] + v[..., 1] * v[..., 1]) + v[..., 2] * v[..., 2])
    return v / ln[..., None]


def sparsity(points, nb, chunk=4096):
    """(s (c,) float32, j* (c,) int) of every row with neighbours nb (c, k), and the candidates (c, k, 3)"""
    p = np.asarray(points, np.float32)
    c, k = nb.shape
    cand = (p[nb] + F2 * p[:, None, :]) / F3                        # (c,k,3)
    s = np.empty(c, np.float32)
    js = np.empty(c, np.int64)
    for a in range(0, c, chunk):
        q = p[nb[a:a + chunk]]                                      # (b,k,3)
        d = cand[a:a + chunk, :, None, :] - q[:, None, :, :]         # (b,j,l,3)
        dist = np.sqrt((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]).min(-1)   # (b,j)
        js[a:a + chunk] = dist.argmax(1)                            # the first j of the largest
        s[a:a + chunk] = dist.max(1)
    return s, js, cand


def upsample_round(points, rows, m, normals=None, features=None):
    """One round of a cloud of c = len(points) points from its K-NN rows (c, k + 1): the m new points, normals,
    features (None without input ones) and parents (m, 2), in the order of the parents' indices"""
    nb = neighbours(rows)
    s, js, cand = sparsity(points, nb)
    c = len(s)
    par = np.sort(np.lexsort((np.arange(c), -s))[:m])             # (s desc, i asc), then by index
    jn = nb[par, js[par]]
    new_p = cand[par, js[par]]
    new_n = new_f = None
    if normals is not None:
        nrm = np.asarray(normals, np.float32)
        new_n = normalize(F2 * normalize(nrm[par]) + normalize(nrm[jn]))
    if features is not None:
        f = np.asarray(features, np.float32)
        new_f = (f[jn] + F2 * f[par]) / F3
    return new_p, new_n, new_f, np.stack([par, jn], 1).astype(np.int32)


def upsample(points, n, k=16, normals=None, features=None, knn=knn_rows):
    """every round of one cloud: (points, normals, features, parents (M,2), sizes per round)"""
    p = np.asarray(points, np.float32)
    if not np.isfinite(p).all():
        raise ValueError("non-finite coordinates")
    sizes = [s[0] for s in schedule([len(p)], [n], k)]
    nrm = None if normals is None else np.asarray(normals, np.float32)
    ftr = None if features is None else np.asarray(features, np.float32)
    par = np.full((len(p), 2), -1, np.int32)
    for c, c1 in zip(sizes[:-1], sizes[1:]):
        new_p, new_n, new_f, new_par = upsample_round(p, knn(p, k + 1), c1 - c, nrm, ftr)
        p = np.concatenate([p, new_p])
        nrm = None if nrm is None else np.concatenate([nrm, new_n])
        ftr = None if ftr is None else np.concatenate([ftr, new_f])
        par = np.concatenate([par, new_par])
    return p, nrm, ftr, par, sizes


def sym3_eigvals(A):
    """ascending eigenvalues (..., 3) of symmetric (..., 3, 3) float64 matrices, closed form (Smith 1961)"""
    A = np.asarray(A, np.float64)
    q = np.trace(A, axis1=-2, axis2=-1) / 3.0
    p1 = A[..., 0, 1] ** 2 + A[..., 0, 2] ** 2 + A[..., 1, 2] ** 2
    B = A - q[..., None, None] * np.eye(3)
    p2 = (B[..., 0, 0] ** 2 + B[..., 1, 1] ** 2 + B[..., 2, 2] ** 2) + 2.0 * p1
    p = np.sqrt(p2 / 6.0)
    safe = np.where(p > 0, p, 1.0)
    r = np.clip(np.linalg.det(B / safe[..., None, None]) / 2.0, -1.0, 1.0)
    phi = np.arccos(r) / 3.0
    l2 = q + 2.0 * p * np.cos(phi)
    l0 = q + 2.0 * p * np.cos(phi + 2.0 * np.pi / 3.0)
    l1 = 3.0 * q - l0 - l2
    return np.stack([l0, l1, l2], -1)


def outlier_ratio(points, idx, tolerance=0.05):
    """(ratio (P,) float64, keep (P,) bool) over the neighbour rows idx (P,k); a row with a -1 neighbour is NaN"""
    pts = np.asarray(points, np.float64)
    ratio = np.full(len(idx), np.nan)
    ok = (idx >= 0).all(1)
    if ok.any():
        q = pts[idx[ok]]
        d = q - q.mean(1, keepdims=True)
        lam = sym3_eigvals(np.einsum("mki,mkj->mij", d, d) / idx.shape[1])
        with np.errstate(invalid="ignore", divide="ignore"):
            ratio[ok] = lam[:, 0] / ((lam[:, 0] + lam[:, 1]) + lam[:, 2])
    with np.errstate(invalid="ignore"):
        keep = ratio < tolerance
    return ratio, keep
