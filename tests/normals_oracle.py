"""Host oracle of dss_estimate_normals (csrc/normals.cu; the rules are in include/dss_b200.h and DESIGN.md).

* ``pca_normals``: float64 PCA with numpy.linalg.eigh over given neighbour rows, the canonical sign.
* ``orient``: given the unoriented float32 normals and the neighbour rows, the float32 weights and the key
  (w, min(i,j), max(i,j)) exactly as the device forms them, Kruskal with union-find on that key, the max-z roots and a
  breadth-first propagation of the signs from them.  It reproduces the device's forest, roots and oriented normals bit
  for bit from the device's unoriented normals.
"""
from collections import deque

import numpy as np


def knn_rows(points, k):
    """(P,k) int32 indices of every point's k nearest points (itself included), by cKDTree; -1 where the cloud is
    smaller than k or the point is non-finite (ties may be ordered differently from the device's search)"""
    from scipy.spatial import cKDTree
    pts = np.asarray(points, np.float64)
    P = pts.shape[0]
    out = np.full((P, k), -1, np.int32)
    ok = np.isfinite(pts).all(1)
    if ok.sum() >= k:
        good = np.nonzero(ok)[0]
        _, idx = cKDTree(pts[good]).query(pts[good], k=k)
        out[good] = good[idx.reshape(len(good), k)]
    return out


def canonical(n):
    """the sign rule without orientation: the component of largest |n_k| (the first such axis) positive"""
    n = np.array(n, np.float32, copy=True)
    axis = np.argmax(np.abs(n), 1)                    # argmax takes the first of equal values
    big = n[np.arange(n.shape[0]), axis]
    n[big < 0] *= -1
    return n


def pca_normals(points, idx):
    """(P,3) float32 canonical PCA normals in float64 over the neighbour rows ``idx`` (-1: the row is NaN), and (P,3)
    float64 eigenvalues in ascending order"""
    pts = np.asarray(points, np.float64)
    P = pts.shape[0]
    n = np.full((P, 3), np.nan, np.float32)
    lam = np.full((P, 3), np.nan)
    ok = (idx >= 0).all(1)
    if ok.any():
        q = pts[idx[ok]]                                  # (M,k,3)
        d = q - q.mean(1, keepdims=True)
        cov = np.einsum("mki,mkj->mij", d, d) / idx.shape[1]
        w, v = np.linalg.eigh(cov)
        lam[ok] = w
        n[ok] = v[:, :, 0].astype(np.float32)
    n[ok] = canonical(n[ok])
    return n, lam


def dot32(a, b):
    """n_a . n_b in float32, each product and sum rounded, in the order x, y, z (no FMA)"""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def graph_edges(normals, idx):
    """(lo, hi, w) of the undirected k-NN graph over the valid rows (a finite normal and a full neighbour row), each
    edge once, sorted by the key (w, lo, hi); w float32"""
    n = np.asarray(normals, np.float32)
    valid = np.isfinite(n).all(1) & (idx >= 0).all(1)
    rows = np.repeat(np.arange(idx.shape[0]), idx.shape[1])
    cols = idx.reshape(-1).astype(np.int64)
    keep = valid[rows] & (cols >= 0) & (cols != rows)
    rows, cols = rows[keep], cols[keep]
    keep = valid[cols]
    rows, cols = rows[keep], cols[keep]
    lo, hi = np.minimum(rows, cols), np.maximum(rows, cols)
    pairs = np.unique(np.stack([lo, hi], 1), axis=0)
    lo, hi = pairs[:, 0], pairs[:, 1]
    w = (np.float32(1) - np.abs(dot32(n[lo], n[hi]))).astype(np.float32)
    order = np.lexsort((hi, lo, w))
    return lo[order], hi[order], w[order]


def kruskal(P, lo, hi):
    """the edges (positions into lo / hi) Kruskal keeps, taking them in the given order"""
    up = np.arange(P)

    def find(x):
        while up[x] != x:
            up[x] = up[up[x]]
            x = up[x]
        return x

    kept = []
    for e in range(len(lo)):
        a, b = find(lo[e]), find(hi[e])
        if a != b:
            up[max(a, b)] = min(a, b)
            kept.append(e)
    return np.asarray(kept, np.int64)


def orient(points, normals, idx):
    """dict(normals (P,3) f32 oriented, root (P,) int32, parent (P,) int32, edges (E,2) the forest, weight float64
    the forest's total weight) from the unoriented ``normals`` (canonical, NaN on invalid rows) and the neighbour rows
    ``idx`` of one cloud"""
    pts = np.asarray(points, np.float32)
    n = np.asarray(normals, np.float32)
    P = n.shape[0]
    valid = np.isfinite(n).all(1) & (idx >= 0).all(1)
    lo, hi, w = graph_edges(n, idx)
    kept = kruskal(P, lo, hi)
    adj = [[] for _ in range(P)]
    for e in kept:
        adj[lo[e]].append(hi[e])
        adj[hi[e]].append(lo[e])
    root = np.full(P, -1, np.int32)
    parent = np.full(P, -1, np.int32)
    out = n.copy()
    # components in order of their root: largest z, then smallest index
    order = sorted(np.nonzero(valid)[0], key=lambda i: (-float(pts[i, 2]), i))
    for r in order:
        if root[r] >= 0:
            continue
        root[r] = r
        if out[r, 2] < 0:
            out[r] = -out[r]
        todo = deque([r])
        while todo:
            u = todo.popleft()
            for v in adj[u]:
                if root[v] < 0:
                    root[v], parent[v] = r, u
                    if dot32(out[v], out[u]) < 0:
                        out[v] = -out[v]
                    todo.append(v)
    edges = np.stack([lo[kept], hi[kept]], 1) if len(kept) else np.zeros((0, 2), np.int64)
    return {"normals": out, "root": root, "parent": parent, "edges": edges,
            "weight": float(np.sum(w[kept].astype(np.float64))) if len(kept) else 0.0}


def parent_edges(parent):
    """the undirected edge set {(min, max)} of a parent array"""
    c = np.nonzero(np.asarray(parent) >= 0)[0]
    p = np.asarray(parent)[c]
    return {(int(min(a, b)), int(max(a, b))) for a, b in zip(c, p)}
