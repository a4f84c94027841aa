"""Time normal estimation (ops.estimate_normals) on a unit sphere of P = 100k and 1M points, k = 20: the K-NN, the PCA
(dss_estimate_normals without orientation), the forest and signs (the oriented call less the PCA), and the whole call,
with the launches per call and the loop lengths; next to a scipy CPU path (cKDTree, eigh, csgraph's minimum spanning
tree) at 100k for context."""
import json
import time

import numpy as np
import torch
from timing import card, launches, median_ms

from dss_b200 import _lib
from dss_b200.frnn_grid import knn_points_packed
from dss_b200.ops import estimate_normals

dev = torch.device("cuda:0")
K = 20


def sphere(P, seed=0):
    p = np.random.default_rng(seed).normal(size=(P, 3))
    return (p / np.linalg.norm(p, axis=1, keepdims=True)).astype(np.float32)


def scipy_path(p):
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import minimum_spanning_tree
    from scipy.spatial import cKDTree
    t0 = time.perf_counter()
    _, idx = cKDTree(p).query(p, k=K)
    t1 = time.perf_counter()
    q = p[idx].astype(np.float64)
    d = q - q.mean(1, keepdims=True)
    n = np.linalg.eigh(np.einsum("pki,pkj->pij", d, d) / K)[1][:, :, 0]
    t2 = time.perf_counter()
    rows = np.repeat(np.arange(len(p)), K - 1)
    cols = idx[:, 1:].reshape(-1)
    w = 1.0 - np.abs(np.sum(n[rows] * n[cols], 1)) + 1.0
    minimum_spanning_tree(coo_matrix((w, (rows, cols)), shape=(len(p), len(p))).tocsr())
    t3 = time.perf_counter()
    return {"knn_s": t1 - t0, "pca_s": t2 - t1, "mst_s": t3 - t2, "total_s": t3 - t0}


res = {}
for P in (100_000, 1_000_000):
    pts = torch.from_numpy(sphere(P)).to(dev)
    first = torch.zeros(1, dtype=torch.int64, device=dev)
    num = torch.full((1,), P, dtype=torch.int64, device=dev)
    idx = knn_points_packed(pts, first, num, K, -1.0)[1]
    out = (torch.empty((P, 3), device=dev), torch.empty(P, dtype=torch.int32, device=dev),
           torch.empty(P, dtype=torch.int32, device=dev))
    lib = lambda orient: _lib.call("dss_estimate_normals", dev, pts, first, num, 1, P, idx, K, orient, *out)
    knn_ms = median_ms(lambda: knn_points_packed(pts, first, num, K, -1.0), 3, 20)
    pca_ms = median_ms(lambda: lib(0), 3, 20)
    oriented_ms = median_ms(lambda: lib(1), 3, 20)
    whole_ms = median_ms(lambda: estimate_normals(pts, K), 3, 20)
    est = estimate_normals(pts, K)
    loop = int(np.ceil(np.log2(P))) + 1
    res[P] = {"knn_ms": knn_ms, "pca_ms": pca_ms, "forest_and_signs_ms": oriented_ms - pca_ms,
              "estimate_normals_ms": whole_ms, "launches_oriented": launches(lambda: lib(1), dev),
              "boruvka_rounds_launched": loop, "jumps_per_round_launched": loop,
              "components": int(torch.unique(est.root).numel()),
              "outward": float((torch.sum(est.normals * pts, 1) > 0).float().mean())}
    if P == 100_000:
        res[P]["scipy_cpu"] = scipy_path(pts.cpu().numpy())
    print(P, json.dumps(res[P]), flush=True)
gpu = card()
res["card"], res["power_limit"], res["max_sm_clock"] = gpu["name"], gpu["power_limit"], gpu["max_sm_clock"]
print(json.dumps(res))
