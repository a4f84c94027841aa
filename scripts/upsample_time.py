"""Time upsampling (ops.upsample_points) on Poisson-disk samples of a torus, k = 16: 8 000 -> 100 000 points (27
rounds) and 100 000 -> 1 000 000; the whole call, the share of it spent in the per-round K-NN calls (the library's
profiled "knn" stage) and the launches per call; and outlier_ratio at both input sizes.  Then the quality of 2 000 ->
20 000 on the same torus: the new points' distance to the mesh, mean and max, relative to the input's mean
nearest-neighbour spacing, and the largest nearest-neighbour distance before and after (DESIGN.md §3)."""
import json

import torch
from meshes import torus
from timing import card, launches, median_ms, stage_ms

from dss_b200.frnn_grid import knn_points_packed
from dss_b200.ops import (outlier_ratio, point_mesh_distance, sample_points_poisson_disk, upsample_points,
                          upsample_schedule)

dev = torch.device("cuda:0")
K = 16
verts, faces = (t.to(dev) for t in torus())


def nn_dist(p):
    first = torch.zeros(1, dtype=torch.int64, device=dev)
    num = torch.full((1,), p.shape[0], dtype=torch.int64, device=dev)
    return knn_points_packed(p, first, num, 2, -1.0)[0][:, 1].sqrt()


res = {}
for P0, P1 in ((8_000, 100_000), (100_000, 1_000_000)):
    p = sample_points_poisson_disk(verts, faces, P0).points.contiguous()
    n = p.shape[0]
    call = lambda: upsample_points(p, P1, K)
    whole = median_ms(call, 2, 10)
    stages = stage_ms(call, 3, dev)
    knn = stages.get("knn", 0.0)
    res["%d->%d" % (n, P1)] = {"upsample_ms": whole, "knn_ms": knn, "knn_share": knn / whole,
                               "rounds": len(upsample_schedule([n], [P1], K)) - 1,
                               "launches": launches(call, dev),
                               "outlier_ratio_ms": median_ms(lambda: outlier_ratio(p, K), 3, 20)}
    print(n, P1, json.dumps(res["%d->%d" % (n, P1)]), flush=True)

s = sample_points_poisson_disk(verts, faces, 2000)
p, nrm = s.points.contiguous(), s.normals.contiguous()
up = upsample_points(p, 20_000, K, nrm)
spacing = float(nn_dist(p).mean())
d = point_mesh_distance(up.points[p.shape[0]:], verts, faces).sq_dists.double().sqrt()
d_in = point_mesh_distance(p, verts, faces).sq_dists.double().sqrt()
res["quality_2000_to_20000"] = {
    "input_points": p.shape[0], "mean_spacing": spacing,
    "new_mesh_dist_mean_rel": float(d.mean()) / spacing, "new_mesh_dist_max_rel": float(d.max()) / spacing,
    "input_mesh_dist_max_rel": float(d_in.max()) / spacing,
    "max_nn_before": float(nn_dist(p).max()), "max_nn_after": float(nn_dist(up.points).max()),
    "mean_nn_after": float(nn_dist(up.points).mean())}
print(json.dumps(res["quality_2000_to_20000"]), flush=True)
gpu = card()
res["card"], res["power_limit"], res["max_sm_clock"] = gpu["name"], gpu["power_limit"], gpu["max_sm_clock"]
print(json.dumps(res))
