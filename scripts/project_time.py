"""Time the RIMLS projection (ops.project_to_surface) and the normal denoising (ops.denoise_normals) on noisy
Poisson-disk samples of a torus, k = 31, at 100k and 1M points: the whole call, the K-NN inside it (the library's
profiled "knn" stage), and the mean and max distance to the torus mesh before and after.  The noise moves each sample
along its normal by N(0, sigma^2) with sigma half the samples' mean nearest-neighbour spacing.  Then the upsample ->
project pipeline on the torus of DESIGN.md §3: 2 000 samples grown to 20 000 (k = 16) and projected (k = 31), with the
new points' and the input points' distance to the mesh relative to the input's spacing (DESIGN.md §3, §6)."""
import json

import torch
from meshes import torus
from timing import card, median_ms, stage_ms

from dss_b200.frnn_grid import knn_points_packed
from dss_b200.ops import (denoise_normals, point_mesh_distance, project_to_surface, sample_points_poisson_disk,
                          upsample_points)

dev = torch.device("cuda:0")
K = 31
verts, faces = (t.to(dev) for t in torus())


def nn_dist(p):
    first = torch.zeros(1, dtype=torch.int64, device=dev)
    num = torch.full((1,), p.shape[0], dtype=torch.int64, device=dev)
    return knn_points_packed(p, first, num, 2, -1.0)[0][:, 1].sqrt()


def mesh_dist(p):
    d = point_mesh_distance(p, verts, faces).sq_dists.double().sqrt()
    return {"mean": float(d.mean()), "max": float(d.max())}


res = {}
for n in (100_000, 1_000_000):
    s = sample_points_poisson_disk(verts, faces, n)
    spacing = float(nn_dist(s.points.contiguous()).mean())
    g = torch.Generator().manual_seed(0)
    noise = (0.5 * spacing * torch.randn((s.points.shape[0], 1), generator=g)).to(dev)
    p, nrm = (s.points + noise * s.normals).contiguous(), s.normals.contiguous()
    call = lambda: project_to_surface(p, nrm, K)
    whole = median_ms(call, 2, 10)
    knn = stage_ms(call, 3, dev).get("knn", 0.0)
    out = call()
    r = {"points": p.shape[0], "spacing": spacing, "sigma": 0.5 * spacing, "project_ms": whole, "knn_ms": knn,
         "knn_share": knn / whole, "denoise_ms": median_ms(lambda: denoise_normals(p, nrm), 2, 10),
         "iterations": torch.bincount(out.iterations.long()).tolist(),
         "dist_before": mesh_dist(p), "dist_after": mesh_dist(out.points)}
    r["mean_dist_factor"] = r["dist_before"]["mean"] / r["dist_after"]["mean"]
    res[str(n)] = r
    print(n, json.dumps(r), flush=True)

s = sample_points_poisson_disk(verts, faces, 2000)
p, nrm = s.points.contiguous(), s.normals.contiguous()
P = p.shape[0]
spacing = float(nn_dist(p).mean())
up = upsample_points(p, 20_000, 16, nrm)
out = project_to_surface(up.points, up.normals, K)
rel = lambda d: {k: v / spacing for k, v in d.items()}
res["upsample_then_project_2000_to_20000"] = {
    "input_points": P, "mean_spacing": spacing,
    "new_before_rel": rel(mesh_dist(up.points[P:])), "new_after_rel": rel(mesh_dist(out.points[P:])),
    "input_after_rel": rel(mesh_dist(out.points[:P]))}
print(json.dumps(res["upsample_then_project_2000_to_20000"]), flush=True)
gpu = card()
res["card"], res["power_limit"], res["max_sm_clock"] = gpu["name"], gpu["power_limit"], gpu["max_sm_clock"]
print(json.dumps(res))
