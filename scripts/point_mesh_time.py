"""Time ops.point_mesh_distance (csrc/mesh_distance.cu) at 8k, 100k and 1M queries against the seeded 631k-face
displaced sphere of scripts/mesh_raster_time.py and a 5k-face torus (both in scripts/meshes.py), with queries on the
surface and spread through the bounding box; next to it a chunked float32 torch brute force where that finishes in
reasonable time.

    python scripts/point_mesh_time.py [--warmup 2] [--iters 5]

CUDA events around each call, median after warm-up.  "build_ms" is the call with a single query (the grid build and
its one host synchronisation, plus one query).  "tests" is the mean / max number of face distances a query evaluated.
Prints one JSON line per case, the card name and its power limit first."""
import argparse
import json

import torch

from timing import card, median_ms
from meshes import displaced_sphere, torus
from dss_b200.ops import point_mesh_distance
from dss_b200.utils.create_mvr_data import sample_points_from_mesh
from tests.point_mesh_oracle import closest_points


def brute_force(q, verts, faces, chunk=1 << 24):
    """float32 squared distance to the nearest face, chunked over queries x faces (the same Voronoi-region formula as
    the oracle, vectorised); for timing only"""
    tri = verts[faces]
    out = torch.full((q.shape[0],), float("inf"), device=q.device)
    step_q = max(1, min(q.shape[0], chunk // faces.shape[0]))
    step_f = max(1, chunk // step_q)
    for s in range(0, q.shape[0], step_q):
        qq = q[s:s + step_q, None, :]
        best = torch.full((qq.shape[0],), float("inf"), device=q.device)
        for fs in range(0, faces.shape[0], step_f):
            t = tri[None, fs:fs + step_f]
            x = closest_points(qq, t[..., 0, :], t[..., 1, :], t[..., 2, :])
            best = torch.minimum(best, ((qq - x) ** 2).sum(-1).min(1).values)
        out[s:s + step_q] = best
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--brute-max", type=float, default=6e9, help="largest queries x faces for the brute force")
    opt = ap.parse_args()
    dev = torch.device("cuda:0")
    gpu = card()
    print(json.dumps({"card": gpu["name"], "power_limit": gpu["power_limit"]}), flush=True)
    for mesh_name, (v, f) in (("displaced_sphere", displaced_sphere()), ("torus", torus())):
        v, f = v.to(dev), f.to(dev)
        lo, hi = v.min(0).values, v.max(0).values
        g = torch.Generator(device=dev).manual_seed(0)
        pools = {"surface": sample_points_from_mesh(v, f, 1_000_000, generator=g)[0],
                 "box": lo + (hi - lo) * torch.rand(1_000_000, 3, device=dev, generator=g)}
        build = median_ms(lambda: point_mesh_distance(pools["surface"][:1], v, f), opt.warmup, opt.iters)
        for kind, pool in pools.items():
            for n in (8_000, 100_000, 1_000_000):
                q = pool[:n].contiguous()
                res = {"mesh": mesh_name, "faces": int(f.shape[0]), "queries": kind, "P": n, "build_ms": build}
                res["ms"] = median_ms(lambda: point_mesh_distance(q, v, f), opt.warmup, opt.iters)
                tests = torch.empty(n, dtype=torch.int32, device=dev)
                r = point_mesh_distance(q, v, f, _face_tests=tests)
                res["tests_mean"], res["tests_max"] = float(tests.double().mean()), int(tests.max())
                if n * f.shape[0] <= opt.brute_max:
                    keep = {}
                    res["brute_ms"] = median_ms(lambda: keep.update(bf=brute_force(q, v, f)), 0, 1)
                    bf = keep["bf"]
                    res["brute_max_rel_diff"] = float(((bf - r.sq_dists).abs() / r.sq_dists.clamp(min=1e-12)).max())
                print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
