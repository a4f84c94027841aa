"""Time ops.sample_points_poisson_disk (csrc/mesh_sample.cu) at N = 8000, 10000 and 100000 on ico_sphere(6) (82k
faces), ico_sphere(8) (1.3M faces) and the 5k-face torus of point_mesh_time.py, Euclidean and geodesic.

    python scripts/poisson_disk_time.py [--warmup 1] [--iters 3] [--out FILE]

Per case: the whole call (median of CUDA-event times after warm-up; the call synchronises the host itself), and from
the last call the stage times the library reports (pool build, radius search, a final selection when the returned
probe was not the last, output), the number of probes and each probe's radius, count and selection rounds.  Prints
one JSON line per case, the card name and its power limit first; --out also writes them to FILE."""
import argparse
import json
import os

import torch

from timing import card, median_ms
from meshes import torus
from dss_b200.ops import poisson_disk_stats, sample_points_poisson_disk
from dss_b200.utils.create_mvr_data import ico_sphere


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--out", default=None)
    opt = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    dev = torch.device("cuda:0")
    gpu = card()
    lines = [{"card": gpu["name"], "power_limit": gpu["power_limit"]}]
    print(json.dumps(lines[0]), flush=True)
    meshes = {"ico_sphere(6)": ico_sphere(6), "ico_sphere(8)": ico_sphere(8), "torus": torus()}
    for mesh, (v, f) in meshes.items():
        v, f = v.to(dev), f.to(dev)
        for geodesic in (False, True):
            for N in (8000, 10000, 100000):
                out = {}

                def call():
                    out["s"] = sample_points_poisson_disk(v, f, N, geodesic=geodesic)
                ms = median_ms(call, opt.warmup, opt.iters)
                st = poisson_disk_stats()
                rec = {"mesh": mesh, "faces": int(f.shape[0]), "geodesic": geodesic, "N": N,
                       "samples": int(out["s"].points.shape[0]), "radius": out["s"].radius, "call_ms": round(ms, 3),
                       "stage_ms": dict(zip(("pool", "search", "reselect", "output"),
                                            [round(x, 3) for x in st["stage_ms"]])),
                       "probes": st["probes"], "rounds": st["rounds"], "counts": st["counts"],
                       "radii": st["radii"]}
                lines.append(rec)
                print(json.dumps(rec), flush=True)
    if opt.out:
        os.makedirs(os.path.dirname(os.path.abspath(opt.out)), exist_ok=True)
        with open(opt.out, "w") as fh:
            fh.write("\n".join(json.dumps(x) for x in lines) + "\n")


if __name__ == "__main__":
    main()
