"""Step time of the point regularisers (ProjectionLoss, RepulsionLoss) with knn_k = 12, as the trainer runs them
(rebuilt every iteration): forward + backward of reduction="mean", the K-NN search included, on noisy spheres of
P = 5 000 (configs/dss.yml), 100 000 and 1 000 000 points.  Two routes, alternated in one process and timed with CUDA
events:
  torch -- the torch body (`torch_body`) in float32 on CUDA, K-NN from frnn_grid.knn_points on the padded cloud
  fused -- the loss module's CUDA route: knn_points_packed + dss_surface_regulariser

    python scripts/regulariser_time.py [--rounds 7] [--steps 10]
"""
import argparse
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dss_b200.core.cloud import PointClouds3D, PointCloudsFilters  # noqa: E402
from dss_b200.training.losses import ProjectionLoss, RepulsionLoss  # noqa: E402
from tests.util import sphere_cloud  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--sizes", default="5000,100000,1000000")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("regulariser_time.py needs a CUDA device")
    dev = torch.device("cuda:0")
    cases = {}
    for P in [int(s) for s in a.sizes.split(",")]:
        pts, nrm, _ = sphere_cloud(P, seed=3)
        g = torch.Generator().manual_seed(P)
        pts = (pts + 0.002 * torch.randn(P, 3, generator=g)).to(dev).requires_grad_(True)
        nrm = torch.nn.functional.normalize(nrm + 0.2 * torch.randn(P, 3, generator=g), dim=1).to(dev)
        vis = (torch.rand(1, P, generator=g) < 0.6).to(dev)
        filt = PointCloudsFilters(device=dev, visibility=vis, inmask=torch.ones_like(vis))
        cases[P] = (pts, nrm, filt)

    def step(route, kind, P):
        pts, nrm, filt = cases[P]
        pts.grad = None
        cloud = PointClouds3D([pts], normals=[nrm])
        loss = (ProjectionLoss if kind == "projection" else RepulsionLoss)(reduction="mean", knn_k=12)
        if route == "torch":
            out = loss.torch_body(cloud, points_filter=filt, rebuild_knn=True).mean()
        else:
            out = loss(cloud, points_filter=filt, rebuild_knn=True)
        out.backward()

    def timed(v, n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            step(*v)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    variants = [(r, k, P) for P in cases for k in ("projection", "repulsion") for r in ("torch", "fused")]
    for v in variants:
        timed(v, 2)                                     # warm-up of every variant
    ms = {v: [] for v in variants}
    for _ in range(a.rounds):
        for v in variants:
            ms[v].append(timed(v, a.steps))
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print("gpu: %s" % (smi or "not measured"))
    for v in variants:
        print("P=%-8d %-10s %-5s step ms: median %.3f  (min %.3f max %.3f)"
              % (v[2], v[1], v[0], statistics.median(ms[v]), min(ms[v]), max(ms[v])))
    for P in cases:
        for k in ("projection", "repulsion"):
            r = [t / f for t, f in zip(ms[("torch", k, P)], ms[("fused", k, P)])]
            print("P=%-8d %-10s torch / fused: median %.1fx  (min %.1f max %.1f)"
                  % (P, k, statistics.median(r), min(r), max(r)))


if __name__ == "__main__":
    main()
