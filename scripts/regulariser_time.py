"""Step time of the point regularisers (ProjectionLoss, RepulsionLoss) with knn_k = 12, as the trainer runs them
(rebuilt every iteration): forward + backward of reduction="mean", the K-NN search included, on noisy spheres of
P = 5 000 (configs/dss.yml), 100 000 and 1 000 000 points.  Two routes, alternated in one process and timed with CUDA
events:
  torch -- the torch body (`torch_body`) in float32 on CUDA, K-NN from frnn_grid.knn_points on the padded cloud
  fused -- the loss module's CUDA route: knn_points_packed + dss_surface_regulariser

    python scripts/regulariser_time.py [--rounds 7] [--steps 10]
"""
import argparse
import sys

import torch

from timing import alternate, card, spread
from dss_b200.core.cloud import PointClouds3D, PointCloudsFilters
from dss_b200.training.losses import ProjectionLoss, RepulsionLoss
from tests.util import sphere_cloud


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

    variants = [(r, k, P) for P in cases for k in ("projection", "repulsion") for r in ("torch", "fused")]
    ms = alternate({v: lambda v=v: step(*v) for v in variants}, a.rounds, a.steps, 2)
    print("gpu: %(name)s, %(power_limit)s, %(max_sm_clock)s" % card())
    for v in variants:
        print("P=%-8d %-10s %-5s step ms: median %.3f  (min %.3f max %.3f)" % (v[2], v[1], v[0], *spread(ms[v])))
    for P in cases:
        for k in ("projection", "repulsion"):
            r = [t / f for t, f in zip(ms[("torch", k, P)], ms[("fused", k, P)])]
            print("P=%-8d %-10s torch / fused: median %.1fx  (min %.1f max %.1f)" % (P, k, *spread(r)))


if __name__ == "__main__":
    main()
