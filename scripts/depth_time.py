"""Time of one graphed training step with and without the dense depth term, at configs/dss.yml's settings: the bunny of
camera_refine_time.py (1 001 points), 512^2 views, K = 5, 8 views per batch, Vrk_invariant splats, learning points and
normals.  The ground-truth depth maps are the renders' own (render_points(..., depth=True) of the unshrunk bunny); both
steps are GraphedTrainStep.from_views on the same cloud and views, the second with lambda_dr_depth = 1.  The two are
alternated in rounds in one process, each round timing --steps replays of each between CUDA events; the median, min and
max per step and the median of the per-round differences are reported with the card's name and power limit.

The difference is what the term adds: the depth map launch, the depth loss (three launches) and the fixed-point depth
backward (three launches) with the z chain it feeds.

    python scripts/depth_time.py [--rounds 21] [--steps 20]
"""
import argparse
import json
import sys

import torch

from camera_refine_time import bunny_views
from timing import alternate, card, paired, spread
from dss_b200.ops import SplatParams, render_points
from dss_b200.training.step import GraphedTrainStep
from tests.util import camera_matrices, random_cameras


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=21)
    ap.add_argument("--steps", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("depth_time.py needs a CUDA device")
    dev = torch.device("cuda:0")
    V, B, S = 32, 8, 512
    prm = SplatParams(image_size=S, points_per_pixel=5, cutoff_threshold=1.0, depth_merging_threshold=0.05,
                      radii_backward_scaler=5.0, clip_pts_grad=0.05, znear=0.1)
    pts, nrm, data = bunny_views(dev, V, S, prm)
    proj, view = camera_matrices(random_cameras(V, 0))
    with torch.no_grad():
        depth = render_points(pts.to(dev), nrm.to(dev), torch.ones_like(pts).to(dev), proj.to(dev), view.to(dev),
                              torch.full((V,), 3e-4, device=dev), prm, depth=True).depth.cpu()
    data.depths = list(depth.numpy())
    views = data.device_views(dev)
    p, n, c = (0.97 * pts).to(dev), nrm.to(dev), torch.ones_like(pts).to(dev)
    kw = dict(Vrk_invariant=True, Vrk_isotropic=False, lambda_dr_proj=0.01, lambda_dr_repel=0.0)
    order = torch.randperm(V, generator=torch.Generator().manual_seed(1)).tolist()
    plain = GraphedTrainStep.from_views(p, n, c, prm, views, order[:B], **kw)
    with_depth = GraphedTrainStep.from_views(p, n, c, prm, views, order[:B], lambda_dr_depth=1.0, **kw)
    batches = [order[i:i + B] for i in range(0, V - B + 1, B)]
    state = {"k": 0}

    def run(step):
        def fn():
            step.load_views(batches[state["k"] % len(batches)])
            state["k"] += 1
            step.replay()
        return fn

    ms = alternate({"plain": run(plain), "depth": run(with_depth)}, a.rounds, a.steps, 10)
    gpu = card()
    res = {"card": gpu["name"], "power_limit": gpu["power_limit"], "points": int(p.shape[0]), "views": V, "batch": B,
           "image_size": S}
    for k, xs in ms.items():
        res[k + "_ms"] = dict(zip(("median", "min", "max"), spread(xs)))
    diff = paired(ms["plain"], ms["depth"])
    res["overhead_ms"] = dict(zip(("median", "min", "max"), spread(diff)))
    res["overhead_pct"] = 100.0 * res["overhead_ms"]["median"] / res["plain_ms"]["median"]
    print(json.dumps(res))


if __name__ == "__main__":
    sys.exit(main())
