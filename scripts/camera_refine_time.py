"""Time of one graphed training step with and without camera refinement, at configs/dss.yml's settings: the bunny of
tests/golden/ply/bunny-8000.ply (1 001 points), 512^2 views, K = 5, 8 views per batch, Vrk_invariant splats, learning points and normals.
The views are 32 renders of the bunny from the test suite's random cameras, resident on the device as the loop holds
them (DeviceViews); both steps are GraphedTrainStep.from_views on the same cloud and views, and the refined one also
learns one pose per view (zero poses: the same images, filters and cloud gradients).  The two are alternated in
rounds in one process, each round timing --steps replays of each between CUDA events; the median, min and max per
step and the median of the per-round differences are reported with the card's name and power limit.

The difference is what refinement adds: the camera backward (its (P,3) NDC gradient and per-view partial sums), the
camera-centre chain of the shading, and the two pose launches.

    python scripts/camera_refine_time.py [--rounds 21] [--steps 20]
"""
import argparse
import json
import os
import sys
import tempfile

import numpy as np
import torch

from timing import alternate, card, paired, spread
from dss_b200.core.lighting import DirectionalLights
from dss_b200.ops import SplatParams, render_points
from dss_b200.training.step import GraphedTrainStep
from dss_b200.utils.dataset import MVRData
from dss_b200.utils.io import read_ply
from tests.util import GOLDEN_DIR, camera_matrices, random_cameras


def bunny_views(dev, V, S, prm):
    """an MVRData of V renders of the bunny (mask: alpha > 0) with per-view directional lights"""
    ply = read_ply(os.path.join(GOLDEN_DIR, "ply", "bunny-8000.ply"))
    pts, nrm = (torch.as_tensor(ply[k], dtype=torch.float32) for k in ("points", "normals"))
    pts = pts - pts.mean(0)
    pts = pts / pts.norm(dim=1).max()
    cams = random_cameras(V, 0)
    proj, view = camera_matrices(cams)
    g = torch.Generator().manual_seed(0)
    light = {"ambient_color": 0.3 * torch.ones(V, 1, 1, 3),
             "diffuse_color": 0.6 * torch.rand(V, 1, 1, 3, generator=g),
             "specular_color": 0.1 * torch.ones(V, 1, 1, 3), "direction": torch.randn(V, 1, 1, 3, generator=g)}
    with torch.no_grad():
        out = render_points(pts.to(dev), nrm.to(dev), torch.ones_like(pts).to(dev), proj.to(dev), view.to(dev),
                            torch.full((V,), 3e-4, device=dev), prm).image.cpu()
    d = {"camera_mat": view.numpy(), "cameras_params": {"znear": 0.1}, "lights_type": "DirectionalLights"}
    for i in range(V):
        d["lights_%d" % i] = {k: t[i].numpy() for k, t in light.items()}
    path = os.path.join(tempfile.mkdtemp(prefix="dss_camera_time_"), "data_dict.npz")
    np.savez(path, **d)
    images = [out[i, :, :, :3].permute(2, 0, 1).contiguous() for i in range(V)]
    masks = [(out[i, :, :, 3] > 0).float()[None] for i in range(V)]
    return pts, nrm, MVRData(path, images=images, masks=masks)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=21)
    ap.add_argument("--steps", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("camera_refine_time.py needs a CUDA device")
    dev = torch.device("cuda:0")
    V, B, S = 32, 8, 512
    prm = SplatParams(image_size=S, points_per_pixel=5, cutoff_threshold=1.0, depth_merging_threshold=0.05,
                      radii_backward_scaler=5.0, clip_pts_grad=0.05, znear=0.1)
    pts, nrm, data = bunny_views(dev, V, S, prm)
    views = data.device_views(dev)
    # the cloud trained: the bunny shrunk a little, so that the images and the cloud disagree
    p, n, c = (0.97 * pts).to(dev), nrm.to(dev), torch.ones_like(pts).to(dev)
    kw = dict(Vrk_invariant=True, Vrk_isotropic=False, lambda_dr_proj=0.01, lambda_dr_repel=0.0)
    order = torch.randperm(V, generator=torch.Generator().manual_seed(1)).tolist()
    plain = GraphedTrainStep.from_views(p, n, c, prm, views, order[:B], **kw)
    refined = GraphedTrainStep.from_views(p, n, c, prm, views, order[:B], poses=torch.zeros(V, 6, device=dev), **kw)
    batches = [order[i:i + B] for i in range(0, V - B + 1, B)]
    state = {"k": 0}

    def run(step):
        def fn():
            step.load_views(batches[state["k"] % len(batches)])
            state["k"] += 1
            step.replay()
        return fn

    ms = alternate({"plain": run(plain), "refined": run(refined)}, a.rounds, a.steps, 10)
    gpu = card()
    res = {"card": gpu["name"], "power_limit": gpu["power_limit"], "points": int(p.shape[0]), "views": V, "batch": B,
           "image_size": S}
    for k, xs in ms.items():
        res[k + "_ms"] = dict(zip(("median", "min", "max"), spread(xs)))
    diff = paired(ms["plain"], ms["refined"])
    res["overhead_ms"] = dict(zip(("median", "min", "max"), spread(diff)))
    res["overhead_pct"] = 100.0 * res["overhead_ms"]["median"] / res["plain_ms"]["median"]
    print(json.dumps(res))


if __name__ == "__main__":
    sys.exit(main())
