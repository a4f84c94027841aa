"""Extra step time of camera gradients at the bench.py headline configuration (1M points x 8 views, 512x512, K=5):
eager forward+backward steps with and without proj / view requiring grad, alternated in one process, timed with CUDA
events; plus the per-stage device time of the camera kernels and of the chain kernel (which writes grad_ndc when
camera gradients are asked for).

    python scripts/camera_grad_time.py [--rounds 10] [--steps 20]
"""
import argparse

import torch

from timing import alternate, card, paired, spread, stage_ms
from dss_b200.core.camera import camera_matrices
from dss_b200.ops import SplatParams, render_points
from tests.util import random_cameras, sphere_cloud


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--steps", type=int, default=20)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    P0, S, K, V = 1_000_000, 512, 5, 8
    prm = SplatParams(image_size=S, points_per_pixel=K, cutoff_threshold=1.0, depth_merging_threshold=0.05,
                      antialiasing_sigma=1.0, radii_backward_scaler=5.0, clip_pts_grad=0.05,
                      backface_culling=False, znear=0.1, zfar=100.0)      # as bench.py
    pts, nrm, col = sphere_cloud(P0, seed=0)
    proj, view = camera_matrices(random_cameras(V, seed=0))
    pts_d, nrm_d, col_d = pts.to(dev).requires_grad_(True), nrm.to(dev), col.to(dev).requires_grad_(True)
    h = torch.full((V,), 5e-5, device=dev)
    grad = (torch.randn(V, S, S, 4, generator=torch.Generator().manual_seed(99)) * 1e-3).to(dev)
    cams = {False: (proj.to(dev), view.to(dev)),
            True: (proj.to(dev).requires_grad_(True), view.to(dev).requires_grad_(True))}

    def step(cam):
        pr, vw = cams[cam]
        pts_d.grad = col_d.grad = pr.grad = vw.grad = None
        render_points(pts_d, nrm_d, col_d, pr, vw, h, prm).image.backward(grad)

    ms = alternate({cam: lambda cam=cam: step(cam) for cam in (False, True)}, a.rounds, a.steps, 3)
    stages = {}
    for cam in (False, True):
        st = stage_ms(lambda: step(cam), a.steps, dev)
        stages[cam] = {k: st[k] for k in ("chain_world", "camera_backward")}
    print("gpu: %(name)s, %(power_limit)s, %(max_sm_clock)s" % card())
    print("step ms without camera grads: median %.4f  (min %.4f max %.4f)" % spread(ms[False]))
    print("step ms with camera grads:    median %.4f  (min %.4f max %.4f)" % spread(ms[True]))
    print("paired difference ms: median %.4f  (min %.4f max %.4f)" % spread(paired(ms[False], ms[True])))
    for cam in (False, True):
        print("stage ms/step (camera grads %s): %s" % (cam, {k: round(v, 4) for k, v in stages[cam].items()}))


if __name__ == "__main__":
    main()
