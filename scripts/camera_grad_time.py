"""Extra step time of camera gradients at the bench.py headline configuration (1M points x 8 views, 512x512, K=5):
eager forward+backward steps with and without proj / view requiring grad, alternated in one process, timed with CUDA
events; plus the per-stage device time of the camera kernels and of the chain kernel (which writes grad_ndc when
camera gradients are asked for).

    python scripts/camera_grad_time.py [--rounds 10] [--steps 20]
"""
import argparse
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dss_b200 import _lib  # noqa: E402
from dss_b200.core.camera import camera_matrices  # noqa: E402
from dss_b200.ops import SplatParams, render_points  # noqa: E402
from tests.util import random_cameras, sphere_cloud  # noqa: E402


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

    def timed(cam, n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            step(cam)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    for cam in (False, True):
        timed(cam, 3)                                   # warm-up of both shapes
    ms = {False: [], True: []}
    for _ in range(a.rounds):
        for cam in (False, True):
            ms[cam].append(timed(cam, a.steps))
    stages = {}
    for cam in (False, True):
        _lib.profile_enable(True, dev)
        _lib.profile_reset(dev)
        for _ in range(a.steps):
            step(cam)
        torch.cuda.synchronize()
        st = _lib.profile_read(dev)
        _lib.profile_enable(False, dev)
        stages[cam] = {k: st[k][0] / a.steps for k in ("chain_world", "camera_backward")}
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    med = {k: statistics.median(v) for k, v in ms.items()}
    diffs = [b - a_ for a_, b in zip(ms[False], ms[True])]
    print("gpu: %s" % smi)
    print("step ms without camera grads: median %.4f  (min %.4f max %.4f)" % (med[False], min(ms[False]), max(ms[False])))
    print("step ms with camera grads:    median %.4f  (min %.4f max %.4f)" % (med[True], min(ms[True]), max(ms[True])))
    print("paired difference ms: median %.4f  (min %.4f max %.4f)" % (statistics.median(diffs), min(diffs), max(diffs)))
    for cam in (False, True):
        print("stage ms/step (camera grads %s): %s" % (cam, {k: round(v, 4) for k, v in stages[cam].items()}))


if __name__ == "__main__":
    main()
