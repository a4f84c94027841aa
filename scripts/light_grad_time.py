"""Step time of per-view lights and of light gradients through the fused shading at the bench.py headline configuration
(1M points x 8 views, 512x512, K=5) with L = 1 and L = 3 directional lights (3: the reference's tri-colour setting).
Eager forward+backward steps of four variants per L -- shared or per-view lights, with or without gradients to the
light directions and colours -- alternated in one process and timed with CUDA events; plus the per-stage device time of
the light kernels (light_backward).

    python scripts/light_grad_time.py [--rounds 10] [--steps 20]
"""
import argparse

import torch

from timing import alternate, card, paired, spread, stage_ms
from dss_b200.core.camera import camera_matrices
from dss_b200.core.lighting import DirectionalLights
from dss_b200.ops import SplatParams, make_shading, render_points
from tests.util import random_cameras, sphere_cloud


def lights(L, V, per_view, grad, dev):
    g = torch.Generator().manual_seed(L)
    diffuse = torch.eye(3)[:L] * 0.5 if L == 3 else torch.full((L, 3), 0.5)       # tri-colour: red, green, blue
    direction = torch.randn(V if per_view else 1, L, 3, generator=g)
    out = DirectionalLights(ambient_color=torch.full((1, 1, 3), 0.3), diffuse_color=diffuse[None],
                            specular_color=torch.full((1, L, 3), 0.2), direction=direction, device=dev)
    if grad:
        out.direction.requires_grad_(True)
        out.diffuse_color.requires_grad_(True)
        out.specular_color.requires_grad_(True)
    return out


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
    proj, view = proj.to(dev), view.to(dev)
    pts_d, nrm_d, alb_d = pts.to(dev).requires_grad_(True), nrm.to(dev).requires_grad_(True), col.to(dev).requires_grad_(True)
    h = torch.full((V,), 5e-5, device=dev)
    grad = (torch.randn(V, S, S, 4, generator=torch.Generator().manual_seed(99)) * 1e-3).to(dev)
    variants = [(L, pv, lg) for L in (1, 3) for pv in (False, True) for lg in (False, True)]
    light_objs = {v: lights(v[0], V, v[1], v[2], dev) for v in variants}

    def step(v):
        lt = light_objs[v]
        pts_d.grad = nrm_d.grad = alb_d.grad = lt.direction.grad = lt.diffuse_color.grad = lt.specular_color.grad = None
        sh = make_shading(lt, view)
        render_points(pts_d, nrm_d, alb_d, proj, view, h, prm, shading=sh).image.backward(grad)

    ms = alternate({v: lambda v=v: step(v) for v in variants}, a.rounds, a.steps, 3)
    stages = {}
    for v in variants:
        st = stage_ms(lambda: step(v), a.steps, dev)
        stages[v] = {k: st[k] for k in ("preprocess", "colour_backward", "light_backward")}
    print("gpu: %(name)s, %(power_limit)s, %(max_sm_clock)s" % card())
    name = lambda v: "L=%d %-8s %s" % (v[0], "per-view" if v[1] else "shared", "light grads" if v[2] else "no light grads")
    for v in variants:
        print("step ms %s: median %.4f  (min %.4f max %.4f)  stage ms/step %s"
              % (name(v), *spread(ms[v]), {k: round(x, 4) for k, x in stages[v].items()}))
    for L in (1, 3):
        for what, (x, y) in (("per-view - shared, no light grads", ((L, False, False), (L, True, False))),
                             ("light grads - none, shared", ((L, False, False), (L, False, True))),
                             ("light grads - none, per-view", ((L, True, False), (L, True, True)))):
            print("L=%d paired difference ms (%s): median %.4f  (min %.4f max %.4f)"
                  % (L, what, *spread(paired(ms[x], ms[y]))))


if __name__ == "__main__":
    main()
