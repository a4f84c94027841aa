"""Step time of shading a batch of different clouds (packed layout) at the bench.py headline size: 8 views, 1M packed rows
per view (jittered copies of the headline sphere), 512x512, K=5, with L = 1 and L = 3 directional lights.  Three routes,
eager forward+backward steps alternated in one process and timed with CUDA events:
  torch  -- the torch shading (dss_b200.core.texture.apply_lighting, what LightingTexture runs, with the per-row view
            index) feeding render_points with the (P,3) shaded colours
  packed -- render_points(..., shading=make_shading(...)) on the packed clouds, (P,3) albedo
  shared -- the fused shading of one shared 1M-point cloud seen by the same 8 cameras (the sphere without jitter)

    python scripts/packed_shading_time.py [--rounds 8] [--steps 15]
"""
import argparse
import sys

import torch

from timing import alternate, card, paired, spread
from dss_b200.core.camera import camera_matrices
from dss_b200.core.lighting import DirectionalLights
from dss_b200.core.texture import apply_lighting, camera_centres
from dss_b200.ops import SplatParams, make_shading, render_points
from tests.util import random_cameras, sphere_cloud


def lights(L, dev):
    g = torch.Generator().manual_seed(L)
    diffuse = torch.eye(3)[:L] * 0.5 if L == 3 else torch.full((L, 3), 0.5)       # tri-colour: red, green, blue
    return DirectionalLights(ambient_color=torch.full((1, 1, 3), 0.3), diffuse_color=diffuse[None],
                             specular_color=torch.full((1, L, 3), 0.2), direction=torch.randn(1, L, 3, generator=g),
                             device=dev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=8)
    ap.add_argument("--steps", type=int, default=15)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("packed_shading_time.py needs a CUDA device")
    dev = torch.device("cuda:0")
    P0, S, K, V, shin = 1_000_000, 512, 5, 8, 64.0
    prm = SplatParams(image_size=S, points_per_pixel=K, cutoff_threshold=1.0, depth_merging_threshold=0.05,
                      antialiasing_sigma=1.0, radii_backward_scaler=5.0, clip_pts_grad=0.05,
                      backface_culling=False, znear=0.1, zfar=100.0)      # as bench.py
    pts, nrm, col = sphere_cloud(P0, seed=0)
    proj, view = camera_matrices(random_cameras(V, seed=0))
    proj, view = proj.to(dev), view.to(dev)
    h = torch.full((V,), 5e-5, device=dev)
    grad = (torch.randn(V, S, S, 4, generator=torch.Generator().manual_seed(99)) * 1e-3).to(dev)
    # packed: view n renders its own jittered copy of the sphere
    g = torch.Generator().manual_seed(7)
    pk_pts = (pts.repeat(V, 1) + 2e-3 * torch.randn(V * P0, 3, generator=g)).to(dev).requires_grad_(True)
    pk_nrm, pk_alb = nrm.repeat(V, 1).to(dev).requires_grad_(True), col.repeat(V, 1).to(dev).requires_grad_(True)
    first = torch.arange(V, device=dev) * P0
    num = torch.full((V,), P0, dtype=torch.int64, device=dev)
    vidx = torch.arange(V, device=dev).repeat_interleave(P0)
    sh_pts, sh_nrm, sh_alb = (t.to(dev).requires_grad_(True) for t in (pts, nrm, col))
    light_objs = {L: lights(L, dev) for L in (1, 3)}
    packed = dict(first_idx=first, num_points=num, shared_cloud=False)

    def step(route, L):
        lt = light_objs[L]
        for t in (pk_pts, pk_nrm, pk_alb, sh_pts, sh_nrm, sh_alb):
            t.grad = None
        if route == "torch":
            cam = camera_centres(view)
            amb, dif, spe = apply_lighting(pk_pts, pk_nrm, lt, cam[vidx], shininess=shin, view_idx=vidx)
            out = render_points(pk_pts, pk_nrm, pk_alb * (amb + dif) + spe, proj, view, h, prm, **packed)
        elif route == "packed":
            out = render_points(pk_pts, pk_nrm, pk_alb, proj, view, h, prm, shading=make_shading(lt, view, shin),
                                **packed)
        else:
            out = render_points(sh_pts, sh_nrm, sh_alb, proj, view, h, prm, shading=make_shading(lt, view, shin))
        out.image.backward(grad)

    variants = [(r, L) for L in (1, 3) for r in ("torch", "packed", "shared")]
    ms = alternate({v: lambda v=v: step(*v) for v in variants}, a.rounds, a.steps, 3)
    print("gpu: %(name)s, %(power_limit)s, %(max_sm_clock)s" % card())
    for v in variants:
        print("step ms L=%d %-6s: median %.3f  (min %.3f max %.3f)" % (v[1], v[0], *spread(ms[v])))
    for L in (1, 3):
        for x, y in (("torch", "packed"), ("packed", "shared")):
            print("L=%d paired difference ms (%s - %s): median %.3f  (min %.3f max %.3f)"
                  % (L, x, y, *spread(paired(ms[(y, L)], ms[(x, L)]))))


if __name__ == "__main__":
    main()
