"""Time of the image loss of the training step (Trainer.calc_dr_loss: masked RGB L1 + silhouette L1 + 0.01 IoU),
forward + backward, at 1 x 256^2, 8 x 512^2 (the headline) and 8 x 1024^2.  The RGBA is a real render of the headline
sphere (1M points, bench.py's scene) and the target a render of the sphere jittered and recoloured, its alpha > 0 the
GT mask, the GT RGB passed as the trainer passes it (a permuted (N,3,H,W) batch).  Two routes, alternated in rounds in
one process and timed with CUDA events:
  torch -- `image_loss_torch` in float32 on CUDA (the reference's calc_dr_loss, its host synchronisations included)
  fused -- `image_loss`'s CUDA route (dss_image_loss_forward / _backward)
and the whole step at the headline size: render + torch loss + backward, render + fused loss + backward, and the
GraphedRenderStep with targets= (one graph replay).  The achieved bandwidth of the fused route counts the algorithmic
bytes (forward: rgba 16 + gt 12 + mask 4 per pixel; backward: the same again + 16 written) over the route's time.

    python scripts/image_loss_time.py [--rounds 7] [--steps 20]
"""
import argparse
import statistics
import sys

import torch

from timing import alternate, card, spread
from dss_b200.graph import GraphedRenderStep
from dss_b200.ops import SplatParams, render_points
from dss_b200.training.losses import image_loss, image_loss_torch
from tests.util import scene


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--steps", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("image_loss_time.py needs a CUDA device")
    dev = torch.device("cuda:0")
    P0 = 1_000_000
    cases, steps = {}, {}
    for N, S in ((1, 256), (8, 512), (8, 1024)):
        pts, nrm, col, proj, view, _ = scene(P0, N, seed=0)
        pts, nrm, col, proj, view = (t.to(dev) for t in (pts, nrm, col, proj, view))
        prm = SplatParams(image_size=S, points_per_pixel=5, znear=0.1, clip_pts_grad=0.05)
        h = torch.full((N,), 5e-5 * (512 / S) ** 2, device=dev)
        g = torch.Generator().manual_seed(S)
        with torch.no_grad():
            rgba = render_points(pts, nrm, col, proj, view, h, prm).image
            tgt = render_points(pts + 0.01 * torch.randn(3, generator=g).to(dev), nrm, col.flip(1), proj, view, h,
                                prm).image
        img = tgt[..., :3].permute(0, 3, 1, 2).contiguous().permute(0, 2, 3, 1)
        mask = (tgt[..., 3] > 0).float()
        cases[(N, S)] = (rgba.clone().requires_grad_(True), img, mask)
        if (N, S) == (8, 512):
            p, c = pts.clone().requires_grad_(True), col.clone().requires_grad_(True)
            steps["render"] = (p, nrm, c, proj, view, h, prm, img, mask)
            steps["graph"] = GraphedRenderStep(p, nrm, c, proj, view, h, prm, targets=(img, mask, 1.0, 1.0))

    def loss_step(route, N, S):
        x, img, mask = cases[(N, S)]
        x.grad = None
        (image_loss_torch if route == "torch" else image_loss)(x, img, mask)["loss"].backward()

    def whole_step(route):
        if route == "graph":
            steps["graph"].replay()
            return
        p, nrm, c, proj, view, h, prm, img, mask = steps["render"]
        p.grad = c.grad = None
        out = render_points(p, nrm, c, proj, view, h, prm)
        (image_loss_torch if route == "torch" else image_loss)(out.image, img, mask)["loss"].backward()

    def run(v):
        if v[0] == "loss":
            loss_step(*v[1:])
        else:
            whole_step(v[1])

    variants = [("loss", r, N, S) for (N, S) in cases for r in ("torch", "fused")]
    variants += [("step", r) for r in ("torch", "fused", "graph")]
    ms = alternate({v: lambda v=v: run(v) for v in variants}, a.rounds, a.steps, 3)
    print("gpu: %(name)s, %(power_limit)s, %(max_sm_clock)s" % card())
    for v in variants:
        what = "%d x %d^2 loss" % (v[2], v[3]) if v[0] == "loss" else "8 x 512^2 whole step"
        print("%-22s %-5s ms: median %.3f  (min %.3f max %.3f)" % (what, v[1], *spread(ms[v])))
    for (N, S) in cases:
        t, f = ms[("loss", "torch", N, S)], ms[("loss", "fused", N, S)]
        r = [x / y for x, y in zip(t, f)]
        gb = N * S * S * (2 * (16 + 12 + 4) + 16) / 1e9
        print("%d x %d^2: torch / fused median %.1fx (min %.1f max %.1f); fused %.0f GB/s algorithmic"
              % (N, S, *spread(r), gb / (statistics.median(f) / 1e3)))


if __name__ == "__main__":
    main()
