"""Time of the anisotropic splat kernel (Vrk_invariant = Vrk_isotropic = false, configs/default.yaml):
  frames -- dss_b200.ops.local_frames (the K = 8 search and dss_local_frames) on the sphere of bench.py's scene at
            P0 = 8 000 (default.yaml's n_points_per_cloud), 100 000 and 1 000 000 points
  eager / graph -- TrainStep and GraphedTrainStep.replay() at 8 views of 512^2, K = 5, in the anisotropic and the
            Vrk_invariant mode (everything else as scripts/train_step_time.py), at P0 = 8 000 and 100 000
Every variant is warmed up, then timed call by call with CUDA events; the median of the samples is reported, with the
library's kernel launches of one eager step and the kernel nodes of the graph.

    python scripts/anisotropic_time.py [--samples 21]
"""
import argparse
import sys

import torch

from timing import card, events_ms, launches, spread
from dss_b200.core.lighting import DirectionalLights
from dss_b200.ops import SplatParams, local_frames, render_points
from dss_b200.training.step import GraphedTrainStep, TrainStep
from tests.util import scene


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=21)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("anisotropic_time.py needs a CUDA device")
    dev = torch.device("cuda:0")
    print("gpu: %(name)s, %(power_limit)s, %(max_sm_clock)s" % card())

    def samples(fn):
        t = [events_ms(fn, 1) for _ in range(3 + a.samples)]
        return spread(t[3:])                            # after 3 warm-up calls

    for P0 in (8000, 100000, 1000000):
        pts = scene(P0, 1, seed=0)[0].to(dev)
        print("local_frames P0 = %7d: median %.3f ms (min %.3f max %.3f)"
              % (P0, *samples(lambda: local_frames(pts))))
    N, S = 8, 512
    prm = SplatParams(image_size=S, points_per_pixel=5, cutoff_threshold=0.5, depth_merging_threshold=0.05,
                      radii_backward_scaler=5.0, clip_pts_grad=0.05, znear=0.1)
    for P0 in (8000, 100000):
        pts, nrm, col, proj, view, _ = scene(P0, N, seed=0)
        pts, nrm, col, proj, view = (t.to(dev) for t in (pts, nrm, col, proj, view))
        g = torch.Generator().manual_seed(P0)
        lights = DirectionalLights(ambient_color=0.2 * torch.rand(N, 1, 3, generator=g),
                                   diffuse_color=0.5 * torch.rand(N, 1, 3, generator=g),
                                   specular_color=0.1 * torch.rand(N, 1, 3, generator=g),
                                   direction=torch.randn(N, 1, 3, generator=g), device=dev)
        with torch.no_grad():
            tgt = render_points(pts + 0.01 * torch.randn(3, generator=g).to(dev), nrm, col.flip(1), proj, view,
                                torch.full((N,), 3e-4, device=dev), prm).image
        batch = (tgt[..., :3].contiguous(), (tgt[..., 3] > 0).float(), proj, view, lights)
        for mode, kw in (("invariant", dict(Vrk_invariant=True)),
                         ("anisotropic", dict(Vrk_invariant=False, Vrk_isotropic=False))):
            eager = TrainStep(pts, nrm, col, prm, **kw)
            n = launches(lambda: eager(*batch), dev)
            te = samples(lambda: eager(*batch))
            graph = GraphedTrainStep(pts, nrm, col, prm, *batch, **kw)
            tg = samples(graph.replay)
            print("P0 = %6d %-11s: %d library launches per eager step, %d graph kernel nodes; eager median %.3f ms "
                  "(min %.3f max %.3f), graph median %.3f ms (min %.3f max %.3f)"
                  % (P0, mode, n, graph.kernel_nodes(), *te, *tg))
            del graph, eager


if __name__ == "__main__":
    main()
