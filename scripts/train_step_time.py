"""Time of one training step on the fused path at the configs/dss.yml configuration (N = 8 views, 512^2, K = 5,
Vrk_invariant, lambda_dr_proj = 0.01, lambda_dr_repel = 0, learning points and normals) for P0 = 5 000 (dss.yml),
100 000 and 1 000 000 points on the sphere of bench.py's scene:
  eager  -- dss_b200.training.step.TrainStep (normalise, splat size, render, image loss, point filters, regularisers,
            backward)
  graph  -- GraphedTrainStep.replay() (the same step, one CUDA graph)
  filter -- dss_point_filters alone (ops.point_filters on a render of the cloud), 50 launches replayed from one CUDA
            graph per sample so that the kernel, not the host, is timed
The targets are a render of the sphere jittered and recoloured, its alpha > 0 the mask.  Every variant is warmed up,
then timed call by call with CUDA events, alternated in rounds in one process; the median of the samples is reported,
with the library's kernel launches of one eager step and the kernel nodes of the graph.

    python scripts/train_step_time.py [--samples 21] [--sizes 5000,100000,1000000]
"""
import argparse
import sys

import torch

from timing import alternate, card, launches, spread
from dss_b200 import _lib
from dss_b200.core.lighting import DirectionalLights
from dss_b200.ops import SplatParams, point_filters, render_points
from dss_b200.training.step import GraphedTrainStep, TrainStep
from tests.util import scene

FILTER_REPS = 50


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=21)
    ap.add_argument("--sizes", default="5000,100000,1000000")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("train_step_time.py needs a CUDA device")
    dev = torch.device("cuda:0")
    N, S = 8, 512
    prm = SplatParams(image_size=S, points_per_pixel=5, cutoff_threshold=1.0, depth_merging_threshold=0.05,
                      radii_backward_scaler=5.0, clip_pts_grad=0.05, znear=0.1)
    runs = {}
    for P0 in (int(s) for s in a.sizes.split(",")):
        pts, nrm, col, proj, view, _ = scene(P0, N, seed=0)
        pts, nrm, col, proj, view = (t.to(dev) for t in (pts, nrm, col, proj, view))
        g = torch.Generator().manual_seed(P0)
        lights = DirectionalLights(ambient_color=0.2 * torch.rand(N, 1, 3, generator=g),
                                   diffuse_color=0.5 * torch.rand(N, 1, 3, generator=g),
                                   specular_color=0.1 * torch.rand(N, 1, 3, generator=g),
                                   direction=torch.randn(N, 1, 3, generator=g), device=dev)
        with torch.no_grad():
            h = torch.full((N,), 3e-4, device=dev)
            tgt = render_points(pts + 0.01 * torch.randn(3, generator=g).to(dev), nrm, col.flip(1), proj, view, h,
                                prm).image
        img = tgt[..., :3].permute(0, 3, 1, 2).contiguous().permute(0, 2, 3, 1)
        mask = (tgt[..., 3] > 0).float()
        eager = TrainStep(pts, nrm, col, prm)
        lib_launches = launches(lambda: eager(img, mask, proj, view, lights), dev)
        with torch.no_grad():
            out = render_points(pts, nrm, col, proj, view, h, prm)
        runs[P0] = {"eager": lambda e=eager, b=(img, mask, proj, view, lights): e(*b),
                    "filter": lambda o=out, m=mask: point_filters(o, m),
                    "_args": (pts, nrm, col, prm, img, mask, proj, view, lights), "_launches": lib_launches}

    def measure(variants):
        return alternate({(P0, v): runs[P0][v] for P0, v in variants}, a.samples, 1, 3)

    # the eager steps are timed before any graph exists: an eager call may reallocate the library's scratch, which a
    # graph then captures again at its next replay
    ms = measure([(P0, "eager") for P0 in runs])
    graphs = {}
    for P0, r in runs.items():
        graphs[P0] = GraphedTrainStep(*r.pop("_args"))
        r["graph"] = graphs[P0].replay
        # the filter kernel alone: FILTER_REPS launches replayed from one graph, so that no host time is counted
        fg = torch.cuda.CUDAGraph()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            r["filter"]()
        torch.cuda.current_stream().wait_stream(s)
        with torch.cuda.graph(fg):
            for _ in range(FILTER_REPS):
                r["filter"]()
        r["filter"] = fg.replay
    # a later capture may have grown the scratch: the earlier graphs capture again here, until a round of replays
    # leaves the scratch as it found it (then every graph holds the current buffers)
    for _ in range(8):
        scratch = _lib.scratch_bytes()
        for P0 in runs:
            runs[P0]["graph"]()
        torch.cuda.synchronize()
        if _lib.scratch_bytes() == scratch:
            break
    else:
        sys.exit("the library's scratch kept growing across the graph captures")
    ms.update(measure([(P0, v) for P0 in runs for v in ("graph", "filter")]))
    assert _lib.scratch_bytes() == scratch, "the scratch moved while the graphs were timed"
    for P0, r in runs.items():
        r["_counts"] = (r.pop("_launches"), graphs[P0].kernel_nodes(), float(graphs[P0].loss["loss"]))
    print("gpu: %(name)s, %(power_limit)s, %(max_sm_clock)s" % card())
    for P0 in runs:
        lib_launches, nodes, loss = runs[P0]["_counts"]
        print("P0 = %d: %d library kernel launches per eager step, %d kernel nodes per graph replay, loss %.6f"
              % (P0, lib_launches, nodes, loss))
        for v in ("eager", "graph", "filter"):
            t = [x / FILTER_REPS for x in ms[(P0, v)]] if v == "filter" else ms[(P0, v)]
            print("  %-6s ms: median %.3f  (min %.3f max %.3f, %d samples)" % (v, *spread(t), len(t)))


if __name__ == "__main__":
    main()
