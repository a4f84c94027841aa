"""Time L0 smoothing (ops.l0_smooth) and one cycle of the image-filter command (dss_b200.utils.image_filter).

    python scripts/l0_smooth_time.py [--out FILE]

1. ms per call of l0_smooth on 8 x 512^2 x 3 and 8 x 1024^2 x 3 float32 images (median of CUDA-event timings), and the
   bytes its 20 rounds move, counted from the shapes by the passes of csrc/l0_smooth.cu, over that time: GB/s and the
   share of the H100 SXM's 3.35 TB/s of HBM3.  Per value and round: the shrink pass reads S (8 B); the forward row
   pass reads I and S (16 B) and writes the complex rows (16 B); the column pass reads and writes them (32 B); the
   inverse row pass reads them (16 B) and writes S (8 B): 96 B, plus 1 B per pixel written and read of the keep flags.
   Loading and storing the images, once per call, add 12 B (float32) per value.
2. One cycle of ``filter_cloud`` at its defaults (64 views, batch 8, 512^2, 20 steps) on the bunny: the time of a
   run of 2 cycles less that of 1 cycle (a cycle after the capture), and, with the same calls, the render of the 64
   views and the filter of their images; the steps are the rest.
The card's name and power limit are read in the same call and printed with the numbers."""
import argparse
import json
import os
import tempfile
import time

import torch
from timing import card, median_ms

from dss_b200.ops import l0_smooth

HBM_BYTES_PER_S = 3.35e12
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def round_bytes(N, H, W, C, rounds=20):
    values, pixels = N * H * W * C, N * H * W
    return rounds * (96 * values + 2 * pixels) + 12 * values


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    res = {"card": card()}
    g = torch.Generator(device=dev).manual_seed(0)
    for S in (512, 1024):
        x = torch.rand((8, S, S, 3), generator=g, device=dev)
        ms = median_ms(lambda: l0_smooth(x, 0.05), 2, 10)
        b = round_bytes(8, S, S, 3)
        res["l0_8x%dx%dx3" % (S, S)] = {"ms": ms, "bytes": b, "GB_per_s": b / ms * 1e-6,
                                        "hbm_share": b / (ms * 1e-3) / HBM_BYTES_PER_S}
        print(json.dumps(res["l0_8x%dx%dx3" % (S, S)]), flush=True)

    from dss_b200.ops import SplatParams, make_shading, render_points, shared_cloud_splats
    from dss_b200.core.camera import CameraSampler, FoVPerspectiveCameras, camera_matrices
    from dss_b200.utils.create_mvr_data import _stack_lights, get_light_for_view
    from dss_b200.utils.image_filter import filter_cloud
    from dss_b200.utils.io import read_ply
    import random
    src = os.path.join(ROOT, "tests", "golden", "ply", "bunny-8000.ply")
    d = read_ply(src)
    pts = torch.from_numpy(d["points"]).double()
    pts = ((pts - pts.mean(0)) / (pts - pts.mean(0)).norm(dim=1).max()).float().to(dev)
    nrm = torch.nn.functional.normalize(torch.from_numpy(d["normals"]).to(dev), dim=-1)
    V, B, S = 64, 8, 512
    sampler = CameraSampler(V, 1, distance_range=((1.2, 2.2),), camera_params={"znear": 0.1},
                            generator=torch.Generator().manual_seed(0))
    rng = random.Random(0)
    lights = [get_light_for_view(c, point_lights=False, has_specular=False, rng=rng) for c in sampler]
    proj, view = (m.to(dev) for m in camera_matrices(FoVPerspectiveCameras(R=sampler.R, T=sampler.T, znear=0.1)))
    prm = SplatParams(image_size=S, points_per_pixel=5, cutoff_threshold=1.0, radii_backward_scaler=5.0,
                      clip_pts_grad=0.05, znear=0.1)
    bl = [_stack_lights(lights[i:i + B]).to(dev) for i in range(0, V, B)]
    rgbs = []

    def render():
        rgbs.clear()
        with torch.no_grad():
            for b in range(V // B):
                sl = slice(b * B, (b + 1) * B)
                h, frames = shared_cloud_splats(pts, B, True, False)
                rgbs.append(render_points(pts, nrm, torch.ones_like(pts), proj[sl], view[sl], h, prm,
                                          shading=make_shading(bl[b], view[sl]), deterministic=True,
                                          frames=frames).image[..., :3])

    render_ms = median_ms(render, 2, 5)
    filter_ms = median_ms(lambda: [l0_smooth(r, 0.05) for r in rgbs], 1, 5)
    walls = {}
    with tempfile.TemporaryDirectory() as tmp:
        for cycles in (1, 2, 1, 2):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            filter_cloud(src, os.path.join(tmp, "out.ply"), cycles=cycles, log=None)
            torch.cuda.synchronize()
            walls.setdefault(cycles, []).append((time.perf_counter() - t0) * 1e3)
    cycle_ms = min(walls[2]) - min(walls[1])
    res["filter_cycle_defaults"] = {"cycle_ms": cycle_ms, "render_64_views_ms": render_ms,
                                    "filter_64_views_ms": filter_ms, "steps_20_ms": cycle_ms - render_ms - filter_ms,
                                    "run_1_cycle_ms": min(walls[1]), "run_2_cycles_ms": min(walls[2])}
    print(json.dumps(res["filter_cycle_defaults"]), flush=True)
    res["card_after"] = card()
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
