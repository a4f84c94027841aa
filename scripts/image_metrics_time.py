"""Time of the image-space validation (Trainer.evaluate_2d's iou / psnr) on 120 views of 512^2 data, the reference's
data size: the torus of scripts/meshes.py rendered by create_mvr_data (120 cameras, 512^2, point lights) into a
temporary directory.
  kernel  -- `image_metrics` alone (dss_image_metrics: resize + sums, two launches) on 120 stored renders at s = 128
             (resolution // 4, what the training loop validates at) and s = 512, the GT passed as the loop passes it
             (a permuted (V,3,H,W) batch and a float mask); its algorithmic bytes are the renders (16 B per output
             pixel) plus the ground-truth rows the bilinear taps touch (16 B per pixel of such a row: all of them at
             s = 512, every other pair at s = 128), each read once
  eval2d  -- `evaluate_2d` of the data's stored cloud over the 120 views at s = 128 and s = 512, --batch views per
             render, host-to-device upload of each batch's ground truth included
Each variant is timed in alternated rounds with CUDA events (scripts/timing.py).

    python scripts/image_metrics_time.py [--rounds 5] [--steps 20] [--batch 8]
"""
import argparse
import sys
import tempfile

import torch

from timing import alternate, card, spread
from meshes import torus
from dss_b200.ops import evaluate_2d, image_metrics, render_data_views
from dss_b200.training.config import DEFAULTS, splat_params
from dss_b200.utils.dataset import MVRData


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--batch", type=int, default=8)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("image_metrics_time.py needs a CUDA device")
    from dss_b200.utils.create_mvr_data import main as create
    from dss_b200.utils.io import save_obj
    dev = torch.device("cuda:0")
    with tempfile.TemporaryDirectory() as tmp:
        verts, faces = torus()
        save_obj(tmp + "/torus.obj", verts.numpy(), faces.numpy())
        data_dir = create(["--points", tmp + "/torus.obj", "--output", tmp + "/data", "--num_cameras", "120",
                           "--image-size", "512", "--point_lights", "--seed", "0"])[0]
        data = MVRData(data_dir)
        V, S = len(data), data.resolution[0]
        pc = data.get_pointclouds()
        pts, nrm = pc.points_packed().to(dev), pc.normals_packed().to(dev)
        col = torch.ones_like(pts)
        cams = data.get_cameras()
        params = splat_params(DEFAULTS, cams.znear, cams.zfar)
        b = data.pinned_batch(list(range(V)))
        rgb, mask = b["img.rgb"].to(dev).permute(0, 2, 3, 1), b["img.mask"].to(dev)
        renders = {}
        for s in (S // 4, S):
            renders[s] = torch.cat([render_data_views(pts, nrm, col, data, params._replace(image_size=s),
                                                      range(i, min(i + a.batch, V))) for i in range(0, V, a.batch)])
        variants = {("kernel", s): (lambda s=s: image_metrics(renders[s], rgb, mask)) for s in renders}
        variants.update({("eval2d", s): (lambda s=s: evaluate_2d(pts, nrm, col, data, params, s, a.batch))
                         for s in renders})
        ms = alternate(variants, a.rounds, a.steps, 2)
        print("gpu: %(name)s, %(power_limit)s, %(max_sm_clock)s" % card())
        print("data: %d views of %d^2, stored cloud of %d points, batch %d" % (V, S, pts.shape[0], a.batch))
        for (what, s), xs in ms.items():
            med, lo, hi = spread(xs)
            line = "%-6s s = %3d: median %.3f ms (min %.3f max %.3f)" % (what, s, med, lo, hi)
            if what == "kernel":
                src = [max((d + 0.5) * S / s - 0.5, 0.0) for d in range(s)]
                rows = {int(x) for x in src} | {min(int(x) + 1, S - 1) for x in src}
                gb = V * (16 * s * s + 16 * len(rows) * S) / 1e9
                line += "; %.3f GB algorithmic, %.0f GB/s" % (gb, gb / (med / 1e3))
            print(line)
        for s in renders:
            ev = evaluate_2d(pts, nrm, col, data, params, s, a.batch)
            print("stored cloud at s = %d: iou %.5f, psnr %.6f" % (s, float(ev["iou"]), float(ev["psnr"])))


if __name__ == "__main__":
    main()
