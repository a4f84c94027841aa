"""Time of the view coverage the training loop prunes on, on 100 views of 512^2 data: the torus of scripts/meshes.py
rendered by create_mvr_data (100 cameras, 512^2, point lights) into a temporary directory, and P0 area-weighted samples
of that torus as the cloud (P0 = 100k and 1M).
  kernel -- `accumulate_coverage` alone (dss_point_coverage, one launch) on one render of all 100 views of the shared
            cloud; its algorithmic bytes are each (view, point) record's x, y, z read as one 16-byte load, its visible
            byte, and the two int32 counters read and written (the mask taps, a few per point and view, are not counted)
  whole  -- `point_coverage` over the 100 views, --batch views per render: the renders, the mask gathers and the kernels
Each is the median of CUDA-event timings after a warm-up (scripts/timing.py), with the card read in the same run.

    python scripts/point_coverage_time.py [--iters 10] [--batch 8]
"""
import argparse
import sys
import tempfile

import torch

from timing import card, median_ms
from meshes import torus
from dss_b200.ops import Coverage, _data_view_renderer, accumulate_coverage, point_coverage
from dss_b200.training.config import DEFAULTS, splat_params
from dss_b200.utils.dataset import MVRData


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--batch", type=int, default=8)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("point_coverage_time.py needs a CUDA device")
    from dss_b200.utils.create_mvr_data import main as create, sample_points_from_mesh
    from dss_b200.utils.io import save_obj
    dev = torch.device("cuda:0")
    print("gpu: %(name)s, %(power_limit)s, %(max_sm_clock)s" % card())
    with tempfile.TemporaryDirectory() as tmp:
        verts, faces = torus()
        save_obj(tmp + "/torus.obj", verts.numpy(), faces.numpy())
        data_dir = create(["--points", tmp + "/torus.obj", "--output", tmp + "/data", "--num_cameras", "100",
                           "--image-size", "512", "--point_lights", "--seed", "0"])[0]
        data = MVRData(data_dir)
        views = data.device_views(dev)
        V = len(views)
        cams = data.get_cameras()
        params = splat_params(DEFAULTS, cams.znear, cams.zfar)
        flags = dict(Vrk_invariant=True, Vrk_isotropic=False)
        print("data: %d views of %d^2, %s store; batch %d" % (V, views.H, str(views.store.dtype), a.batch))
        g = torch.Generator(device=dev).manual_seed(0)
        for P0 in (100_000, 1_000_000):
            pts, nrm = sample_points_from_mesh(verts.float().to(dev), faces.to(dev), P0, generator=g)
            out = _data_view_renderer(pts, nrm, torch.ones_like(pts), views, True, False, 0.2, 64.0)(params, range(V))
            _, mask = views.gather(views.upload(range(V)))
            cov = Coverage(*(torch.zeros((P0,), dtype=torch.int32, device=dev) for _ in range(2)))
            k_ms = median_ms(lambda: accumulate_coverage(out, mask, *cov), 3, a.iters)
            gb = (V * P0 * 17 + 16 * P0) / 1e9
            del out
            torch.cuda.empty_cache()
            w_ms = median_ms(lambda: point_coverage(pts, nrm, views, params, a.batch, **flags), 1, a.iters)
            c = point_coverage(pts, nrm, views, params, a.batch, **flags)
            print("P0 = %7d: kernel %.3f ms (%.3f GB algorithmic, %.0f GB/s); whole point_coverage %.1f ms; "
                  "seen in no view %d, outside in some view %d"
                  % (P0, k_ms, gb, gb / (k_ms / 1e3), w_ms, int((c.seen == 0).sum()), int((c.outside > 0).sum())))


if __name__ == "__main__":
    main()
