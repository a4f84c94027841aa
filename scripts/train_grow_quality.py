"""Quality and time of growing the cloud during training against training the final size from the start: the loop of
dss_b200.training.train at configs/dss.yml's settings (512^2 views, 8 per batch, Vrk_invariant splats) on data that
create_mvr_data renders from a torus, run twice for the same number of iterations from the same seed:

  fixed  -- n_points_per_cloud 8000 throughout;
  grown  -- 2000 points, grown to 4000 and 8000 at --milestones (training.grow_milestones / grow_points).

    python scripts/train_grow_quality.py [--its 900] [--milestones 300 600] [--views 64] [--out results.json]

For each run: chamfer_point, chamfer_normal (against 8000 area-weighted samples of the mesh, the loop's validation)
and p2f_avg (mean distance of the cloud's points to the mesh) after the last iteration; the wall-clock time of the
iterations (Trainer.run between two device synchronisations, without the data upload and the first capture, with no
validation or checkpoint inside); and the cost of each growth event (upsample_points plus the new step's capture, host
clock to a device synchronisation).  Prints one JSON line with the card name and its power limit."""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

import torch
import yaml

from timing import card


def make_data(tmp, views):
    from dss_b200.utils.create_mvr_data import main as create
    from dss_b200.utils.io import save_obj
    from tests.test_mesh_data import torus
    verts, faces = torus(nu=192, nv=96)
    save_obj(os.path.join(tmp, "torus.obj"), verts.numpy(), faces.numpy())
    return create(["--points", os.path.join(tmp, "torus.obj"), "--output", os.path.join(tmp, "data"),
                   "--num_cameras", str(views), "--image-size", "512", "--tri_color_light", "--point_lights",
                   "--seed", "3"])[0]


def run(name, data_dir, tmp, its, n0, milestones, sizes):
    from dss_b200.training.config import load_config
    from dss_b200.training.train import Trainer
    path = os.path.join(tmp, name + ".yml")
    with open(path, "w") as f:
        yaml.safe_dump({
            "name": name, "data": {"data_dir": data_dir},
            "model": {"model_kwargs": {"n_points_per_cloud": n0, "learn_colors": False}},
            "renderer": {"raster_params": {"Vrk_invariant": True, "Vrk_isotropic": False, "clip_pts_grad": 0.05,
                                           "cutoff_threshold": 1.0, "depth_merging_threshold": 0.05,
                                           "image_size": 512, "points_per_pixel": 5, "radii_backward_scaler": 5}},
            "training": {"out_dir": os.path.join(tmp, "out"), "batch_size": 8, "lambda_dr_proj": 0.01,
                         "lambda_dr_repel": 0.0, "steps_dss_backward_radii": 200, "print_every": 100,
                         "validate_every": 0, "checkpoint_every": 0, "model_selection_metric": "p2f_avg",
                         "grow_milestones": list(milestones), "grow_points": list(sizes)}}, f)
    t = Trainer(load_config(path))
    events = []
    grow = t.grow

    def timed(n):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        grow(n)
        torch.cuda.synchronize()
        events.append({"it": t.it, "points": n, "ms": (time.perf_counter() - t0) * 1e3})

    t.grow = timed
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    t.run(exit_after=-1, max_it=its)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    ev = t.evaluate()
    res = {"points_start": n0, "points_end": int(t.step.points.shape[0]), "its": its, "wall_s": wall,
           "chamfer_point": ev["chamfer_point"], "chamfer_normal": ev["chamfer_normal"], "p2f_avg": ev["p2f_avg"],
           "growth_events": events}
    del t
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--its", type=int, default=900)
    ap.add_argument("--milestones", type=int, nargs=2, default=[300, 600])
    ap.add_argument("--views", type=int, default=64)
    ap.add_argument("--out", default=None)
    opt = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    tmp = tempfile.mkdtemp(prefix="dss_grow_quality_")
    try:
        data_dir = make_data(tmp, opt.views)
        res = {"fixed": run("fixed", data_dir, tmp, opt.its, 8000, [], []),
               "grown": run("grown", data_dir, tmp, opt.its, 2000, opt.milestones, [4000, 8000])}
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    gpu = card()
    res["card"], res["power_limit"] = gpu["name"], gpu["power_limit"]
    print(json.dumps(res))
    if opt.out:
        with open(opt.out, "w") as f:
            json.dump(res, f)


if __name__ == "__main__":
    sys.exit(main())
