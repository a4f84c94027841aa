"""Quality of training with and without the dense depth term: the loop of dss_b200.training.train at configs/dss.yml's
settings (512^2 views, 8 per batch, Vrk_invariant splats, 8000 points) on the torus data of
scripts/train_grow_quality.py, written once by create_mvr_data (which also writes the views' depth/%06d.exr), run twice
for the same iterations from the same seed:

  plain  -- training.lambda_dr_depth 0 (the depth maps are loaded but not read);
  depth  -- training.lambda_dr_depth --lambda-depth.

    python scripts/train_depth_quality.py [--its 900] [--views 64] [--lambda-depth 1.0] [--out results.json]

For each run, after the last iteration: chamfer_point and chamfer_normal against 8000 area-weighted samples of the mesh
(the loop's validation), p2f_avg (mean distance of the cloud's points to the mesh), iou (evaluate_2d at 128^2 on the
views), the last logged loss_dr_depth of the depth run, and the wall time.  Prints one JSON line with the card name and
its power limit."""
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


def run(name, data_dir, tmp, its, lam):
    from dss_b200.core.cloud import PointClouds3D
    from dss_b200.ops import chamfer_distance, evaluate_2d
    from dss_b200.training.config import load_config
    from dss_b200.training.train import Trainer
    from dss_b200.utils.evaluate import p2f_stats
    path = os.path.join(tmp, name + ".yml")
    with open(path, "w") as f:
        yaml.safe_dump({
            "name": name, "data": {"data_dir": data_dir, "load_dense_depth": True},
            "model": {"model_kwargs": {"n_points_per_cloud": 8000, "learn_colors": False}},
            "renderer": {"raster_params": {"Vrk_invariant": True, "Vrk_isotropic": False, "clip_pts_grad": 0.05,
                                           "cutoff_threshold": 1.0, "depth_merging_threshold": 0.05,
                                           "image_size": 512, "points_per_pixel": 5, "radii_backward_scaler": 5}},
            "training": {"out_dir": os.path.join(tmp, "out"), "batch_size": 8, "lambda_dr_proj": 0.01,
                         "lambda_dr_repel": 0.0, "steps_dss_backward_radii": 200, "print_every": 100,
                         "validate_every": 0, "checkpoint_every": 0, "model_selection_metric": "p2f_avg",
                         "lambda_dr_depth": lam}}, f)
    t = Trainer(load_config(path))
    torch.cuda.synchronize()
    t0 = time.time()
    t.run(exit_after=-1, max_it=its)
    torch.cuda.synchronize()
    res = {"lambda_dr_depth": lam, "seconds": time.time() - t0}
    points, normals = t.cloud()
    with torch.no_grad():
        cd_p, cd_n = chamfer_distance(PointClouds3D([t.gt[0]], [t.gt[1]]), PointClouds3D([points], [normals]))
    _, p2f, _ = p2f_stats(points, t.mesh)
    res.update(chamfer_point=float(cd_p), chamfer_normal=float(cd_n), p2f_avg=float(p2f))
    st = t.step
    ev = evaluate_2d(st.points, st.normals, st.colours, t.views, t.params, 128, 8, st.Vrk_invariant, st.Vrk_isotropic,
                     st.frnn_radius, st.shininess)
    res["iou"] = float(ev["iou"])
    if lam > 0:
        with open(os.path.join(tmp, "out", name, "metrics.jsonl")) as f:
            res["last_loss_dr_depth"] = [json.loads(line) for line in f][-1]["loss_dr_depth"]
    del t
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--its", type=int, default=900)
    ap.add_argument("--views", type=int, default=64)
    ap.add_argument("--lambda-depth", type=float, default=1.0)
    ap.add_argument("--out", default=None)
    opt = ap.parse_args()
    if not opt.lambda_depth > 0:
        raise SystemExit("--lambda-depth must be > 0")
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    tmp = tempfile.mkdtemp(prefix="dss_depth_quality_")
    try:
        data = make_data(tmp, opt.views)
        res = {"its": opt.its, "views": opt.views}
        for name, lam in (("plain", 0.0), ("depth", opt.lambda_depth)):
            res[name] = run(name, data, tmp, opt.its, lam)
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
