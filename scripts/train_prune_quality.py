"""Quality and time of pruning the cloud during training: the loop of dss_b200.training.train on the data, settings
and iterations of scripts/train_grow_quality.py (a rendered torus, 512^2 views, 8 per batch, Vrk_invariant splats),
three runs from the same seed:

  fixed  -- n_points_per_cloud 8000 throughout;
  grown  -- 2000 points, grown to 4000 and 8000 at --milestones (training.grow_milestones / grow_points);
  pruned -- the same growth with a prune at each growth milestone (training.prune_milestones, the default tests:
            seen in at least 1 view, over background in none), run before the growth.

    python scripts/train_prune_quality.py [--its 900] [--milestones 300 600] [--views 64] [--out results.json]

For each run: chamfer_point, chamfer_normal and p2f_avg after the last iteration and the wall-clock time of the
iterations, as train_grow_quality.py measures them.  For the grown runs, at each growth: the mean squared distance to
the mesh of the points that were there and of the new ones; for the pruned run, at each prune: the points removed, how
many failed each test, and the event's time (host clock to a device synchronisation).  Prints one JSON line with the
card name and its power limit."""
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
from train_grow_quality import make_data


def run(name, data_dir, tmp, its, n0, milestones, sizes, prune):
    from dss_b200.ops import point_coverage, point_mesh_distance
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
                         "grow_milestones": list(milestones), "grow_points": list(sizes),
                         "prune_milestones": list(milestones) if prune else []}}, f)
    t = Trainer(load_config(path))
    events = []
    grow, prune_event = t.grow, t.prune

    def sq_dist(points):
        return float(point_mesh_distance(points.float(), t.mesh[0], t.mesh[1]).sq_dists.double().mean())

    def timed_grow(n):
        P = t.step.points.shape[0]
        grow(n)
        pts = t.step.points.detach()
        events.append({"event": "grow", "it": t.it, "from": P, "to": n, "old_sq_dist": sq_dist(pts[:P]),
                       "new_sq_dist": sq_dist(pts[P:])})

    def timed_prune():
        st = t.step
        P = st.points.shape[0]
        # the counts the event decides on, taken apart by test (outside the timed event)
        cov = point_coverage(st.points.detach(), st.normals.detach(), t.views, t.params, t.batch_size, None,
                             st.Vrk_invariant, st.Vrk_isotropic, st.frnn_radius)
        few, over = cov.seen < t.prune_min_views, cov.outside > t.prune_max_outside
        st = None
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        prune_event()
        torch.cuda.synchronize()
        events.append({"event": "prune", "it": t.it, "from": P, "to": int(t.step.points.shape[0]),
                       "unseen": int(few.sum()), "outside": int(over.sum()), "both": int((few & over).sum()),
                       "ms": (time.perf_counter() - t0) * 1e3})

    t.grow, t.prune = timed_grow, timed_prune
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    t.run(exit_after=-1, max_it=its)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    ev = t.evaluate()
    res = {"points_start": n0, "points_end": int(t.step.points.shape[0]), "its": its, "wall_s": wall,
           "chamfer_point": ev["chamfer_point"], "chamfer_normal": ev["chamfer_normal"], "p2f_avg": ev["p2f_avg"],
           "events": events}
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
    tmp = tempfile.mkdtemp(prefix="dss_prune_quality_")
    try:
        data_dir = make_data(tmp, opt.views)
        res = {"fixed": run("fixed", data_dir, tmp, opt.its, 8000, [], [], False),
               "grown": run("grown", data_dir, tmp, opt.its, 2000, opt.milestones, [4000, 8000], False),
               "pruned": run("pruned", data_dir, tmp, opt.its, 2000, opt.milestones, [4000, 8000], True)}
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
