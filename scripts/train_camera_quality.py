"""Quality of training from perturbed cameras, with and without camera refinement: the loop of
dss_b200.training.train at configs/dss.yml's settings (512^2 views, 8 per batch, Vrk_invariant splats, 8000 points) on
the torus data of scripts/train_grow_quality.py, written once with ``create_mvr_data --camera-noise DEG FRAC`` (every
pose off by a rotation of DEG degrees and a translation of FRAC of its distance to the origin), run three ways for the
same iterations from the same seed:

  true     -- the exact cameras (camera_mat_true), no refinement;
  noisy    -- the perturbed cameras, no refinement;
  refined  -- the perturbed cameras with model.model_kwargs.learn_cameras (--lr-cameras, --cameras-from-it).

    python scripts/train_camera_quality.py [--its 900] [--views 64] [--noise 1 0.01] [--lr-cameras 1e-4]
                                           [--cameras-from-it 300] [--runs true,noisy,refined] [--out results.json]

For each run, after the last iteration: chamfer_point and chamfer_normal against 8000 area-weighted samples of the mesh
(the loop's validation), p2f_avg (mean distance of the cloud's points to the mesh), and iou, evaluate_2d at 128^2 on
the views with the exact cameras; and the median and maximum rotation (degrees) and camera-centre errors of the cameras
the run ends with (refined or not) against the exact ones.  The views and the regularisers are invariant to a
similarity transform of the cloud and the cameras together, so the refined run may drift by one: its errors are also
reported after a 7-DoF Umeyama alignment of its camera centres to the true ones, and its chamfer and p2f numbers after
applying the same transform to the cloud ("aligned").  Prints one JSON line with the card name and its power limit."""
import argparse
import json
import os
import shutil
import sys
import tempfile

import numpy as np
import torch
import yaml
from scipy.spatial.transform import Rotation

from timing import card


def make_data(tmp, views, noise):
    from dss_b200.utils.create_mvr_data import main as create
    from dss_b200.utils.io import save_obj
    from tests.test_mesh_data import torus
    verts, faces = torus(nu=192, nv=96)
    save_obj(os.path.join(tmp, "torus.obj"), verts.numpy(), faces.numpy())
    noisy = create(["--points", os.path.join(tmp, "torus.obj"), "--output", os.path.join(tmp, "data"),
                    "--num_cameras", str(views), "--image-size", "512", "--tri_color_light", "--point_lights",
                    "--seed", "3", "--camera-noise", str(noise[0]), str(noise[1])])[0]
    exact = os.path.join(tmp, "exact")
    shutil.copytree(noisy, exact)
    d = dict(np.load(os.path.join(noisy, "data_dict.npz"), allow_pickle=True))
    d["camera_mat"] = d.pop("camera_mat_true")
    np.savez(os.path.join(exact, "data_dict.npz"), **d)
    return noisy, exact


def umeyama(x, y):
    """(s, A, b) of the similarity y ~ s A x + b minimising the squared error over the rows of x, y (V,3)"""
    mx, my = x.mean(0), y.mean(0)
    xc, yc = x - mx, y - my
    cov = yc.T @ xc / len(x)
    U, D, Vt = np.linalg.svd(cov)
    S = np.eye(3)
    if np.linalg.det(U) * np.linalg.det(Vt) < 0:
        S[2, 2] = -1
    A = U @ S @ Vt
    s = np.trace(np.diag(D) @ S) / (xc ** 2).sum(1).mean()
    return s, A, my - s * A @ mx


def centres(m):
    return -np.einsum("vj,vij->vi", m[:, 3, :3], m[:, :3, :3])


def pose_errors(cams, true, sim=None):
    """(rotation errors in degrees, centre distances) of world-to-view matrices (V,4,4), row-vector convention, against
    the true ones; ``sim`` = (s, A, b) maps the cameras' world into the true one first"""
    R, c = cams[:, :3, :3], centres(cams)
    if sim is not None:
        s, A, b = sim
        R, c = np.einsum("ij,vjk->vik", A, R), s * c @ A.T + b
    rel = np.einsum("vji,vjk->vik", true[:, :3, :3], R)
    return np.degrees(Rotation.from_matrix(rel).magnitude()), np.linalg.norm(c - centres(true), axis=1)


def summary(rot, tr):
    return {"rot_median_deg": float(np.median(rot)), "rot_max_deg": float(rot.max()),
            "trans_median": float(np.median(tr)), "trans_max": float(tr.max())}


def run(name, data_dir, exact_dir, true, tmp, opt, learn):
    from dss_b200.core.cloud import PointClouds3D
    from dss_b200.ops import chamfer_distance, evaluate_2d
    from dss_b200.training.config import load_config
    from dss_b200.training.train import Trainer
    from dss_b200.utils.dataset import MVRData
    from dss_b200.utils.evaluate import p2f_stats
    path = os.path.join(tmp, name + ".yml")
    with open(path, "w") as f:
        yaml.safe_dump({
            "name": name, "data": {"data_dir": data_dir},
            "model": {"model_kwargs": {"n_points_per_cloud": 8000, "learn_colors": False, "learn_cameras": learn}},
            "renderer": {"raster_params": {"Vrk_invariant": True, "Vrk_isotropic": False, "clip_pts_grad": 0.05,
                                           "cutoff_threshold": 1.0, "depth_merging_threshold": 0.05,
                                           "image_size": 512, "points_per_pixel": 5, "radii_backward_scaler": 5}},
            "training": {"out_dir": os.path.join(tmp, "out"), "batch_size": 8, "lambda_dr_proj": 0.01,
                         "lambda_dr_repel": 0.0, "steps_dss_backward_radii": 200, "print_every": 100,
                         "validate_every": 0, "checkpoint_every": 0, "model_selection_metric": "p2f_avg",
                         "lr_cameras": opt.lr_cameras, "cameras_from_it": opt.cameras_from_it}}, f)
    t = Trainer(load_config(path))
    t.run(exit_after=-1, max_it=opt.its)
    cams = (t.views_now().camera_mat if learn else t.views.camera_mat).cpu().numpy().astype(np.float64)
    points, normals = t.cloud()
    res = {"raw": {}, "aligned": {}}
    res["poses_before"] = summary(*pose_errors(t.views.camera_mat.cpu().numpy().astype(np.float64), true))
    res["poses_after"] = summary(*pose_errors(cams, true))
    sim = umeyama(centres(cams), centres(true))
    res["poses_after_aligned"] = summary(*pose_errors(cams, true, sim))
    res["similarity"] = {"scale": float(sim[0]), "rotation_deg": float(np.degrees(Rotation.from_matrix(sim[1]).magnitude())),
                         "translation": float(np.linalg.norm(sim[2]))}
    s, A, b = (torch.as_tensor(v, dtype=torch.float32, device=points.device) for v in sim)
    for key, (p, n) in (("raw", (points, normals)), ("aligned", (s * points @ A.T + b, normals @ A.T))):
        with torch.no_grad():
            cd_p, cd_n = chamfer_distance(PointClouds3D([t.gt[0]], [t.gt[1]]), PointClouds3D([p], [n]))
        _, p2f, _ = p2f_stats(p, t.mesh)
        res[key] = {"chamfer_point": float(cd_p), "chamfer_normal": float(cd_n), "p2f_avg": float(p2f)}
    st = t.step
    ev = evaluate_2d(st.points, st.normals, st.colours, MVRData(exact_dir), t.params, 128, 8, st.Vrk_invariant,
                     st.Vrk_isotropic, st.frnn_radius, st.shininess)
    res["iou"] = float(ev["iou"])
    del t
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--its", type=int, default=900)
    ap.add_argument("--views", type=int, default=64)
    ap.add_argument("--noise", type=float, nargs=2, default=[1.0, 0.01])
    ap.add_argument("--lr-cameras", type=float, default=1e-4)
    ap.add_argument("--cameras-from-it", type=int, default=300)
    ap.add_argument("--runs", default="true,noisy,refined", help="which of the three runs to make")
    ap.add_argument("--out", default=None)
    opt = ap.parse_args()
    runs = opt.runs.split(",")
    if not set(runs) <= {"true", "noisy", "refined"}:
        raise SystemExit("--runs takes true, noisy and refined, got %r" % opt.runs)
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    tmp = tempfile.mkdtemp(prefix="dss_camera_quality_")
    try:
        noisy, exact = make_data(tmp, opt.views, opt.noise)
        true = np.load(os.path.join(noisy, "data_dict.npz"), allow_pickle=True)["camera_mat_true"].astype(np.float64)
        res = {"noise": opt.noise, "its": opt.its, "lr_cameras": opt.lr_cameras,
               "cameras_from_it": opt.cameras_from_it}
        for name, src, learn in (("true", exact, False), ("noisy", noisy, False), ("refined", noisy, True)):
            if name in runs:
                res[name] = run(name, src, exact, true, tmp, opt, learn)
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
