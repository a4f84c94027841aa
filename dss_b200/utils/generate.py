"""Export a trained cloud and its surface: the reference's ``Generator`` (DSS/models/point_modeling.py:248-326).

    python -m dss_b200.utils.generate --config CFG [--depth 8] [--model FILE] [--images]

Loads the checkpoint ``Trainer.save`` writes (``<training.out_dir>/<name>/<test.model_file>``, ``model_best.pt`` by
default, or ``--model``), keeps the points whose ``points_activation`` is set, normalises their normals and writes into
``<training.out_dir>/<name>/<generation.generation_dir>/``:
  - ``pointcloud.ply``: the points, with normals / colours as ``generation.with_normals`` / ``with_colors`` say
    (``generate_pointclouds``);
  - ``mesh.<generation.mesh_extension>`` (``ply`` or ``obj``): the screened Poisson surface of the points and their
    normals at ``--depth`` (``generate_mesh``; ``ops.poisson_reconstruction`` on the device);
  - with ``--images`` (:func:`generate_images`): ``images/%04d.png``, the renders of the data's first
    ``generation.vis_n_outputs`` views at the data's resolution S, clipped to [0, 1] (``generate_images``,
    point_modeling.py:335-348), and ``image_metrics.json``, the ``evaluate_2d`` metrics of every view at S // 4 (the
    training loop's validation size) and at S.  When the checkpoint holds camera poses (a run with
    ``model.model_kwargs.learn_cameras``), the views are rendered and scored with the refined cameras, and
    ``cameras.npz`` holds their ``camera_mat`` (V,4,4) float32, in ``data_dict.npz``'s layout.
The ``generation`` block is read over ``configs/default.yaml``'s values (:data:`GENERATION_DEFAULTS`)."""
import argparse
import copy
import os
import sys
import warnings

import torch

__all__ = ["GENERATION_DEFAULTS", "generation_settings", "load_cloud", "load_poses", "generate", "generate_images",
           "main"]

# configs/default.yaml's generation block (refinement_step and points_batch_size have no effect on a point model's
# export; batch_size is the number of views --images renders at once, vis_n_outputs how many it writes)
GENERATION_DEFAULTS = {"batch_size": 1, "vis_n_outputs": 30, "generation_dir": "generation", "refinement_step": -1,
                       "points_batch_size": 100000, "with_colors": True, "with_normals": True, "mesh_extension": "ply"}


def generation_settings(cfg):
    """the configuration's ``generation`` block over :data:`GENERATION_DEFAULTS`"""
    g = copy.deepcopy(GENERATION_DEFAULTS)
    g.update(cfg.get("generation") or {})
    if str(g["mesh_extension"]).lower() not in ("ply", "obj"):
        raise ValueError("generation.mesh_extension must be 'ply' or 'obj', got %r" % g["mesh_extension"])
    return g


def load_cloud(path, device):
    """(points, unit normals, colours) of the active points of a ``Trainer.save`` checkpoint, on ``device``"""
    ckpt = torch.load(path, map_location=device, weights_only=False)
    m = ckpt["model"]
    points, normals, colours = m["points"][0], m["normals"][0], m["colors"][0]
    active = m.get("points_activation")
    if active is not None:
        keep = active[0].to(torch.bool)
        points, normals, colours = points[keep], normals[keep], colours[keep]
    normals = torch.nn.functional.normalize(normals, dim=-1)
    return points.float().contiguous(), normals.float().contiguous(), colours.float().contiguous()


def load_poses(path, device):
    """the (V,6) camera poses of a ``Trainer.save`` checkpoint on ``device``, or None when it holds none"""
    ckpt = torch.load(path, map_location=device, weights_only=False)
    cams = ckpt.get("cameras")
    return None if cams is None else cams["poses"].float().contiguous()


def generate(cfg, depth=8, model=None, images=False):
    """write pointcloud.ply and mesh.<ext> (and, with ``images``, what :func:`generate_images` writes); returns (cloud
    path, mesh path, number of points, PoissonMesh)"""
    from ..ops import poisson_reconstruction
    from .io import save_obj, save_ply
    out_dir = os.path.join(str(cfg["training"]["out_dir"]), str(cfg["name"]))
    g = generation_settings(cfg)
    path = model if model is not None else os.path.join(out_dir, str((cfg.get("test") or {}).get("model_file",
                                                                                                 "model_best.pt")))
    points, normals, colours = load_cloud(path, torch.device("cuda", torch.cuda.current_device()))
    gen_dir = os.path.join(out_dir, str(g["generation_dir"]))
    os.makedirs(gen_dir, exist_ok=True)
    cloud_path = os.path.join(gen_dir, "pointcloud.ply")
    save_ply(cloud_path, points.cpu().numpy(), colors=colours.cpu().numpy() if g["with_colors"] else None,
             normals=normals.cpu().numpy() if g["with_normals"] else None)
    mesh = poisson_reconstruction(points, normals, depth=depth)
    ext = str(g["mesh_extension"]).lower()
    mesh_path = os.path.join(gen_dir, "mesh." + ext)
    if ext == "ply":
        save_ply(mesh_path, mesh.verts.cpu().numpy(), faces=mesh.faces.cpu().numpy())
    else:
        save_obj(mesh_path, mesh.verts.cpu().numpy(), mesh.faces.cpu().numpy())
    if images:
        generate_images(cfg, points, normals, colours, gen_dir, load_poses(path, points.device))
    return cloud_path, mesh_path, points.shape[0], mesh


def generate_images(cfg, points, normals, colours, gen_dir, poses=None):
    """``<gen_dir>/images/%04d.png`` (RGBA, ``uint8(255 c)`` of c clipped to [0, 1]) for the first ``vis_n_outputs``
    views of the configuration's data at its resolution S, rendered as the training step renders them, and
    ``<gen_dir>/image_metrics.json``: for s = S // 4 and s = S, ``iou`` and ``psnr`` (the reference's names: 1 - IoU
    and the squared RGB error summed over the channels, per pixel) and ``psnr_db`` = -10 log10(psnr / 3), the PSNR in
    dB of the per-channel mean squared error of images in [0, 1] (null when the error is 0), per view and as their means
    over the views.  ``poses``: (V,6) camera corrections of the data's views; the views are then rendered and scored
    with the refined cameras (``DeviceViews.with_poses``), whose world-to-view matrices go to ``<gen_dir>/cameras.npz``
    as ``camera_mat`` (V,4,4) float32.  With the images, ``<gen_dir>/depth/%04d.exr``: their depth maps
    (``render_points(..., depth=True)``: the blend's view-space depth, 0 where no splat covers the pixel), one float32
    ``Y`` channel, ZIP compressed.  Returns (the PNG paths, the JSON path)."""
    import json
    import math

    import numpy as np
    from PIL import Image

    from ..ops import evaluate_2d, render_data_views
    from .io import write_exr
    from ..training.config import splat_params, step_settings
    from ..training.train import load_data
    g = generation_settings(cfg)
    data = load_data(cfg)
    cams = data.get_cameras()
    S = int(data.resolution[0])
    params = splat_params(cfg, cams.znear, cams.zfar)._replace(image_size=S)
    st = step_settings(cfg)
    flags = (st["Vrk_invariant"], st["Vrk_isotropic"])
    V, B = len(data), max(1, int(g["batch_size"]))
    if poses is not None:
        if tuple(poses.shape) != (V, 6):
            raise ValueError("the checkpoint holds camera poses of shape %s, but the data has %d views"
                             % (tuple(poses.shape), V))
        data = data.device_views(points.device).with_poses(poses)
        np.savez(os.path.join(gen_dir, "cameras.npz"), camera_mat=data.camera_mat.cpu().numpy())
    img_dir, depth_dir = os.path.join(gen_dir, "images"), os.path.join(gen_dir, "depth")
    os.makedirs(img_dir, exist_ok=True)
    os.makedirs(depth_dir, exist_ok=True)
    pngs = []
    n_out = min(max(0, int(g["vis_n_outputs"])), V)
    for i in range(0, n_out, B):
        views = list(range(i, min(i + B, n_out)))
        rgba, depth = render_data_views(points, normals, colours, data, params, views, *flags, depth=True)
        rgba, depth = rgba.clamp(0, 1).cpu().numpy(), depth.cpu().numpy()
        for v, img, d in zip(views, rgba, depth):
            pngs.append(os.path.join(img_dir, "%04d.png" % v))
            Image.fromarray((255 * img).astype(np.uint8)).save(pngs[-1])
            write_exr(os.path.join(depth_dir, "%04d.exr" % v), d)
    db = lambda e: -10.0 * math.log10(e / 3.0) if e > 0 else None
    report = {"views": V, "resolution": S, "metrics": []}
    for s in (max(1, S // 4), S):
        ev = evaluate_2d(points, normals, colours, data, params, s, B, *flags)
        rows = ev["per_view"].cpu().tolist()
        per_db = [db(r[4]) for r in rows]
        finite = [d for d in per_db if d is not None]
        report["metrics"].append({
            "image_size": s, "iou": float(ev["iou"]), "psnr": float(ev["psnr"]),
            "psnr_db": sum(finite) / len(finite) if finite else None,
            "per_view": {"iou": [r[3] for r in rows], "psnr": [r[4] for r in rows], "psnr_db": per_db}})
    path = os.path.join(gen_dir, "image_metrics.json")
    with open(path, "w") as f:
        json.dump(report, f, indent=1)
    return pngs, path


def main(argv=None):
    from ..training.config import load_config
    p = argparse.ArgumentParser(description="Export a trained cloud and its screened Poisson surface (Generator).")
    p.add_argument("--config", required=True, help="the training configuration (inherit_from chains over the defaults)")
    p.add_argument("--depth", type=int, default=8, help="octree depth of the reconstruction: a 2^depth grid (2 .. 9)")
    p.add_argument("--model", default=None, help="checkpoint to export (default <out_dir>/<name>/<test.model_file>)")
    p.add_argument("--images", action="store_true",
                   help="also write images/%%04d.png (the first generation.vis_n_outputs views) and image_metrics.json")
    args = p.parse_args(argv)
    if not torch.cuda.is_available():
        raise RuntimeError("the export needs a CUDA device (sm_90a)")
    with warnings.catch_warnings():
        # the training loop's warning about keys it ignores names the generation block this export reads
        warnings.simplefilter("ignore")
        cfg = load_config(args.config)
    cloud_path, mesh_path, n, mesh = generate(cfg, depth=args.depth, model=args.model, images=args.images)
    print("%s: %d points\n%s: %d vertices, %d faces (CG: %d iterations, relative residual %.2e)"
          % (cloud_path, n, mesh_path, mesh.verts.shape[0], mesh.faces.shape[0], mesh.iterations, mesh.residual))
    return 0


if __name__ == "__main__":
    sys.exit(main())
