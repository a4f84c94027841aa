"""Export a trained cloud and its surface: the reference's ``Generator`` (DSS/models/point_modeling.py:248-326).

    python -m dss_b200.utils.generate --config CFG [--depth 8] [--model FILE]

Loads the checkpoint ``Trainer.save`` writes (``<training.out_dir>/<name>/<test.model_file>``, ``model_best.pt`` by
default, or ``--model``), keeps the points whose ``points_activation`` is set, normalises their normals and writes into
``<training.out_dir>/<name>/<generation.generation_dir>/``:
  - ``pointcloud.ply``: the points, with normals / colours as ``generation.with_normals`` / ``with_colors`` say
    (``generate_pointclouds``);
  - ``mesh.<generation.mesh_extension>`` (``ply`` or ``obj``): the screened Poisson surface of the points and their
    normals at ``--depth`` (``generate_mesh``; ``ops.poisson_reconstruction`` on the device).
The ``generation`` block is read over ``configs/default.yaml``'s values (:data:`GENERATION_DEFAULTS`)."""
import argparse
import copy
import os
import sys
import warnings

import torch

__all__ = ["GENERATION_DEFAULTS", "generation_settings", "load_cloud", "generate", "main"]

# configs/default.yaml's generation block (batch_size, vis_n_outputs, refinement_step and points_batch_size have no
# effect on a point model's export)
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


def generate(cfg, depth=8, model=None):
    """write pointcloud.ply and mesh.<ext>; returns (cloud path, mesh path, number of points, PoissonMesh)"""
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
    return cloud_path, mesh_path, points.shape[0], mesh


def main(argv=None):
    from ..training.config import load_config
    p = argparse.ArgumentParser(description="Export a trained cloud and its screened Poisson surface (Generator).")
    p.add_argument("--config", required=True, help="the training configuration (inherit_from chains over the defaults)")
    p.add_argument("--depth", type=int, default=8, help="octree depth of the reconstruction: a 2^depth grid (2 .. 9)")
    p.add_argument("--model", default=None, help="checkpoint to export (default <out_dir>/<name>/<test.model_file>)")
    args = p.parse_args(argv)
    if not torch.cuda.is_available():
        raise RuntimeError("the export needs a CUDA device (sm_90a)")
    with warnings.catch_warnings():
        # the training loop's warning about keys it ignores names the generation block this export reads
        warnings.simplefilter("ignore")
        cfg = load_config(args.config)
    cloud_path, mesh_path, n, mesh = generate(cfg, depth=args.depth, model=args.model)
    print("%s: %d points\n%s: %d vertices, %d faces (CG: %d iterations, relative residual %.2e)"
          % (cloud_path, n, mesh_path, mesh.verts.shape[0], mesh.faces.shape[0], mesh.iterations, mesh.residual))
    return 0


if __name__ == "__main__":
    sys.exit(main())
