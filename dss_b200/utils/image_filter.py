"""Filter a point cloud through its renders: render it from many views, L0-smooth the renders, fit the cloud to the
smoothed images with the differentiable renderer, and repeat -- the reference's image-filter application
(learn_image_filter.py with DSS/misc/imageFilters.py's ``L0Smooth``), on the fused training step.

    python -m dss_b200.utils.image_filter IN OUT [--views 64] [--batch 8] [--image-size 512] [--cycles 10]
                                                 [--steps 20] [--lmd 0.05] [--lambda-proj 0.01] [--seed 0]
                                                 [--save-images DIR [--save-views 4]]

IN is a PLY with normals (``python -m dss_b200.utils.normals`` estimates them for a cloud without); its colours are
used as the albedo when present, ones otherwise, and are not learnt.  The cloud is centred on its mean and scaled by
its largest point norm (as ``create_mvr_data.normalize_mesh`` does a mesh) and seen by ``--views`` cameras drawn by
``CameraSampler`` at distances 1.2 .. 2.2, each with one white directional light from ``get_light_for_view``; every
draw comes from ``--seed``.  The splats use the settings of the reference's ``configs/dss.yml`` (one h per view,
anisotropic off, cutoff 1, 5 points per pixel).  Each cycle:

1. renders every view of the current cloud (no gradients), ``--batch`` views at a time;
2. takes as targets ``l0_smooth(rgb, lmd)`` and the render's ``alpha > 0.5``;
3. runs ``--steps`` steps of the graphed training step on batches of a seeded permutation of the views, cycled
   through, with Adam (lr 0.01, betas (0.5, 0.9)) on the points and normals: RGB and silhouette losses with weight 1,
   the projection regulariser with ``--lambda-proj``, no repulsion.

OUT gets the points, mapped back to IN's frame, their unit normals and the colours, in IN's order.  ``--save-images``
writes ``c%03d_v%02d_{render,target,diff}.png`` of the first ``--save-views`` views of every cycle.  One GPU."""
import argparse
import os
import random
import sys

import numpy as np
import torch
import torch.nn.functional as F

__all__ = ["filter_cloud", "main"]


def _png(path, rgb):
    from PIL import Image
    Image.fromarray((np.clip(rgb, 0.0, 1.0) * np.float32(255.0)).astype(np.uint8)).save(path)


def filter_cloud(src, dst, views=64, batch=8, image_size=512, cycles=10, steps=20, lmd=0.05, lambda_proj=0.01,
                 seed=0, save_images=None, save_views=4, log=print):
    """``src`` -> ``dst`` as the command line does it.  Returns a list of (first, last) mean image losses, one pair per
    cycle.  Raises ValueError for a cloud without normals, ``views`` not a multiple of ``batch`` and an image size
    ``l0_smooth`` does not take, before anything is rendered."""
    from ..core.camera import CameraSampler, FoVPerspectiveCameras, camera_matrices
    from ..ops import SplatParams, l0_size_error, l0_smooth, make_shading, render_points, shared_cloud_splats
    from ..training.step import GraphedTrainStep
    from ..training.train import make_optimizer
    from .create_mvr_data import _stack_lights, get_light_for_view
    from .io import read_ply, save_ply
    views, batch, image_size, cycles, steps = int(views), int(batch), int(image_size), int(cycles), int(steps)
    if views < 1 or batch < 1 or views % batch != 0:
        raise ValueError("--views (%d) must be a positive multiple of --batch (%d)" % (views, batch))
    msg = l0_size_error(image_size)
    if msg is not None:
        raise ValueError("--image-size: " + msg)
    if cycles < 0 or steps < 0:
        raise ValueError("--cycles and --steps must be >= 0")
    d = read_ply(src)
    pts_in, nrm_in, col_in = d["points"], d["normals"], d["colors"]
    if nrm_in is None:
        raise ValueError("%s has no normals, which the renderer needs: estimate them first with "
                         "python -m dss_b200.utils.normals" % src)
    col_out = col_in if col_in is not None else np.ones_like(pts_in)
    if cycles == 0:
        save_ply(dst, pts_in, colors=col_out, normals=nrm_in)
        return []
    dev = torch.device("cuda")
    # the frame of create_mvr_data.normalize_mesh, in float64; OUT is mapped back to IN's
    p64 = pts_in.astype(np.float64)
    centre = p64.mean(0)
    scale = np.linalg.norm(p64 - centre, axis=1).max()
    points = torch.from_numpy(((p64 - centre) / scale).astype(np.float32)).to(dev)
    normals = torch.from_numpy(np.ascontiguousarray(nrm_in, dtype=np.float32)).to(dev)
    albedo = torch.from_numpy(np.ascontiguousarray(col_out[:, :3], dtype=np.float32)).to(dev)

    g = torch.Generator().manual_seed(int(seed))
    rng = random.Random(int(seed))
    cam_params = {"znear": 0.1}
    sampler = CameraSampler(views, 1, distance_range=((1.2, 2.2),), sort_distance=True,
                            camera_type=FoVPerspectiveCameras, camera_params=cam_params, generator=g)
    lights = [get_light_for_view(cam, point_lights=False, has_specular=False, rng=rng) for cam in sampler]
    proj, view = (m.to(dev) for m in camera_matrices(FoVPerspectiveCameras(R=sampler.R, T=sampler.T, **cam_params)))
    batch_lights = [_stack_lights(lights[i:i + batch]).to(dev) for i in range(0, views, batch)]
    order = torch.randperm(views, generator=g)
    params = SplatParams(image_size=image_size, points_per_pixel=5, cutoff_threshold=1.0, radii_backward_scaler=5.0,
                         clip_pts_grad=0.05, znear=0.1)
    settings = dict(learn=("points", "normals"), Vrk_invariant=True, Vrk_isotropic=False, lambda_dr_rgb=1.0,
                    lambda_dr_silhouette=1.0, lambda_dr_proj=float(lambda_proj), lambda_dr_repel=0.0)
    if save_images:
        os.makedirs(save_images, exist_ok=True)

    step = opt = None
    cursor = 0
    losses = []
    for cyc in range(cycles):
        # 1-2. the targets: the renders of the current cloud, L0-smoothed, and their silhouettes
        cur_p = points if step is None else step.points.detach()
        cur_n = normals if step is None else step.normals.detach()
        img = torch.empty((views, image_size, image_size, 3), dtype=torch.float32, device=dev)
        mask = torch.empty((views, image_size, image_size), dtype=torch.float32, device=dev)
        with torch.no_grad():
            nrm = F.normalize(cur_n, dim=-1)
            for b, v0 in enumerate(range(0, views, batch)):
                sl = slice(v0, v0 + batch)
                h, frames = shared_cloud_splats(cur_p, batch, settings["Vrk_invariant"], settings["Vrk_isotropic"])
                shading = make_shading(batch_lights[b], view[sl])
                out = render_points(cur_p, nrm, albedo, proj[sl], view[sl], h, params, shading=shading,
                                    deterministic=True, frames=frames)
                rgb = out.image[..., :3]
                img[sl] = l0_smooth(rgb, lmd)
                mask[sl] = (out.image[..., 3] > 0.5).float()
                if save_images and v0 < save_views:
                    for v in range(v0, min(v0 + batch, save_views)):
                        r, t = rgb[v - v0].cpu().numpy(), img[v].cpu().numpy()
                        base = os.path.join(save_images, "c%03d_v%02d_" % (cyc, v))
                        _png(base + "render.png", r)
                        _png(base + "target.png", t)
                        _png(base + "diff.png", np.abs(r - t))
        # 3. fit the cloud to the targets
        first = last = None
        for it in range(steps):
            idx = order[cursor * batch:(cursor + 1) * batch].to(dev)
            b_lights = _stack_lights([lights[int(i)] for i in order[cursor * batch:(cursor + 1) * batch]]).to(dev)
            cursor = (cursor + 1) % (views // batch)
            args = (img[idx], mask[idx], proj[idx], view[idx], b_lights)
            if step is None:
                step = GraphedTrainStep(points, normals, albedo, params, *args, **settings)
                opt = make_optimizer({"points": step.points, "normals": step.normals, "colours": step.colours})
            else:
                step.load(*args)
            step.replay()
            opt.step()
            if it == 0 or it == steps - 1:
                val = float(step.loss["loss_dr_rgb"] + step.loss["loss_dr_silhouette"])
                first = val if it == 0 else first
                last = val
        losses.append((first, last))
        if log is not None:
            log("cycle %d: image loss %s -> %s" % (cyc, "n/a" if first is None else "%.6f" % first,
                                                    "n/a" if last is None else "%.6f" % last))

    p_out = points if step is None else step.points.detach()
    n_out = normals if step is None else step.normals.detach()
    p_np = (p_out.double().cpu().numpy() * scale + centre).astype(np.float32)
    n_np = F.normalize(n_out, dim=-1).cpu().numpy()
    save_ply(dst, p_np, colors=col_out, normals=n_np)
    return losses


def main(argv=None):
    p = argparse.ArgumentParser(description="Filter a point cloud through its renders: render it from many views, "
                                            "L0-smooth the renders and fit the cloud to them, in cycles.")
    p.add_argument("input", help="PLY point cloud with normals (colours optional)")
    p.add_argument("output", help="PLY file of the filtered cloud")
    p.add_argument("--views", type=int, default=64, help="number of cameras (a multiple of --batch)")
    p.add_argument("--batch", type=int, default=8, help="views per render and per training step")
    p.add_argument("--image-size", type=int, default=512,
                   help="render size: 2 .. 2048 with no prime factor above 5")
    p.add_argument("--cycles", type=int, default=10, help="render-filter-fit cycles (0: write IN back unchanged)")
    p.add_argument("--steps", type=int, default=20, help="training steps per cycle")
    p.add_argument("--lmd", type=float, default=0.05, help="L0 smoothing weight: larger flattens more")
    p.add_argument("--lambda-proj", type=float, default=0.01, help="weight of the projection regulariser")
    p.add_argument("--seed", type=int, default=0, help="seed of the cameras, lights and batch order")
    p.add_argument("--save-images", default=None, metavar="DIR",
                   help="write c%%03d_v%%02d_{render,target,diff}.png of the first views of every cycle")
    p.add_argument("--save-views", type=int, default=4, help="views written per cycle with --save-images")
    args = p.parse_args(argv)
    if args.cycles > 0 and not torch.cuda.is_available():
        raise RuntimeError("filtering needs a CUDA device (sm_90a)")
    filter_cloud(args.input, args.output, args.views, args.batch, args.image_size, args.cycles, args.steps, args.lmd,
                 args.lambda_proj, args.seed, args.save_images, args.save_views)
    print(args.output)
    return 0


if __name__ == "__main__":
    sys.exit(main())
