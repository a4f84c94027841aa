"""Time ops.render_mesh (csrc/mesh_raster.cu) on a seeded displaced sphere of about 630k faces, the face count of the
reference's yoga6 mesh: 128 views at 512^2 with and without flat shading, and 8 views at 1024^2.

    python scripts/mesh_raster_time.py [--warmup 3] [--iters 10] [--save-mesh out.ply]

CUDA events around each call, median after warm-up.  Prints one JSON line with the card name and its power limit."""
import argparse
import json

import torch

from timing import card, median_ms
from meshes import displaced_sphere
from dss_b200.core.camera import CameraSampler, FoVPerspectiveCameras, camera_matrices
from dss_b200.core.lighting import PointLights
from dss_b200.ops import make_shading, render_mesh


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--save-mesh", default=None)
    opt = ap.parse_args()
    dev = torch.device("cuda:0")
    verts, faces = displaced_sphere()
    if opt.save_mesh:
        from dss_b200.utils.io import save_obj
        save_obj(opt.save_mesh, verts.numpy(), faces.numpy())
    v, f = verts.to(dev), faces.to(dev)
    sampler = CameraSampler(128, 128, distance_range=((2.4, 4.4),), camera_type=FoVPerspectiveCameras,
                            camera_params={"znear": 0.1}, generator=torch.Generator().manual_seed(1))
    proj, view = (t.to(dev) for t in camera_matrices(next(sampler)))
    lights = PointLights(location=torch.randn(128, 3, 3, generator=torch.Generator().manual_seed(2)) * 5,
                         diffuse_color=torch.full((1, 3, 3), 0.3), specular_color=torch.full((1, 3, 3), 0.1), device=dev)
    sh = make_shading(lights, view)
    res = {"faces": int(faces.shape[0]), "verts": int(verts.shape[0])}
    timed = lambda fn: median_ms(fn, opt.warmup, opt.iters)
    res["ms_128x512_shaded"] = timed(lambda: render_mesh(v, f, proj, view, 512, shading=sh))
    res["ms_128x512_unshaded"] = timed(lambda: render_mesh(v, f, proj, view, 512))
    res["ms_8x1024_shaded"] = timed(lambda: render_mesh(v, f, proj[:8], view[:8], 1024, shading=make_shading(
        PointLights(location=lights.location[:8], diffuse_color=lights.diffuse_color,
                    specular_color=lights.specular_color, device=dev), view[:8])))
    r = render_mesh(v, f, proj, view, 512)
    res["coverage_128x512"] = float((r.pix_to_face >= 0).float().mean())
    gpu = card()
    res["card"], res["power_limit"] = gpu["name"], gpu["power_limit"]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
