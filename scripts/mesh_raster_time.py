"""Time ops.render_mesh (csrc/mesh_raster.cu) on a seeded displaced sphere of about 630k faces, the face count of the
reference's yoga6 mesh: 128 views at 512^2 with and without flat shading, and 8 views at 1024^2.

    python scripts/mesh_raster_time.py [--warmup 3] [--iters 10] [--save-mesh out.ply]

CUDA events around each call, median after warm-up.  Prints one JSON line with the card name and its power limit."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from dss_b200.core.camera import CameraSampler, FoVPerspectiveCameras, camera_matrices  # noqa: E402
from dss_b200.core.lighting import PointLights  # noqa: E402
from dss_b200.ops import make_shading, render_mesh  # noqa: E402


def displaced_sphere(n=562, seed=0):
    """UV sphere of n x n quads (2 n^2 triangles, 631 688 for n = 562), radius 1 + 0.05 * seeded smooth noise"""
    g = torch.Generator().manual_seed(seed)
    th = torch.linspace(0.02, 3.12, n + 1)
    ph = torch.arange(n) * (2 * torch.pi / n)
    T, P = torch.meshgrid(th, ph, indexing="ij")
    k = torch.randint(1, 8, (6, 3), generator=g).float()
    a = torch.rand(6, generator=g) - 0.5
    r = 1 + 0.05 * sum(a[i] * torch.sin(k[i, 0] * T + k[i, 1] * P + k[i, 2]) for i in range(6))
    verts = torch.stack([r * torch.sin(T) * torch.cos(P), r * torch.cos(T), r * torch.sin(T) * torch.sin(P)], -1)
    idx = torch.arange((n + 1) * n).view(n + 1, n)
    a0, a1 = idx[:-1], idx[:-1].roll(-1, 1)
    b0, b1 = idx[1:], idx[1:].roll(-1, 1)
    faces = torch.cat([torch.stack([a0, b0, b1], -1).reshape(-1, 3), torch.stack([a0, b1, a1], -1).reshape(-1, 3)])
    return verts.reshape(-1, 3).contiguous(), faces.contiguous()


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def timed(fn, warmup, iters):
    for _ in range(warmup):
        fn()
    ms = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return sorted(ms)[len(ms) // 2]


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
    res["ms_128x512_shaded"] = timed(lambda: render_mesh(v, f, proj, view, 512, shading=sh), opt.warmup, opt.iters)
    res["ms_128x512_unshaded"] = timed(lambda: render_mesh(v, f, proj, view, 512), opt.warmup, opt.iters)
    res["ms_8x1024_shaded"] = timed(lambda: render_mesh(v, f, proj[:8], view[:8], 1024, shading=make_shading(
        PointLights(location=lights.location[:8], diffuse_color=lights.diffuse_color,
                    specular_color=lights.specular_color, device=dev), view[:8])), opt.warmup, opt.iters)
    r = render_mesh(v, f, proj, view, 512)
    res["coverage_128x512"] = float((r.pix_to_face >= 0).float().mean())
    res["card"], res["power_limit"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
