"""Multi-view training data from a triangle mesh: the twin of the reference's scripts/create_mvr_data_from_mesh.py.

    python -m dss_b200.utils.create_mvr_data --points mesh.ply --output data --num_cameras 128 --image-size 512 \\
        --tri_color_light --point_lights --has_specular [--seed 0]

For every mesh it writes ``<output>/<name>_variational_light/``, the directory ``MVRData`` reads:

- ``mesh.obj``: the mesh centred on its vertex mean and scaled by its largest vertex norm;
- ``image/%06d.png``: RGBA, ``uint8(255 c)`` truncated as the reference's ``astype('uint8')``, c clamped to [0, 1]
  first (the reference's cast of values above 1 is undefined);
- ``mask/%06d.png``: 8-bit 0 / 255 coverage;
- ``depth/%06d.exr``: the view-space depth of the closest face (``render_mesh``'s z-buffer) where the mesh covers the
  pixel and the cameras' ``zfar`` elsewhere, one float32 ``Y`` channel, ZIP compressed (``utils.io.write_exr``), as
  the reference writes it (create_mvr_data_from_mesh.py:215-219, 240-242);
- ``data_dict.npz``: ``points``, ``normals``, ``colors`` (ones) of 20 000 surface samples, ``camera_mat`` (V,4,4)
  row-vector world-to-view matrices, ``lights_%d`` per image, ``cameras_type``, ``cameras_params`` and ``lights_type``.

The images are rendered on the GPU by ``render_mesh`` (flat shading, one light set per image).  Not written: the
DVR-only ``cameras.npz`` / ``pcl.npz``.  All randomness comes from ``--seed`` (a ``torch.Generator`` for the cameras, the
tri-colour light frames and the surface samples, a ``random.Random`` for the single-light draws); the reference's own
random draws are not reproduced.
"""
import argparse
import glob
import math
import os
import random

import numpy as np
import torch
import torch.nn.functional as F

from ..core.camera import CameraSampler, FoVPerspectiveCameras, camera_matrices, look_at_rotation
from ..core.lighting import DirectionalLights, PointLights
from .io import read_mesh, save_obj, write_exr

__all__ = ["get_tri_color_lights_for_view", "get_light_for_view", "light_value_dict", "sample_points_from_mesh",
           "ico_sphere", "normalize_mesh", "write_mvr_data", "create_mvr_data", "main"]

CAMERAS_TYPE = "pytorch3d.renderer.cameras.FoVPerspectiveCameras"
LIGHTS_TYPE = {False: "DSS.core.lighting.DirectionalLights", True: "DSS.core.lighting.PointLights"}


def get_tri_color_lights_for_view(cams, has_specular=False, point_lights=True, generator=None):
    """Three lights (blue right, green left, red bottom) at elevation 30 and azimuths -60, 60, 180 degrees of a frame
    that looks from the origin along normalize(cross(C, u)), u uniform in [0, 1)^3, with C the camera centre as its up
    vector (the reference's common.py:47-98).  Ambient 0.2; diffuse 0.8 per channel, or 0.68 with a specular 0.12
    (``has_specular``).  Point lights sit at 5x the direction.  ``cams`` of batch 1."""
    elev = torch.tensor(((30.0, 30.0, 30.0),)) * (math.pi / 180.0)
    azim = torch.tensor(((-60.0, 60.0, 180.0),)) * (math.pi / 180.0)
    dirs = torch.stack([torch.cos(elev) * torch.sin(azim), torch.sin(elev), torch.cos(elev) * torch.cos(azim)], -1)
    cam_pos = cams.get_camera_center().float().cpu()
    u = torch.rand(cam_pos.shape, generator=generator)
    R = look_at_rotation(torch.zeros_like(cam_pos), at=F.normalize(torch.cross(cam_pos, u, dim=-1), dim=-1), up=cam_pos)
    dirs = dirs @ R.transpose(1, 2)   # pytorch3d Rotate(R=R^T).transform_points: X @ R^T
    ambient = torch.tensor((((0.2, 0.2, 0.2),),))
    diffuse = torch.tensor((((0.0, 0.0, 0.8), (0.0, 0.8, 0.0), (0.8, 0.0, 0.0)),))
    if has_specular:
        specular = 0.15 * diffuse
        diffuse = diffuse * 0.85
    else:
        specular = torch.zeros(1, 3, 3)
    if point_lights:
        return PointLights(ambient_color=ambient, diffuse_color=diffuse, specular_color=specular, location=dirs * 5)
    return DirectionalLights(ambient_color=ambient, diffuse_color=diffuse, specular_color=specular, direction=dirs)


def get_light_for_view(cams, point_lights, has_specular, rng=random):
    """One white light (ambient 0.6, diffuse 0.2, or 0.17 with a specular 0.03) at an elevation drawn from
    randint(10, 90) and an azimuth from randint(0, 360) degrees (the reference's common.py:100-124, draws from ``rng``).

    The direction is drawn in the camera's frame and taken to the world with the inverse world-to-view transform
    applied as to a POINT: the camera's translation is added to a direction.  That is the reference's behaviour and is
    kept, so that the data match; the light then need not point where the camera-frame angles say."""
    ambient = torch.tensor((((0.6, 0.6, 0.6),),))
    diffuse = torch.tensor((((0.2, 0.2, 0.2),),))
    if has_specular:
        specular = 0.15 * diffuse
        diffuse = diffuse * 0.85
    else:
        specular = torch.zeros(1, 1, 3)
    elev = torch.tensor(((float(rng.randint(10, 90)),),)) * (math.pi / 180.0)
    azim = torch.tensor(((float(rng.randint(0, 360)),),)) * (math.pi / 180.0)
    d = torch.stack([torch.cos(elev) * torch.sin(azim), torch.sin(elev), torch.cos(elev) * torch.cos(azim)], -1)
    w2v = cams.get_world_to_view_transform().get_matrix().float().cpu()
    hom = torch.cat([d, torch.ones_like(d[..., :1])], -1) @ torch.inverse(w2v)
    d = hom[..., :3] / hom[..., 3:]
    if point_lights:
        return PointLights(ambient_color=ambient, diffuse_color=diffuse, specular_color=specular, location=d * 5)
    return DirectionalLights(ambient_color=ambient, diffuse_color=diffuse, specular_color=specular, direction=d)


def light_value_dict(lights):
    """The dict the reference's ``convert_tensor_property_to_value_dict`` stores per image (DSS/utils/__init__.py:
    102-117): the lights' tensors as numpy arrays of shape (1, L, 3)."""
    vec = "location" if isinstance(lights, PointLights) else "direction"
    return {"ambient_color": lights.ambient_color.detach().cpu().numpy(),
            "diffuse_color": lights.diffuse_color.detach().cpu().numpy(),
            "specular_color": lights.specular_color.detach().cpu().numpy(),
            vec: lights._vec.detach().cpu().numpy()}


def _stack_lights(lights_list):
    """lights of batch 1 per view -> one lights object of batch N (one set per view)"""
    cat = lambda name: torch.cat([getattr(l, name) for l in lights_list], 0)
    kind = type(lights_list[0])
    kw = {"location" if kind is PointLights else "direction": cat("_vec")}
    return kind(ambient_color=cat("ambient_color"), diffuse_color=cat("diffuse_color"),
                specular_color=cat("specular_color"), **kw)


def sample_points_from_mesh(verts, faces, num_samples, generator=None):
    """Uniform surface samples as pytorch3d's ``sample_points_from_meshes`` draws them: faces with probability
    proportional to their area, then w0 = 1 - sqrt(u), w1 = sqrt(u)(1 - v), w2 = sqrt(u) v; each sample's normal is its
    face's unit normal normalize(cross(v1 - v0, v2 - v0)).  Runs on the tensors' device.  Returns (points, normals)."""
    v0, v1, v2 = (verts[faces[:, k]] for k in range(3))
    cross = torch.cross(v1 - v0, v2 - v0, dim=1)
    areas = cross.norm(dim=1) * 0.5
    fidx = torch.multinomial(areas, num_samples, replacement=True, generator=generator)
    u = torch.rand(num_samples, 1, device=verts.device, generator=generator)
    v = torch.rand(num_samples, 1, device=verts.device, generator=generator)
    su = u.sqrt()
    w0, w1, w2 = 1.0 - su, su * (1.0 - v), su * v
    points = w0 * v0[fidx] + w1 * v1[fidx] + w2 * v2[fidx]
    normals = F.normalize(cross, dim=1, eps=1e-6)[fidx]
    return points, normals


_ICO_T = (1.0 + 5.0 ** 0.5) / 2.0
_ICO_VERTS = ((-1, _ICO_T, 0), (1, _ICO_T, 0), (-1, -_ICO_T, 0), (1, -_ICO_T, 0), (0, -1, _ICO_T), (0, 1, _ICO_T),
              (0, -1, -_ICO_T), (0, 1, -_ICO_T), (_ICO_T, 0, -1), (_ICO_T, 0, 1), (-_ICO_T, 0, -1), (-_ICO_T, 0, 1))
_ICO_FACES = ((0, 11, 5), (0, 5, 1), (0, 1, 7), (0, 7, 10), (0, 10, 11), (1, 5, 9), (5, 11, 4), (11, 10, 2),
              (10, 7, 6), (7, 1, 8), (3, 9, 4), (3, 4, 2), (3, 2, 6), (3, 6, 8), (3, 8, 9), (4, 9, 5), (2, 4, 11),
              (6, 2, 10), (8, 6, 7), (9, 8, 1))


def ico_sphere(level=0):
    """Unit icosphere as pytorch3d's ``ico_sphere(level)`` builds it: the icosahedron, then ``level`` times every face
    split into four at its edge midpoints, the new vertices pushed onto the unit sphere.  10 4^level + 2 vertices,
    20 4^level faces, counter-clockwise seen from outside.  Returns (verts (V,3) float32, faces (F,3) int64) on the
    CPU."""
    verts = torch.tensor(_ICO_VERTS, dtype=torch.float64)
    verts = verts / verts.norm(dim=1, keepdim=True)
    faces = torch.tensor(_ICO_FACES, dtype=torch.int64)
    for _ in range(int(level)):
        F_, V = faces.shape[0], verts.shape[0]
        edges = torch.cat([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]]).sort(dim=1).values
        unique, inverse = torch.unique(edges, dim=0, return_inverse=True)
        mid = verts[unique[:, 0]] + verts[unique[:, 1]]
        verts = torch.cat([verts, mid / mid.norm(dim=1, keepdim=True)])
        ab, bc, ca = (inverse[k * F_:(k + 1) * F_] + V for k in range(3))
        a, b, c = faces.unbind(1)
        faces = torch.cat([torch.stack(f, 1) for f in ((a, ab, ca), (b, bc, ab), (c, ca, bc), (ab, bc, ca))])
    return verts.float(), faces


def normalize_mesh(verts):
    """Centre on the vertex mean and scale by the largest vertex norm (the reference's 'unit sphere' normalisation)."""
    verts = verts - verts.mean(0)
    return verts / verts.norm(dim=1).max()


def perturb_cameras(camera_mat, degrees, frac, seed=0):
    """``camera_mat`` (V,4,4) world-to-view matrices (row-vector convention) with every pose perturbed in its camera
    frame, as the pose refinement corrects it (``view E``, E = [[R, 0], [t, 1]]): R a rotation of exactly ``degrees``
    about a uniformly random axis and t a uniformly random direction of length ``frac`` times the camera's distance to
    the origin, which is then how far the camera centre moves.  Drawn from ``numpy.random.default_rng(seed)``,
    computed in float64; returns float32 (V,4,4)."""
    m = np.asarray(camera_mat, dtype=np.float64)
    V = m.shape[0]
    rng = np.random.default_rng(int(seed))
    unit = lambda x: x / np.linalg.norm(x, axis=1, keepdims=True)
    axis, direction = unit(rng.standard_normal((V, 3))), unit(rng.standard_normal((V, 3)))
    centres = -np.einsum("vj,vij->vi", m[:, 3, :3], m[:, :3, :3])          # c R + t = 0
    th = np.deg2rad(float(degrees))
    out = m.copy()
    for v in range(V):
        k = axis[v]
        K = np.array([[0.0, -k[2], k[1]], [k[2], 0.0, -k[0]], [-k[1], k[0], 0.0]])
        E = np.eye(4)
        E[:3, :3] = np.eye(3) + np.sin(th) * K + (1.0 - np.cos(th)) * (K @ K)
        E[3, :3] = float(frac) * np.linalg.norm(centres[v]) * direction[v]
        out[v] = m[v] @ E
    return out.astype(np.float32)


def write_mvr_data(output_dir, verts, faces, images, masks, camera_mat, lights, points, normals, point_lights,
                   camera_params, camera_mat_true=None, depths=None):
    """Write the data directory from renders already made (host arrays): images (N,S,S,4) float in [0,1]-ish, masks
    (N,S,S) bool, camera_mat (N,4,4), lights a list of N ``light_value_dict`` dicts, points / normals (P,3),
    ``camera_mat_true`` (N,4,4), the cameras the images were rendered from when ``camera_mat`` is not, and ``depths``
    (N,S,S) float32, the dense depth maps, written to ``depth/%06d.exr`` when given.  Returns ``output_dir``."""
    from PIL import Image
    rgb_dir, mask_dir = os.path.join(output_dir, "image"), os.path.join(output_dir, "mask")
    os.makedirs(rgb_dir, exist_ok=True)
    os.makedirs(mask_dir, exist_ok=True)
    save_obj(os.path.join(output_dir, "mesh.obj"), verts, faces)
    images = np.asarray(images, dtype=np.float32)
    masks = np.asarray(masks).astype(bool)
    for i in range(len(images)):
        rgba = (np.clip(images[i], 0.0, 1.0) * np.float32(255.0)).astype(np.uint8)
        Image.fromarray(rgba).save(os.path.join(rgb_dir, "%06d.png" % i))
        Image.fromarray(masks[i].astype(np.uint8) * 255).save(os.path.join(mask_dir, "%06d.png" % i))
    if depths is not None:
        depth_dir = os.path.join(output_dir, "depth")
        os.makedirs(depth_dir, exist_ok=True)
        for i, d in enumerate(np.asarray(depths, dtype=np.float32)):
            write_exr(os.path.join(depth_dir, "%06d.exr" % i), d)
    points = np.asarray(points, dtype=np.float32)
    data = {"cameras_type": CAMERAS_TYPE, "cameras_params": dict(camera_params), "lights_type": LIGHTS_TYPE[bool(point_lights)],
            "points": points, "normals": np.asarray(normals, dtype=np.float32),
            "colors": np.ones_like(points, dtype=np.float32), "camera_mat": np.asarray(camera_mat, dtype=np.float32)}
    if camera_mat_true is not None:
        data["camera_mat_true"] = np.asarray(camera_mat_true, dtype=np.float32)
    for i, d in enumerate(lights):
        data["lights_%d" % i] = d
    np.savez(os.path.join(output_dir, "data_dict.npz"), **data)
    return output_dir


def create_mvr_data(mesh_path, output, num_cameras=120, image_size=512, tri_color_light=False, point_lights=False,
                    has_specular=False, min_dist=1.2, max_dist=2.2, znear=0.1, seed=0, num_points=20000,
                    device="cuda", views_per_call=32, camera_noise=None):
    """Render one mesh into ``<output>/<name>_variational_light/`` (see the module docstring).  ``camera_noise``:
    ``(degrees, frac)``, the data's ``camera_mat`` are then those of :func:`perturb_cameras` (seeded with ``seed``) and
    ``camera_mat_true`` the cameras the images are rendered from.  Returns the directory."""
    from ..ops import make_shading, render_mesh
    dev = torch.device(device)
    name = os.path.splitext(os.path.basename(mesh_path))[0]
    out_dir = os.path.join(output, name + "_variational_light")
    verts_np, faces_np = read_mesh(mesh_path)
    verts = normalize_mesh(torch.from_numpy(verts_np))
    faces = torch.from_numpy(faces_np)
    g = torch.Generator().manual_seed(int(seed))
    rng = random.Random(int(seed))
    camera_params = {"znear": float(znear)}
    sampler = CameraSampler(num_cameras, 1, distance_range=((min_dist, max_dist),), sort_distance=True,
                            camera_type=FoVPerspectiveCameras, camera_params=camera_params, generator=g)
    cams, lights = [], []
    for cam in sampler:
        cams.append(cam)
        if tri_color_light:
            lights.append(get_tri_color_lights_for_view(cam, has_specular=has_specular, point_lights=point_lights,
                                                        generator=g))
        else:
            lights.append(get_light_for_view(cam, point_lights=point_lights, has_specular=has_specular, rng=rng))
    all_cams = FoVPerspectiveCameras(R=sampler.R, T=sampler.T, **camera_params)
    proj, view = camera_matrices(all_cams)
    vd, fd = verts.to(dev), faces.to(dev)
    images, masks, depths = [], [], []
    zfar = torch.tensor(all_cams.zfar, dtype=torch.float32, device=dev)
    for n0 in range(0, num_cameras, views_per_call):
        sl = slice(n0, min(n0 + views_per_call, num_cameras))
        view_n = view[sl].to(dev)
        shading = make_shading(_stack_lights(lights[sl]), view_n)
        r = render_mesh(vd, fd, proj[sl].to(dev), view_n, image_size, shading=shading)
        images.append(r.image.cpu())
        masks.append((r.pix_to_face >= 0).cpu())
        depths.append(torch.where(r.pix_to_face >= 0, r.zbuf, zfar).cpu())
    gd = torch.Generator(device=dev).manual_seed(int(seed))
    points, normals = sample_points_from_mesh(vd, fd, num_points, generator=gd)
    cams_out, cams_true = view.numpy(), None
    if camera_noise is not None:
        cams_out, cams_true = perturb_cameras(view.numpy(), camera_noise[0], camera_noise[1], seed), view.numpy()
    return write_mvr_data(out_dir, verts.numpy(), faces_np, torch.cat(images).numpy(), torch.cat(masks).numpy(),
                          cams_out, [light_value_dict(l) for l in lights], points.cpu().numpy(),
                          normals.cpu().numpy(), point_lights, camera_params, cams_true, torch.cat(depths).numpy())


def main(argv=None):
    p = argparse.ArgumentParser("Create multi-view training data from meshes: RGBA images, masks, cameras, lights")
    p.add_argument("--points", required=True, nargs="+", help="mesh files or globs (.ply, .obj)")
    p.add_argument("--num_cameras", type=int, default=120)
    p.add_argument("--image-size", type=int, default=512)
    p.add_argument("--output", type=str, default="data")
    p.add_argument("--tri_color_light", action="store_true")
    p.add_argument("--point_lights", action="store_true")
    p.add_argument("--has_specular", action="store_true")
    p.add_argument("--min_dist", type=float, default=1.2)
    p.add_argument("--max_dist", type=float, default=2.2)
    p.add_argument("--znear", type=float, default=0.1)
    p.add_argument("--seed", type=int, default=0)
    p.add_argument("--camera-noise", type=float, nargs=2, metavar=("DEG", "FRAC"), default=None,
                   help="store every camera perturbed by a random rotation of DEG degrees and a translation of FRAC "
                        "times its distance to the origin (the exact ones as camera_mat_true)")
    opt = p.parse_args(argv)
    if opt.camera_noise is not None and (opt.camera_noise[0] < 0 or opt.camera_noise[1] < 0):
        p.error("--camera-noise takes DEG >= 0 and FRAC >= 0")
    paths = sorted({q for pat in opt.points for q in (glob.glob(pat) or [pat])})
    out = []
    for path in paths:
        out.append(create_mvr_data(path, opt.output, opt.num_cameras, opt.image_size, opt.tri_color_light,
                                   opt.point_lights, opt.has_specular, opt.min_dist, opt.max_dist, opt.znear,
                                   opt.seed, camera_noise=opt.camera_noise))
        print(out[-1])
    return out


if __name__ == "__main__":
    main()
