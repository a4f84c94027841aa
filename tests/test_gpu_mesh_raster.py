"""GPU: the mesh rasterizer (dss_rasterize_mesh / ops.render_mesh) against the float32 oracle of tests/mesh_oracle.py,
bit for bit; its flat shading against a float64 restatement; the data directory end to end through MVRData and the
training step."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from dss_b200 import _lib
from dss_b200.core.camera import camera_matrices
from dss_b200.core.lighting import DirectionalLights, PointLights
from dss_b200.ops import Shading, SplatParams, make_shading, preprocess_points, render_mesh
from tests.mesh_oracle import rasterize_mesh_naive
from tests.test_mesh_data import HAND_CASES, icosphere, torus
from tests.util import random_cameras

pytestmark = pytest.mark.gpu


def screen_verts(verts, proj, view):
    """(N,V,3) {NDC x, NDC y, view z} from the splat preprocess, the expression the mesh kernel uses"""
    V, N = verts.shape[0], proj.shape[0]
    prm = SplatParams(image_size=8, znear=-3e38, zfar=3e38)
    nrm = torch.zeros_like(verts)
    nrm[:, 2] = 1
    out = preprocess_points(verts, nrm, proj, view, torch.full((N,), 1e-3, device=verts.device), prm)
    scr = out["ndc"].view(N, V, 3).cpu().numpy().copy()
    # the preprocess writes z = -1 for a non-finite depth (its depth filter); the mesh kernel keeps the value
    vz = torch.einsum("vk,nk->nv", torch.cat([verts, torch.ones_like(verts[:, :1])], 1).double(),
                      view[:, :, 2].double()).cpu().numpy()
    bad = ~np.isfinite(vz)
    scr[..., 2][bad] = vz[bad]
    return scr


def check_against_oracle(verts, faces, proj, view, S):
    d = torch.device("cuda:0")
    verts, faces, proj, view = verts.to(d), faces.to(d), proj.to(d), view.to(d)
    r = render_mesh(verts, faces, proj, view, S)
    want_f, want_z = rasterize_mesh_naive(screen_verts(verts, proj, view), faces.cpu().numpy(), S)
    got_f, got_z = r.pix_to_face.cpu().numpy(), r.zbuf.cpu().numpy()
    assert np.array_equal(got_f, want_f), np.argwhere(got_f != want_f)[:5]
    assert np.array_equal(got_z, want_z)                      # == : -0 and +0 compare equal
    assert not np.signbit(got_z[got_f >= 0]).any()            # the kernel writes depth 0 as +0
    r2 = render_mesh(verts, faces, proj, view, S)
    assert torch.equal(r.pix_to_face, r2.pix_to_face) and torch.equal(r.zbuf.view(torch.int32), r2.zbuf.view(torch.int32))
    return got_f


def soup(F, seed, scale=1.0, spread=0.7):
    g = torch.Generator().manual_seed(seed)
    centres = (torch.rand(F, 1, 3, generator=g) * 2 - 1) * spread
    verts = (centres + (torch.rand(F, 3, 3, generator=g) - 0.5) * scale).reshape(-1, 3).contiguous()
    return verts, torch.arange(3 * F).reshape(F, 3)


def cams(N, seed):
    return camera_matrices(random_cameras(N, seed))


@pytest.mark.parametrize("S,N", [(1, 3), (15, 129), (17, 3), (512, 1), (1024, 1)])
def test_soup_matches_oracle(cuda_device, S, N):
    verts, faces = soup(60 if N < 100 else 12, seed=S + N)
    proj, view = cams(N, seed=S)
    f = check_against_oracle(verts, faces, proj, view, S)
    assert S < 8 or (f >= 0).mean() > 0.01


@pytest.mark.parametrize("S", [17, 512])
def test_sphere_mesh_matches_oracle(cuda_device, S):
    verts, faces = icosphere(3)
    proj, view = cams(3, seed=7)
    f = check_against_oracle(verts * 0.5, faces, proj, view, S)
    assert (f >= 0).any()


def test_faces_larger_than_the_image(cuda_device):
    # a few faces many times the image across, mixed with small ones: the item kernel spreads them over the grid
    big, fb = soup(4, seed=3, scale=30.0, spread=0.2)
    small, fs = soup(40, seed=4)
    verts = torch.cat([big, small])
    faces = torch.cat([fb, fs + big.shape[0]])
    proj, view = cams(2, seed=11)
    f = check_against_oracle(verts, faces, proj, view, 256)
    assert (f >= 0).mean() > 0.5


def test_several_view_chunks(cuda_device):
    # 1024^2 pixels: 32 views per chunk of the pixel keys, so 40 views take two chunks
    verts, faces = soup(8, seed=21, scale=0.3)
    proj, view = cams(40, seed=21)
    check_against_oracle(verts, faces, proj, view, 1024)


@pytest.mark.parametrize("case", sorted(HAND_CASES))
def test_hand_built_cases_match_oracle(cuda_device, case):
    verts, faces, S, _ = HAND_CASES[case]()
    eye = torch.eye(4)[None]
    check_against_oracle(torch.as_tensor(verts, dtype=torch.float32), torch.as_tensor(faces), eye, eye, S)


def test_invalid_input_is_refused(cuda_device):
    d = cuda_device
    verts, faces = soup(2, seed=0)
    proj, view = (t.to(d) for t in cams(1, seed=0))
    with pytest.raises(ValueError):
        render_mesh(verts.to(d), torch.tensor([[0, 1, 6]], device=d), proj, view, 8)
    with pytest.raises(ValueError):
        render_mesh(verts.to(d), torch.tensor([[0, -1, 2]], device=d), proj, view, 8)
    lib, p2f, z = _lib.load(), torch.empty(64, dtype=torch.int32, device=d), torch.empty(64, device=d)
    f32 = faces.to(d).int()
    common = (_lib.ctx(d), _lib.ptr(verts.to(d)), 6, _lib.ptr(f32), 2, _lib.ptr(proj), _lib.ptr(view), 1)
    shade0 = (0, 0, 0, C.c_float(0.0), None, None, None)
    assert lib.dss_rasterize_mesh(*common, 0, *shade0, _lib.ptr(p2f), _lib.ptr(z), None, None) == -1
    assert lib.dss_rasterize_mesh(*common, 8, *shade0, None, _lib.ptr(z), None, None) == -1
    assert lib.dss_rasterize_mesh(_lib.ctx(d), None, 6, _lib.ptr(f32), 2, _lib.ptr(proj), _lib.ptr(view), 1, 8,
                                  *shade0, _lib.ptr(p2f), _lib.ptr(z), None, None) == -1
    assert lib.dss_rasterize_mesh(*common[:2], 2 ** 31, *common[3:], 8, *shade0, _lib.ptr(p2f), _lib.ptr(z), None,
                                  None) == -1
    # rgba without lights
    rgba = torch.empty(256, device=d)
    assert lib.dss_rasterize_mesh(*common, 8, *shade0, _lib.ptr(p2f), _lib.ptr(z), _lib.ptr(rgba), None) == -1
    torch.cuda.synchronize()


# ---- flat shading --------------------------------------------------------------------------------------------------

def flat_shading_f64(verts, faces, p2f, sh: Shading):
    """float64: (ambient + diffuse) + specular of the face at every covered pixel (white vertices, unit materials),
    with the normal normalize(cross(v1 - v0, v2 - v0)) renormalised by the lighting (F.normalize, eps 1e-6)"""
    Fn = torch.nn.functional.normalize
    v = verts.double()
    tri = v[faces.long()]
    centroid = tri.mean(1)
    nrm = Fn(torch.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0], dim=1), dim=1, eps=1e-6)
    N = p2f.shape[0]
    lights = sh.lights.double() if sh.lights.dim() == 3 else sh.lights.double()[None].expand(N, -1, -1)
    amb = sh.ambient.double() if sh.ambient.dim() == 2 else sh.ambient.double()[None].expand(N, -1)
    out = torch.ones(p2f.shape + (4,), dtype=torch.float64, device=p2f.device)
    out[..., 3] = 0
    for n in range(N):
        m = p2f[n] >= 0
        f = p2f[n][m].long()
        p, nn = centroid[f], Fn(nrm[f], dim=1, eps=1e-6)
        vdir = Fn(sh.cam_centres[n].double() - p, dim=1, eps=1e-6)
        col = amb[n].expand_as(p).clone()
        spec = torch.zeros_like(p)
        for l in range(lights.shape[1]):
            L = lights[n, l]
            d = Fn((L[:3] - p) if sh.light_type else L[:3].expand_as(p), dim=1, eps=1e-6)
            cos = (nn * d).sum(1)
            col += L[3:6] * cos.clamp(min=0)[:, None]
            r = -d + 2 * cos[:, None] * nn
            a = (vdir * r).sum(1).clamp(min=0) * (cos > 0)
            spec += L[6:9] * torch.where(a > 0, a.pow(sh.shininess), torch.zeros_like(a))[:, None]
        out[n][m] = torch.cat([col + spec, torch.ones_like(col[:, :1])], 1)
    return out


def lights_of(kind, N, per_view, specular, seed):
    g = torch.Generator().manual_seed(seed)
    B = N if per_view else 1
    vec = torch.randn(B, 3, 3, generator=g) * (2.0 if kind else 1.0)
    dif = torch.rand(B, 3, 3, generator=g) * 0.6
    spe = torch.rand(B, 3, 3, generator=g) * 0.3 if specular else torch.zeros(B, 3, 3)
    amb = torch.rand(B, 1, 3, generator=g) * 0.3
    cls = PointLights if kind else DirectionalLights
    key = "location" if kind else "direction"
    return cls(ambient_color=amb, diffuse_color=dif, specular_color=spe, **{key: vec})


WORST = {}


@pytest.mark.parametrize("kind", [0, 1])
@pytest.mark.parametrize("per_view", [False, True])
@pytest.mark.parametrize("specular", [False, True])
def test_flat_shading_against_float64(cuda_device, kind, per_view, specular):
    d = cuda_device
    verts, faces = icosphere(3)
    verts = (verts * 0.6).to(d)
    faces = faces.to(d)
    N, S = 3, 128
    proj, view = (t.to(d) for t in cams(N, seed=31))
    sh = make_shading(lights_of(kind, N, per_view, specular, seed=kind + 2 * per_view), view)
    r = render_mesh(verts, faces, proj, view, S, shading=sh)
    want = flat_shading_f64(verts, faces, r.pix_to_face, sh)
    mask = r.pix_to_face >= 0
    assert mask.any() and (~mask).any()
    assert torch.equal(r.image[..., 3], mask.float())
    assert bool((r.image[~mask][:, :3] == 1).all())
    err = float((r.image[..., :3].double() - want[..., :3]).abs().max())
    WORST[(kind, per_view, specular)] = err
    print("flat shading worst |rgb - f64| = %.3g" % err)
    assert err <= 1e-5
    # the plain render gives the same faces and depths
    r0 = render_mesh(verts, faces, proj, view, S)
    assert torch.equal(r0.pix_to_face, r.pix_to_face) and torch.equal(r0.zbuf, r.zbuf)


def test_shared_lights_expanded_per_view_give_the_same_bits(cuda_device):
    d = cuda_device
    verts, faces = icosphere(2)
    verts, faces = verts.to(d), faces.to(d)
    N = 4
    proj, view = (t.to(d) for t in cams(N, seed=5))
    sh = make_shading(lights_of(1, N, False, True, seed=9), view)
    per = Shading(sh.lights[None].expand(N, -1, -1).contiguous(), sh.ambient[None].expand(N, -1).contiguous(),
                  sh.cam_centres, sh.light_type, sh.shininess)
    a = render_mesh(verts, faces, proj, view, 64, shading=sh)
    b = render_mesh(verts, faces, proj, view, 64, shading=per)
    assert torch.equal(a.image.view(torch.int32), b.image.view(torch.int32))


def test_empty_mesh_and_empty_views_are_background(cuda_device):
    d = cuda_device
    N, S = 2, 32
    proj, view = (t.to(d) for t in cams(N, seed=2))
    sh = make_shading(lights_of(0, N, False, True, seed=1), view)
    empty = render_mesh(torch.zeros(0, 3, device=d), torch.zeros(0, 3, dtype=torch.int64, device=d), proj, view, S,
                        shading=sh)
    # a mesh behind every camera: nothing in view
    verts, faces = icosphere(1)
    centre = sh.cam_centres[0] * 3.0
    far = render_mesh((verts.to(d) * 0.01 - centre), faces.to(d), proj[:1], view[:1], S,
                      shading=Shading(sh.lights, sh.ambient, sh.cam_centres[:1], sh.light_type, sh.shininess))
    for r in (empty, far):
        assert bool((r.pix_to_face == -1).all()) and bool((r.zbuf == -1).all())
        bg = torch.ones_like(r.image)
        bg[..., 3] = 0
        assert torch.equal(r.image, bg)


# ---- end to end: data directory -> MVRData -> training step ------------------------------------------------------

def test_generated_data_trains_a_cloud(cuda_device, tmp_path):
    from dss_b200.training.step import TrainStep
    from dss_b200.utils.create_mvr_data import main
    from dss_b200.utils.dataset import MVRData
    from dss_b200.utils.io import save_obj
    d = cuda_device
    verts, faces = torus()
    mesh = tmp_path / "torus.obj"
    save_obj(str(mesh), verts.numpy(), faces.numpy())
    out = main(["--points", str(mesh), "--output", str(tmp_path / "data"), "--num_cameras", "16", "--image-size", "128",
                "--tri_color_light", "--point_lights", "--seed", "3"])
    data = MVRData(out[0])
    assert len(data) == 16 and data.resolution == (128, 128)
    cloud = data.get_pointclouds()
    assert cloud.points_packed().shape == (20000, 3)
    cams_all = data.get_cameras()
    proj, view = (t.to(d) for t in camera_matrices(cams_all))
    items = [data[i] for i in range(16)]
    # the INTEGRATION recipe: stack the items' light dicts into one lights object of batch N
    lights = PointLights(**{k: torch.stack([torch.as_tensor(it["lights"][k]) for it in items])
                            for k in items[0]["lights"]}, device=d)
    img = torch.stack([im.permute(1, 2, 0) for im in data.images]).to(d).contiguous()
    mask = torch.stack([m[0] for m in data.masks]).to(d)
    g = torch.Generator().manual_seed(0)
    P0 = 4000
    p = torch.nn.functional.normalize(torch.randn(P0, 3, generator=g), dim=1)
    prm = SplatParams(image_size=128, points_per_pixel=5, znear=0.1, clip_pts_grad=0.05, radii_backward_scaler=5.0)
    step = TrainStep((0.5 * p).to(d), p.to(d), torch.ones(P0, 3, device=d), prm, lambda_dr_proj=0.0)
    opt = torch.optim.Adam([{"params": [step.normals], "lr": 0.01}, {"params": [step.points], "lr": 0.01}],
                           betas=(0.5, 0.9))
    hist = []
    for it in range(60):
        sel = torch.arange(it % 4, 16, 4, device=d)
        loss = step(img[sel], mask[sel], proj[sel], view[sel], PointLights(
            ambient_color=lights.ambient_color[sel.cpu()], diffuse_color=lights.diffuse_color[sel.cpu()],
            specular_color=lights.specular_color[sel.cpu()], location=lights.location[sel.cpu()], device=d))
        hist.append((float(loss["loss_dr_silhouette"]), float(loss["loss_dr_rgb"])))
        opt.step()
    first = np.mean(hist[:4], 0)
    last = np.mean(hist[-4:], 0)
    print("silhouette %.4f -> %.4f, rgb %.4f -> %.4f" % (first[0], last[0], first[1], last[1]))
    # measured on an H100: silhouette 0.491 -> 0.214 (0.44x), rgb 0.743 -> 0.643 (0.87x); see DESIGN.md
    assert last[0] <= 0.6 * first[0] and last[1] <= 0.95 * first[1]
