"""GPU: the camera pose map (csrc/poses.cu, ``ops.pose_cameras``) against the float64 restatement of
tests/pose_oracle.py, its chain through the renderer, and pose recovery with the cloud fixed.

What must hold:
  - forward within one float32 ulp of the float64 map, and ``view0`` / ``proj0`` bit for bit at zero poses;
  - backward within 1e-6 of the largest float64 autograd gradient, over V = 1, 7, 129, B = 0, 1, 8, repeated views, the
    small-angle joins and angles near pi, on random and looked-at cameras; the same bits twice, rows outside the batch
    exactly 0;
  - the pose gradient through ``render_points`` with fused shading (camera centres included) equals the one of the
    float64 map feeding the same render, within 1e-5 of the largest;
  - learning the poses alone, against renders of the true cloud from the true cameras, shrinks their errors."""
import math

import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

from dss_b200.core.lighting import DirectionalLights
from dss_b200.ops import SplatParams, make_shading, pose_cameras, render_points
from tests import pose_oracle as po
from tests.util import camera_matrices, random_cameras

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
ANGLES = [0.0, 1e-12, 1e-4, 0.1 * (1 - 1e-7), 0.1, 0.1 * (1 + 1e-7), 0.5, math.pi - 1e-3]


def cameras(V, kind, seed):
    """(view0, proj0) (V,4,4) float32 on the CPU: the test suite's random look-at cameras, or cameras of
    pose_oracle.look_at at random places looking at jittered targets"""
    if kind == "random":
        proj, view = camera_matrices(random_cameras(V, seed))
        return view.float(), proj.float()
    g = torch.Generator().manual_seed(seed)
    K = torch.zeros(4, 4, dtype=torch.float64)
    K[0, 0] = K[1, 1] = 1.7320508
    K[2, 2], K[2, 3], K[3, 2] = 1.001, 1.0, -0.1001
    views = []
    for _ in range(V):
        eye = torch.randn(3, generator=g, dtype=torch.float64)
        views.append(po.look_at(eye / eye.norm() * 1.8, at=0.05 * torch.randn(3, generator=g, dtype=torch.float64)))
    view = torch.stack(views)
    return view.float(), (view @ K).float()


def poses_at(V, theta, seed):
    g = torch.Generator().manual_seed(seed)
    p = torch.randn(V, 6, generator=g, dtype=torch.float64)
    p[:, :3] = p[:, :3] / p[:, :3].norm(dim=1, keepdim=True) * theta
    p[:, 3:] *= 0.05
    return p.float()


def within_one_ulp(got, ref64):
    ref32 = ref64.float()
    ulp = torch.from_numpy(np.spacing(np.abs(ref32.numpy())))
    return bool(((got.double() - ref64).abs() <= ulp.double()).all())


@pytest.mark.parametrize("kind", ["random", "look_at"])
@pytest.mark.parametrize("V, B", [(1, 0), (1, 1), (1, 8), (7, 1), (7, 8), (129, 8), (129, 1)])
@pytest.mark.parametrize("theta", ANGLES)
def test_kernel_matches_the_oracle(kind, V, B, theta):
    view0, proj0 = cameras(V, kind, V + B)
    poses = poses_at(V, theta, V * 10 + B)
    g = torch.Generator().manual_seed(B)
    idx = torch.randint(0, V, (B,), generator=g)
    if B >= 2:
        idx[1] = idx[0]                                    # a repeated view
    view, proj = pose_cameras(poses.to(DEV).requires_grad_(True), idx.to(DEV), view0.to(DEV), proj0.to(DEV))
    p64 = poses.double().requires_grad_(True)
    rv, rp = po.pose_map(p64, idx, view0, proj0)
    assert within_one_ulp(view.detach().cpu(), rv.detach()) and within_one_ulp(proj.detach().cpu(), rp.detach())
    # backward against float64 autograd of the same weights
    gv, gp = torch.randn(B, 4, 4, generator=g), torch.randn(B, 4, 4, generator=g)
    pd = poses.to(DEV).requires_grad_(True)
    v, q = pose_cameras(pd, idx.to(DEV), view0.to(DEV), proj0.to(DEV))
    ((v * gv.to(DEV)).sum() + (q * gp.to(DEV)).sum()).backward()
    if B:
        ((rv * gv.double()).sum() + (rp * gp.double()).sum()).backward()
        ref = p64.grad
    else:
        ref = torch.zeros(V, 6, dtype=torch.float64)
    got = pd.grad.cpu()
    scale = max(float(ref.abs().max()), 1e-30)
    assert float((got.double() - ref).abs().max()) <= 1e-6 * scale, (got, ref)
    outside = torch.ones(V, dtype=torch.bool)
    outside[idx] = False
    assert (got[outside] == 0).all() and not torch.signbit(got[outside]).any()
    # the same bits again
    pd2 = poses.to(DEV).requires_grad_(True)
    v, q = pose_cameras(pd2, idx.to(DEV), view0.to(DEV), proj0.to(DEV))
    ((v * gv.to(DEV)).sum() + (q * gp.to(DEV)).sum()).backward()
    assert torch.equal(pd.grad, pd2.grad)


@pytest.mark.parametrize("kind", ["random", "look_at"])
def test_zero_poses_give_the_cameras_bit_for_bit(kind):
    view0, proj0 = cameras(33, kind, 2)
    view0[0, 0, 1] = -0.0                                  # a negative zero keeps its sign
    idx = torch.tensor([5, 0, 32, 5, 17], device=DEV)
    view, proj = pose_cameras(torch.zeros(33, 6, device=DEV), idx, view0.to(DEV), proj0.to(DEV))
    assert torch.equal(view.view(torch.int32), view0.to(DEV)[idx].view(torch.int32))
    assert torch.equal(proj.view(torch.int32), proj0.to(DEV)[idx].view(torch.int32))


def test_arguments_are_checked():
    view0, proj0 = (t.to(DEV) for t in cameras(3, "random", 0))
    idx = torch.tensor([0, 2], device=DEV)
    with pytest.raises(RuntimeError, match="poses must be a float32"):
        pose_cameras(torch.zeros(3, 6, device=DEV, dtype=torch.float64), idx, view0, proj0)
    with pytest.raises(RuntimeError, match="idx must be an int64"):
        pose_cameras(torch.zeros(3, 6, device=DEV), idx.int(), view0, proj0)
    with pytest.raises(RuntimeError, match="view0 must be a float32 tensor of shape"):
        pose_cameras(torch.zeros(3, 6, device=DEV), idx, view0[:2], proj0)
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        pose_cameras(torch.zeros(3, 6), idx, view0, proj0)


def test_pose_gradient_through_the_renderer():
    """the kernel's map and the float64 map feed the same render with fused shading; their pose gradients agree"""
    from tests.util import sphere_cloud
    N, V, S = 4, 6, 64
    pts, nrm, col = (t.to(DEV) for t in sphere_cloud(3000, 1))
    view0, proj0 = cameras(V, "random", 4)
    poses = poses_at(V, 0.02, 3)
    idx = torch.tensor([3, 0, 3, 5])
    prm = SplatParams(image_size=S, points_per_pixel=5, znear=0.1, clip_pts_grad=0.05)
    h = torch.full((N,), 3e-4, device=DEV)
    lights = DirectionalLights(direction=(((0.3, 0.8, -0.5),),), device=DEV)
    g = torch.randn(N, S, S, 4, generator=torch.Generator().manual_seed(0)).to(DEV)

    def loss(view, proj):
        sh = make_shading(lights, view)
        out = render_points(pts, nrm, col, proj, view, h, prm, shading=sh, deterministic=True)
        return (out.image * g).sum()

    pd = poses.to(DEV).requires_grad_(True)
    loss(*pose_cameras(pd, idx.to(DEV), view0.to(DEV), proj0.to(DEV))).backward()
    p64 = poses.double().requires_grad_(True)
    rv, rp = po.pose_map(p64, idx, view0, proj0)
    loss(rv.float().to(DEV), rp.float().to(DEV)).backward()
    ref, got = p64.grad, pd.grad.cpu().double()
    assert float(ref.abs().max()) > 0
    assert float((got - ref).abs().max()) <= 1e-5 * float(ref.abs().max()), (got, ref)


# ---- recovery with the cloud fixed --------------------------------------------------------------------------------
# Measured on an H100 with these settings (2 degrees and 2 %, 16 views at 128^2, batch 4): the median rotation error
# fell from 2.00 to 0.80 degrees (0.40 of its start) and the median camera-centre error from 0.0322 to 0.0220 (0.68)
# after 300 iterations.  The rotations are well observed in silhouettes; a camera's shift along its optical axis much
# less, and the splats of the sampled cloud are not the mesh, so the translations stop short.  The bounds keep a margin.
RECOVERY_ITERS = 300
RECOVERY_LR = 3e-4
RECOVERY_ROTATION = 0.6      # the median rotation error after RECOVERY_ITERS must fall below this fraction of its start
RECOVERY_TRANSLATION = 0.85  # and the median camera-centre error below this one


def pose_errors(cams, true):
    """(rotation errors in degrees, camera-centre distances) (V,) of world-to-view matrices against the true ones"""
    c, t = cams.double().cpu().numpy(), true.astype(np.float64)
    rel = np.einsum("vji,vjk->vik", t[:, :3, :3], c[:, :3, :3])
    centre = lambda m: -np.einsum("vj,vij->vi", m[:, 3, :3], m[:, :3, :3])
    return np.degrees(Rotation.from_matrix(rel).magnitude()), np.linalg.norm(centre(c) - centre(t), axis=1)


def test_poses_alone_recover_from_noise(tmp_path):
    from dss_b200.training.step import GraphedTrainStep
    from dss_b200.utils.create_mvr_data import main as create
    from dss_b200.utils.dataset import MVRData
    from dss_b200.utils.io import save_obj
    from tests.test_mesh_data import torus
    verts, faces = torus()
    save_obj(str(tmp_path / "torus.obj"), verts.numpy(), faces.numpy())
    d = create(["--points", str(tmp_path / "torus.obj"), "--output", str(tmp_path / "data"), "--num_cameras", "16",
                "--image-size", "128", "--tri_color_light", "--point_lights", "--seed", "3",
                "--camera-noise", "2", "0.02"])[0]
    data = MVRData(d)
    true = np.asarray(data.data_dict["camera_mat_true"])
    views = data.device_views(DEV)
    pc = data.get_pointclouds()
    pts, nrm = pc.points_packed().to(DEV), pc.normals_packed().to(DEV)
    cams = data.get_cameras()
    prm = SplatParams(image_size=128, points_per_pixel=5, cutoff_threshold=1.0, clip_pts_grad=0.05,
                      znear=float(cams.znear), zfar=float(cams.zfar))
    V = len(views)
    step = GraphedTrainStep.from_views(pts, nrm, torch.ones_like(pts), prm, views, [0, 1, 2, 3], learn=(),
                                       Vrk_invariant=True, Vrk_isotropic=False, lambda_dr_proj=0.0,
                                       poses=torch.zeros(V, 6, device=DEV))
    opt = torch.optim.Adam([step.poses], lr=RECOVERY_LR, betas=(0.5, 0.9))
    rot0, tr0 = pose_errors(views.camera_mat, true)
    g = torch.Generator().manual_seed(0)
    for _ in range(RECOVERY_ITERS):
        step.load_views(torch.randperm(V, generator=g)[:4].tolist())
        step.replay()
        opt.step()
    rot1, tr1 = pose_errors(views.with_poses(step.poses).camera_mat, true)
    print("median rotation error %.4f -> %.4f deg, translation %.5f -> %.5f"
          % (np.median(rot0), np.median(rot1), np.median(tr0), np.median(tr1)))
    assert np.median(rot1) < RECOVERY_ROTATION * np.median(rot0)
    assert np.median(tr1) < RECOVERY_TRANSLATION * np.median(tr0)
