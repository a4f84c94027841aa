"""CPU: camera refinement's settings (model.model_kwargs.learn_cameras, training.lr_cameras, training.cameras_from_it)
and their refusals, the seeded camera noise of create_mvr_data --camera-noise, the rigidity check of the cameras the
pose map takes, and the optimizer's pose group."""
import copy
import math

import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

from dss_b200.ops import check_rigid_cameras
from dss_b200.training.config import DEFAULTS, check_config
from dss_b200.training.train import CAMERA_GROUP, make_optimizer, pose_stats
from dss_b200.utils.create_mvr_data import main as create_main
from dss_b200.utils.create_mvr_data import perturb_cameras
from tests import pose_oracle as po


def config(learn=True, lr=1e-3, start=0):
    cfg = copy.deepcopy(DEFAULTS)
    cfg["model"]["model_kwargs"]["learn_cameras"] = learn
    cfg["training"]["lr_cameras"], cfg["training"]["cameras_from_it"] = lr, start
    return cfg


def check(cfg):
    check_config(cfg, (512, 512), True)


def test_defaults_learn_no_cameras():
    assert DEFAULTS["model"]["model_kwargs"]["learn_cameras"] is False
    assert DEFAULTS["training"]["lr_cameras"] > 0 and DEFAULTS["training"]["cameras_from_it"] >= 0
    check(copy.deepcopy(DEFAULTS))


@pytest.mark.parametrize("learn, lr, start", [(True, 1e-3, 0), (True, 1, 500), (False, 0.5, 3)])
def test_accepted_settings(learn, lr, start):
    check(config(learn, lr, start))


@pytest.mark.parametrize("learn, lr, start, match", [
    ("yes", 1e-3, 0, "learn_cameras must be true or false"),
    (1, 1e-3, 0, "learn_cameras must be true or false"),
    (True, 0, 0, "lr_cameras must be a number > 0"),
    (True, -1e-3, 0, "lr_cameras must be a number > 0"),
    (True, float("nan"), 0, "lr_cameras must be a number > 0"),
    (True, float("inf"), 0, "lr_cameras must be a number > 0"),
    (True, "0.001", 0, "lr_cameras must be a number > 0"),
    (True, True, 0, "lr_cameras must be a number > 0"),
    (True, 1e-3, -1, "cameras_from_it must be an integer >= 0"),
    (True, 1e-3, 2.0, "cameras_from_it must be an integer >= 0"),
    (True, 1e-3, None, "cameras_from_it must be an integer >= 0"),
    (True, 1e-3, False, "cameras_from_it must be an integer >= 0"),
])
def test_refused_settings(learn, lr, start, match):
    with pytest.raises(ValueError, match=match):
        check(config(learn, lr, start))


def cameras(V, seed=0):
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(V):
        eye = torch.randn(3, generator=g, dtype=torch.float64)
        out.append(po.look_at(eye / eye.norm() * (1.2 + torch.rand(1, generator=g, dtype=torch.float64))))
    return torch.stack(out).float().numpy()


@pytest.mark.parametrize("deg, frac", [(1.0, 0.01), (2.0, 0.02), (0.0, 0.05), (30.0, 0.0)])
def test_camera_noise_is_exact_and_seeded(deg, frac):
    true = cameras(12)
    noisy = perturb_cameras(true, deg, frac, seed=4)
    assert noisy.dtype == np.float32 and noisy.shape == true.shape
    assert np.array_equal(noisy, perturb_cameras(true, deg, frac, seed=4))
    assert deg == frac == 0 or not np.array_equal(noisy, perturb_cameras(true, deg, frac, seed=5))
    t, n = true.astype(np.float64), noisy.astype(np.float64)
    rel = np.einsum("vji,vjk->vik", t[:, :3, :3], n[:, :3, :3])                 # R0^T R: the perturbation
    angle = np.degrees(Rotation.from_matrix(rel).magnitude())
    assert np.abs(angle - deg).max() <= 1e-4
    centre = lambda m: -np.einsum("vj,vij->vi", m[:, 3, :3], m[:, :3, :3])
    moved = np.linalg.norm(centre(n) - centre(t), axis=1)
    assert np.abs(moved - frac * np.linalg.norm(centre(t), axis=1)).max() <= 1e-5
    check_rigid_cameras(noisy)


def test_camera_noise_refuses_negative_values():
    with pytest.raises(SystemExit):
        create_main(["--points", "mesh.obj", "--camera-noise", "-1", "0.01"])


def test_rigidity_check():
    good = cameras(5)
    check_rigid_cameras(good)
    scaled = good.copy()
    scaled[3, :3, :3] *= 1.01
    with pytest.raises(ValueError, match="camera 3 is not a rigid world-to-view transform"):
        check_rigid_cameras(scaled)
    mirrored = good.copy()
    mirrored[1, :3, 0] *= -1
    with pytest.raises(ValueError, match="camera 1 is not a rigid"):
        check_rigid_cameras(mirrored)
    projective = good.copy()
    projective[2, 0, 3] = 0.5
    with pytest.raises(ValueError, match="camera 2 is not a rigid"):
        check_rigid_cameras(projective)


def test_optimizer_pose_group_and_stats():
    t = {k: torch.zeros(4, 3, requires_grad=True) for k in ("points", "normals", "colours")}
    t["colours"].requires_grad_(False)
    poses = torch.zeros(3, 6, requires_grad=True)
    opt = make_optimizer(t, poses, 0.002)
    groups = opt.param_groups
    assert len(groups) == 3 and groups[-1]["name"] == CAMERA_GROUP and groups[-1]["params"][0] is poses
    assert groups[-1]["lr"] == 0.002 and groups[-1]["betas"] == (0.5, 0.9)
    assert len(make_optimizer(t).param_groups) == 2
    with torch.no_grad():
        poses[0, :3] = torch.tensor([0.0, 0.0, math.radians(2.0)])
        poses[1, 3:] = torch.tensor([0.3, 0.4, 0.0])
    mean_a, max_a, mean_t, max_t = pose_stats(poses).tolist()
    assert abs(max_a - 2.0) < 1e-5 and abs(mean_a - 2.0 / 3) < 1e-5
    assert abs(max_t - 0.5) < 1e-6 and abs(mean_t - 0.5 / 3) < 1e-6
