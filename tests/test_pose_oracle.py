"""CPU: the float64 pose map of tests/pose_oracle.py, the restatement the GPU tests pin csrc/poses.cu to: its rotation
against scipy, its gradient against finite differences, E(0) = I, and the joins of the small-angle series."""
import math

import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

from tests import pose_oracle as po


def random_cameras(V, seed):
    g = torch.Generator().manual_seed(seed)
    views, projs = [], []
    for _ in range(V):
        eye = torch.randn(3, generator=g, dtype=torch.float64)
        eye = eye / eye.norm() * (1.5 + torch.rand(1, generator=g, dtype=torch.float64))
        v = po.look_at(eye, at=0.05 * torch.randn(3, generator=g, dtype=torch.float64))
        K = torch.zeros(4, 4, dtype=torch.float64)
        K[0, 0] = K[1, 1] = 1.7
        K[2, 2], K[2, 3], K[3, 2] = 1.01, 1.0, -0.101
        views.append(v)
        projs.append(v @ K)
    return torch.stack(views), torch.stack(projs)


@pytest.mark.parametrize("theta", [0.0, 1e-12, 1e-4, 0.05, 0.0999999, 0.1, 0.1000001, 0.7, 2.0, math.pi - 1e-6,
                                   math.pi, 4.0])
def test_rotation_is_scipys(theta):
    g = torch.Generator().manual_seed(int(theta * 1000) + 1)
    axis = torch.randn(3, generator=g, dtype=torch.float64)
    w = axis / axis.norm() * theta
    R = po.rotation(w).numpy()
    ref = Rotation.from_rotvec(w.numpy()).as_matrix()
    assert np.abs(R - ref).max() <= 4e-16
    assert np.abs(R @ R.T - np.eye(3)).max() <= 4e-16


def test_zero_pose_is_the_identity():
    D = po.delta(torch.zeros(6, dtype=torch.float64))
    assert torch.equal(D, torch.zeros(4, 4, dtype=torch.float64))
    view0, proj0 = random_cameras(3, 0)
    view, proj = po.pose_map(torch.zeros(3, 6, dtype=torch.float64), [2, 0, 2], view0, proj0)
    assert torch.equal(view, view0[[2, 0, 2]]) and torch.equal(proj, proj0[[2, 0, 2]])


@pytest.mark.parametrize("th2", [0.0, 1e-24, 1e-8, 1e-4, 0.01 * (1 - 1e-12), 0.01, 0.01 * (1 + 1e-12)])
def test_series_and_closed_forms_agree(th2):
    """both branches of s and c at the same angle: the series below 0.1, the closed forms above, within float64"""
    t = torch.tensor([th2], dtype=torch.float64)
    th = math.sqrt(th2)
    if th2 > 0:
        s_cl, c_cl = math.sin(th) / th, 2 * math.sin(th / 2) ** 2 / th2
    else:
        s_cl, c_cl = 1.0, 0.5
    s, c = po.coeffs(t)
    assert abs(float(s) - s_cl) <= 2e-16 and abs(float(c) - c_cl) <= 2e-16


def test_branches_join_continuously():
    """s and c on both sides of the series' bound differ by their slope alone"""
    for f in (lambda x: po.coeffs(x)[0], lambda x: po.coeffs(x)[1]):
        lo = f(torch.tensor([0.01 * (1 - 1e-9)], dtype=torch.float64))
        hi = f(torch.tensor([0.01 * (1 + 1e-9)], dtype=torch.float64))
        assert abs(float(hi - lo)) <= 1e-11


@pytest.mark.parametrize("theta", [0.0, 1e-12, 1e-4, 0.3, 0.1, math.pi - 1e-3])
def test_gradient_matches_finite_differences(theta):
    view0, proj0 = random_cameras(4, 3)
    g = torch.Generator().manual_seed(7)
    poses = torch.randn(4, 6, generator=g, dtype=torch.float64)
    poses[:, :3] = poses[:, :3] / poses[:, :3].norm(dim=1, keepdim=True) * theta
    poses[:, 3:] *= 0.05
    gv = torch.randn(5, 4, 4, generator=g, dtype=torch.float64)
    gp = torch.randn(5, 4, 4, generator=g, dtype=torch.float64)
    idx = [1, 3, 1, 0, 1]

    def loss(p):
        v, q = po.pose_map(p, idx, view0, proj0)
        return (v * gv).sum() + (q * gp).sum()

    assert torch.autograd.gradcheck(loss, (poses.clone().requires_grad_(True),), eps=1e-6, atol=1e-6, rtol=1e-5)


def test_map_is_the_composed_transform():
    """view = view0 E and proj = view0 E view0^-1 proj0 with E from scipy"""
    view0, proj0 = random_cameras(3, 5)
    g = torch.Generator().manual_seed(1)
    poses = torch.randn(3, 6, generator=g, dtype=torch.float64) * 0.3
    view, proj = po.pose_map(poses, [0, 1, 2], view0, proj0)
    for v in range(3):
        E = np.eye(4)
        E[:3, :3] = Rotation.from_rotvec(poses[v, :3].numpy()).as_matrix()
        E[3, :3] = poses[v, 3:].numpy()
        V0 = view0[v].numpy()
        assert np.abs(view[v].numpy() - V0 @ E).max() <= 1e-14
        assert np.abs(proj[v].numpy() - V0 @ E @ np.linalg.inv(V0) @ proj0[v].numpy()).max() <= 1e-13
