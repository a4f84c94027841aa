"""CPU: the float64 depth restatement (tests/depth_oracle.py) against a brute-force loop and finite differences, and the
torch body of the depth loss (losses.depth_loss_torch) against it."""
import numpy as np
import torch

from dss_b200.training.losses import depth_loss, depth_loss_torch
from tests import depth_oracle as O


def _lists(rng, N=2, S=5, K=4, P=30):
    idx = rng.integers(0, P, size=(N, S, S, K)).astype(np.int32)
    # ragged lists: empty tails, whole empty lists, and a stale id after an empty slot (not read)
    cut = rng.integers(0, K + 1, size=(N, S, S))
    for k in range(K):
        idx[..., k][k >= cut] = -1
    idx[0, 0, 0] = [-1, 7, -1, 3]
    w = rng.random((N, S, S, K)).astype(np.float32)
    z = (rng.random(P) * 3 + 0.5).astype(np.float32)
    return idx, w, z


def test_depth_map_and_record_gradient_against_brute_force():
    rng = np.random.default_rng(0)
    idx, w, z = _lists(rng)
    N, S, _, K = idx.shape
    g = rng.standard_normal((N, S, S))
    D, gz = O.depth_map(idx, w, z), O.depth_record_grad(idx, w, g, 30)
    want_D, want_gz = np.zeros((N, S, S)), np.zeros(30)
    for n in range(N):
        for y in range(S):
            for x in range(S):
                for k in range(K):
                    p = idx[n, y, x, k]
                    if p < 0:
                        break
                    want_D[n, y, x] += float(w[n, y, x, k]) * float(z[p])
                    want_gz[p] += g[n, y, x] * float(w[n, y, x, k])
    assert np.array_equal(D == 0, want_D == 0) and D[0, 0, 0] == 0.0
    np.testing.assert_allclose(D, want_D, rtol=1e-14, atol=0)
    np.testing.assert_allclose(gz, want_gz, rtol=1e-12, atol=1e-14)


def test_record_gradient_is_the_derivative_of_the_depth_map():
    rng = np.random.default_rng(1)
    idx, w, z = _lists(rng)
    g = rng.standard_normal(idx.shape[:3])
    z64 = z.astype(np.float64)
    f = lambda zz: float((O.depth_map(idx, w, zz) * g).sum())
    gz = O.depth_record_grad(idx, w, g, z.size)
    for s in range(z.size):
        e = np.zeros_like(z64)
        e[s] = 1e-6
        assert abs((f(z64 + e) - f(z64 - e)) / 2e-6 - gz[s]) < 1e-6


def _loss_case(rng, N=3, S=6, znear=0.5, zfar=10.0):
    depth = rng.random((N, S, S)) * 4 + 1
    gt = depth + rng.standard_normal((N, S, S)) * 0.3
    gt[0, 0, :3] = [np.nan, np.inf, -np.inf]
    gt[0, 1, :4] = [znear, zfar, znear * 0.5, zfar * 2]        # on and outside the open range
    gt[1, 2, 2] = depth[1, 2, 2]                                # |d| = 0: sign 0
    alpha = (rng.random((N, S, S)) > 0.2).astype(np.float64)
    mask = (rng.random((N, S, S)) > 0.2).astype(np.float64)
    mask[2, 0, 0] = np.nan                                      # NaN counts as set
    return depth, alpha, gt, mask, znear, zfar


def test_loss_gradient_against_finite_differences():
    rng = np.random.default_rng(2)
    depth, alpha, gt, mask, zn, zf = _loss_case(rng)
    gt[1, 2, 2] += 0.01                                         # keep away from the kink here
    lam = 0.7
    grad = O.depth_loss_grad(depth, alpha, gt, mask, lam, zn, zf, g=1.0)
    for i in zip(*np.nonzero(np.ones_like(depth))):
        e = np.zeros_like(depth)
        e[i] = 1e-7
        fd = (O.depth_loss(depth + e, alpha, gt, mask, lam, zn, zf) - O.depth_loss(depth - e, alpha, gt, mask, lam, zn, zf)) / 2e-7
        assert abs(fd - grad[i]) < 1e-6, i


def test_torch_body_against_the_restatement():
    rng = np.random.default_rng(3)
    depth, alpha, gt, mask, zn, zf = _loss_case(rng)
    rgba = np.concatenate([rng.random(depth.shape + (3,)), alpha[..., None]], -1)
    t = lambda a: torch.tensor(a, dtype=torch.float64)
    for lam in (1.0, 0.25):
        d = t(depth).requires_grad_(True)
        for fn in (depth_loss_torch, depth_loss):                 # CPU tensors take the torch body
            d.grad = None
            loss = fn(d, t(rgba), t(gt), t(mask), lam, zn, zf)
            loss.backward()
            assert abs(float(loss.detach()) - O.depth_loss(depth, alpha, gt, mask, lam, zn, zf)) < 1e-12
            np.testing.assert_allclose(d.grad.numpy(), O.depth_loss_grad(depth, alpha, gt, mask, lam, zn, zf),
                                       rtol=1e-12, atol=1e-15)
    # M = 0: zero, and no gradient
    d = t(depth).requires_grad_(True)
    loss = depth_loss_torch(d, t(rgba), t(gt), t(np.zeros_like(mask)), 1.0, zn, zf)
    assert float(loss) == 0.0 and O.depth_loss(depth, alpha, gt, np.zeros_like(mask), 1.0, zn, zf) == 0.0
