"""A float64 torch restatement of the camera pose map of csrc/poses.cu (the map is in include/dss_b200.h), for the
tests: differentiable with torch's autograd, so that its gradients check the kernel's backward.

    view = view0 + view0 D,   proj = proj0 + view0 D K,   D = E(xi) - I,   K = view0^-1 proj0 (rigid inverse)

with E(xi) = [[R(w), 0], [t, 1]] (row-vector convention), R(w) = I + s [w]x + c [w]x^2 scipy's
``Rotation.from_rotvec(w).as_matrix()``.  s and c take their Taylor series below th = SERIES_BELOW, as the kernel does."""
import torch

SERIES_BELOW = 0.1


def coeffs(th2):
    """(s, c) = (sin th / th, (1 - cos th) / th^2) of th^2, float64, differentiable at 0 too"""
    small = th2 < SERIES_BELOW ** 2
    x = torch.where(small, th2, torch.zeros_like(th2))
    s_ser = 1 + x * (-1 / 6 + x * (1 / 120 + x * (-1 / 5040 + x * (1 / 362880 + x * (-1 / 39916800)))))
    c_ser = 0.5 + x * (-1 / 24 + x * (1 / 720 + x * (-1 / 40320 + x * (1 / 3628800 + x * (-1 / 479001600)))))
    th = torch.sqrt(torch.where(small, torch.ones_like(th2), th2))
    s_cl = torch.sin(th) / th
    c_cl = 2 * torch.sin(0.5 * th) ** 2 / th ** 2
    return torch.where(small, s_ser, s_cl), torch.where(small, c_ser, c_cl)


def skew(w):
    z = torch.zeros_like(w[..., 0])
    return torch.stack([torch.stack([z, -w[..., 2], w[..., 1]], -1),
                        torch.stack([w[..., 2], z, -w[..., 0]], -1),
                        torch.stack([-w[..., 1], w[..., 0], z], -1)], -2)


def delta(xi):
    """D = E(xi) - I, (..., 4, 4) float64, formed directly"""
    xi = xi.double()
    w, t = xi[..., :3], xi[..., 3:]
    th2 = (w * w).sum(-1)
    s, c = coeffs(th2)
    W = skew(w)
    A = s[..., None, None] * W + c[..., None, None] * (w[..., :, None] * w[..., None, :]
                                                       - th2[..., None, None] * torch.eye(3, dtype=torch.float64))
    D = torch.zeros(xi.shape[:-1] + (4, 4), dtype=torch.float64)
    D[..., :3, :3] = A
    D[..., 3, :3] = t
    return D


def rotation(w):
    """R(w) = I + A, (..., 3, 3)"""
    return torch.eye(3, dtype=torch.float64) + delta(torch.cat([w.double(), torch.zeros_like(w.double())], -1))[..., :3, :3]


def rigid_inverse(view0):
    v = view0.double()
    R, t = v[..., :3, :3], v[..., 3, :3]
    inv = torch.zeros_like(v)
    inv[..., :3, :3] = R.transpose(-1, -2)
    inv[..., 3, :3] = -(t[..., None, :] @ R.transpose(-1, -2))[..., 0, :]
    inv[..., 3, 3] = 1.0
    return inv


def pose_map(poses, idx, view0, proj0):
    """(view, proj) (B,4,4) float64 of the batch ``idx`` (a host list or int64 tensor): the kernel's map in float64,
    differentiable in ``poses``"""
    idx = torch.as_tensor(idx, dtype=torch.int64)
    v0, p0 = view0.double()[idx], proj0.double()[idx]
    D = delta(poses[idx])
    M = v0 @ D
    K = rigid_inverse(v0) @ p0
    return v0 + M, p0 + M @ K


def look_at(eye, at=(0.0, 0.0, 0.0), up=(0.0, 1.0, 0.0)):
    """a world-to-view matrix (4,4) float64, row-vector convention, of a camera at ``eye`` looking at ``at`` (the
    camera's +z towards ``at``)"""
    eye, at, up = (torch.as_tensor(x, dtype=torch.float64) for x in (eye, at, up))
    z = at - eye
    z = z / z.norm()
    x = torch.linalg.cross(up, z)
    x = x / x.norm()
    y = torch.linalg.cross(z, x)
    R = torch.stack([x, y, z], 1)       # columns: world -> view is p R
    m = torch.eye(4, dtype=torch.float64)
    m[:3, :3] = R
    m[3, :3] = -(eye @ R)
    return m
