"""Minimal camera model for the hot path (pytorch3d is not a dependency of this package).

Restates the pytorch3d 0.4.0 conventions DSS relies on (SURVEY.md Appendix D; call sites
DSS/core/rasterizer.py:138,188,465-466, config.py:259, scripts/create_mvr_data_from_mesh.py:137-143):
row-vector transforms ``X_view = X_world @ R + T``; NDC +X left, +Y up, camera looks along +Z;
``get_full_projection_transform = world_to_view o projection``.  Any object exposing the same four
members (``R``, ``T``, ``get_world_to_view_transform()``, ``get_full_projection_transform()`` with
``.get_matrix()``) -- e.g. a real ``pytorch3d.renderer.FoVPerspectiveCameras`` -- can be passed to the
rasterizer instead.
"""
import math

import torch

__all__ = ["FoVPerspectiveCameras", "look_at_view_transform", "look_at_rotation", "camera_matrices", "CameraSampler"]


class _Transform:
    def __init__(self, matrix):
        self._m = matrix

    def get_matrix(self):
        return self._m

    def compose(self, other):
        return _Transform(self._m @ other.get_matrix())

    def transform_points(self, points, eps=None):
        """points (N,P,3) or (P,3) -> same shape; homogeneous divide like pytorch3d Transform3d."""
        squeeze = points.dim() == 2
        pts = points[None] if squeeze else points
        ones = torch.ones_like(pts[..., :1])
        out = torch.cat([pts, ones], dim=-1) @ self._m
        denom = out[..., 3:]
        if eps is not None:
            sign = denom.sign() + (denom == 0.0).type_as(denom)
            denom = sign * torch.clamp(denom.abs(), eps)
        out = out[..., :3] / denom
        return out[0] if squeeze else out

    def transform_normals(self, normals):
        """Normals transform with the inverse-transpose of the linear part (pytorch3d Transform3d)."""
        squeeze = normals.dim() == 2
        nrm = normals[None] if squeeze else normals
        mat = self._m[:, :3, :3]
        out = nrm @ torch.inverse(mat).transpose(1, 2)
        return out[0] if squeeze else out


def look_at_rotation(camera_position, at=((0.0, 0.0, 0.0),), up=((0.0, 1.0, 0.0),)):
    camera_position = torch.as_tensor(camera_position, dtype=torch.float32).reshape(-1, 3)
    at = torch.as_tensor(at, dtype=torch.float32).reshape(-1, 3).expand_as(camera_position)
    up = torch.as_tensor(up, dtype=torch.float32).reshape(-1, 3).expand_as(camera_position)
    z_axis = torch.nn.functional.normalize(at - camera_position, eps=1e-5)
    x_axis = torch.nn.functional.normalize(torch.cross(up, z_axis, dim=1), eps=1e-5)
    y_axis = torch.nn.functional.normalize(torch.cross(z_axis, x_axis, dim=1), eps=1e-5)
    is_close = torch.isclose(x_axis, torch.tensor(0.0), atol=5e-3).all(dim=1, keepdim=True)
    if is_close.any():
        replacement = torch.nn.functional.normalize(torch.cross(y_axis, z_axis, dim=1), eps=1e-5)
        x_axis = torch.where(is_close, replacement, x_axis)
    R = torch.cat((x_axis[:, None, :], y_axis[:, None, :], z_axis[:, None, :]), dim=1)
    return R.transpose(1, 2)


def look_at_view_transform(dist=1.0, elev=0.0, azim=0.0, degrees=True, at=((0.0, 0.0, 0.0),),
                           up=((0.0, 1.0, 0.0),)):
    """(R (N,3,3), T (N,3)) of cameras on a sphere around ``at`` (pytorch3d look_at_view_transform)."""
    dist = torch.as_tensor(dist, dtype=torch.float32).reshape(-1)
    elev = torch.as_tensor(elev, dtype=torch.float32).reshape(-1)
    azim = torch.as_tensor(azim, dtype=torch.float32).reshape(-1)
    n = max(dist.numel(), elev.numel(), azim.numel())
    dist, elev, azim = dist.expand(n), elev.expand(n), azim.expand(n)
    at = torch.as_tensor(at, dtype=torch.float32).reshape(-1, 3).expand(n, 3)
    if degrees:
        elev, azim = elev * (math.pi / 180.0), azim * (math.pi / 180.0)
    x = dist * torch.cos(elev) * torch.sin(azim)
    y = dist * torch.sin(elev)
    z = dist * torch.cos(elev) * torch.cos(azim)
    C = torch.stack([x, y, z], dim=1) + at
    R = look_at_rotation(C, at=at, up=up)
    T = -torch.bmm(R.transpose(1, 2), C[:, :, None])[:, :, 0]
    return R, T


class FoVPerspectiveCameras(torch.nn.Module):
    """Field-of-view perspective camera batch (fov 60 deg, znear 1.0, zfar 100, aspect 1 by default)."""

    def __init__(self, znear=1.0, zfar=100.0, aspect_ratio=1.0, fov=60.0, degrees=True, R=None, T=None,
                 device="cpu"):
        super().__init__()
        if R is None:
            R = torch.eye(3)[None]
        if T is None:
            T = torch.zeros(1, 3)
        R = torch.as_tensor(R, dtype=torch.float32).reshape(-1, 3, 3)
        T = torch.as_tensor(T, dtype=torch.float32).reshape(-1, 3)
        n = max(R.shape[0], T.shape[0])
        self.R = R.expand(n, 3, 3).clone().to(device)
        self.T = T.expand(n, 3).clone().to(device)
        self.znear, self.zfar = float(znear), float(zfar)
        self.aspect_ratio, self.fov, self.degrees = float(aspect_ratio), float(fov), bool(degrees)

    def __len__(self):
        return self.R.shape[0]

    @property
    def device(self):
        return self.R.device

    def to(self, device):
        self.R, self.T = self.R.to(device), self.T.to(device)
        return self

    def clone(self):
        return FoVPerspectiveCameras(self.znear, self.zfar, self.aspect_ratio, self.fov, self.degrees,
                                     self.R.clone(), self.T.clone(), device=self.R.device)

    def get_camera_center(self):
        return -torch.bmm(self.R, self.T[:, :, None])[:, :, 0]   # C = -R T  (X_view = X R + T)

    def get_world_to_view_transform(self, **kwargs):
        R, T = kwargs.get("R", self.R), kwargs.get("T", self.T)
        n = R.shape[0]
        m = torch.zeros(n, 4, 4, dtype=R.dtype, device=R.device)
        m[:, :3, :3] = R
        m[:, 3, :3] = T
        m[:, 3, 3] = 1.0
        return _Transform(m)

    def get_projection_transform(self, **kwargs):
        n, dev = self.R.shape[0], self.R.device
        fov = self.fov * math.pi / 180.0 if self.degrees else self.fov
        t = math.tan(fov / 2.0)
        m = torch.zeros(n, 4, 4, dtype=torch.float32, device=dev)
        m[:, 0, 0] = 1.0 / (self.aspect_ratio * t)
        m[:, 1, 1] = 1.0 / t
        m[:, 2, 2] = self.zfar / (self.zfar - self.znear)
        m[:, 3, 2] = -(self.zfar * self.znear) / (self.zfar - self.znear)
        m[:, 2, 3] = 1.0
        return _Transform(m)

    def get_full_projection_transform(self, **kwargs):
        return self.get_world_to_view_transform(**kwargs).compose(self.get_projection_transform(**kwargs))

    def transform_points(self, points, eps=None, **kwargs):
        return self.get_full_projection_transform(**kwargs).transform_points(points, eps=eps)


def camera_matrices(cameras, **kwargs):
    """(proj (N,4,4), view (N,4,4)) float32 contiguous, row-vector convention, from any camera object."""
    proj = cameras.get_full_projection_transform().get_matrix()
    view = cameras.get_world_to_view_transform().get_matrix()
    return proj.float().contiguous(), view.float().contiguous()


class CameraSampler:
    """Random cameras looking at (about) the origin from varying distances, in batches (DSS/core/camera.py:6-71):
    distances uniform in ``distance_range`` (sorted descending with ``sort_distance``), azimuth uniform in [-180, 180),
    elevation in [-90, 90) degrees and ``at`` uniform in [-0.05, 0.05)^3, through :func:`look_at_view_transform`.
    Iterating yields ``camera_type(R=..., T=..., **camera_params)`` of ``num_cams_batch`` cameras (the last batch may be
    smaller).  All draws come from ``generator`` (a ``torch.Generator``; None: torch's global one)."""

    def __init__(self, num_cams_total, num_cams_batch, distance_range=(5, 10), sort_distance=True,
                 camera_type=FoVPerspectiveCameras, camera_params=None, generator=None):
        self.num_cams_total, self.num_cams_batch = int(num_cams_total), int(num_cams_batch)
        self.sort_distance = sort_distance
        self.camera_type = camera_type
        self.camera_params = {} if camera_params is None else dict(camera_params)
        rng = torch.as_tensor(distance_range, dtype=torch.float32).reshape(-1, 2)
        n, g = self.num_cams_total, generator
        distances = torch.rand(n, generator=g) * (rng[:, 1] - rng[:, 0]) + rng[:, 0]
        if sort_distance:
            distances, _ = distances.sort(descending=True)
        azim = torch.rand(n, generator=g) * 360 - 180
        elev = torch.rand(n, generator=g) * 180 - 90
        at = torch.rand((n, 3), generator=g) * 0.1 - 0.05
        self.distances, self.azim, self.elev, self.at = distances, azim, elev, at
        self.R, self.T = look_at_view_transform(distances, elev, azim, at=at, degrees=True)
        self._idx = 0

    def __len__(self):
        return (self.R.shape[0] + self.num_cams_batch - 1) // self.num_cams_batch

    def __iter__(self):
        return self

    def __next__(self):
        if self._idx >= len(self):
            raise StopIteration
        start = self._idx * self.num_cams_batch
        end = min(start + self.num_cams_batch, self.R.shape[0])
        self._idx += 1
        return self.camera_type(R=self.R[start:end], T=self.T[start:end], **self.camera_params)
