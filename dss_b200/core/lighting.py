"""Lights and the per-point lighting terms -- the torch twin of DSS/core/lighting.py (which derives from
pytorch3d.renderer.lighting, absent here) for the unfused route and as the autograd reference of the fused CUDA
shading (dss_render_args.shade, csrc/render.cu: shade_point).

Conventions of the reference: colours / directions / locations are (N, L, 3) or (1, L, 3) tensors (N views, L lights);
`diffuse` is Lambert's law with the renormalised normal and light direction summed over the lights
(lighting.py:10-69), `specular` the reflected ray against the view direction, zero where the light is behind the
surface (lighting.py:72-172).  Packed inputs (P,3) take per-point properties gathered by the caller.
"""
import torch
import torch.nn.functional as F

__all__ = ["diffuse", "specular", "DirectionalLights", "PointLights", "pack_lights"]


def _as_nl3(x, device=None):
    t = torch.as_tensor(x, dtype=torch.float32, device=device)
    if t.dim() == 1:
        t = t.view(1, 1, 3)
    elif t.dim() == 2:
        t = t.unsqueeze(0)
    if t.dim() != 3 or t.shape[-1] != 3:
        raise ValueError("expected (N,L,3), got %s" % (tuple(t.shape),))
    return t


def diffuse(normals, color, direction) -> torch.Tensor:
    """normals (..., 3); color, direction (..., L, 3) broadcastable against normals[..., None, :] -> (..., 3)
    (lighting.py:62-69)."""
    n = F.normalize(normals, p=2, dim=-1, eps=1e-6).unsqueeze(-2)
    d = F.normalize(direction, p=2, dim=-1, eps=1e-6)
    angle = F.relu((n * d).sum(-1))
    return (color * angle[..., None]).sum(-2)


def specular(points, normals, direction, color, camera_position, shininess) -> torch.Tensor:
    """points, normals, camera_position (..., 3); direction, color (..., L, 3) -> (..., 3)  (lighting.py:139-172)."""
    n = F.normalize(normals, p=2, dim=-1, eps=1e-6).unsqueeze(-2)
    d = F.normalize(direction, p=2, dim=-1, eps=1e-6)
    cos_angle = (n * d).sum(-1)
    mask = (cos_angle > 0).to(points.dtype)
    view_direction = F.normalize(camera_position - points, p=2, dim=-1, eps=1e-6).unsqueeze(-2)
    reflect_direction = -d + 2 * (cos_angle[..., None] * n)
    alpha = F.relu((view_direction * reflect_direction).sum(-1)) * mask
    return (color * torch.pow(alpha, shininess)[..., None]).sum(-2)


class _Lights(torch.nn.Module):
    """ambient / diffuse / specular colours (N|1, L, 3) + a direction or a location per light."""
    kind = None

    def __init__(self, ambient_color=(((0.5, 0.5, 0.5),),), diffuse_color=(((0.3, 0.3, 0.3),),),
                 specular_color=(((0.2, 0.2, 0.2),),), vec=(((0, 1, 0),),), device="cpu"):
        super().__init__()
        self.register_buffer("ambient_color", _as_nl3(ambient_color, device))
        self.register_buffer("diffuse_color", _as_nl3(diffuse_color, device))
        self.register_buffer("specular_color", _as_nl3(specular_color, device))
        self.register_buffer("_vec", _as_nl3(vec, device))
        for prop in ("diffuse_color", "specular_color", "_vec"):
            if getattr(self, prop).dim() != 3:
                raise ValueError("%s must be an (N,L,3) tensor" % prop)
        if not (self.diffuse_color.shape[1] == self.specular_color.shape[1] == self._vec.shape[1]):
            raise ValueError("diffuse_color, specular_color and the direction/location need the same number of lights")

    @property
    def device(self):
        return self._vec.device

    def _per_point(self, t, view_idx):
        """(N|1, L, 3) -> (P, L, 3) for packed points of views `view_idx` (P,) or broadcast (1, L, 3)."""
        return t if (view_idx is None or t.shape[0] == 1) else t[view_idx]


class DirectionalLights(_Lights):
    """DSS/core/lighting.py:175-225."""
    kind = 0

    def __init__(self, ambient_color=(((0.5, 0.5, 0.5),),), diffuse_color=(((0.3, 0.3, 0.3),),),
                 specular_color=(((0.2, 0.2, 0.2),),), direction=(((0, 1, 0),),), device="cpu", **kwargs):
        super().__init__(ambient_color, diffuse_color, specular_color, direction, device)

    @property
    def direction(self):
        return self._vec

    def diffuse(self, normals, points=None, view_idx=None):
        return diffuse(normals, self._per_point(self.diffuse_color, view_idx), self._per_point(self._vec, view_idx))

    def specular(self, normals, points, camera_position, shininess, view_idx=None):
        return specular(points, normals, self._per_point(self._vec, view_idx),
                        self._per_point(self.specular_color, view_idx), camera_position, shininess)


class PointLights(_Lights):
    """DSS/core/lighting.py:228-300."""
    kind = 1

    def __init__(self, ambient_color=(((0.5, 0.5, 0.5),),), diffuse_color=(((0.3, 0.3, 0.3),),),
                 specular_color=(((0.2, 0.2, 0.2),),), location=(((0, 1, 0),),), device="cpu", **kwargs):
        super().__init__(ambient_color, diffuse_color, specular_color, location, device)

    @property
    def location(self):
        return self._vec

    def diffuse(self, normals, points, view_idx=None):
        direction = self._per_point(self._vec, view_idx) - points.unsqueeze(-2)
        return diffuse(normals, self._per_point(self.diffuse_color, view_idx), direction)

    def specular(self, normals, points, camera_position, shininess, view_idx=None):
        direction = self._per_point(self._vec, view_idx) - points.unsqueeze(-2)
        return specular(points, normals, direction, self._per_point(self.specular_color, view_idx), camera_position,
                        shininess)


def pack_lights(lights):
    """-> (rows, ambient, light_type) for the fused path: rows {direction|location, diffuse rgb, specular rgb}.

    Lights whose properties all have batch 1 (one set for every view) give rows (L,9) and ambient (3,).  Otherwise the
    set is per view, as the reference's data gives every image its own light: properties of batch 1 broadcast against
    those of batch N (as pytorch3d's TensorProperties do) and the result is rows (N,L,9), ambient (N,3).  The ambient
    colours are summed over the lights (texture.py:52-55).  The result is differentiable w.r.t. the light tensors."""
    props = (lights._vec, lights.diffuse_color, lights.specular_color, lights.ambient_color)
    batches = sorted({int(t.shape[0]) for t in props})
    if batches == [1]:
        rows = torch.cat([lights._vec[0], lights.diffuse_color[0], lights.specular_color[0]], dim=1).contiguous().float()
        ambient = lights.ambient_color[0].sum(0).contiguous().float()
        return rows, ambient, int(lights.kind)
    N = batches[-1]
    if len(batches) > 2 or (len(batches) == 2 and batches[0] != 1):
        raise ValueError("light properties must have batch 1 or N, got batches %s" % batches)
    vec, dif, spe, amb = (t.expand(N, -1, -1) for t in props)
    rows = torch.cat([vec, dif, spe], dim=2).contiguous().float()
    return rows, amb.sum(1).contiguous().float(), int(lights.kind)
