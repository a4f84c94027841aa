"""Surface-splatting renderer -- host-side mirror of DSS/core/renderer.py (same class name, constructor and
forward signature; returns (N,H,W,4) RGBA).  Select it from YAML with
``renderer.renderer_type: dss_b200.core.renderer.SurfaceSplattingRenderer`` (config.py:241-262).

By default ``forward`` runs the FUSED path: one call into libdss_b200.so per direction
(dss_render_forward / dss_render_backward) covering per-point EWA preprocess, tile binning, top-K
rasterization, the normalised blend and the alpha channel -- i.e. rasterizer.forward + the weights /
compositor / concat code of renderer.py:53-78.  Passing ``fragments=`` (or ``fused=False``) takes the
unfused route through ``SurfaceSplatting.forward`` and the compositor, like the reference.
"""
import torch
import torch.nn as nn

from ..ops import render_points
from .camera import camera_matrices
from .cloud import clouds_equal_sized, clouds_share_points
from .rasterizer import PointFragments, _splat_params

__all__ = ["SurfaceSplattingRenderer", "NormWeightedCompositor"]


class NormWeightedCompositor(nn.Module):
    """pytorch3d ``NormWeightedCompositor`` [ext] restated with torch indexing (SURVEY.md Appendix D):
    forward(idx (N,K,H,W) int64, alphas (N,K,H,W), features (C,P)) -> (N,C,H,W),
    sum_k alpha_k f[:, idx_k] / max(sum_k alpha_k, 1e-4), fragments with idx < 0 ignored."""

    def forward(self, fragments, alphas, ptclds, **kwargs):
        valid = (fragments >= 0)
        w = alphas * valid
        f = ptclds[:, fragments.clamp(min=0)]                    # (C,N,K,H,W)
        num = (f * w[None]).sum(dim=2)                           # (C,N,H,W)
        den = w.sum(dim=1).clamp(min=1e-4)                       # (N,H,W)
        return (num / den[None]).permute(1, 0, 2, 3)


class SurfaceSplattingRenderer(nn.Module):
    """renderer.py:14-82"""

    def __init__(self, rasterizer, compositor=None, antialiasing_sigma: float = 1.0, density: float = 1e-4,
                 frnn_radius=-1, fused: bool = True):
        super().__init__()
        self.rasterizer = rasterizer
        self.compositor = compositor if compositor is not None else NormWeightedCompositor()
        self.cameras = self.rasterizer.cameras
        self._Vrk_h = None
        self.antialiasing_sigma = antialiasing_sigma
        self.density = density
        self.frnn_radius = frnn_radius
        self.fused = fused

    def to(self, device):
        self.rasterizer.to(device)
        self.cameras = self.rasterizer.cameras
        return self

    def _forward_fused(self, point_clouds, **kwargs):
        rast = self.rasterizer
        rs = kwargs.get("raster_settings", rast.raster_settings)
        cameras = rast._cameras(kwargs)
        point_clouds = rast._prepare_clouds(point_clouds, kwargs.get("point_clouds_filter", None), cameras)
        dev = point_clouds.device
        proj, view = camera_matrices(cameras)
        prm = _splat_params(rs, cameras, kwargs)
        shared = clouds_share_points(point_clouds) and clouds_equal_sized(point_clouds)
        frames = None
        with torch.no_grad():
            h = kwargs.get("Vrk_h", None)
            if h is None:
                h = rast._compute_h(point_clouds, **kwargs)
            if h is None:
                # anisotropic splats: the frames of the one cloud (shared) or of every packed cloud
                frames = rast._compute_frames(point_clouds, shared)
            else:
                h = h.to(dev)
        feats = point_clouds.features_packed()[:, :3].contiguous()
        verbose = kwargs.get("verbose", False)
        if shared:
            out = render_points(point_clouds.points_list()[0], point_clouds.normals_list()[0], feats, proj.to(dev),
                                view.to(dev), h, prm, shared_cloud=True, return_fragments=verbose, frames=frames)
        else:
            out = render_points(point_clouds.points_packed(), point_clouds.normals_packed(), feats, proj.to(dev),
                                view.to(dev), h, prm, first_idx=point_clouds.cloud_to_packed_first_idx(),
                                num_points=point_clouds.num_points_per_cloud(), shared_cloud=False,
                                return_fragments=verbose, frames=frames)
        pcf = kwargs.get("point_clouds_filter", None)
        if pcf is not None:
            num = point_clouds.num_points_per_cloud()
            first = point_clouds.cloud_to_packed_first_idx()
            padded = torch.zeros((len(point_clouds), int(num.max())), dtype=torch.bool, device=dev)
            vis = out.visible.bool()
            for n in range(len(point_clouds)):
                padded[n, : int(num[n])] = vis[int(first[n]): int(first[n]) + int(num[n])]
            pcf.set_filter(visibility=padded)
        if verbose:
            frag_scaler = torch.where(out.idx >= 0, out.scaler[out.idx.clamp(min=0).long()],
                                      torch.zeros_like(out.qvalue))
            return out.image, PointFragments(idx=out.idx, zbuf=out.zbuf, qvalue=out.qvalue, scaler=frag_scaler,
                                             occupancy=out.image[..., 3])
        return out.image

    def forward(self, point_clouds, **kwargs) -> torch.Tensor:
        """point_clouds_filter: used to get the activation mask and receive the visibility mask."""
        if point_clouds.isempty():
            return None
        fragments = kwargs.get("fragments", None)
        if fragments is None and kwargs.get("fused", self.fused):
            return self._forward_fused(point_clouds, **kwargs)
        if fragments is None:
            out = self.rasterizer(point_clouds, **kwargs)
            fragments, point_clouds = out[0], out[1]
        # weight: scalar * exp(-0.5 Q)   (renderer.py:53-54)
        weights = (torch.exp(-0.5 * fragments.qvalue) * fragments.scaler).permute(0, 3, 1, 2)
        pts_rgb = point_clouds.features_packed()[:, :3]
        images = self.compositor(fragments.idx.long().permute(0, 3, 1, 2), weights, pts_rgb.permute(1, 0), **kwargs)
        images = images.permute(0, 2, 3, 1)
        images = torch.cat([images, fragments.occupancy.unsqueeze(-1)], dim=-1)
        if kwargs.get("verbose", False):
            return images, fragments
        return images
