"""Point-cloud regularisers of the training step -- twins of DSS/training/losses.py:24-62 (BaseLoss), :148-277
(SurfaceLoss), :282-397 (ProjectionLoss) and :400-497 (RepulsionLoss), same class names, constructor arguments,
``forward(point_clouds, points_filter=..., rebuild_knn=..., knn_tree=...)`` signature and reductions.

They are rebuilt every iteration by the trainer (trainer.py:134-137, 321-326 with ``knn_k = 12``) and start with a
K-nearest-neighbour search over the cloud: pytorch3d ``knn_points`` in the reference, here
``dss_b200.frnn_grid.knn_points_packed`` (csrc/knn.cu: density-sized grid, ring search).

Two routes compute the same formulas, chosen by device and dtype:

* float32 CUDA points and normals take the fused route: the K-NN rows of the packed cloud go to
  ``dss_surface_regulariser`` (csrc/regularisers.cu), which writes each row's loss and its gradient with respect to the
  row's own position in two or three kernels (the neighbour positions, the weights and the denoised normals are
  detached in the reference, so the gradient is a closed form).  No padded round trip, no host synchronisation.
* every other dtype or device runs the torch body below (autograd gives the position gradients), which is also the
  float64 reference of the tests.

CUDA tensors take the CUDA K-NN; a caller on another device passes ``knn_tree=(dists, idx, knn)`` (the reference has
the same keyword) -- there is no CPU search in this package.
"""
from typing import NamedTuple, Optional

import torch
import torch.nn as nn

from .. import _lib

__all__ = ["BaseLoss", "L1Loss", "L2Loss", "SurfaceLoss", "ProjectionLoss", "RepulsionLoss", "KNN",
           "surface_regulariser"]


class KNN(NamedTuple):
    """pytorch3d's ``_KNN``: squared distances (N,P,K), indices (N,P,K) int64, neighbour positions (N,P,K,3)."""
    dists: torch.Tensor
    idx: torch.Tensor
    knn: Optional[torch.Tensor]


def eps_denom(denom, eps=1e-17):
    """DSS/utils/mathHelper.py:10-14: sign-preserving clamp, zero counts as positive."""
    sign = denom.sign().detach()
    sign = torch.where(sign == 0, torch.ones_like(sign), sign)
    return sign * torch.clamp(denom.abs(), min=eps)


def knn_gather(x, idx, lengths=None):
    """pytorch3d.ops.knn_gather: x (N,M,U), idx (N,P,K) -> (N,P,K,U); rows past `lengths` are zero."""
    N, P, K = idx.shape
    U = x.shape[-1]
    out = torch.gather(x[:, None].expand(-1, P, -1, -1), 2, idx[..., None].expand(-1, -1, -1, U))
    if lengths is not None:
        # pytorch3d zeroes neighbours that do not exist (k >= length of the cloud)
        need = torch.arange(K, device=idx.device)[None, None, :] >= lengths[:, None, None]
        out = torch.where(need[..., None], torch.zeros_like(out), out)
    return out


class BaseLoss(nn.Module):
    """losses.py:24-62."""

    def __init__(self, reduction: str = "mean", channel_dim: Optional[int] = -1):
        super().__init__()
        self.reduction = reduction
        self.channel_dim = channel_dim
        self.hooks = []

    def compute(self, *args, **kwargs):
        raise NotImplementedError

    def _reduce(self, loss, reduction=None):
        reduction = reduction or self.reduction
        if reduction == "none":
            return loss
        if reduction == "sum":
            return torch.sum(loss)
        if reduction == "mean":
            return torch.mean(loss)
        raise ValueError("Invalid reduction method ({})".format(self.reduction))

    def forward(self, *args, **kwargs):
        reduction = kwargs.pop("reduction", self.reduction)
        self.channel_dim = kwargs.pop("channel_dim", self.channel_dim)
        loss = self.compute(*args, **kwargs)
        if self.channel_dim is not None:
            loss = torch.sum(loss, dim=self.channel_dim)
        return self._reduce(loss, reduction=reduction)


class L1Loss(BaseLoss):
    def compute(self, x, y, weights=None, mask=None, **kwargs):
        loss = torch.abs(x - y)
        if weights is not None:
            loss = loss * weights
        return loss[mask] if mask is not None else loss


class L2Loss(BaseLoss):
    def compute(self, x, y, weights=None, mask=None, **kwargs):
        loss = (x - y) ** 2
        if weights is not None:
            loss = loss * weights
        return loss[mask] if mask is not None else loss


def _padded_to_packed(x, lengths):
    """(N, Pmax, ...) -> (sum lengths, ...)"""
    keep = torch.arange(x.shape[1], device=x.device)[None, :] < lengths[:, None]
    return x[keep]


# -- fused route (float32 CUDA) ------------------------------------------------------------------------------------------
_KINDS = {"projection": 0, "repulsion": 1}


class _SurfaceRegulariser(torch.autograd.Function):
    """dss_surface_regulariser forward; the backward contracts the saved per-row gradient coefficients."""

    @staticmethod
    def forward(ctx, points, normals, first_idx, num_points, knn_dists, knn_idx, K, self_col, knn_points,
                neighbour_points, reliable, visible, kind, sharpness_sigma, filter_scale):
        dev = points.device
        P, N = points.shape[0], num_points.shape[0]
        loss = torch.empty((P,) if kind == 0 else (P, 3), dtype=torch.float32, device=dev)
        coef = torch.empty((P, 3 if kind == 0 else 9), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            rc = _lib.load().dss_surface_regulariser(
                _lib.ctx(dev), kind, _lib.ptr(points), _lib.ptr(normals), _lib.ptr(first_idx), _lib.ptr(num_points), N,
                P, _lib.ptr(knn_dists), _lib.ptr(knn_idx), K, self_col, _lib.ptr(knn_points), _lib.ptr(neighbour_points),
                _lib.ptr(reliable), _lib.ptr(visible),
                float(sharpness_sigma), float(filter_scale), _lib.ptr(loss), _lib.ptr(coef), _lib.stream_ptr(dev))
        _lib.check(rc, "dss_surface_regulariser")
        ctx.kind = kind
        ctx.save_for_backward(coef)
        return loss

    @staticmethod
    def backward(ctx, grad_loss):
        coef, = ctx.saved_tensors
        if ctx.kind == 0:
            grad = grad_loss[:, None] * coef
        else:
            grad = (coef.view(-1, 3, 3) * grad_loss[:, None, :]).sum(dim=-1)
        return (grad,) + (None,) * 14


def surface_regulariser(kind, points, normals, first_idx, num_points, knn_dists, knn_idx, self_col=True,
                        knn_points=None, neighbour_points=None, reliable=None, visible=None, sharpness_sigma=0.75,
                        filter_scale=1.0):
    """Packed ProjectionLoss (``kind="projection"``, loss (P,)) or RepulsionLoss (``"repulsion"``, loss (P,3)) of
    float32 CUDA clouds, before the reduction, differentiable with respect to ``points`` only.

    ``points``, ``normals`` (P,3); cloud n owns rows [first_idx[n], first_idx[n] + num_points[n]) (int64, contiguous
    clouds).  ``knn_dists`` (P,W) float32 and ``knn_idx`` (P,W) int32, contiguous: each row's neighbours local to its
    cloud, ascending, as ``knn_points_packed`` returns them; ``self_col``: column 0 is the query itself (W = knn_k) or
    not (W = knn_k - 1); 2 <= knn_k <= 32.  Neighbour positions: ``knn_points`` (P,W,3) float32, one per column, used
    as given (pytorch3d's ``knn``), or else read at the neighbour's index from ``neighbour_points`` (P,3) float32 (the
    positions the rows were built on; ``points`` when None), zero for columns past the cloud's length as
    ``knn_gather(..., lengths)`` gives them.  ``reliable`` (P,) bool: rows that keep their own normal in the denoise
    (visibility & inmask); ``visible`` (P,) bool, projection only: neighbours outside it weigh 0.1."""
    if kind not in _KINDS:
        raise RuntimeError("kind must be 'projection' or 'repulsion'")
    _lib.require_cuda(points, normals, first_idx, num_points, knn_dists, knn_idx, reliable, visible)
    if points.dim() != 2 or points.shape[1] != 3 or normals.shape != points.shape:
        raise RuntimeError("points and normals must both have shape (P, 3)")
    if points.dtype != torch.float32 or normals.dtype != torch.float32:
        raise RuntimeError("points and normals must be float32")
    if first_idx.dim() != 1 or first_idx.shape != num_points.shape or first_idx.dtype != torch.int64 \
            or num_points.dtype != torch.int64:
        raise RuntimeError("first_idx and num_points must be int64 of shape (N,)")
    P = points.shape[0]
    if knn_dists.dim() != 2 or knn_dists.shape[0] != P or knn_idx.shape != knn_dists.shape:
        raise RuntimeError("knn_dists and knn_idx must both have shape (P, W) with P = %d" % P)
    if knn_dists.dtype != torch.float32 or knn_idx.dtype != torch.int32:
        raise RuntimeError("knn_dists must be float32 and knn_idx int32")
    if not (knn_dists.is_contiguous() and knn_idx.is_contiguous()):
        raise RuntimeError("knn_dists and knn_idx must be contiguous")
    K = knn_dists.shape[1] + (0 if self_col else 1)
    if not 2 <= K <= 32:
        raise RuntimeError("knn_k must be in [2, 32], got %d" % K)
    W = knn_dists.shape[1]
    for name, t, shape in (("knn_points", knn_points, (P, W, 3)), ("neighbour_points", neighbour_points, (P, 3))):
        if t is not None and (t.shape != shape or t.dtype != torch.float32 or not t.is_contiguous()):
            raise RuntimeError("%s must be a contiguous float32 tensor of shape %s" % (name, shape))
    masks = []
    for name, m in (("reliable", reliable), ("visible", visible)):
        if m is not None and (m.shape != (P,) or m.dtype not in (torch.bool, torch.uint8)):
            raise RuntimeError("%s must be a (P,) bool tensor" % name)
        masks.append(None if m is None else m.contiguous())
    return _SurfaceRegulariser.apply(points.contiguous(), normals.detach().contiguous(), first_idx.contiguous(),
                                     num_points.contiguous(), knn_dists, knn_idx, K, int(bool(self_col)),
                                     None if knn_points is None else knn_points.detach(),
                                     None if neighbour_points is None else neighbour_points.detach(), masks[0],
                                     masks[1], _KINDS[kind], sharpness_sigma, filter_scale)


class _KnnRows(NamedTuple):
    """The fused route's K-NN of a packed cloud: (P,W) rows, whether column 0 is the query, the neighbour positions
    (per column, or the (P,3) points the rows were built on) and the (N, P_max, P) sizes they belong to."""
    dists: torch.Tensor
    idx: torch.Tensor
    self_col: bool
    knn_points: Optional[torch.Tensor]
    neighbour_points: Optional[torch.Tensor]
    shape: tuple


def _use_fused(point_clouds):
    """the fused route serves float32 CUDA clouds; other dtypes and devices run the torch body"""
    pts, nrm = point_clouds.points_packed(), point_clouds.normals_packed()
    return nrm is not None and pts.is_cuda and nrm.is_cuda and pts.dtype == torch.float32 \
        and nrm.dtype == torch.float32


def _packed_mask(mask, N, Pmax, cloud, local, broadcast):
    """padded (B, Pmax) filter -> (P,) bool of the packed rows: a gather of known shape, no boolean indexing.  A batch
    of B > 1 over one cloud is or-ed over B, as the torch body does; a batch of 1 over N > 1 clouds applies to every
    cloud where the torch body broadcasts it (``broadcast``)."""
    if mask.dim() != 2 or mask.shape[1] != Pmax:
        raise RuntimeError("filter must have shape (B, %d), got %s" % (Pmax, tuple(mask.shape)))
    if mask.shape[0] != N and N == 1:
        mask = mask.any(dim=0, keepdim=True)
    if mask.shape[0] == N:
        flat = cloud * Pmax + local
    elif mask.shape[0] == 1 and broadcast:
        flat = local
    else:
        raise RuntimeError("filter of batch %d does not match %d clouds" % (mask.shape[0], N))
    return mask.reshape(-1).index_select(0, flat).bool()


class SurfaceLoss(BaseLoss):
    """losses.py:148-277: neighbourhood weights shared by the two regularisers."""

    def __init__(self, reduction="mean", knn_k: int = 33, filter_scale: float = 1.0, sharpness_sigma: float = 0.75):
        super().__init__(reduction=reduction, channel_dim=None)
        self.knn_tree = None
        self.knn_mask = None
        self.knn_rows = None      # fused route: _KnnRows of the packed cloud, kept for rebuild_knn=False
        self.knn_k = knn_k
        self.filter_scale = filter_scale
        self.sharpness_sigma = sharpness_sigma

    # -- neighbourhood ---------------------------------------------------------------------------
    def _build_knn(self, point_clouds):
        """losses.py:157-180: K nearest neighbours of every point inside its own cloud, the point itself dropped."""
        from ..frnn_grid import knn_points
        points_padded = point_clouds.points_padded()
        lengths = point_clouds.num_points_per_cloud()
        dists, idx, knn = knn_points(points_padded.detach(), points_padded.detach(), lengths, lengths, K=self.knn_k,
                                     return_nn=True)
        self._set_tree(KNN(dists, idx, knn), lengths)

    def _set_tree(self, tree, lengths):
        dists, idx, knn = tree
        K = dists.shape[-1]
        mask = torch.arange(idx.shape[1], device=idx.device)[None, :, None] < lengths[:, None, None]
        mask = mask & (torch.arange(K, device=idx.device)[None, None, :] < lengths.clamp(max=K)[:, None, None])
        self.knn_tree = KNN(dists[:, :, 1:], idx[:, :, 1:], None if knn is None else knn[:, :, 1:, :])
        self.knn_mask = mask[:, :, 1:]

    def _ensure_tree(self, point_clouds, rebuild_knn, kwargs):
        tree = kwargs.get("knn_tree", None)
        points = point_clouds.points_padded()
        lengths = point_clouds.num_points_per_cloud()
        if tree is not None:
            tree = KNN(*tree)
            if tree.dists.shape[-1] == self.knn_k:          # full result incl. the query itself (pytorch3d layout)
                if tree.knn is None:
                    tree = KNN(tree.dists, tree.idx, knn_gather(points.detach(), tree.idx, lengths))
                self._set_tree(tree, lengths)
            else:                                           # already without the query point (losses.py:305)
                self.knn_tree = tree if tree.knn is not None else KNN(tree.dists, tree.idx,
                                                                      knn_gather(points.detach(), tree.idx, lengths))
                self.knn_mask = kwargs.get("knn_mask", self.knn_mask)
        elif rebuild_knn or self.knn_tree is None or self.knn_tree.idx.shape[:2] != points.shape[:2]:
            self._build_knn(point_clouds)

    # -- fused route -------------------------------------------------------------------------------
    def _fused(self, kind, point_clouds, points_filter, rebuild_knn, kwargs):
        """The loss of every packed row through dss_surface_regulariser.  The K-NN rows come from knn_points_packed,
        from a caller's ``knn_tree`` (padded, with or without the query column, as ``_ensure_tree`` takes it) or, when
        ``rebuild_knn=False``, from an earlier call.  Like the torch body's stored tree, the rows keep the neighbour
        positions they were built with: the tree's ``knn`` when given, else a copy of the points of that call.  The
        CUDA search and the kernel take at most 32 columns; wider rows raise instead of running the torch body."""
        from ..frnn_grid import knn_points_packed
        self.sharpness_sigma = kwargs.get("sharpness_sigma", self.sharpness_sigma)
        self.filter_scale = kwargs.get("filter_scale", self.filter_scale)
        points, normals = point_clouds.points_packed(), point_clouds.normals_packed()
        first, num = point_clouds.cloud_to_packed_first_idx(), point_clouds.num_points_per_cloud()
        P, N = points.shape[0], len(point_clouds)
        Pmax = max(p.shape[0] for p in point_clouds.points_list())
        gather = []

        def padded_index():        # packed row -> (cloud, row inside the cloud)
            if not gather:
                cloud = torch.repeat_interleave(torch.arange(N, device=points.device), num, output_size=P)
                gather.extend([cloud, torch.arange(P, device=points.device) - first[cloud]])
            return gather

        tree = kwargs.get("knn_tree", None)
        if tree is not None:
            tree = KNN(*tree)
            W = tree.dists.shape[-1]
            if tree.dists.shape[:2] != (N, Pmax) or tree.idx.shape != tree.dists.shape:
                raise RuntimeError("knn_tree must be padded (N, P_max, K) = (%d, %d, K)" % (N, Pmax))
            cloud, local = padded_index()
            flat = cloud * Pmax + local
            d = tree.dists.reshape(-1, W).index_select(0, flat).to(torch.float32)
            i = tree.idx.reshape(-1, W).index_select(0, flat).to(torch.int32)
            if tree.knn is not None:
                knn = tree.knn.detach().reshape(-1, W, 3).index_select(0, flat).to(torch.float32)
                self.knn_rows = _KnnRows(d, i, W == self.knn_k, knn, None, (N, Pmax, P))
            else:
                self.knn_rows = _KnnRows(d, i, W == self.knn_k, None, points.detach().clone(), (N, Pmax, P))
        elif rebuild_knn or self.knn_rows is None or self.knn_rows.shape != (N, Pmax, P):
            if not 2 <= self.knn_k <= 32:
                raise RuntimeError("knn_k must be in [2, 32] for the CUDA K-NN, got %d" % self.knn_k)
            d, i = knn_points_packed(points, first, num, self.knn_k)
            self.knn_rows = _KnnRows(d, i, True, None, points.detach().clone(), (N, Pmax, P))
        rows = self.knn_rows
        reliable = visible = None
        vis = getattr(points_filter, "visibility", None) if points_filter is not None else None
        if vis is not None:
            inmask = getattr(points_filter, "inmask", None)
            rel = vis & inmask if inmask is not None else vis
            reliable = _packed_mask(rel, N, Pmax, *padded_index(), broadcast=True)
            if kind == "projection":      # knn_gather needs a filter per cloud (losses.py:335)
                visible = _packed_mask(vis, N, Pmax, *padded_index(), broadcast=False)
        return surface_regulariser(kind, points, normals, first, num, rows.dists, rows.idx, rows.self_col,
                                   rows.knn_points, rows.neighbour_points, reliable, visible, self.sharpness_sigma,
                                   self.filter_scale)

    # -- weights ---------------------------------------------------------------------------------
    def get_phi(self, point_clouds, **kwargs):
        """(1 - |x - xi|^2 / h^2)^4 with h^2 = 4 x the mean squared neighbour distance (losses.py:258-277)."""
        h = self.knn_tree.dists.mean(dim=-1, keepdim=True) * 4
        w = (1 - self.knn_tree.dists / h).clamp(min=0)
        w = w * w
        return w * w

    def _denoise_normals(self, point_clouds, weights, point_clouds_filter=None):
        """robust normal mollification (losses.py:182-222): padded (N,P,3) weighted neighbour average; points that are
        visible AND inside the mask keep their own normal."""
        lengths = point_clouds.num_points_per_cloud()
        normals = point_clouds.normals_padded()
        knn_normals = knn_gather(normals, self.knn_tree.idx, lengths)
        den = torch.sum(knn_normals * weights[..., None], dim=-2) / eps_denom(torch.sum(weights, dim=-1, keepdim=True))
        if point_clouds_filter is not None and getattr(point_clouds_filter, "visibility", None) is not None:
            reliable = point_clouds_filter.visibility
            if getattr(point_clouds_filter, "inmask", None) is not None:
                reliable = reliable & point_clouds_filter.inmask
            if reliable.shape[0] != normals.shape[0] and normals.shape[0] == 1:
                reliable = reliable.any(dim=0, keepdim=True)
            den = torch.where(reliable[..., None], normals, den)
        return den

    def get_normal_w(self, normals, **kwargs):
        """exp(-|n - ni|^2 / sigma^2) over the neighbourhood, both renormalised (losses.py:224-246)."""
        self.sharpness_sigma = kwargs.get("sharpness_sigma", self.sharpness_sigma)
        inv = 1.0 / (self.sharpness_sigma * self.sharpness_sigma)
        knn_normals = torch.nn.functional.normalize(knn_gather(normals, self.knn_tree.idx), dim=-1)
        n = torch.nn.functional.normalize(normals, dim=-1)
        diff = knn_normals - n[:, :, None, :]
        return torch.exp(-torch.sum(diff * diff, dim=-1) * inv)

    def get_spatial_w(self, point_clouds, points=None, **kwargs):
        """exp(-|p - pi|^2 * (P / diag^2) * filter_scale) (losses.py:248-256)."""
        pts = point_clouds.points_padded()
        lengths = point_clouds.num_points_per_cloud()
        valid = torch.arange(pts.shape[1], device=pts.device)[None, :, None] < lengths[:, None, None]
        lo = torch.where(valid, pts, torch.full_like(pts, float("inf"))).min(dim=1)[0]
        hi = torch.where(valid, pts, torch.full_like(pts, float("-inf"))).max(dim=1)[0]
        diag2 = torch.sum((hi - lo) ** 2, dim=-1)
        inv_sigma = lengths.float() / diag2
        self.filter_scale = kwargs.get("filter_scale", self.filter_scale)
        if points is None:
            points = pts
        d = self.knn_tree.knn - points[:, :, None, :]
        return torch.exp(-torch.sum(d * d, dim=-1) * inv_sigma[:, None, None] * self.filter_scale)


class ProjectionLoss(SurfaceLoss):
    """losses.py:282-397: squared distance to the local plane of every neighbour, weighted (Oztireli et al.)."""

    def get_spatial_w(self, point_clouds, **kwargs):
        return torch.ones_like(self.knn_tree.dists)                       # losses.py:293-298

    def compute(self, point_clouds, points_filter=None, rebuild_knn=False, **kwargs):
        self.sharpness_sigma = kwargs.get("sharpness_sigma", self.sharpness_sigma)
        self.filter_scale = kwargs.get("filter_scale", self.filter_scale)
        if _use_fused(point_clouds):
            return self._fused("projection", point_clouds, points_filter, rebuild_knn, kwargs)
        return self.torch_body(point_clouds, points_filter, rebuild_knn, **kwargs)

    def torch_body(self, point_clouds, points_filter=None, rebuild_knn=False, **kwargs):
        """the loss in torch ops (any dtype and device; autograd gives the position gradients)"""
        lengths = point_clouds.num_points_per_cloud()
        points = point_clouds.points_padded()
        with torch.no_grad():
            self._ensure_tree(point_clouds, rebuild_knn, kwargs)
            phi = self.get_phi(point_clouds, **kwargs)
            normals = self._denoise_normals(point_clouds, phi, points_filter)          # Eq. (11)
            normal_w = self.get_normal_w(normals, **kwargs)
            if points_filter is not None and getattr(points_filter, "visibility", None) is not None:
                vis = points_filter.visibility
                if vis.shape[0] != points.shape[0] and points.shape[0] == 1:
                    vis = vis.any(dim=0, keepdim=True)
                vis_nb = knn_gather(vis.unsqueeze(-1), self.knn_tree.idx, lengths).squeeze(-1)
                visibility_w = torch.where(vis_nb, torch.ones_like(phi), torch.full_like(phi, 0.1))   # :335-337
            else:
                visibility_w = torch.ones_like(phi)
            weights = phi * normal_w * visibility_w
            knn_normals = knn_gather(normals, self.knn_tree.idx, lengths)
        sdf = torch.sum((self.knn_tree.knn.detach() - points.unsqueeze(-2)) * knn_normals, dim=-1)   # :373-374
        weights = _padded_to_packed(weights, lengths)
        sdf = _padded_to_packed(sdf, lengths)
        return torch.sum(weights * sdf * sdf, dim=-1) / eps_denom(torch.sum(weights, dim=-1))         # :390-395


class RepulsionLoss(SurfaceLoss):
    """losses.py:400-497: pushes a point away from the weighted centre of its neighbours inside the local plane."""

    def compute(self, point_clouds, points_filter=None, rebuild_knn=True, **kwargs):
        if _use_fused(point_clouds):
            return self._fused("repulsion", point_clouds, points_filter, rebuild_knn, kwargs)
        return self.torch_body(point_clouds, points_filter, rebuild_knn, **kwargs)

    def torch_body(self, point_clouds, points_filter=None, rebuild_knn=True, **kwargs):
        """the loss in torch ops (any dtype and device; autograd gives the position gradients)"""
        lengths = point_clouds.num_points_per_cloud()
        points = point_clouds.points_padded()
        with torch.no_grad():
            self._ensure_tree(point_clouds, rebuild_knn, kwargs)
            phi = self.get_phi(point_clouds, **kwargs)
            normals = self._denoise_normals(point_clouds, phi, points_filter)
        knn_diff = points.unsqueeze(-2) - self.knn_tree.knn.detach()                                   # :432
        knn_normals = knn_gather(normals, self.knn_tree.idx, lengths)
        proj = knn_diff - (knn_diff * knn_normals).sum(dim=-1, keepdim=True) * knn_normals            # :436-437
        with torch.no_grad():
            spatial_w = self.get_spatial_w(point_clouds, **kwargs)
            normal_w = self.get_normal_w(normals, **kwargs)
            density_w = torch.sum(spatial_w, dim=-1, keepdim=True) + 1.0                               # :470
            weights = spatial_w * normal_w
        weights = _padded_to_packed(weights, lengths)
        proj = _padded_to_packed(proj, lengths)
        density_w = _padded_to_packed(density_w, lengths)
        repel = torch.sum(proj * weights.unsqueeze(-1), dim=1) / eps_denom(torch.sum(weights, dim=1).unsqueeze(-1))
        repel = repel * density_w                                                                      # :482-485
        return torch.exp(-repel.abs())                                                                 # :487
