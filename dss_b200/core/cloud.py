"""Minimal point-cloud container and filter for the hot path.

The reference's ``PointClouds3D`` subclasses ``pytorch3d.structures.Pointclouds`` (DSS/core/cloud.py:23-79)
and ``PointCloudsFilters`` subclasses ``TensorProperties`` (:285-360).  Only the accessors the rasterizer and
renderer touch are restated here (SURVEY.md section 2.1 row 6): ``points_packed / normals_packed /
features_packed / points_padded / extend / num_points_per_cloud / cloud_to_packed_first_idx /
packed_to_cloud_idx / isempty / len``.  Real pytorch3d ``Pointclouds`` objects expose the same members and
can be passed to the rasterizer instead.
"""
from typing import List, Optional, Sequence, Tuple

import torch

__all__ = ["PointClouds3D", "PointCloudsFilters", "upsample", "remove_outliers", "denoise_normals",
           "project_to_latent_surface"]


def _as_list(x, name):
    if x is None:
        return None
    if torch.is_tensor(x):
        if x.dim() != 3:
            raise ValueError("%s must be a list of (P_i, D) tensors or a padded (N, P, D) tensor" % name)
        return [x[i] for i in range(x.shape[0])]
    return list(x)


class PointClouds3D:
    """Batch of N point clouds (possibly of different sizes) with optional normals and features."""

    def __init__(self, points, normals=None, features=None):
        self._points: List[torch.Tensor] = _as_list(points, "points")
        self._normals: Optional[List[torch.Tensor]] = _as_list(normals, "normals")
        self._features: Optional[List[torch.Tensor]] = _as_list(features, "features")
        for name, lst in (("normals", self._normals), ("features", self._features)):
            if lst is not None and [t.shape[0] for t in lst] != [t.shape[0] for t in self._points]:
                raise ValueError("%s must match points in the number of points per cloud" % name)
        self._cache = {}

    # ---- sizes -------------------------------------------------------------------------------
    def __len__(self):
        return len(self._points)

    @property
    def device(self):
        return self._points[0].device if self._points else torch.device("cpu")

    def isempty(self):
        return len(self._points) == 0 or all(p.shape[0] == 0 for p in self._points)

    def num_points_per_cloud(self):
        if "num" not in self._cache:
            self._cache["num"] = torch.tensor([p.shape[0] for p in self._points], dtype=torch.int64,
                                              device=self.device)
        return self._cache["num"]

    def cloud_to_packed_first_idx(self):
        if "first" not in self._cache:
            num = self.num_points_per_cloud()
            first = torch.zeros_like(num)
            if num.numel() > 1:
                first[1:] = torch.cumsum(num, 0)[:-1]
            self._cache["first"] = first
        return self._cache["first"]

    def packed_to_cloud_idx(self):
        if "p2c" not in self._cache:
            num = self.num_points_per_cloud()
            self._cache["p2c"] = torch.repeat_interleave(torch.arange(len(self), device=self.device), num)
        return self._cache["p2c"]

    def equal_sized(self):
        return len({p.shape[0] for p in self._points}) <= 1

    def shares_points(self):
        """True when every cloud aliases the same point / normal storage (the result of ``extend``)."""
        p0 = self._points[0]
        same = all(p.data_ptr() == p0.data_ptr() and p.shape == p0.shape for p in self._points)
        if same and self._normals is not None:
            n0 = self._normals[0]
            same = all(n.data_ptr() == n0.data_ptr() for n in self._normals)
        return same

    # ---- data --------------------------------------------------------------------------------
    def points_list(self):
        return self._points

    def normals_list(self):
        return self._normals

    def features_list(self):
        return self._features

    def _packed(self, lst, key):
        if lst is None:
            return None
        if key not in self._cache:
            self._cache[key] = torch.cat(lst, dim=0) if len(lst) > 1 else lst[0]
        return self._cache[key]

    def points_packed(self):
        return self._packed(self._points, "pp")

    def normals_packed(self):
        return self._packed(self._normals, "np")

    def features_packed(self):
        return self._packed(self._features, "fp")

    def _padded(self, lst, key):
        if lst is None:
            return None
        if key not in self._cache:
            if self.equal_sized():
                self._cache[key] = torch.stack(lst, dim=0)
            else:
                P = max(t.shape[0] for t in lst)
                out = lst[0].new_zeros((len(lst), P) + tuple(lst[0].shape[1:]))
                for i, t in enumerate(lst):
                    out[i, : t.shape[0]] = t
                self._cache[key] = out
        return self._cache[key]

    def points_padded(self):
        return self._padded(self._points, "ppad")

    def normals_padded(self):
        return self._padded(self._normals, "npad")

    def features_padded(self):
        return self._padded(self._features, "fpad")

    # ---- transforms --------------------------------------------------------------------------
    def extend(self, N: int):
        """N copies of every cloud, aliasing the same tensors (pytorch3d ``Pointclouds.extend``)."""
        if N <= 0:
            raise ValueError("N must be > 0")
        rep = lambda lst: None if lst is None else [t for t in lst for _ in range(N)]
        return PointClouds3D(rep(self._points), rep(self._normals), rep(self._features))

    def to(self, device):
        mv = lambda lst: None if lst is None else [t.to(device) for t in lst]
        return PointClouds3D(mv(self._points), mv(self._normals), mv(self._features))

    def clone(self):
        cp = lambda lst: None if lst is None else [t.clone() for t in lst]
        return PointClouds3D(cp(self._points), cp(self._normals), cp(self._features))

    def update_features(self, features):
        """Same geometry, new per-point features (what LightingTexture produces: texture.py:118-127)."""
        return PointClouds3D(self._points, self._normals, features)

    def estimate_normals(self, neighborhood_size: int = 20, disambiguate_directions: bool = True,
                         assign_to_self: bool = False):
        """The clouds' normals by :func:`dss_b200.ops.estimate_normals` (DSS/core/cloud.py:210-258), as a padded
        (N, P, 3) tensor; with ``assign_to_self`` they also replace the clouds' normals.

        Two departures from the reference: ``neighborhood_size`` defaults to 20 (meshlab's K; the reference's 50 is above
        the device K-NN's limit of 32), and ``disambiguate_directions=True`` orients the normals along a minimum spanning
        forest from each component's topmost point, so that their signs agree across the surface (outwards on a closed
        one), where the reference's per-point vote (Tombari et al.) only agrees locally.  ``False`` gives the canonical
        sign (the largest component positive).  The clouds must be on a CUDA device."""
        from ..ops import estimate_normals
        pts = self.points_packed()
        est = estimate_normals(pts, neighborhood_size, disambiguate_directions, self.cloud_to_packed_first_idx(),
                               self.num_points_per_cloud())
        normals = list(est.normals.split([p.shape[0] for p in self._points]))
        if assign_to_self:
            self._normals = normals
            for key in ("np", "npad"):
                self._cache.pop(key, None)
        return PointClouds3D(self._points, normals).normals_padded()

    def upsample(self, n, neighborhood_size: int = 16):
        """A denser copy by :func:`dss_b200.ops.upsample_points`: every cloud grown to ``n`` points (an int or one per
        cloud), its normals and features carried to the new points.  The input points keep their indices in every
        cloud.  The clouds must be on a CUDA device."""
        from ..ops import upsample_points
        up = upsample_points(self.points_packed(), n, neighborhood_size, self.normals_packed(), self.features_packed(),
                             self.cloud_to_packed_first_idx(), self.num_points_per_cloud())
        sizes = up.num_points.tolist()
        split = lambda t: None if t is None else list(t.split(sizes))
        return PointClouds3D(split(up.points), split(up.normals), split(up.features))

    def project_to_latent_surface(self, neighborhood_size: int = 31, max_proj_iters: int = 10, max_est_iter: int = 5):
        """A copy with every point moved onto the RIMLS surface of its cloud by :func:`dss_b200.ops.project_to_surface`,
        the normals and features carried unchanged.  The clouds need normals and must be on a CUDA device."""
        from ..ops import project_to_surface
        if self._normals is None:
            raise ValueError("projecting onto the surface needs normals (see PointClouds3D.estimate_normals)")
        out = project_to_surface(self.points_packed(), self.normals_packed(), neighborhood_size, max_proj_iters,
                                 max_est_iter, self.cloud_to_packed_first_idx(), self.num_points_per_cloud())
        sizes = self.num_points_per_cloud().tolist()
        return PointClouds3D(list(out.points.split(sizes)), self.normals_list(), self.features_list())


class PointCloudsFilters:
    """Named per-point boolean masks, padded (N, P_max) (DSS/core/cloud.py:285-360): ``activation`` selects
    the points that take part, ``visibility`` is written back by the rasterizer (rasterizer.py:643-653)."""

    def __init__(self, device="cpu", activation=None, visibility=None, inmask=None):
        self.device = torch.device(device)
        self.activation, self.visibility, self.inmask = activation, visibility, inmask

    def set_filter(self, **kwargs):
        for k, v in kwargs.items():
            if k not in ("activation", "visibility", "inmask"):
                raise ValueError("unknown filter %r" % k)
            setattr(self, k, v.to(self.device) if v is not None else None)

    def to(self, device):
        self.device = torch.device(device)
        for k in ("activation", "visibility", "inmask"):
            v = getattr(self, k)
            if v is not None:
                setattr(self, k, v.to(device))
        return self

    def filter_with(self, point_clouds: PointClouds3D, filter_names: Sequence[str]):
        """Keep the points for which every named filter is true (``filter_with``: cloud.py:318-360)."""
        mask = None
        for name in filter_names:
            f = getattr(self, name)
            if f is not None:
                mask = f if mask is None else (mask & f)
        if mask is None:
            return point_clouds
        if mask.shape[0] != len(point_clouds):
            mask = mask.expand(len(point_clouds), -1)
        sel = lambda lst: None if lst is None else [t[mask[i, : t.shape[0]]] for i, t in enumerate(lst)]
        return PointClouds3D(sel(point_clouds.points_list()), sel(point_clouds.normals_list()),
                             sel(point_clouds.features_list()))


def upsample(points, n_points, num_points=None, neighborhood_size=16, knn_result=None):
    """The reference's ``upsample`` (DSS/core/cloud.py:555-632) on :func:`dss_b200.ops.upsample_points`: padded
    ``points`` (N, P, 3) with ``num_points`` (N,) (default: all P) grown to ``n_points`` (an int or (N,)) ->
    ``(points_padded (N, max n, 3), num_points (N,))``, zero-padded.  Each cloud's input points come first, where the
    reference puts each round's points in front.  ``knn_result`` must be None: the neighbourhoods are recomputed on the
    device every round.  Raises ValueError where the reference would loop forever or pad neighbourhoods with zeros (see
    ``upsample_points``)."""
    from ..ops import upsample_points
    if knn_result is not None:
        raise ValueError("knn_result is not supported: the neighbourhoods are recomputed on the device every round")
    if points.dim() != 3 or points.shape[2] != 3:
        raise ValueError("points must be padded (N, P, 3)")
    N, P = points.shape[0], points.shape[1]
    dev = points.device
    if num_points is None:
        num_points = torch.full((N,), P, dtype=torch.int64, device=dev)
    first = torch.arange(N, dtype=torch.int64, device=dev) * P
    up = upsample_points(points.reshape(N * P, 3), n_points, neighborhood_size, first_idx=first,
                         num_points=num_points.to(device=dev, dtype=torch.int64))
    return PointClouds3D(list(up.points.split(up.num_points.tolist()))).points_padded(), up.num_points


def remove_outliers(pointclouds, neighborhood_size=16, tolerance=0.05):
    """The reference's ``remove_outliers`` (DSS/core/cloud.py:363-378) on :func:`dss_b200.ops.outlier_ratio`: the points
    whose ``neighborhood_size`` nearest neighbours (themselves included) are planar, i.e. whose covariance has its
    smallest eigenvalue below ``tolerance`` of the three's sum, with their normals and features, as a new
    :class:`PointClouds3D`.  Like the reference, raises ValueError for a cloud of at most ``neighborhood_size`` points;
    ``neighborhood_size`` is at most 32, the device K-NN's limit.  The clouds must be on a CUDA device."""
    from ..ops import outlier_ratio
    sizes = [int(p.shape[0]) for p in pointclouds.points_list()]
    if any(n <= neighborhood_size for n in sizes):
        raise ValueError("every cloud needs more than neighborhood_size = %d points, got %s" % (neighborhood_size, sizes))
    nl, fl = getattr(pointclouds, "normals_list", None), getattr(pointclouds, "features_list", None)
    normals, features = (nl() if callable(nl) else None), (fl() if callable(fl) else None)
    num = torch.tensor(sizes, dtype=torch.int64, device=pointclouds.points_list()[0].device)
    first = torch.cumsum(num, 0) - num
    keep = outlier_ratio(torch.cat(pointclouds.points_list(), 0), neighborhood_size, tolerance, first, num).keep
    masks = keep.split(sizes)
    sel = lambda lst: None if lst is None else [t[m] for t, m in zip(lst, masks)]
    return PointClouds3D(sel(pointclouds.points_list()), sel(normals), sel(features))


def _padded_layout(points, normals, num_points):
    if points.dim() != 3 or points.shape[2] != 3 or tuple(normals.shape) != tuple(points.shape):
        raise ValueError("points and normals must be padded (N, P, 3)")
    N, P = points.shape[0], points.shape[1]
    dev = points.device
    if num_points is None:
        num_points = torch.full((N,), P, dtype=torch.int64, device=dev)
    first = torch.arange(N, dtype=torch.int64, device=dev) * P
    return N, P, first, num_points.to(device=dev, dtype=torch.int64)


def denoise_normals(points, normals, num_points=None, sharpness_sigma=30, knn_result=None, neighborhood_size=16):
    """The reference's ``denoise_normals`` (DSS/core/cloud.py:515-553) on :func:`dss_b200.ops.denoise_normals`: padded
    ``points`` and ``normals`` (N, P, 3) with ``num_points`` (N,) (default: all P) -> the denoised unit normals (N, P, 3);
    rows past a cloud's size are returned as given.  Each cloud uses its own size and bounding box, where the
    reference uses the padded size and the whole batch's box; a row whose weights are all zero keeps its own normal,
    where the reference returns zero.  ``knn_result`` must be None: the neighbourhoods are computed on the device."""
    from ..ops import denoise_normals as _denoise
    if knn_result is not None:
        raise ValueError("knn_result is not supported: the neighbourhoods are computed on the device")
    N, P, first, num = _padded_layout(points, normals, num_points)
    out = _denoise(points.reshape(N * P, 3), normals.reshape(N * P, 3), neighborhood_size, float(sharpness_sigma),
                   first, num)
    return out.view_as(normals)


def project_to_latent_surface(points, normals, sharpness_angle=60, neighborhood_size=31, max_proj_iters=10,
                              max_est_iter=5):
    """The reference's ``project_to_latent_surface`` (DSS/core/cloud.py:442-513, RIMLS) on
    :func:`dss_b200.ops.project_to_surface`: padded ``points`` and ``normals`` (N, P, 3), every cloud of P points ->
    the projected points (N, P, 3).  The surface is fitted to the input samples throughout, where the reference reads
    the neighbours from the points it is moving; ``points`` is not modified, where the reference overwrites it.
    ``sharpness_angle`` is accepted and unused, as in the reference."""
    from ..ops import project_to_surface
    N, P, first, num = _padded_layout(points, normals, None)
    out = project_to_surface(points.reshape(N * P, 3), normals.reshape(N * P, 3), neighborhood_size, max_proj_iters,
                             max_est_iter, first, num)
    return out.points.view(N, P, 3)

# ---- duck typing for foreign cloud containers --------------------------------------------------------------------
# The reference hands pytorch3d ``Pointclouds`` (or its own ``PointClouds3D`` subclass) to the renderer; the filter's
# ``filter_with`` returns exactly that type (DSS/core/cloud.py).  Those objects have ``points_list`` / ``normals_list`` /
# ``equisized`` but neither ``shares_points`` nor ``equal_sized``, and their ``extend()`` CLONES the tensors, so storage
# aliasing never identifies a shared cloud there: fall back to shapes and, for clouds of equal shape, to the contents.
def clouds_equal_sized(point_clouds) -> bool:
    f = getattr(point_clouds, "equal_sized", None)
    if callable(f):
        return bool(f())
    eq = getattr(point_clouds, "equisized", None)
    if eq is not None:
        return bool(eq() if callable(eq) else eq)
    return len({int(p.shape[0]) for p in point_clouds.points_list()}) <= 1


def clouds_share_points(point_clouds) -> bool:
    f = getattr(point_clouds, "shares_points", None)
    if callable(f):
        return bool(f())
    pts = point_clouds.points_list()
    if len(pts) <= 1:
        return True
    if any(p.shape != pts[0].shape for p in pts):
        return False
    nl = getattr(point_clouds, "normals_list", None)
    nrm = nl() if callable(nl) else None

    def same(group):
        g0 = group[0]
        return all(t.data_ptr() == g0.data_ptr() or torch.equal(t, g0) for t in group[1:])

    return same(pts) and (nrm is None or same(nrm))
