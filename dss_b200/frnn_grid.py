"""Drop-ins for the FRNN entry points DSS uses.

* ``frnn_grid_points`` / ``knn_points_packed``: K nearest neighbours within a radius on a 3-D grid
  (external/FRNN/frnn/frnn.py:176-301), which sizes the splats (DSS/core/rasterizer.py:313-326, 369-388) -- SURVEY.md
  section 8(f) row 1, backed by ``dss_knn_points`` (dss_b200/csrc/knn.cu).
* ``insert_points_cuda`` / ``counting_sort_cuda`` (external/FRNN/frnn/csrc/grid/grid.h:43-50, counting_sort.h:4-11),
  D = 2: the radius-binning primitives the reference's backward used.  This package's backward does not need them (it
  gathers per point, see _C.occ_backward); they are kept so code written against them keeps working."""
import torch

from . import _lib

__all__ = ["insert_points_cuda", "counting_sort_cuda", "frnn_grid_points", "knn_points_packed", "knn_points"]


def insert_points_cuda(points, lengths, params, grid_cnt, grid_cell, grid_idx, G):
    dev = _lib.require_cuda(points, lengths, params, grid_cnt, grid_cell, grid_idx)
    if points.dim() != 3 or points.shape[2] != 2:
        raise RuntimeError("for now only 2D is supported by this build (got D=%s)" % (points.shape[-1],))
    if not (grid_cnt.dtype == grid_cell.dtype == grid_idx.dtype == torch.int32):
        raise RuntimeError("grid_cnt, grid_cell, grid_idx must be int32")
    for t in (grid_cnt, grid_cell, grid_idx):
        if not t.is_contiguous():
            raise RuntimeError("output tensors must be contiguous")
    N, P = points.shape[0], points.shape[1]
    _lib.call("dss_grid_insert_points_2d", dev, _lib.as_f32(points, "points"), lengths.contiguous(),
              _lib.as_f32(params, "params"), grid_cnt, grid_cell, grid_idx, N, P, int(G))


def counting_sort_cuda(points, lengths, grid_cell, grid_idx, grid_off, sorted_points, sorted_points_idxs):
    dev = _lib.require_cuda(points, lengths, grid_cell, grid_idx, grid_off, sorted_points, sorted_points_idxs)
    if points.dim() != 3 or points.shape[2] != 2:
        raise RuntimeError("for now only 2D is supported by this build")
    for t in (sorted_points, sorted_points_idxs):
        if not t.is_contiguous():
            raise RuntimeError("output tensors must be contiguous")
    N, P, G = points.shape[0], points.shape[1], grid_off.shape[1]
    _lib.call("dss_grid_counting_sort_2d", dev, _lib.as_f32(points, "points"), lengths.contiguous(),
              grid_cell.contiguous(), grid_idx.contiguous(), grid_off.contiguous(), sorted_points, sorted_points_idxs,
              N, P, G)


def knn_points_packed(points, first_idx, num_points, K, r=-1.0, queries=None, query_first_idx=None, query_num=None,
                      return_idx=True):
    """Packed form: ``points`` (P,3) f32, cloud n owns rows [first_idx[n], first_idx[n] + num_points[n]) (both None: one
    cloud).  The ranges may leave gaps between them (padded storage passed as packed: first_idx = n * Pmax, num_points =
    lengths) but must not overlap; rows outside every query range are left unwritten.  ``queries`` (Pq,3) f32 take the
    points' offsets unless both ``query_first_idx`` and ``query_num`` are given.  Returns ``(sq_dists (Pq,K) f32
    ascending, idxs (Pq,K) int32 local to the cloud or None)``, -1 padded.  Rows of points or queries with a NaN or
    infinite coordinate are all -1, and such points are nobody's neighbour."""
    dev = _lib.require_cuda(points, first_idx, num_points, queries, query_first_idx, query_num)
    pts, first_idx, num_points = _lib.packed_cloud(points, first_idx, num_points)
    if not (1 <= int(K) <= 32):
        raise RuntimeError("K must be in [1, 32]")
    P, N = pts.shape[0], num_points.shape[0]
    query_args = (None, None, None)
    if queries is not None:
        if query_first_idx is None and query_num is None:
            query_first_idx, query_num = first_idx, num_points
        query_args = _lib.packed_cloud(queries, query_first_idx, query_num, N)
    Pq = P if queries is None else query_args[0].shape[0]
    d = torch.empty((Pq, K), dtype=torch.float32, device=dev)
    i = torch.empty((Pq, K), dtype=torch.int32, device=dev) if return_idx else None
    _lib.call("dss_knn_points", dev, *query_args, pts, first_idx, num_points, N, Pq, P, int(K), float(r), d, i)
    return d, i


def frnn_grid_points(points1, points2, lengths1=None, lengths2=None, K=-1, r=-1, grid=None, return_nn=False,
                     return_sorted=True, radius_cell_ratio=2.0):
    """``frnn.frnn_grid_points`` (external/FRNN/frnn/frnn.py:176-301) for D = 3: padded (N,P1,3) queries against padded
    (N,P2,3) points -> ``(dists (N,P1,K), idxs (N,P1,K) int64, nn or None, grid=None)``; -1 where there is no
    neighbour (fewer than K points inside the radius, or padding rows).  ``grid`` / ``radius_cell_ratio`` are accepted
    for signature parity and ignored: the grid is rebuilt in a few tens of microseconds and sized by the density."""
    if points1.dim() != 3 or points1.shape[2] != 3 or points2.dim() != 3 or points2.shape[2] != 3:
        raise RuntimeError("for now only (N, P, 3) inputs are supported by this build")
    if K < 1:
        raise RuntimeError("K must be positive")
    dev = _lib.require_cuda(points1, points2, lengths1, lengths2)
    N, P1, P2 = points1.shape[0], points1.shape[1], points2.shape[1]
    if lengths1 is None:
        lengths1 = torch.full((N,), P1, dtype=torch.int64, device=dev)
    if lengths2 is None:
        lengths2 = torch.full((N,), P2, dtype=torch.int64, device=dev)
    same = points1 is points2 and lengths1 is lengths2
    m2 = torch.arange(P2, device=dev)[None, :] < lengths2[:, None]
    first2 = torch.cumsum(lengths2, 0) - lengths2
    packed2 = points2[m2].contiguous()
    if same:
        d, i = knn_points_packed(packed2, first2, lengths2.contiguous(), K, float(r))
        m1 = m2
    else:
        m1 = torch.arange(P1, device=dev)[None, :] < lengths1[:, None]
        first1 = torch.cumsum(lengths1, 0) - lengths1
        d, i = knn_points_packed(packed2, first2, lengths2.contiguous(), K, float(r), points1[m1].contiguous(), first1,
                                 lengths1.contiguous())
    dists = torch.full((N, P1, K), -1.0, dtype=torch.float32, device=dev)
    idxs = torch.full((N, P1, K), -1, dtype=torch.int64, device=dev)
    dists[m1] = d
    idxs[m1] = i.long()
    nn = None
    if return_nn:
        nn = torch.gather(points2[:, None].expand(-1, P1, -1, -1), 2, idxs.clamp(min=0)[..., None].expand(-1, -1, -1, 3))
        nn = torch.where((idxs >= 0)[..., None], nn, torch.zeros_like(nn))
    return dists, idxs, nn, None


def knn_points(p1, p2, lengths1=None, lengths2=None, K=1, version=-1, return_nn=False, return_sorted=True):
    """``pytorch3d.ops.knn_points`` [ext, pytorch3d 0.4.0] as DSS calls it (DSS/core/rasterizer.py:308-312 when
    ``frnn_radius <= 0``; DSS/training/losses.py:157-180 with K = 12): the K nearest neighbours without a radius.
    Returns ``(dists (N,P1,K), idx (N,P1,K) int64, knn (N,P1,K,3) or None)``; where a cloud has fewer than K points the
    entries are zero-padded, as pytorch3d documents (not -1 as frnn does)."""
    dists, idxs, nn, _ = frnn_grid_points(p1, p2, lengths1, lengths2, K=K, r=-1.0, return_nn=return_nn)
    missing = idxs < 0
    dists = torch.where(missing, torch.zeros_like(dists), dists)
    idxs = torch.where(missing, torch.zeros_like(idxs), idxs)
    return dists, idxs, nn
