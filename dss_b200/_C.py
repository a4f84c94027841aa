"""Drop-in for the reference's native module ``DSS._C`` (pybind surface: DSS/csrc/ext.cpp:5-18).

Same function names, argument order and tensor shapes/dtypes; every function calls libdss_b200.so
through its C ABI (include/dss_b200.h) on the current CUDA stream.  CUDA tensors only: the reference
dispatches CPU tensors to its *Cpu twins (rasterize_points.h:77-124); this build has no CPU path and
raises RuntimeError instead.
"""
import ctypes as C

import torch

from . import _lib

__all__ = ["splat_points", "_splat_points_naive", "_rasterize_coarse", "_rasterize_coarse_csr",
           "_rasterize_fine", "_splat_points_occ_backward", "_splat_points_occ_fast_cuda_backward", "_backward_zbuf"]


def _check_packed(points, ellipse_params, cutoff_thres, radii, first_idx, num_points):
    """rasterize_points.h:483-488 -> (points, first_idx, num_points) of _lib.packed_cloud"""
    points, first_idx, num_points = _lib.packed_cloud(points, first_idx, num_points)
    P = points.shape[0]
    if radii is not None and tuple(radii.shape) != (P, 2):
        raise RuntimeError("radii must have shape (%d, 2), got %s" % (P, tuple(radii.shape)))
    if ellipse_params is not None and tuple(ellipse_params.shape) != (P, 3):
        raise RuntimeError("ellipse_params must have shape (%d, 3), got %s" % (P, tuple(ellipse_params.shape)))
    if cutoff_thres is not None and tuple(cutoff_thres.shape) != (P,):
        raise RuntimeError("cutoff_thres must have shape (%d,), got %s" % (P, tuple(cutoff_thres.shape)))
    return points, first_idx, num_points


def splat_points(points, ellipse_params, cutoff_thres, radii, cloud_to_packed_first_idx,
                 num_points_per_cloud, depth_merging_thres, image_size, points_per_pixel,
                 bin_size=0, max_points_per_bin=0):
    """``_C.splat_points`` (ext.cpp:8; rasterize_points.h:461-525).

    Returns ``(idx int32 (N,S,S,K), zbuf f32, qvalue f32, occupancy f32 (N,S,S))``, -1 padded.
    ``bin_size`` / ``max_points_per_bin`` are accepted and ignored: tiling is internal and tile lists
    are exact-size, so the reference's "more than max_points_per_bin points in a bin" overflow and its
    ``num_bins >= 22`` error (rasterize_points.cu:462-468) cannot occur."""
    dev = _lib.require_cuda(points, ellipse_params, cutoff_thres, radii, cloud_to_packed_first_idx,
                            num_points_per_cloud)
    points, fi, npts = _check_packed(points, ellipse_params, cutoff_thres, radii, cloud_to_packed_first_idx,
                                     num_points_per_cloud)
    K, S = int(points_per_pixel), int(image_size)
    if K > _lib.MAX_POINTS_PER_PIXEL:
        raise RuntimeError("Must have points_per_pixel <= %d" % _lib.MAX_POINTS_PER_PIXEL)
    N, P = npts.shape[0], points.shape[0]
    ellipse_params = _lib.as_f32(ellipse_params.detach(), "ellipse_params")
    cutoff_thres = _lib.as_f32(cutoff_thres.detach(), "cutoff_thres")
    radii = _lib.as_f32(radii.detach(), "radii")
    idx = torch.empty((N, S, S, K), dtype=torch.int32, device=dev)
    zbuf = torch.empty((N, S, S, K), dtype=torch.float32, device=dev)
    qvalue = torch.empty((N, S, S, K), dtype=torch.float32, device=dev)
    occ = torch.empty((N, S, S), dtype=torch.float32, device=dev)
    _lib.call("dss_splat_points", dev, points, ellipse_params, cutoff_thres, radii, fi, npts, N, P,
              float(depth_merging_thres), S, K, int(bin_size or 0), idx, zbuf, qvalue, occ)
    return idx, zbuf, qvalue, occ


def _splat_points_naive(points, ellipse_params, cutoff_thres, radii, cloud_to_packed_first_idx,
                        num_points_per_cloud, depth_merging_thres, image_size, points_per_pixel):
    """``_C._splat_points_naive`` (ext.cpp:9): same outputs as ``splat_points`` (the naive and the
    coarse-to-fine reference paths compute the same function; there is one kernel here)."""
    return splat_points(points, ellipse_params, cutoff_thres, radii, cloud_to_packed_first_idx,
                        num_points_per_cloud, depth_merging_thres, image_size, points_per_pixel, 0, 0)


def _rasterize_coarse_csr(points, radii, cloud_to_packed_first_idx, num_points_per_cloud, image_size, bin_size):
    """Bin membership as CSR: ``(bin_offsets int32 (N*B*B+1,), bin_ids int32 (total,))``."""
    dev = _lib.require_cuda(points, radii, cloud_to_packed_first_idx, num_points_per_cloud)
    points, fi, npts = _check_packed(points, None, None, radii, cloud_to_packed_first_idx, num_points_per_cloud)
    S, bs = int(image_size), int(bin_size)
    if bs <= 0:
        raise RuntimeError("bin_size must be positive")
    N, P = npts.shape[0], points.shape[0]
    B = 1 + (S - 1) // bs
    radii = _lib.as_f32(radii.detach(), "radii")
    off = torch.empty(N * B * B + 1, dtype=torch.int32, device=dev)
    cap = max(2 * P, 1024)
    for first in (True, False):
        ids = torch.empty(cap, dtype=torch.int32, device=dev)
        need = C.c_int64(0)
        if _lib.call("dss_rasterize_coarse", dev, points, radii, fi, npts, N, P, S, bs, off, ids, cap, C.byref(need),
                     capacity=first) != _lib.DSS_E_CAPACITY:
            break
        cap = int(need.value)
    return off, ids[: int(need.value)]


def _rasterize_coarse(points, radii, cloud_to_packed_first_idx, num_points_per_cloud, image_size, bin_size,
                      max_points_per_bin):
    """``_C._rasterize_coarse`` (ext.cpp:11): dense ``(N,B,B,M)`` int32, -1 padded, for callers that want
    the reference layout.  Ids inside a bin are ascending.  Prefer ``_rasterize_coarse_csr``: the dense
    tensor is what makes the reference need 8 GB per call at 1M points."""
    off, ids = _rasterize_coarse_csr(points, radii, cloud_to_packed_first_idx, num_points_per_cloud,
                                     image_size, bin_size)
    N = num_points_per_cloud.shape[0]
    B = 1 + (int(image_size) - 1) // int(bin_size)
    M = int(max_points_per_bin)
    counts = (off[1:] - off[:-1]).long()
    if counts.numel() and int(counts.max()) > M:
        raise RuntimeError("a bin holds %d points > max_points_per_bin=%d" % (int(counts.max()), M))
    dense = torch.full((N * B * B, M), -1, dtype=torch.int32, device=points.device)
    if ids.numel():
        bin_of = torch.repeat_interleave(torch.arange(N * B * B, device=points.device), counts)
        # ascending ids per bin: sort by (bin, id)
        order = torch.argsort(bin_of * (int(points.shape[0]) + 1) + ids.long())
        ids_s, bin_s = ids[order], bin_of[order]
        rank = torch.arange(ids.numel(), device=points.device) - off[:-1].long()[bin_s]
        dense[bin_s, rank] = ids_s
    return dense.view(N, B, B, M)


def _rasterize_fine(points, ellipse_params, cutoff_thres, radii, bin_points, depth_merging_thres, image_size,
                    bin_size, points_per_pixel):
    """``_C._rasterize_fine`` (ext.cpp:12).  ``bin_points`` is taken to be the output of
    ``_rasterize_coarse`` for the same inputs (it always is in the reference: rasterize_points.h:503-523),
    in which case the result equals ``splat_points``; only the number of views is read from it."""
    N = bin_points.shape[0]
    P = points.shape[0]
    if N != 1:
        raise RuntimeError("_rasterize_fine: pass cloud offsets through splat_points for batches (N=%d)" % N)
    fi = torch.zeros(1, dtype=torch.int64, device=points.device)
    npts = torch.full((1,), P, dtype=torch.int64, device=points.device)
    return splat_points(points, ellipse_params, cutoff_thres, radii, fi, npts, depth_merging_thres, image_size,
                        points_per_pixel, bin_size, 0)


def _splat_points_occ_backward(points, radii, grad_occ, cloud_to_packed_first_idx, num_points_per_cloud, radii_s,
                               depth_merging_thres=0.05):
    """``_C._splat_points_occ_backward`` (ext.cpp:10,16; rasterize_points.cu:673-821), the reference's SLOW occupancy
    backward (rectangular window ``radii * radii_s``, every renderable point): -> ``(P,2)``.  ``depth_merging_thres`` is
    accepted and unused, as in the reference kernel.  The training path uses the fast variant (rasterizer.py:816)."""
    dev = _lib.require_cuda(points, radii, grad_occ, cloud_to_packed_first_idx, num_points_per_cloud)
    points, fi, npts = _check_packed(points, None, None, radii, cloud_to_packed_first_idx, num_points_per_cloud)
    if grad_occ.dim() != 3 or grad_occ.shape[1] != grad_occ.shape[2]:
        raise RuntimeError("grad_occ must have shape (N, S, S)")
    N, S, P = grad_occ.shape[0], grad_occ.shape[1], points.shape[0]
    radii = _lib.as_f32(radii.detach(), "radii")
    grad_occ = _lib.as_f32(grad_occ.detach(), "grad_occ")
    out = torch.empty((P, 2), dtype=torch.float32, device=dev)
    _lib.call("dss_occ_backward_slow", dev, points, radii, grad_occ, 1, 0, fi, npts, N, P, S, float(radii_s), out)
    return out


def _splat_points_occ_fast_cuda_backward(points_sorted, radii_sorted, rs, grad_occ, num_points_per_cloud,
                                         cloud_to_packed_first_idx, points_grid_off=None, grid_params=None):
    """``_C._splat_points_occ_fast_cuda_backward`` (ext.cpp:13-15; rasterize_points_backward.cu:227-322).

    Every given point is treated as visible (the reference passes the visible, grid-sorted subset).
    ``points_grid_off`` / ``grid_params`` are accepted and ignored: the grid only accelerates the
    reference's pixel->point scatter; this gathers per point and needs none.  Returns ``(P,2)``."""
    dev = _lib.require_cuda(points_sorted, radii_sorted, rs, grad_occ, num_points_per_cloud,
                            cloud_to_packed_first_idx)
    _check_packed(points_sorted, None, None, radii_sorted, cloud_to_packed_first_idx, num_points_per_cloud)
    if grad_occ.dim() != 3 or grad_occ.shape[1] != grad_occ.shape[2]:
        raise RuntimeError("grad_occ must have shape (N, S, S)")
    if rs.shape != num_points_per_cloud.shape:
        raise RuntimeError("rs must have shape (N,)")
    P = points_sorted.shape[0]
    visible = torch.ones(P, dtype=torch.uint8, device=dev)
    return occ_backward(points_sorted, radii_sorted, visible, rs, grad_occ, cloud_to_packed_first_idx,
                        num_points_per_cloud)


def occ_backward(points, radii, visible, rs, grad_occ, cloud_to_packed_first_idx, num_points_per_cloud):
    """Occupancy gather on unsorted packed points with an explicit visibility mask -> ``(P,2)``."""
    dev = _lib.require_cuda(points, radii, visible, rs, grad_occ)
    N, S = grad_occ.shape[0], grad_occ.shape[1]
    points, fi, npts = _lib.packed_cloud(points, cloud_to_packed_first_idx, num_points_per_cloud, N)
    P = points.shape[0]
    radii = _lib.as_f32(radii.detach(), "radii")
    grad_occ = _lib.as_f32(grad_occ.detach(), "grad_occ")
    rs = _lib.as_f32(rs.detach(), "rs")
    visible = visible.to(torch.uint8).contiguous()
    out = torch.empty((P, 2), dtype=torch.float32, device=dev)
    _lib.call("dss_occ_backward", dev, points, radii, visible, rs, grad_occ, 1, 0, fi, npts, N, P, S, out)
    return out


def visibility_from_idx(idx, P):
    """(P,) uint8: points appearing in ``idx`` at pixels whose first slot is occupied (rasterizer.py:854-860)."""
    dev = _lib.require_cuda(idx)
    idx = idx.contiguous()
    if idx.dtype != torch.int32:
        raise RuntimeError("idx must be int32")
    K = idx.shape[-1]
    vis = torch.empty(P, dtype=torch.uint8, device=dev)
    _lib.call("dss_visibility_from_idx", dev, idx, idx.numel() // K, K, P, vis)
    return vis


def search_radius(radii, visible, cloud_to_packed_first_idx, num_points_per_cloud, radii_s):
    """(N,) f32: ``radii_s * lower_median(radii of the view's visible points)`` (rasterizer.py:888)."""
    dev = _lib.require_cuda(radii, visible, cloud_to_packed_first_idx, num_points_per_cloud)
    fi, npts = _lib.cloud_offsets(cloud_to_packed_first_idx, num_points_per_cloud)
    N = npts.shape[0]
    rs = torch.empty(N, dtype=torch.float32, device=dev)
    radii = _lib.as_f32(radii.detach(), "radii")
    _lib.call("dss_search_radius", dev, radii, visible.contiguous(), fi, npts, N, radii.shape[0], float(radii_s), rs)
    return rs


def _backward_zbuf(idx, grad_zbuf, point_z_grad):
    """``_C._backward_zbuf`` (ext.cpp:17): in-place ``point_z_grad[idx_k] += grad_zbuf_k``; returns None."""
    dev = _lib.require_cuda(idx, grad_zbuf, point_z_grad)
    if idx.shape != grad_zbuf.shape or idx.dim() != 4:
        raise RuntimeError("idx and grad_zbuf must both have shape (N, H, W, K)")
    if not point_z_grad.is_contiguous() or point_z_grad.dtype != torch.float32:
        raise RuntimeError("point_z_grad must be a contiguous float32 tensor")
    K = idx.shape[-1]
    _lib.call("dss_zbuf_backward", dev, idx.contiguous(), _lib.as_f32(grad_zbuf, "grad_zbuf"), idx.numel() // K, K,
              point_z_grad)
    return None
