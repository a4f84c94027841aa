"""Drop-in for the reference's ``prefix_sum`` module (external/prefix_sum/prefix_sum.h:6-21)."""
import torch

from . import _lib

__all__ = ["prefix_sum_cuda"]


def prefix_sum_cuda(grid_cnt, num_grids, grid_off):
    """Exclusive int32 scan of the first ``num_grids`` elements of ``grid_cnt`` into ``grid_off``
    (prefix_sum.cu:74-87).  Single-pass decoupled look-back on the current stream; unlike the reference
    (cudaMalloc/cudaFree per level, legacy default stream: prefix_sum.cu:176-205) it neither allocates
    nor synchronises.  Returns None."""
    dev = _lib.require_cuda(grid_cnt, grid_off)
    n = int(num_grids)
    if grid_cnt.dtype != torch.int32 or grid_off.dtype != torch.int32:
        raise RuntimeError("prefix_sum_cuda expects int32 tensors")
    if not grid_off.is_contiguous():
        raise RuntimeError("grid_off must be contiguous (it is written in place)")
    if n < 0 or n > grid_cnt.numel() or n > grid_off.numel():
        raise RuntimeError("num_grids=%d out of range" % n)
    src = grid_cnt.contiguous()
    _lib.call("dss_exclusive_scan_i32", dev, src, grid_off, n)
    return None
