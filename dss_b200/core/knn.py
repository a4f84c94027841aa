"""K nearest neighbours within a radius, for the splat-size rule h_k (rasterizer.py:313-326, 369-388).

SURVEY.md section 8(f) row 1: the reference calls ``frnn.frnn_grid_points(K=7, r=0.2)`` (a 3-D grid search) in every
forward.  This module routes to ``dss_knn_points`` (dss_b200/csrc/knn.cu, a density-sized 3-D grid with ring-by-ring
search) -- CUDA only, like everything else in the package."""
import torch

from ..frnn_grid import knn_points_packed

__all__ = ["knn_sq_dists"]


def knn_sq_dists(points: torch.Tensor, K: int = 7, radius: float = 0.2) -> torch.Tensor:
    """(P, K) ascending squared distances from every point to its K nearest points of the same cloud (self
    included, distance 0).  Neighbours farther than ``radius`` (when radius > 0) are reported as -1 like frnn
    does for missing neighbours (frnn.py:176-301); the callers take ``max`` over the row, so -1 never wins
    as long as one neighbour exists."""
    return knn_points_packed(points, None, None, K, radius if radius is not None else -1.0, return_idx=False)[0]
