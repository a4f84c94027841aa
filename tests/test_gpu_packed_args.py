"""Every operator that takes a packed cloud (``first_idx`` / ``num_points``) refuses malformed offsets before it
launches anything: the kernels read both as int64[N] and index rows with them, so int32 or (N,1) offsets, offsets of
different lengths, one offset without the other and offsets on another device must never reach them."""
from types import SimpleNamespace

import pytest
import torch

from dss_b200 import _lib
from dss_b200.frnn_grid import knn_points_packed
from dss_b200.ops import (SplatParams, denoise_normals, estimate_normals, local_frames, outlier_ratio,
                          preprocess_points, project_to_surface, render_points, upsample_points)
from dss_b200.training.losses import surface_regulariser
from tests.util import scene

pytestmark = pytest.mark.gpu

P0, N = 300, 2      # two clouds of P0 rows each, packed without gaps


@pytest.fixture(scope="module")
def cloud(cuda_device):
    pts, nrm, col, proj, view, _ = scene(P0, N, seed=3)
    dev = cuda_device
    p, n = pts.repeat(N, 1).to(dev), nrm.repeat(N, 1).to(dev)
    first = torch.arange(N, dtype=torch.int64, device=dev) * P0
    num = torch.full((N,), P0, dtype=torch.int64, device=dev)
    d, i = knn_points_packed(p, first, num, 12)
    return SimpleNamespace(p=p, n=n, col=col.repeat(N, 1).to(dev), proj=proj.to(dev), view=view.to(dev),
                           h=torch.full((N,), 3e-4, device=dev), prm=SplatParams(image_size=32, znear=0.1),
                           first=first, num=num, d=d, i=i)


OPERATORS = {
    "knn_points_packed": lambda c, f, n: knn_points_packed(c.p, f, n, 8),
    "knn_points_packed_queries": lambda c, f, n: knn_points_packed(c.p, c.first, c.num, 8, queries=c.p,
                                                                   query_first_idx=f, query_num=n),
    "local_frames": lambda c, f, n: local_frames(c.p, f, n),
    "estimate_normals": lambda c, f, n: estimate_normals(c.p, 16, True, f, n),
    "outlier_ratio": lambda c, f, n: outlier_ratio(c.p, 16, 0.05, f, n),
    "upsample_points": lambda c, f, n: upsample_points(c.p, P0 + 30, 16, first_idx=f, num_points=n),
    "denoise_normals": lambda c, f, n: denoise_normals(c.p, c.n, 16, first_idx=f, num_points=n),
    "project_to_surface": lambda c, f, n: project_to_surface(c.p, c.n, 16, 2, 2, first_idx=f, num_points=n),
    "render_points": lambda c, f, n: render_points(c.p, c.n, c.col, c.proj, c.view, c.h, c.prm, first_idx=f,
                                                   num_points=n, shared_cloud=False),
    "preprocess_points": lambda c, f, n: preprocess_points(c.p, c.n, c.proj, c.view, c.h, c.prm, first_idx=f,
                                                           num_points=n, shared_cloud=False),
    "surface_regulariser": lambda c, f, n: surface_regulariser("projection", c.p, c.n, f, n, c.d, c.i),
}

BAD_OFFSETS = {
    "int32": lambda f, n: (f.int(), n.int()),
    "column": lambda f, n: (f[:, None], n[:, None]),
    "lengths_differ": lambda f, n: (f, n[:1]),
    "first_idx_only": lambda f, n: (f, None),
    "num_points_only": lambda f, n: (None, n),
    "cpu": lambda f, n: (f.cpu(), n.cpu()),
}


@pytest.mark.parametrize("op", sorted(OPERATORS))
def test_valid_offsets_run(cloud, op):
    """the calls below fail only through their offsets"""
    OPERATORS[op](cloud, cloud.first, cloud.num)
    torch.cuda.synchronize()


@pytest.mark.parametrize("bad", sorted(BAD_OFFSETS))
@pytest.mark.parametrize("op", sorted(OPERATORS))
def test_malformed_offsets_raise_before_any_launch(cloud, op, bad):
    f, n = BAD_OFFSETS[bad](cloud.first, cloud.num)
    torch.cuda.synchronize()
    before = _lib.launch_count(cloud.p.device)
    with pytest.raises(RuntimeError):
        OPERATORS[op](cloud, f, n)
    assert _lib.launch_count(cloud.p.device) == before
