"""GPU: with ``deterministic=True`` (what the training step passes) the shaded render's backward gives the same bits on
every run.  Its colour scatter into d L / d shaded then sums in 64-bit fixed point (csrc/backward.cu,
colour_backward_fixed), so the albedo, normal and position gradients of a shaded cloud do not depend on the order of the
scatter's atomics; the training loop's exact resume rests on it.  The accuracy of those gradients against float64 is checked in test_gpu_light_grad.py and
test_gpu_packed_shading.py."""
import pytest
import torch

from dss_b200.ops import SplatParams, make_shading, render_points
from tests.test_shading import _lights
from tests.util import scene

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("kind", ["sun", "point"])
@pytest.mark.parametrize("h", [3e-4, 3e-3])
def test_shaded_backward_is_bit_reproducible(cuda_device, kind, h):
    d = cuda_device
    P0, N, S = 3000, 4, 128
    pts, nrm, col, proj, view, _ = scene(P0, N, seed=5)
    prm = SplatParams(image_size=S, points_per_pixel=5, znear=0.1, clip_pts_grad=0.05)
    sh = make_shading(_lights(kind, d), view.to(d), shininess=20.0)
    g = torch.randn(N, S, S, 4, generator=torch.Generator().manual_seed(1)).to(d)
    runs = []
    # the first call is not compared: the occupancy backward sizes its staged window from the previous call's search
    # radii (DESIGN.md section 3), so each compared call follows a call of the same scene
    for _ in range(4):
        p, n, a = (t.to(d).clone().requires_grad_(True) for t in (pts, nrm, col))
        out = render_points(p, n, a, proj.to(d), view.to(d), torch.full((N,), h, device=d), prm, shading=sh,
                            deterministic=True)
        out.image.backward(g)
        runs.append((out.image.detach(), p.grad, n.grad, a.grad))
    runs = runs[1:]
    diff = {name: int(sum((x != y).sum() for x, y in zip([r0] * 2, [r[i] for r in runs[1:]])))
            for i, (name, r0) in enumerate(zip(("image", "points", "normals", "albedo"), runs[0]))}
    print(kind, h, "entries differing from the first compared call:", diff)
    assert all(v == 0 for v in diff.values()), diff
    # large splats put many pixels' terms into one record: the gradients are there, finite and non-zero
    for t in runs[0][1:]:
        assert torch.isfinite(t).all() and t.abs().max() > 0


def test_shaded_backward_non_finite_term(cuda_device):
    """a NaN in the image gradient reaches exactly the records it touches, as a float sum would"""
    d = cuda_device
    P0, N, S = 2000, 2, 64
    pts, nrm, col, proj, view, _ = scene(P0, N, seed=6)
    prm = SplatParams(image_size=S, points_per_pixel=5, znear=0.1)
    sh = make_shading(_lights("sun", d), view.to(d))
    g = torch.randn(N, S, S, 4, generator=torch.Generator().manual_seed(2)).to(d)
    p, n, a = (t.to(d).clone().requires_grad_(True) for t in (pts, nrm, col))
    out = render_points(p, n, a, proj.to(d), view.to(d), torch.full((N,), 3e-4, device=d), prm, shading=sh,
                        return_fragments=True, deterministic=True)
    hit = (out.idx[0] >= 0).any(-1).nonzero()[0]
    g[0, hit[0], hit[1], 0] = float("nan")
    out.image.backward(g)
    rows = out.idx[0, hit[0], hit[1]]
    rows = rows[rows >= 0].long()               # view 0's records are the world points 0..P0-1
    assert torch.isnan(a.grad[rows, 0]).all()
    others = torch.ones(P0, dtype=torch.bool, device=d)
    others[rows] = False
    assert torch.isfinite(a.grad[others]).all()
