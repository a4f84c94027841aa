"""GPU parity tests of the fused renderer path (dss_render_forward / dss_render_backward) against the
CPU oracle on seeded synthetic scenes (SURVEY.md section 8d), plus size-independent properties."""
import numpy as np
import pytest
import torch

import oracle
from dss_b200.ops import SplatParams, preprocess_points, render_points
from tests.util import assert_blend_matches, assert_fragments_exact, packed_offsets, render_backward_f64_of, scene

pytestmark = pytest.mark.gpu

IMAGE_MSE_TOL = 1e-5        # north_star: image MSE vs reference < 1e-5


def _np(t):
    return t.detach().cpu().numpy()


def _oracle_forward(pre, colours, first, num, prm):
    """oracle raster + blend on the per-point info produced by the CUDA preprocess (so that raster parity
    is exact and preprocess parity is a separate tolerance test)."""
    S, K = prm.image_size, prm.points_per_pixel
    idx, zbuf, q, occ = oracle.splat_points_binned(pre["ndc"], pre["ellipse_params"], pre["cutoff_threshold"],
                                                   pre["radii"], first, num, prm.depth_merging_threshold, S, K,
                                                   16, fma_mode=1)
    img = oracle.blend_forward(idx, q, occ, pre["scaler"], colours)
    return idx, zbuf, q, occ, img


@pytest.mark.parametrize("P0,N,S", [(5000, 1, 256), (20000, 2, 128), (3000, 3, 64)])
def test_preprocess_matches_f64_oracle(cuda_device, P0, N, S):
    pts, nrm, col, proj, view, cams = scene(P0, N, seed=S)
    prm = SplatParams(image_size=S, znear=0.1)
    h = torch.full((N,), 2e-4)
    pre = preprocess_points(pts.to(cuda_device), nrm.to(cuda_device), proj.to(cuda_device), view.to(cuda_device),
                            h.to(cuda_device), prm)
    want = oracle.preprocess_f64(_np(proj), _np(view), _np(pts), _np(nrm), _np(h), 1.0, 1.0, S)
    np.testing.assert_allclose(_np(pre["ndc"]), want["ndc"], rtol=2e-5, atol=2e-6)
    np.testing.assert_allclose(_np(pre["radii"]), want["radii"], rtol=2e-4, atol=1e-7)
    # conic entries scale like 1/pixel^2: compare relative to the per-splat magnitude
    mag = np.abs(want["ellipse"]).max(axis=1, keepdims=True)
    assert (np.abs(_np(pre["ellipse_params"]) - want["ellipse"]) <= 5e-4 * mag).all()
    np.testing.assert_allclose(_np(pre["scaler"]), want["scaler"], rtol=2e-3, atol=2e-3 * want["scaler"].max())


@pytest.mark.parametrize("P0,N,S,K", [(5000, 1, 256, 5), (30000, 2, 128, 5), (8000, 2, 96, 8)])
def test_render_forward_matches_oracle(cuda_device, P0, N, S, K):
    pts, nrm, col, proj, view, cams = scene(P0, N, seed=K + S)
    prm = SplatParams(image_size=S, points_per_pixel=K, znear=0.1)
    h = torch.full((N,), 3e-4)
    colours = col.repeat(N, 1) * torch.linspace(0.5, 1.0, N).repeat_interleave(P0)[:, None]
    d = cuda_device
    out = render_points(pts.to(d), nrm.to(d), colours.to(d), proj.to(d), view.to(d), h.to(d), prm,
                        return_fragments=True)
    pre = preprocess_points(pts.to(d), nrm.to(d), proj.to(d), view.to(d), h.to(d), prm)
    pre_np = {k: _np(v) for k, v in pre.items()}
    first, num = packed_offsets(N, P0)
    widx, wz, wq, wocc, wimg = _oracle_forward(pre_np, _np(colours), _np(first), _np(num), prm)
    idx = _np(out.idx)
    # bit-exact fragments except rim pixels (a fragment within a few ulp of the cutoff), image and weights within the
    # fp32 error bound of the blend (tests/util.py: assert_blend_matches)
    rim, same = assert_fragments_exact((out.idx, out.zbuf, out.qvalue, out.image[..., 3]), (widx, wz, wq, wocc),
                                       pre_np["cutoff_threshold"])
    print("rim exemptions: %d" % rim)
    img = _np(out.image)
    mse = float(((img - wimg) ** 2).mean())
    assert mse < IMAGE_MSE_TOL, mse
    assert_blend_matches(out.image, out.weights, widx, wq, wocc, pre_np["scaler"], _np(colours), same)
    # visibility written by the forward pass == reference definition on its own idx
    assert np.array_equal(_np(out.visible), oracle.visibility(idx, N * P0))
    # records carry the same numbers as the standalone preprocess
    rec = _np(out.records)
    assert np.array_equal(rec[:, :3], pre_np["ndc"]) and np.array_equal(rec[:, 3], pre_np["radii"][:, 0])


def test_render_depth_filter_and_empty_views(cuda_device):
    """points outside [znear, zfar] are never rendered (rasterizer.py:183-217); a view that sees nothing
    yields an empty image."""
    P0, N, S = 4000, 2, 64
    pts, nrm, col, proj, view, cams = scene(P0, N, seed=1)
    d = cuda_device
    prm = SplatParams(image_size=S, znear=0.1, zfar=100.0)
    h = torch.full((N,), 3e-4)
    colours = col.repeat(N, 1)
    full = render_points(pts.to(d), nrm.to(d), colours.to(d), proj.to(d), view.to(d), h.to(d), prm)
    assert full.image[..., 3].sum() > 0
    far = render_points(pts.to(d), nrm.to(d), colours.to(d), proj.to(d), view.to(d), h.to(d),
                        prm._replace(znear=50.0))
    assert far.image.abs().sum() == 0 and (far.idx == -1).all() and far.visible.sum() == 0
    assert (far.records[:, 2] == -1).all()


@pytest.mark.parametrize("P0,N,S", [(6000, 2, 128), (2000, 1, 64)])
def test_render_backward_matches_oracle(cuda_device, P0, N, S):
    K = 5
    pts, nrm, col, proj, view, cams = scene(P0, N, seed=S)
    prm = SplatParams(image_size=S, points_per_pixel=K, znear=0.1, radii_backward_scaler=5.0, clip_pts_grad=0.05)
    h = torch.full((N,), 3e-4)
    colours = col.repeat(N, 1)
    d = cuda_device
    p = pts.to(d).requires_grad_(True)
    c = colours.to(d).requires_grad_(True)
    out = render_points(p, nrm.to(d), c, proj.to(d), view.to(d), h.to(d), prm, return_fragments=True)
    g = torch.Generator().manual_seed(9)
    grad_image = (torch.randn(N, S, S, 4, generator=g) * 1e-3)
    out.image.backward(grad_image.to(d))
    # ---- float64 reference on the CUDA forward's own fragments ----
    ref = render_backward_f64_of(out, pts, proj, view, prm, grad_image)
    assert np.array_equal(_np(out.visible), ref["vis"])
    np.testing.assert_allclose(_np(c.grad), ref["colours"], rtol=2e-4, atol=1e-7)
    want = ref["world"]
    got = _np(p.grad)
    scale = np.abs(want).max()
    assert scale > 0
    assert np.abs(got - want).max() <= 2e-4 * scale, (np.abs(got - want).max(), scale)


def test_backward_is_deterministic_and_linear_in_grad(cuda_device):
    """size-independent properties: position gradients are bit-reproducible (gather, no atomics; the same shape, so the
    same staged-window hint) and,
    with clipping off and a single-signed grad image, linear in the upstream gradient."""
    P0, N, S = 20000, 2, 128
    pts, nrm, col, proj, view, cams = scene(P0, N, seed=5)
    d = cuda_device
    prm = SplatParams(image_size=S, znear=0.1, clip_pts_grad=-1.0)
    h = torch.full((N,), 2e-4).to(d)
    colours = col.repeat(N, 1).to(d)
    g = -torch.rand(N, S, S, 4, generator=torch.Generator().manual_seed(2)).to(d)

    def run(scale):
        p = pts.to(d).requires_grad_(True)
        out = render_points(p, nrm.to(d), colours, proj.to(d), view.to(d), h, prm)
        out.image.backward(g * scale)
        return p.grad.clone()

    a, b, c2 = run(1.0), run(1.0), run(2.0)
    assert torch.equal(a, b)
    torch.testing.assert_close(c2, 2 * a, rtol=1e-5, atol=1e-9)


def test_shared_point_colours_equal_repeated_colours(cuda_device):
    """colours given once per POINT (P0,3) render exactly like the same rows repeated for every view, and their
    gradient is the sum over the views of the per-(view,point) gradient."""
    P0, N, S = 12000, 3, 96
    pts, nrm, col, proj, view, cams = scene(P0, N, seed=11)
    d = cuda_device
    prm = SplatParams(image_size=S, znear=0.1, clip_pts_grad=0.05)
    h = torch.full((N,), 3e-4).to(d)
    g = (torch.randn(N, S, S, 4, generator=torch.Generator().manual_seed(4)) * 1e-3).to(d)
    p1 = pts.to(d).requires_grad_(True)
    c1 = col.repeat(N, 1).to(d).requires_grad_(True)
    o1 = render_points(p1, nrm.to(d), c1, proj.to(d), view.to(d), h, prm)
    o1.image.backward(g)
    p2 = pts.to(d).requires_grad_(True)
    c2 = col.to(d).requires_grad_(True)
    o2 = render_points(p2, nrm.to(d), c2, proj.to(d), view.to(d), h, prm)
    o2.image.backward(g)
    assert torch.equal(o1.image, o2.image) and torch.equal(o1.idx, o2.idx)
    assert torch.equal(p1.grad, p2.grad)
    assert tuple(c2.grad.shape) == (P0, 3)
    torch.testing.assert_close(c2.grad, c1.grad.view(N, P0, 3).sum(0), rtol=1e-4, atol=1e-9)


def test_grad_sync_path_equals_plain_backward(cuda_device):
    """render_points(grad_sync=GradSync()) splits the backward into dss_colour_backward (side stream) and
    dss_render_backward without the colour half (dss_b200/parallel.py); on one rank the collectives are no-ops and the
    gradients must be those of the single-call backward: positions bit for bit, colours up to atomic order."""
    from dss_b200.parallel import GradSync
    P0, N, S = 15000, 3, 96
    pts, nrm, col, proj, view, cams = scene(P0, N, seed=17)
    d = cuda_device
    prm = SplatParams(image_size=S, znear=0.1, clip_pts_grad=0.05)
    h = torch.full((N,), 3e-4).to(d)
    g = (torch.randn(N, S, S, 4, generator=torch.Generator().manual_seed(6)) * 1e-3).to(d)
    res = []
    for sync in (None, GradSync(timing=True)):
        p = pts.to(d).requires_grad_(True)
        c = col.to(d).requires_grad_(True)
        o = render_points(p, nrm.to(d), c, proj.to(d), view.to(d), h, prm, grad_sync=sync)
        o.image.backward(g)
        torch.cuda.synchronize()
        res.append((p.grad.clone(), c.grad.clone()))
    assert torch.equal(res[0][0], res[1][0])
    torch.testing.assert_close(res[0][1], res[1][1], rtol=1e-4, atol=1e-10)


def test_more_than_256_shared_views_is_refused_before_any_launch(cuda_device):
    d = cuda_device
    pts, nrm, col, proj, view, cams = scene(100, 1, seed=1)
    N = 257
    with pytest.raises(RuntimeError, match="at most 256 views"):
        render_points(pts.to(d), nrm.to(d), col.to(d), proj.repeat(N, 1, 1).to(d), view.repeat(N, 1, 1).to(d),
                      torch.full((N,), 3e-4, device=d), SplatParams(image_size=32, znear=0.1))


def test_graphed_step_replays_the_eager_step(cuda_device):
    """dss_b200.graph.GraphedRenderStep: forward + backward captured once in a CUDA graph (the library neither
    synchronises nor allocates in steady state); replays must give the eager results, also after the static inputs
    were updated in place."""
    from dss_b200.graph import GraphedRenderStep
    P0, N, S = 30000, 3, 128
    pts, nrm, col, proj, view, cams = scene(P0, N, seed=23)
    d = cuda_device
    prm = SplatParams(image_size=S, znear=0.1, clip_pts_grad=0.05)
    h = torch.full((N,), 3e-4, device=d)
    g = (torch.randn(N, S, S, 4, generator=torch.Generator().manual_seed(8)) * 1e-3).to(d)
    p0 = pts.to(d).requires_grad_(True)
    c0 = col.to(d).requires_grad_(True)
    # leaves that have already been through an eager backward on the default stream (as in a training script that
    # switches to the graph after a few steps)
    render_points(p0, nrm.to(d), c0, proj.to(d), view.to(d), h, prm).image.backward(g)
    step = GraphedRenderStep(p0, nrm.to(d), c0, proj.to(d), view.to(d), h, prm, g)
    p, c = step.points, step.colours

    def eager():
        pe = p.detach().clone().requires_grad_(True)
        ce = c.detach().clone().requires_grad_(True)
        o = render_points(pe, nrm.to(d), ce, proj.to(d), view.to(d), h, prm)
        o.image.backward(g)
        return o.image.detach(), pe.grad, ce.grad

    for it in range(3):
        img = step.replay()
        torch.cuda.synchronize()
        wi, wp, wc = eager()
        assert torch.equal(img, wi)
        assert torch.equal(step.grad_points, wp)                       # deterministic gather
        torch.testing.assert_close(step.grad_colours, wc, rtol=1e-4, atol=1e-9)   # float atomics
        with torch.no_grad():                                          # "optimizer step" on the static tensors
            p.add_(0.002 * torch.randn(P0, 3, generator=torch.Generator().manual_seed(it)).to(d))
            c.mul_(0.9)
    assert not step.stale()


@pytest.fixture
def fresh_context(cuda_device):
    """A library context of the test's own in place of the process's one, so that its scratch starts empty whatever
    earlier tests rendered; destroyed afterwards, and the process's context restored."""
    from dss_b200 import _lib
    index = torch.device(cuda_device).index or 0
    torch.cuda.synchronize()
    saved = _lib._ctx.pop(index, None)
    try:
        yield
    finally:
        torch.cuda.synchronize()
        own = _lib._ctx.pop(index, None)
        if own is not None:
            _lib.load().dss_destroy(own)
        if saved is not None:
            _lib._ctx[index] = saved


def test_graphed_step_captures_again_when_the_scratch_moved(cuda_device, fresh_context):
    """A library call that needs more scratch than a captured GraphedRenderStep reallocates the buffers the graph
    reads; the next replay() must capture again (once) and still give the eager results."""
    from dss_b200 import _lib
    from dss_b200.graph import GraphedRenderStep
    P0, N, S = 20000, 2, 64
    pts, nrm, col, proj, view, cams = scene(P0, N, seed=29)
    d = cuda_device
    prm = SplatParams(image_size=S, znear=0.1, clip_pts_grad=0.05)
    h = torch.full((N,), 3e-4, device=d)
    g = (torch.randn(N, S, S, 4, generator=torch.Generator().manual_seed(9)) * 1e-3).to(d)
    step = GraphedRenderStep(pts.to(d), nrm.to(d), col.to(d), proj.to(d), view.to(d), h, prm, g)
    p, c = step.points, step.colours
    graph, scratch = step.graph, _lib.scratch_bytes()
    # an eager render at a larger image size and cloud grows the tile lists and the per-splat buffers
    bp, bn, bc, bproj, bview, _ = scene(4 * P0, N, seed=30)
    render_points(bp.to(d), bn.to(d), bc.to(d), bproj.to(d), bview.to(d), h, prm._replace(image_size=4 * S))
    torch.cuda.synchronize()
    assert _lib.scratch_bytes() > scratch

    def eager():
        pe = p.detach().clone().requires_grad_(True)
        ce = c.detach().clone().requires_grad_(True)
        o = render_points(pe, nrm.to(d), ce, proj.to(d), view.to(d), h, prm)
        o.image.backward(g)
        return o.image.detach(), pe.grad, ce.grad

    graphs = []
    for it in range(2):
        img = step.replay()
        graphs.append(step.graph)
        torch.cuda.synchronize()
        wi, wp, wc = eager()
        assert img is step.image and torch.equal(img, wi)
        assert torch.equal(step.grad_points, wp) and step.points.grad is step.grad_points
        torch.testing.assert_close(step.grad_colours, wc, rtol=1e-4, atol=1e-9)
        with torch.no_grad():
            p.add_(0.002 * torch.randn(P0, 3, generator=torch.Generator().manual_seed(it)).to(d))
    assert graphs[0] is not graph and graphs[1] is graphs[0]    # captured again over the moved scratch, and only once
    assert not step.stale()
