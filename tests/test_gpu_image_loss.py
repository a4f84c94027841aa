"""The fused image loss (`dss_image_loss_forward` / `_backward`, csrc/image_loss.cu) against the torch body
`image_loss_torch` run in float64 on the same float32 inputs, per element.

Bounds (DESIGN.md section 6), from the kernels' operation sequence: every per-pixel term is formed in fp64 from exact
float32 inputs and summed in fp64, so the totals carry relative errors of a few 2^-50; each output is rounded to float32
once.  Hence
  - an RGB gradient entry (sign * the float32 weight) and the loss scalars' rounding: within 1 ulp of the float64 value
    rounded to float32;
  - an alpha gradient entry: 1 ulp of the rounded value plus 2^-24 * (|m A_n| + |(1 - m) B_n|), the IoU terms'
    magnitudes (A_n = w / E_n, B_n = w I_n / E_n^2);
  - a loss scalar: 1 ulp plus 2^-23 * the sum of its terms' magnitudes.
"""
import os

import pytest
import torch

from dss_b200 import _lib
from dss_b200.ops import SplatParams, make_shading, render_points
from dss_b200.training.losses import image_loss, image_loss_torch
from dss_b200.utils.io import read_ply
from tests.test_shading import _lights
from tests.util import GOLDEN_DIR, camera_matrices, random_cameras

pytestmark = pytest.mark.gpu

KEYS = ("loss", "loss_dr_rgb", "loss_dr_silhouette")
U = 2.0 ** -24
WORST = {}


@pytest.fixture(autouse=True)
def _cuda(cuda_device):
    return cuda_device


def ulp32(x):
    """ulp of x (float64) rounded to float32"""
    a = x.abs().float()
    return (torch.nextafter(a, torch.full_like(a, float("inf"))) - a).double()


def random_case(N, H, W, seed, dev, fractional=True, ties=0.1):
    g = torch.Generator().manual_seed(seed)
    rgba = torch.rand(N, H, W, 4, generator=g)
    a = rgba[..., 3]
    a[torch.rand(N, H, W, generator=g) < 0.3] = 0.0
    a[torch.rand(N, H, W, generator=g) < 0.3] = 1.0
    img = torch.rand(N, H, W, 3, generator=g)
    tie = torch.rand(N, H, W, 3, generator=g) < ties
    img[tie] = rgba[..., :3][tie]
    mask = (torch.rand(N, H, W, generator=g) < 0.5).float()
    if fractional:
        mask = torch.where(torch.rand(N, H, W, generator=g) < 0.3, torch.rand(N, H, W, generator=g), mask)
    return rgba.to(dev), img.to(dev), mask.to(dev)


def upstream(seed, dev):
    """float32-exact upstream gradients of (loss, loss_dr_rgb, loss_dr_silhouette)"""
    g = torch.Generator().manual_seed(seed)
    return [(torch.rand((), generator=g) + 0.5).to(dev) for _ in KEYS]


def fused(rgba, img, mask, lr=1.0, ls=1.0, ups=None):
    x = rgba.detach().clone().requires_grad_(True)
    out = image_loss(x, img, mask, lr, ls)
    ups = ups or [torch.ones((), device=rgba.device), torch.zeros((), device=rgba.device),
                  torch.zeros((), device=rgba.device)]
    torch.autograd.backward([out[k] for k in KEYS], ups)
    return [out[k].detach() for k in KEYS], x.grad


def reference(rgba, img, mask, lr=1.0, ls=1.0, ups=None):
    """float64 torch body on the same inputs; also the magnitudes the bounds scale with"""
    x = rgba.detach().double().requires_grad_(True)
    m = mask.reshape(rgba.shape[:3]).float().double()
    out = image_loss_torch(x, img.double(), m, lr, ls)
    ups = [u.double() for u in ups] if ups else [torch.ones((), device=rgba.device, dtype=torch.float64),
                                                  torch.zeros((), device=rgba.device, dtype=torch.float64),
                                                  torch.zeros((), device=rgba.device, dtype=torch.float64)]
    outs = [(o, u) for o, u in zip((out[k] for k in KEYS), ups) if o.requires_grad]
    if outs:
        torch.autograd.backward([o for o, _ in outs], [u for _, u in outs])
    grad = x.grad if x.grad is not None else torch.zeros_like(x)
    N, H, W = rgba.shape[:3]
    a = x.detach()[..., 3]
    gl, gr, gs = (float(u) for u in ups)
    ws = ls * (gl + gs) if ls > 0 else 0.0
    I = (m * a).sum((1, 2))
    Un = (m + a - m * a).sum((1, 2))
    E = torch.where(Un < 0, -1.0, 1.0) * Un.abs().clamp(min=1e-17)
    A = 0.01 * ws / N / E
    B = 0.01 * ws / N * I / (E * E)
    iou_mag = (m * A[:, None, None]).abs() + ((1 - m) * B[:, None, None]).abs() if ws != 0 else torch.zeros_like(m)
    mp = (m != 0) & (a != 0)
    M = int(mp.sum())
    d = (img.double() - x.detach()[..., :3]).abs().sum(-1)
    rgb_mag = lr * float(torch.where(mp, d, torch.zeros_like(d)).sum()) / M if (lr > 0 and M > 0) else 0.0
    sil_mag = ls * (0.01 * float((1 - I / E).abs().sum()) / N + float((m - a).abs().sum()) / (N * H * W)) \
        if ls > 0 else 0.0
    return [out[k].detach() for k in KEYS], grad, iou_mag, (rgb_mag + sil_mag, rgb_mag, sil_mag)


def compare(name, rgba, img, mask, lr=1.0, ls=1.0, ups=None, nan_ok=False):
    losses, grad = fused(rgba, img, mask, lr, ls, ups)
    check(name, losses, grad, rgba, img, mask, lr, ls, ups, nan_ok)
    return losses, grad


def check(name, losses, grad, rgba, img, mask, lr=1.0, ls=1.0, ups=None, nan_ok=False):
    """the three loss scalars and the RGBA gradient of a fused loss against `reference`, within the docstring's bounds"""
    rlosses, rgrad, iou_mag, mags = reference(rgba, img, mask, lr, ls, ups)
    worst = WORST.setdefault(name, [0.0, 0.0, 0.0])
    # gradient: NaN at the same places, the rest within the bound
    nan = torch.isnan(rgrad)
    assert torch.equal(torch.isnan(grad), nan), name
    assert nan_ok or not nan.any()
    g, r = grad.double(), rgrad
    ok = ~nan
    err = (g - r).abs()
    b_rgb = ulp32(r[..., :3])
    b_a = ulp32(r[..., 3]) + U * iou_mag
    e_rgb, e_a = err[..., :3][ok[..., :3]], err[..., 3][ok[..., 3]]
    assert (e_rgb <= b_rgb[ok[..., :3]]).all(), (name, float((e_rgb - b_rgb[ok[..., :3]]).max()))
    assert (e_a <= b_a[ok[..., 3]]).all(), (name, float((e_a - b_a[ok[..., 3]]).max()))
    if e_rgb.numel():
        worst[0] = max(worst[0], float((e_rgb / b_rgb[ok[..., :3]]).max()))
    if e_a.numel():
        worst[1] = max(worst[1], float((e_a / b_a[ok[..., 3]]).max()))
    for k, got, want, mag in zip(KEYS, losses, rlosses, mags):
        if torch.isnan(want):
            assert nan_ok and torch.isnan(got), (name, k)
            continue
        bound = float(ulp32(want)) + 2 * U * mag
        e = abs(float(got) - float(want))
        assert e <= bound, (name, k, float(got), float(want), bound)
        worst[2] = max(worst[2], e / bound if bound > 0 else 0.0)
    print("%s: worst error / bound  rgb grad %.3f  alpha grad %.3f  losses %.3f" % (name, *worst))


# ---- 1. random images, every size --------------------------------------------------------------------------------
@pytest.mark.parametrize("N,S", [(1, 1), (8, 1), (33, 1), (1, 17), (8, 17), (33, 17), (1, 256), (8, 256), (33, 256),
                                 (8, 512), (33, 512), (1, 1024), (8, 1024)])
def test_random_images_match_float64(N, S, cuda_device):
    rgba, img, mask = random_case(N, S, S, N * 1000 + S, cuda_device)
    compare("random", rgba, img, mask, ups=upstream(S, cuda_device))
    compare("random", rgba, img, mask, 0.7, 2.5, ups=upstream(S + 1, cuda_device))


def test_rectangular_images(cuda_device):
    rgba, img, mask = random_case(3, 17, 40, 3, cuda_device)
    compare("random", rgba, img, mask, ups=upstream(3, cuda_device))


# ---- 2. renders of the golden bunny against a jittered target -----------------------------------------------------
def bunny(dev):
    ply = read_ply(os.path.join(GOLDEN_DIR, "ply", "bunny-8000.ply"))
    pts = torch.as_tensor(ply["points"], dtype=torch.float32)
    pts = (pts - pts.mean(0)) / (pts - pts.mean(0)).norm(dim=1).max() * 0.6
    nrm = torch.nn.functional.normalize(torch.as_tensor(ply["normals"], dtype=torch.float32), dim=1)
    col = torch.rand(pts.shape, generator=torch.Generator().manual_seed(3))
    return pts.to(dev), nrm.to(dev), col.to(dev)


def render(pts, nrm, col, N, S, seed, dev, **kw):
    proj, view = (m.to(dev) for m in camera_matrices(random_cameras(N, seed, dist=(1.6, 2.2))))
    prm = SplatParams(image_size=S, points_per_pixel=5, znear=0.1, clip_pts_grad=0.05)
    h = torch.full((N,), 1e-3, device=dev)
    return render_points(pts, nrm, col.repeat(N, 1) if "shading" not in kw else col, proj, view, h, prm, **kw)


def bunny_targets(N, S, dev):
    """the target: the bunny moved a little, other colours; mask = its alpha > 0"""
    pts, nrm, col = bunny(dev)
    g = torch.Generator().manual_seed(5)
    with torch.no_grad():
        out = render(pts + 0.01 * torch.randn(3, generator=g).to(dev), nrm, col.flip(1), N, S, 0, dev)
    return out.image[..., :3].contiguous(), (out.image[..., 3] > 0).float()


@pytest.mark.parametrize("N,S", [(1, 17), (8, 256), (8, 512), (33, 256), (1, 1024)])
def test_bunny_renders_match_float64(N, S, cuda_device):
    pts, nrm, col = bunny(cuda_device)
    with torch.no_grad():
        rgba = render(pts, nrm, col, N, S, 0, cuda_device).image
    img, mask = bunny_targets(N, S, cuda_device)
    assert 0 < int(((mask != 0) & (rgba[..., 3] != 0)).sum()) < mask.numel()
    compare("bunny", rgba, img, mask, ups=upstream(N, cuda_device))


# ---- 3. edge cases -----------------------------------------------------------------------------------------------
def test_no_overlap_gives_zero_rgb_term(cuda_device):
    rgba, img, mask = random_case(4, 20, 20, 11, cuda_device)
    rgba[..., 3] = torch.where(mask != 0, 0.0, rgba[..., 3])
    losses, grad = compare("edges", rgba, img, mask)
    assert float(losses[1]) == 0.0 and not grad[..., :3].any()


def test_empty_view(cuda_device):
    rgba, img, mask = random_case(3, 16, 16, 12, cuda_device)
    rgba[1, ..., 3] = 0.0
    mask[1] = 0.0
    _, grad = compare("edges", rgba, img, mask)
    assert not grad[1].any()


def test_exact_ties_give_zero_gradient(cuda_device):
    rgba, img, mask = random_case(2, 32, 32, 13, cuda_device, fractional=False, ties=0.0)
    img = rgba[..., :3].clone()
    mask = rgba[..., 3].clone()
    _, grad = compare("edges", rgba, img, mask)
    assert not grad[..., :3].any()


def test_fractional_masks(cuda_device):
    rgba, img, _ = random_case(4, 64, 64, 14, cuda_device)
    mask = torch.rand(4, 64, 64, generator=torch.Generator().manual_seed(14)).to(cuda_device)
    compare("edges", rgba, img, mask, ups=upstream(14, cuda_device))


def bits(t):
    return t.reshape(-1).view(torch.int32)


@pytest.mark.parametrize("absent", ["rgb", "silhouette"])
def test_zero_lambda_drops_the_term_bit_for_bit(absent, cuda_device):
    """lambda = 0 (or < 0): the term is 0, its channels get an exact +0 gradient, and NaN in the inputs only that term
    reads -- planted inside mask_pred, where a term computed with weight 0 would read it -- reaches nothing: every
    output has the bits of a call with lambda = -1 on the clean inputs"""
    rgba, img, mask = random_case(3, 48, 48, 15, cuda_device)
    planted = ((0, 3, 4), (1, 5, 6), (2, 7, 7))
    for n, y, x in planted:                    # inside mask_pred on both sides: m != 0, alpha != 0
        mask[n, y, x] = 1.0
        rgba[n, y, x, 3] = 0.5
    ups = upstream(15, cuda_device)
    lr, ls = (0.0, 1.5) if absent == "rgb" else (1.5, 0.0)
    compare("edges", rgba, img, mask, lr, ls, ups=ups)
    base_losses, base_grad = fused(rgba, img, mask, -1.0 if absent == "rgb" else lr, -1.0 if absent != "rgb" else ls,
                                   ups)
    dirty, img = rgba.clone(), img.clone()
    if absent == "rgb":
        dirty[0, 3, 4, :3] = float("nan")      # read only by the RGB term
        img[1, 5, 6] = float("nan")
    else:
        dirty[2, 7, 7, 3] = float("nan")       # NaN.bool() is true: still inside mask_pred, read by the silhouette terms
    assert all(bool((mask[p] != 0) & (dirty[p][3] != 0)) for p in planted)
    losses, grad = fused(dirty, img, mask, lr, ls, ups)
    assert all(bool(torch.isfinite(x)) for x in losses) and torch.isfinite(grad).all()
    k, ch = (1, slice(0, 3)) if absent == "rgb" else (2, slice(3, 4))
    assert torch.equal(bits(losses[k]), bits(torch.zeros((), device=cuda_device)))
    assert torch.equal(bits(grad[..., ch]), bits(torch.zeros_like(grad[..., ch])))          # +0, not -0
    assert all(torch.equal(bits(a), bits(b)) for a, b in zip(losses, base_losses))
    assert torch.equal(bits(grad), bits(base_grad))
    assert torch.equal(bits(losses[0]), bits(losses[2 if absent == "rgb" else 1]))
    compare("edges", dirty, img, mask, lr, ls, ups=ups)


def test_nan_in_prediction(cuda_device):
    """NaN in pred behaves as in torch: NaN.bool() is true, NaN reaches the losses, abs' backward has sign(NaN) = 0,
    and a NaN alpha makes its view's IoU gradient NaN"""
    rgba, img, mask = random_case(3, 24, 24, 16, cuda_device)
    mask[0, 1, 1] = 1.0
    rgba[0, 1, 1, 3] = 0.5
    mask[1, 2, 3] = 1.0
    mask[2, 9, 9] = 1.0
    rgba[0, 1, 1, 0] = float("nan")
    rgba[1, 2, 3, 3] = float("nan")            # inside the GT mask: counts in M
    rgba[2, 9, 9, 1] = float("nan")
    rgba[2, 9, 9, 3] = 0.0                     # alpha 0: outside mask_pred, the NaN rgb is never read
    compare("nan", rgba, img, mask, ups=upstream(16, cuda_device), nan_ok=True)
    _, grad = fused(rgba, img, mask)
    assert torch.isnan(grad[1, ..., 3]).all() and torch.isfinite(grad[0]).all() and torch.isfinite(grad[2]).all()


# ---- 4. input layouts ----------------------------------------------------------------------------------------------
def test_layouts_and_mask_dtypes_give_identical_bits(cuda_device):
    rgba, img, mask = random_case(4, 40, 56, 17, cuda_device, fractional=False)
    ref = fused(rgba, img, mask)
    perm = img.permute(0, 3, 1, 2).contiguous().permute(0, 2, 3, 1)
    assert not perm.is_contiguous()
    for i, m in ((perm, mask), (img, mask[:, None]), (img, mask.bool()), (img, mask.to(torch.uint8)),
                 (perm, mask.bool()[:, None])):
        got = fused(rgba, i, m)
        assert all(torch.equal(a, b) for a, b in zip(got[0], ref[0])) and torch.equal(got[1], ref[1])
    compare("layout", rgba, perm, mask)


def test_uint8_mask_values_are_used(cuda_device):
    rgba, img, mask = random_case(2, 20, 20, 18, cuda_device, fractional=False)
    m8 = (mask * torch.randint(0, 4, mask.shape, generator=torch.Generator().manual_seed(1)).to(mask.device)).to(
        torch.uint8)
    compare("layout", rgba, img, m8, ups=upstream(18, cuda_device))


def test_targets_that_require_grad_take_the_torch_body(cuda_device):
    """the fused route differentiates the RGBA only: a GT image or a float mask that requires grad runs the torch body,
    which gives it its gradient"""
    rgba, img, mask = random_case(2, 16, 16, 21, cuda_device)
    for which in ("img", "mask"):
        i, m = img.clone().requires_grad_(which == "img"), mask.clone().requires_grad_(which == "mask")
        x = rgba.clone().requires_grad_(True)
        before = _lib.launch_count(cuda_device)
        image_loss(x, i, m)["loss"].backward()
        assert _lib.launch_count(cuda_device) == before
        t = i if which == "img" else m
        want = t.detach().clone().requires_grad_(True)
        args = (want, mask) if which == "img" else (img, want)
        image_loss_torch(rgba, *args)["loss"].backward()
        assert t.grad is not None and torch.equal(t.grad, want.grad)


# ---- 5. end to end through the render backward --------------------------------------------------------------------
def test_render_loss_backward_end_to_end(cuda_device):
    d, N, S = cuda_device, 4, 128
    pts, nrm, col = bunny(d)
    img, mask = bunny_targets(N, S, d)
    proj, view = (m.to(d) for m in camera_matrices(random_cameras(N, 0, dist=(1.6, 2.2))))
    sh = make_shading(_lights("sun", d), view)

    def run(grad_image=None):
        p, n, c = (t.clone().requires_grad_(True) for t in (pts, nrm, col))
        out = render(p, n, c, N, S, 0, d, shading=sh)
        if grad_image is None:
            image_loss(out.image, img, mask, 1.0, 2.0)["loss"].backward()
        else:
            out.image.backward(grad_image)
        return out.image.detach(), (p.grad, n.grad, c.grad)

    rgba, got = run()
    x = rgba.double().requires_grad_(True)
    image_loss_torch(x, img.double(), mask.double(), 1.0, 2.0)["loss"].backward()
    _, want = run(x.grad.float())
    for name, g, w in zip(("points", "normals", "albedo"), got, want):
        scale = w.abs().max().item()
        err = (g.double() - w.double()).abs().max().item()
        assert scale > 0 and err <= 2e-4 * scale, (name, err, scale)


# ---- 6. determinism, host synchronisation, launches ---------------------------------------------------------------
def test_two_calls_are_bit_identical(cuda_device):
    rgba, img, mask = random_case(8, 256, 256, 19, cuda_device)
    ups = upstream(19, cuda_device)
    a, b = fused(rgba, img, mask, ups=ups), fused(rgba, img, mask, ups=ups)
    assert all(torch.equal(x, y) for x, y in zip(a[0], b[0])) and torch.equal(a[1], b[1])


def test_no_host_sync_and_fixed_launch_count(cuda_device):
    """after a warm-up, forward + backward do not synchronise the host and the library launches 2 + 1 kernels at any
    size"""
    dev = cuda_device
    counts = []
    for N, S in ((1, 64), (8, 512)):
        rgba, img, mask = random_case(N, S, S, 20, dev)
        x = rgba.clone().requires_grad_(True)
        perm = img.permute(0, 3, 1, 2).contiguous().permute(0, 2, 3, 1)

        def step():
            image_loss(x, perm, mask.bool(), 1.0, 1.0)["loss"].backward()

        step()
        torch.cuda.synchronize()
        before = _lib.launch_count(dev)
        torch.cuda.set_sync_debug_mode("error")
        try:
            step()
        finally:
            torch.cuda.set_sync_debug_mode("default")
        counts.append(_lib.launch_count(dev) - before)
    assert counts == [3, 3]


# ---- 7. a captured training step -----------------------------------------------------------------------------------
def test_graphed_step_with_targets_replays_the_eager_step(cuda_device):
    from dss_b200.graph import GraphedRenderStep
    d, N, S = cuda_device, 3, 128
    pts, nrm, col = bunny(d)
    proj, view = (m.to(d) for m in camera_matrices(random_cameras(N, 0, dist=(1.6, 2.2))))
    prm = SplatParams(image_size=S, points_per_pixel=5, znear=0.1, clip_pts_grad=0.05)
    h = torch.full((N,), 1e-3, device=d)
    img, mask = bunny_targets(N, S, d)
    img = img.permute(0, 3, 1, 2).contiguous().permute(0, 2, 3, 1)       # the trainer's layout
    cols = col.repeat(N, 1)
    with pytest.raises(ValueError):
        GraphedRenderStep(pts, nrm, cols, proj, view, h, prm)
    with pytest.raises(ValueError):
        GraphedRenderStep(pts, nrm, cols, proj, view, h, prm, torch.zeros(N, S, S, 4, device=d),
                          targets=(img, mask, 1.0, 1.0))
    for bad in ((img.double(), mask), (img, mask.double())):
        with pytest.raises(TypeError):                                 # would run the torch body inside the capture
            GraphedRenderStep(pts, nrm, cols, proj, view, h, prm, targets=(*bad, 1.0, 1.0))
    step = GraphedRenderStep(pts, nrm, cols, proj, view, h, prm, targets=(img, mask, 1.0, 2.0))
    for it in range(3):
        step.replay()
        torch.cuda.synchronize()
        pe, ce = (t.detach().clone().requires_grad_(True) for t in (step.points, step.colours))
        o = render_points(pe, nrm, ce, proj, view, h, prm)
        loss = image_loss(o.image, step.img, step.mask_img, 1.0, 2.0)
        loss["loss"].backward()
        assert torch.equal(step.image, o.image.detach())
        assert all(torch.equal(step.loss[k], loss[k]) for k in KEYS)
        assert torch.equal(step.grad_points, pe.grad)                      # deterministic gather
        torch.testing.assert_close(step.grad_colours, ce.grad, rtol=1e-4, atol=1e-9)   # float atomics
        with torch.no_grad():                                              # the next batch and an optimizer step
            g = torch.Generator().manual_seed(it)
            step.img.copy_(torch.rand(step.img.shape, generator=g).to(d))
            step.mask_img.copy_(torch.roll(step.mask_img, 1 + it, dims=2))
            step.points.add_(0.002 * torch.randn(step.points.shape, generator=g).to(d))
