"""The image loss of the training step on the CPU: the torch body `image_loss_torch` and `IouLoss` against a per-pixel
float64 loop that restates Trainer.calc_dr_loss (DSS/training/trainer.py:349-376) with L1Loss and IouLoss
(DSS/training/losses.py:130-137, 498-513), its gradient with respect to the RGBA image included, and the input checks
that both routes share."""
import math

import numpy as np
import pytest
import torch

from dss_b200.training import IouLoss, image_loss, image_loss_torch


def loop_reference(rgba, img, mask, lambda_rgb, lambda_sil):
    """(loss, loss_rgb, loss_sil), d loss / d rgba: pixel by pixel in float64, eps_denom as mathHelper.py:10-14"""
    rgba, img, mask = (np.asarray(t, np.float64) for t in (rgba, img, mask))
    N, H, W, _ = rgba.shape
    grad = np.zeros_like(rgba)
    loss_rgb = loss_sil = 0.0
    if lambda_rgb > 0:
        M, s = 0, 0.0
        for n in range(N):
            for y in range(H):
                for x in range(W):
                    if mask[n, y, x] != 0 and rgba[n, y, x, 3] != 0:
                        M += 1
                        s += sum(abs(img[n, y, x, c] - rgba[n, y, x, c]) for c in range(3))
        if M > 0:
            loss_rgb = lambda_rgb * s / M
            for n in range(N):
                for y in range(H):
                    for x in range(W):
                        if mask[n, y, x] != 0 and rgba[n, y, x, 3] != 0:
                            for c in range(3):
                                grad[n, y, x, c] = np.sign(rgba[n, y, x, c] - img[n, y, x, c]) * lambda_rgb / M
    if lambda_sil > 0:
        l1, iou = 0.0, 0.0
        for n in range(N):
            I = U = 0.0
            for y in range(H):
                for x in range(W):
                    m, a = mask[n, y, x], rgba[n, y, x, 3]
                    l1 += abs(m - a)
                    I += m * a
                    U += m + a - m * a
            E = (1.0 if U >= 0 else -1.0) * max(abs(U), 1e-17)
            dE = 1.0 if abs(U) >= 1e-17 else 0.0
            iou += 1.0 - I / E
            for y in range(H):
                for x in range(W):
                    m, a = mask[n, y, x], rgba[n, y, x, 3]
                    grad[n, y, x, 3] = lambda_sil * (np.sign(a - m) / (N * H * W)
                                                     - 0.01 * (m * E - I * (1 - m) * dE) / (E * E) / N)
        loss_sil = lambda_sil * (0.01 * iou / N + l1 / (N * H * W))
    return (loss_rgb + loss_sil, loss_rgb, loss_sil), grad


def random_case(N, H, W, seed, fractional=False, ties=0.0):
    g = torch.Generator().manual_seed(seed)
    rgba = torch.rand(N, H, W, 4, generator=g, dtype=torch.float64)
    alpha = rgba[..., 3]
    alpha[torch.rand(N, H, W, generator=g) < 0.3] = 0.0
    alpha[torch.rand(N, H, W, generator=g) < 0.3] = 1.0
    img = torch.rand(N, H, W, 3, generator=g, dtype=torch.float64)
    tie = torch.rand(N, H, W, 3, generator=g) < ties
    img[tie] = rgba[..., :3][tie]
    mask = (torch.rand(N, H, W, generator=g) < 0.5).double()
    if fractional:
        mask = torch.where(torch.rand(N, H, W, generator=g) < 0.5, torch.rand(N, H, W, generator=g).double(), mask)
    return rgba, img, mask


def check(rgba, img, mask, lambda_rgb=1.0, lambda_sil=1.0):
    want, want_grad = loop_reference(rgba, img, mask, lambda_rgb, lambda_sil)
    x = rgba.clone().requires_grad_(True)
    out = image_loss_torch(x, img, mask, lambda_rgb, lambda_sil)
    assert set(out) == {"loss", "loss_dr_rgb", "loss_dr_silhouette", "loss_image_gradients"}
    assert float(out["loss_image_gradients"]) == 0.0
    got = [float(out[k].detach()) for k in ("loss", "loss_dr_rgb", "loss_dr_silhouette")]
    for g, w in zip(got, want):
        assert math.isclose(g, w, rel_tol=1e-12, abs_tol=1e-15), (got, want)
    if out["loss"].requires_grad:
        out["loss"].backward()
        np.testing.assert_allclose(x.grad.numpy(), want_grad, rtol=1e-12, atol=1e-15)
    else:
        assert not want_grad.any()
    return out, x.grad


@pytest.mark.parametrize("N,H,W,seed", [(1, 1, 1, 0), (2, 5, 7, 1), (3, 8, 8, 2), (1, 13, 4, 3)])
@pytest.mark.parametrize("fractional", [False, True])
def test_torch_body_matches_the_loop(N, H, W, seed, fractional):
    check(*random_case(N, H, W, seed, fractional=fractional, ties=0.2))


def test_real_shaped_masks():
    """a disc silhouette against a shifted disc, alpha smooth at the rim, the target image a constant colour"""
    N, S = 2, 16
    yy, xx = torch.meshgrid(torch.arange(S, dtype=torch.float64), torch.arange(S, dtype=torch.float64), indexing="ij")
    rgba = torch.zeros(N, S, S, 4, dtype=torch.float64)
    mask = torch.zeros(N, S, S, dtype=torch.float64)
    for n in range(N):
        r = ((yy - 7.5 - n) ** 2 + (xx - 7.5) ** 2).sqrt()
        rgba[n, ..., 3] = (5.0 - r).clamp(0, 1)
        rgba[n, ..., :3] = torch.stack([xx / S, yy / S, 0.5 * torch.ones_like(xx)], -1) * rgba[n, ..., 3:]
        mask[n] = (((yy - 7.5) ** 2 + (xx - 8.5 + n) ** 2).sqrt() < 5.0).double()
    img = torch.full((N, S, S, 3), 0.3, dtype=torch.float64)
    check(rgba, img, mask)


def test_no_overlap_drops_the_rgb_term():
    """M = 0: the reference's ``if mask_pred.sum() > 0`` leaves the RGB term at 0 and without a gradient"""
    rgba, img, mask = random_case(2, 6, 6, 4)
    rgba[..., 3] = torch.where(mask != 0, torch.zeros_like(mask), rgba[..., 3])
    out, grad = check(rgba, img, mask)
    assert float(out["loss_dr_rgb"]) == 0.0 and not grad[..., :3].any()


def test_empty_ground_truth_and_empty_prediction():
    """an empty view: the IoU term is 1 (union clamped to eps_denom's 1e-17) and its gradient 0"""
    rgba, img, mask = random_case(2, 5, 5, 5)
    rgba[1, ..., 3] = 0.0
    mask[1] = 0.0
    out, grad = check(rgba, img, mask)
    assert not grad[1].any()
    iou = IouLoss(reduction="none", channel_dim=None)(mask, rgba[..., 3])
    assert float(iou[1]) == 1.0


@pytest.mark.parametrize("lambda_rgb,lambda_sil", [(0.0, 1.0), (1.0, 0.0), (-1.0, 2.5), (3.0, -0.5), (0.0, 0.0)])
def test_lambdas_at_or_below_zero_drop_the_term(lambda_rgb, lambda_sil):
    rgba, img, mask = random_case(2, 6, 5, 6, fractional=True)
    out, grad = check(rgba, img, mask, lambda_rgb, lambda_sil)
    if lambda_rgb <= 0:
        assert float(out["loss_dr_rgb"]) == 0.0 and (grad is None or not grad[..., :3].any())
    if lambda_sil <= 0:
        assert float(out["loss_dr_silhouette"]) == 0.0 and (grad is None or not grad[..., 3].any())


@pytest.mark.parametrize("absent", ["rgb", "silhouette"])
def test_zero_lambda_never_reads_the_absent_term(absent):
    """NaN planted inside mask_pred, where only the absent term reads it: a term computed with weight 0 would give a
    NaN loss; the dropped term leaves the loss finite and the channels it owns without a gradient"""
    rgba, img, mask = random_case(2, 6, 5, 11)
    mask[0, 2, 3] = 1.0
    rgba[0, 2, 3, 3] = 0.5
    if absent == "rgb":
        rgba[0, 2, 3, 0] = float("nan")
        lambdas = (0.0, 1.0)
    else:
        rgba[0, 2, 3, 3] = float("nan")          # NaN.bool() is true: the pixel stays in mask_pred for the RGB term
        lambdas = (1.0, 0.0)
    x = rgba.clone().requires_grad_(True)
    out = image_loss_torch(x, img, mask, *lambdas)
    assert all(bool(torch.isfinite(v)) for v in out.values())
    out["loss"].backward()
    assert torch.isfinite(x.grad).all()
    assert not x.grad[..., :3].any() if absent == "rgb" else not x.grad[..., 3].any()


def test_iou_loss_matches_the_loop():
    g = torch.Generator().manual_seed(7)
    p = torch.rand(3, 4, 5, generator=g, dtype=torch.float64)
    t = torch.rand(3, 4, 5, generator=g, dtype=torch.float64)
    want = [1.0 - float((p[n] * t[n]).sum()) / float((p[n] + t[n] - p[n] * t[n]).sum()) for n in range(3)]
    iou = IouLoss(reduction="none", channel_dim=None)
    np.testing.assert_allclose(iou(p, t).numpy(), want, rtol=1e-14)
    assert math.isclose(float(IouLoss(reduction="mean", channel_dim=None)(p, t)), sum(want) / 3, rel_tol=1e-14)
    assert iou(p.float(), t.float()).dtype == torch.float32


def test_mask_layouts_and_dtypes_agree():
    """(N,1,H,W) and (N,H,W) masks, bool / uint8 / float 0-1 masks, a permuted (N,3,H,W) target: the same loss"""
    rgba, img, mask = random_case(2, 6, 7, 8)
    ref = image_loss_torch(rgba, img, mask)
    perm = img.permute(0, 3, 1, 2).contiguous().permute(0, 2, 3, 1)
    for m in (mask[:, None], mask.bool(), mask.to(torch.uint8)):
        out = image_loss_torch(rgba, perm, m)
        assert all(torch.equal(out[k], ref[k]) for k in ref)


def test_cpu_inputs_take_the_torch_body():
    rgba, img, mask = random_case(1, 4, 4, 9)
    out = image_loss(rgba.float(), img.float(), mask.float())
    ref = image_loss_torch(rgba.float(), img.float(), mask.float())
    assert all(torch.equal(out[k], ref[k]) for k in ref)


@pytest.mark.parametrize("case", ["rgba_rank", "rgba_channels", "empty", "img_shape", "mask_shape"])
def test_input_checks_raise(case):
    rgba, img, mask = random_case(2, 4, 5, 10)
    if case == "rgba_rank":
        rgba = rgba[0]
    elif case == "rgba_channels":
        rgba = rgba[..., :3]
    elif case == "empty":
        rgba, img, mask = rgba[:, :0], img[:, :0], mask[:, :0]
    elif case == "img_shape":
        img = img.permute(0, 3, 1, 2)
    elif case == "mask_shape":
        mask = mask[:, None, :, :, None]
    with pytest.raises(RuntimeError):
        image_loss(rgba, img, mask)
    with pytest.raises(RuntimeError):
        image_loss_torch(rgba, img, mask)
