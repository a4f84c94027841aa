"""CPU: tests/image_metrics_oracle.py against torch's own CPU operators -- the resize against F.interpolate(
mode='bilinear', align_corners=False) and the per-view terms against the reference's IouLoss and L2Loss(channel_dim=1)
restated in torch -- and the oracle's edges."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import image_metrics_oracle as im

SIZES = [(64, 64, 64), (64, 64, 16), (100, 100, 37), (64, 64, 96), (20, 31, 8), (7, 5, 2), (1, 1, 3), (9, 9, 1)]


@pytest.mark.parametrize("H,W,s", SIZES)
def test_resize_equals_torch_interpolate(H, W, s):
    rng = np.random.default_rng(H * 1000 + W * 10 + s)
    img = rng.random((3, H, W, 3))
    ref = F.interpolate(torch.from_numpy(img).permute(0, 3, 1, 2), size=(s, s), mode="bilinear",
                        align_corners=False).permute(0, 2, 3, 1).numpy()
    got = im.resize(img, s)
    assert got.shape == (3, s, s, 3)
    np.testing.assert_allclose(got, ref, rtol=0, atol=1e-12)
    mask = rng.random((3, H, W))
    ref_m = F.interpolate(torch.from_numpy(mask)[:, None], size=(s, s), mode="bilinear", align_corners=False)[:, 0]
    np.testing.assert_allclose(im.resize(mask, s), ref_m.numpy(), rtol=0, atol=1e-12)


def test_resize_at_the_same_size_is_the_identity():
    img = np.random.default_rng(0).random((2, 33, 33, 3))
    assert np.array_equal(im.resize(img, 33), img)


def eps_denom_torch(denom, eps=1e-17):
    """DSS/utils/mathHelper.py:10-14"""
    sign = denom.sign() + (denom == 0.0).type_as(denom)
    return sign * torch.clamp(denom.abs(), eps)


def eval_step_torch(pred, img, mask, s):
    """Trainer.eval_step's two terms (trainer.py:196-210) restated in torch, per view: IouLoss(mask_gt, alpha) and
    L2Loss(channel_dim=1) of the resized ground truth against the render, float64"""
    rgba = torch.from_numpy(pred).permute(0, 3, 1, 2)
    mask_gt = F.interpolate(torch.from_numpy(mask)[:, None].double(), s, mode="bilinear", align_corners=False)[:, 0]
    alpha = rgba[:, 3]
    inter = (mask_gt * alpha).sum((1, 2))
    union = (mask_gt + alpha - mask_gt * alpha).sum((1, 2))
    iou = 1.0 - inter / eps_denom_torch(union)
    rgb_gt = F.interpolate(torch.from_numpy(img).permute(0, 3, 1, 2), s, mode="bilinear", align_corners=False)
    # L2Loss with channel_dim=1: the squared error summed over the channels, then the mean over the pixels
    psnr = ((rgb_gt - rgba[:, :3]) ** 2).sum(1).mean((1, 2))
    return iou.numpy(), psnr.numpy()


@pytest.mark.parametrize("H,s", [(32, 32), (32, 8), (50, 19), (24, 36)])
def test_metrics_equal_the_reference_losses(H, s):
    rng = np.random.default_rng(H + s)
    V = 5
    pred = rng.random((V, s, s, 4)) * 1.2 - 0.1          # unclamped renders
    img = rng.random((V, H, H, 3))
    mask = (rng.random((V, H, H)) > 0.4).astype(np.float64)
    mask[1] = 0.0
    pred[1, ..., 3] = 0.0                                 # an all-empty view: I = U = 0
    per_view, iou, psnr = im.image_metrics(pred, img, mask)
    ref_iou, ref_psnr = eval_step_torch(pred, img, mask, s)
    np.testing.assert_allclose(per_view[:, 3], ref_iou, rtol=0, atol=1e-12)
    np.testing.assert_allclose(per_view[:, 4], ref_psnr, rtol=1e-12, atol=0)
    assert per_view[1, 0] == 0 and per_view[1, 1] == 0 and per_view[1, 3] == 1.0     # an empty union scores iou 1
    assert abs(iou - ref_iou.mean()) < 1e-12 and abs(psnr - ref_psnr.mean()) < 1e-12 * ref_psnr.mean()
