"""float64 numpy restatement of dss_image_metrics (csrc/image_metrics.cu; the rule is in include/dss_b200.h): the
ground truth resized as torch's upsample_bilinear2d (align_corners=False, no antialias) resizes it, then per view the
IouLoss and L2Loss(channel_dim=1) terms of the reference's Trainer.eval_step.  The kernel forms the resize in float32,
so it agrees with this oracle to float32 rounding, not bit for bit (except at s == H, where both return the input)."""
import numpy as np


def taps(size_in, size_out):
    """(i0, i1, l0, l1) per output index: src = max((dst + 0.5) size_in / size_out - 0.5, 0), i0 = floor(src),
    i1 = min(i0 + 1, size_in - 1), l1 = src - i0, l0 = 1 - l1"""
    src = np.maximum((np.arange(size_out, dtype=np.float64) + 0.5) * (size_in / size_out) - 0.5, 0.0)
    i0 = np.floor(src).astype(np.int64)
    i1 = np.minimum(i0 + 1, size_in - 1)
    l1 = src - i0
    return i0, i1, 1.0 - l1, l1


def resize(img, s):
    """(V, H, W[, C]) -> (V, s, s[, C]) float64, bilinear with torch's source-index rule"""
    a = np.asarray(img, dtype=np.float64)
    y0, y1, ly0, ly1 = taps(a.shape[1], s)
    x0, x1, lx0, lx1 = taps(a.shape[2], s)
    extra = (1,) * (a.ndim - 3)
    ly0, ly1 = ly0.reshape((1, s, 1) + extra), ly1.reshape((1, s, 1) + extra)
    lx0, lx1 = lx0.reshape((1, 1, s) + extra), lx1.reshape((1, 1, s) + extra)
    r0, r1 = a[:, y0], a[:, y1]
    return ly0 * (lx0 * r0[:, :, x0] + lx1 * r0[:, :, x1]) + ly1 * (lx0 * r1[:, :, x0] + lx1 * r1[:, :, x1])


def eps_denom(u, eps=1e-17):
    """DSS/utils/mathHelper.py:10-14: sign(u) max(|u|, eps), zero counted as positive"""
    sign = np.where(u < 0, -1.0, 1.0)
    return sign * np.maximum(np.abs(u), eps)


def image_metrics(pred, gt_rgb, gt_mask):
    """pred (V, s, s, 4), gt_rgb (V, H, W, 3), gt_mask (V, H, W) -> (per_view (V, 5) rows (I, U, E, iou, psnr),
    mean iou, mean psnr), all float64"""
    p = np.asarray(pred, dtype=np.float64)
    s = p.shape[1]
    g = resize(gt_rgb, s)
    m = resize(np.asarray(gt_mask, dtype=np.float64), s)
    alpha = p[..., 3]
    inter = (m * alpha).sum((1, 2))
    union = (m + alpha - m * alpha).sum((1, 2))
    err = ((g - p[..., :3]) ** 2).sum((1, 2, 3))
    iou = 1.0 - inter / eps_denom(union)
    psnr = err / (s * s)
    per_view = np.stack([inter, union, err, iou, psnr], 1)
    return per_view, iou.mean(), psnr.mean()
