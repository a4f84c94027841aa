"""Float64 restatement of the dense depth of the splat blend and of the depth loss (csrc/depth.cu).

  D[pix]          = sum_k w_k z_k over the pixel's K-list up to its first empty slot; 0 for an empty list
  dL/dz[s]        = sum over the (pixel, k) slots holding record s of g_D[pix] w_k   (the weights held constant)
  loss            = lam sum_valid |D - D_gt| / M, valid = mask != 0 & alpha != 0 & D_gt finite & znear < D_gt < zfar
  dL/dD           = lam g sign(D - D_gt) / M on valid pixels, 0 elsewhere (sign(0) = 0); loss = 0 and no gradient
                    when M = 0
"""
import numpy as np


def _live(idx):
    """slots up to the first empty one of each list"""
    return np.cumprod(np.asarray(idx) >= 0, axis=-1).astype(bool)


def depth_map(idx, weights, z):
    """D (...,) from idx / weights (..., K) and the records' view depth z (P,)"""
    idx, w = np.asarray(idx), np.asarray(weights, np.float64)
    live = _live(idx)
    zk = np.where(live, np.asarray(z, np.float64)[np.where(live, idx, 0)], 0.0)
    return (np.where(live, w, 0.0) * zk).sum(-1)


def depth_record_grad(idx, weights, grad_depth, P):
    """dL/dz (P,) of the records"""
    idx, w = np.asarray(idx), np.asarray(weights, np.float64)
    live = _live(idx)
    terms = np.asarray(grad_depth, np.float64)[..., None] * w
    out = np.zeros(P)
    np.add.at(out, idx[live], terms[live])
    return out


def valid_pixels(alpha, depth_gt, mask, znear, zfar):
    gt = np.asarray(depth_gt, np.float64)
    with np.errstate(invalid="ignore"):
        return (np.asarray(mask) != 0) & (np.asarray(alpha) != 0) & np.isfinite(gt) & (gt > znear) & (gt < zfar)


def depth_loss(depth, alpha, depth_gt, mask, lam, znear, zfar):
    v = valid_pixels(alpha, depth_gt, mask, znear, zfar)
    M = int(v.sum())
    if M == 0:
        return 0.0
    return lam * float(np.abs(np.asarray(depth, np.float64)[v] - np.asarray(depth_gt, np.float64)[v]).sum()) / M


def depth_loss_grad(depth, alpha, depth_gt, mask, lam, znear, zfar, g=1.0):
    v = valid_pixels(alpha, depth_gt, mask, znear, zfar)
    M = int(v.sum())
    out = np.zeros(np.shape(depth))
    if M:
        d = np.asarray(depth, np.float64) - np.asarray(depth_gt, np.float64)
        out[v] = lam * g * np.sign(d[v]) / M
    return out
