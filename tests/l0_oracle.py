"""Float64 numpy restatement of L0 gradient-minimisation smoothing (Xu et al. 2011, as the reference's ``L0Smooth``
runs it, DSS/misc/imageFilters.py:133-180), the oracle of ``dss_b200.ops.l0_smooth``.

Per image I (H, W, C), S = I, beta = 0.1; every round:
  hp, vp = periodic forward differences of S along x and y;
  (hp, vp) = 0 where sum_c(hp^2 + vp^2) < lmd / beta;
  hv = periodic adjoint difference of (hp, vp);
  S = real(ifft2(fft2(I + beta hv) / (1 + beta D))), D = (2 - 2 cos 2 pi u / W) + (2 - 2 cos 2 pi v / H);
  beta *= 2, and the loop ends once beta > 1e5 (at most 40 rounds: 20 at the default schedule).
"""
import numpy as np

BETA0, BETA_MAX, BETA_RATE, MAX_ROUNDS = 0.1, 1e5, 2.0, 40


def denominator(H, W):
    """D (H, W): |fft2 of the forward difference along x|^2 + the same along y, in closed form"""
    u, v = np.arange(W), np.arange(H)
    return (2.0 - 2.0 * np.cos(2.0 * np.pi * u / W))[None, :] + (2.0 - 2.0 * np.cos(2.0 * np.pi * v / H))[:, None]


def betas():
    """the beta of every round"""
    out, beta = [], BETA0
    for _ in range(MAX_ROUNDS):
        out.append(beta)
        beta *= BETA_RATE
        if beta > BETA_MAX:
            break
    return out


def l0_smooth_image(I, lmd=0.05):
    """One image (H, W, C) -> (S (H, W, C) float64, margins): margins[r] is round r's smallest relative distance of a
    pixel's sum_c(hp^2 + vp^2) from the threshold lmd / beta (inf when lmd = 0), i.e. how far the round's shrink
    decisions are from flipping."""
    I = np.asarray(I, dtype=np.float64)
    H, W = I.shape[:2]
    D = denominator(H, W)[..., None]
    S = I
    margins = []
    for beta in betas():
        hp = np.roll(S, -1, axis=1) - S
        vp = np.roll(S, -1, axis=0) - S
        energy = np.sum(hp * hp + vp * vp, axis=2)
        thr = lmd / beta
        margins.append(float(np.min(np.abs(energy - thr)) / thr) if thr > 0 else np.inf)
        zero = energy < thr
        hp[zero] = 0.0
        vp[zero] = 0.0
        hv = (np.roll(hp, 1, axis=1) - hp) + (np.roll(vp, 1, axis=0) - vp)
        S = np.real(np.fft.ifft2(np.fft.fft2(I + beta * hv, axes=(0, 1)) / (1.0 + beta * D), axes=(0, 1)))
    return S, margins


def l0_smooth(images, lmd=0.05):
    """(N, H, W, C) -> (S (N, H, W, C) float64, the smallest margin of every image over all its rounds (N,))"""
    out, margins = [], []
    for I in np.asarray(images, dtype=np.float64):
        S, m = l0_smooth_image(I, lmd)
        out.append(S)
        margins.append(min(m))
    return np.stack(out), np.asarray(margins)
