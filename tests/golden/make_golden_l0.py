"""Mint the L0-smoothing golden vectors from the REFERENCE's own ``L0Smooth`` (DSS/misc/imageFilters.py:133-180),
imported from where the reference lies, never copied.  Run in the build container:

    python -m tests.golden.make_golden_l0

The inputs are seeded float64 numpy images, so that the reference runs in float64 end to end (scipy.fftpack keeps a
float32 input in single precision).  ``skimage``, which the module imports at its top and ``L0Smooth`` does not use,
is stubbed as tests/shim stubs the reference's other third-party imports.  Writes tests/golden/ref_l0_smooth.npz
(``ref_``: the reference's outputs, which the rasterizer's golden-file tests skip), packed to stay small (``load``
unpacks it): ``<case>_in`` (N, H, W, C) uint16 codes of the inputs, which are multiples of
2^-12 and so stored exactly, and ``<case>_lmd<lmd>`` the reference's output for each lmd as multiples of 2^-40
(rounded: within 4.6e-13 of the reference's float64 values, which lie in [0, 1)), stored as 5 planes of bytes,
least significant first.  The low planes are noise that no compressor shrinks: about 5 bytes a value is what 1e-12
costs."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get("DSS_REFERENCE", "/root/reference")
sys.path.insert(0, ROOT)

# (name, N, H, W, C, seed)
CASES = (("n2_40x48x3", 2, 40, 48, 3, 1), ("n1_64x64x1", 1, 64, 64, 1, 2), ("n1_60x60x3", 1, 60, 60, 3, 3))
LMDS = (0.01, 0.05, 0.2)


def case_images(N, H, W, C, seed):
    """piecewise-constant blocks plus a smooth ramp and small noise, in [0, 0.75] (so that the filter's overshoot stays
    below 1): edges for the filter to keep and texture for it to flatten"""
    rng = np.random.default_rng(seed)
    y, x = np.meshgrid(np.arange(H) / H, np.arange(W) / W, indexing="ij")
    out = np.empty((N, H, W, C))
    for n in range(N):
        blocks = rng.random((4, 4, C))[np.minimum((y * 4).astype(int), 3), np.minimum((x * 4).astype(int), 3)]
        ramp = (0.2 * (x + y))[..., None]
        out[n] = 0.75 * np.clip(0.7 * blocks + ramp + 0.03 * rng.standard_normal((H, W, C)), 0.0, 1.0)
    return np.round(out * IN_SCALE) / IN_SCALE


IN_SCALE, OUT_SCALE = 2.0 ** 12, 2.0 ** 40


def load(path=None):
    """{case: (images (N, H, W, C) float64, {lmd: the reference's output (N, H, W, C) float64})}"""
    d = np.load(path or os.path.join(HERE, "ref_l0_smooth.npz"))
    out = {}
    for name, *_ in CASES:
        planes = {lmd: d["%s_lmd%g" % (name, lmd)].astype(np.int64) for lmd in LMDS}
        codes = {lmd: sum(p[b] << (8 * b) for b in range(5)) for lmd, p in planes.items()}
        out[name] = (d[name + "_in"] / IN_SCALE, {lmd: c / OUT_SCALE for lmd, c in codes.items()})
    return out


def main():
    from tests import shim
    shim.install()
    sys.path.insert(0, REF)
    from DSS.misc.imageFilters import L0Smooth
    data = {}
    for name, N, H, W, C, seed in CASES:
        images = case_images(N, H, W, C, seed)
        data[name + "_in"] = np.round(images * IN_SCALE).astype(np.uint16)
        for lmd in LMDS:
            code = np.round(np.stack(L0Smooth(list(images), lmd)) * OUT_SCALE).astype(np.int64)
            assert code.min() >= 0 and code.max() < 2 ** 40
            data["%s_lmd%g" % (name, lmd)] = np.stack([(code >> (8 * b)) & 255 for b in range(5)]).astype(np.uint8)
    path = os.path.join(HERE, "ref_l0_smooth.npz")
    np.savez_compressed(path, **data)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
