"""The float64 L0-smoothing oracle (tests/l0_oracle.py) against the reference's own L0Smooth
(tests/golden/ref_l0_smooth.npz, minted by tests/golden/make_golden_l0.py), and its properties; the host-side refusals of l0_smooth and of the image
filter command, which come before any device work."""
import numpy as np
import pytest

from tests import l0_oracle
from tests.golden.make_golden_l0 import load


@pytest.mark.parametrize("case", ["n2_40x48x3", "n1_64x64x1", "n1_60x60x3"])
def test_oracle_equals_reference(case):
    images, outputs = load()[case]
    for lmd, want in outputs.items():
        got, margins = l0_oracle.l0_smooth(images, lmd)
        assert got.shape == want.shape
        np.testing.assert_allclose(got, want, rtol=0, atol=1e-12, err_msg="lmd %g" % lmd)
        # the oracle's decisions are far from their thresholds, so the device's rounding cannot flip them
        assert margins.min() >= 1e-8


@pytest.mark.parametrize("H,W", [(40, 48), (48, 40), (64, 64), (60, 60), (2, 2048), (7, 9), (30, 50)])
def test_closed_form_denominator_equals_kernel_spectrum(H, W):
    # the reference's construction: difference kernels placed at the image centre, |fft2|^2 of each
    dx = np.zeros((H, W))
    dy = np.zeros((H, W))
    dx[H // 2, W // 2 - 1:W // 2 + 1] = [-1, 1]
    dy[H // 2 - 1:H // 2 + 1, W // 2] = [-1, 1]
    want = np.abs(np.fft.fft2(dx)) ** 2 + np.abs(np.fft.fft2(dy)) ** 2
    np.testing.assert_allclose(l0_oracle.denominator(H, W), want, rtol=0, atol=1e-12)


def test_twenty_rounds_at_the_default_schedule():
    b = l0_oracle.betas()
    assert len(b) == 20
    assert b[0] == 0.1 and b[-1] == 0.1 * 2 ** 19 and b[-1] * 2 > 1e5


def test_zero_lambda_returns_the_input():
    rng = np.random.default_rng(5)
    images = rng.random((2, 30, 50, 3))
    got, _ = l0_oracle.l0_smooth(images, 0.0)
    np.testing.assert_allclose(got, images, rtol=0, atol=1e-12)


def test_two_colour_square_keeps_its_step_edge():
    img = np.full((40, 40, 3), 0.2)
    img[10:30, 10:30] = (0.9, 0.6, 0.1)
    rng = np.random.default_rng(6)
    noisy = img + 0.02 * rng.standard_normal(img.shape)
    got, _ = l0_oracle.l0_smooth(noisy[None], 0.05)
    got = got[0]
    # the noise is gone: both regions are flat and at their colours ...
    assert np.abs(got[12:28, 12:28] - img[20, 20]).max() < 0.01
    assert np.abs(got[:8] - img[0, 0]).max() < 0.01
    # ... and the step keeps its full height across a single pixel, not spread over a ramp
    step = got[20, 10] - got[20, 9]
    np.testing.assert_allclose(step, img[20, 10] - img[20, 9], atol=0.02)
    np.testing.assert_allclose(got[20, 9] - got[20, 8], 0.0, atol=0.005)


@pytest.mark.parametrize("n,nearest", [(49, 48), (4096, 2048), (1, 2), (7, 6), (2049, 2048)])
def test_size_refusal_names_the_nearest_size(n, nearest):
    from dss_b200.ops import l0_size_error
    msg = l0_size_error(n)
    assert msg is not None and str(n) in msg and "nearest: %d" % nearest in msg


@pytest.mark.parametrize("n", [2, 40, 48, 64, 256, 384, 512, 1000, 1024, 2048])
def test_accepted_sizes(n):
    from dss_b200.ops import l0_size_error
    assert l0_size_error(n) is None


def _ply(tmp_path, normals=True):
    from dss_b200.utils.io import save_ply
    rng = np.random.default_rng(0)
    pts = rng.standard_normal((50, 3)).astype(np.float32)
    path = str(tmp_path / "in.ply")
    save_ply(path, pts, normals=pts / np.linalg.norm(pts, axis=1, keepdims=True) if normals else None)
    return path


@pytest.mark.parametrize("kw,match", [({"views": 10, "batch": 4}, "multiple"), ({"image_size": 49}, "nearest: 48"),
                                      ({"image_size": 4096}, "nearest: 2048")])
def test_image_filter_refuses_before_rendering(tmp_path, kw, match):
    from dss_b200.utils.image_filter import filter_cloud
    with pytest.raises(ValueError, match=match):
        filter_cloud(_ply(tmp_path), str(tmp_path / "out.ply"), **kw)
    assert not (tmp_path / "out.ply").exists()


def test_image_filter_needs_normals(tmp_path):
    from dss_b200.utils.image_filter import filter_cloud
    with pytest.raises(ValueError, match="dss_b200.utils.normals"):
        filter_cloud(_ply(tmp_path, normals=False), str(tmp_path / "out.ply"))
