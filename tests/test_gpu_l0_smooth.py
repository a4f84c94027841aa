"""dss_l0_smooth on the device (csrc/l0_smooth.cu) against the float64 oracle (tests/l0_oracle.py): parity on the
reference's golden cases and on rectangular sizes, a full-size batch of renders, the identity at lmd = 0, the refusals,
and bit-identical results, also from a CUDA graph replay."""
import os

import numpy as np
import pytest
import torch

from tests import l0_oracle
from tests.golden.make_golden_l0 import load

pytestmark = pytest.mark.gpu


def _parity(images, lmd, dev):
    want, margins = l0_oracle.l0_smooth(images, lmd)
    assert margins.min() >= 1e-8, "fixture too close to a threshold: change its seed"
    from dss_b200.ops import l0_smooth
    got = l0_smooth(torch.from_numpy(images).to(dev), lmd)
    assert got.dtype == torch.float64 and tuple(got.shape) == images.shape
    np.testing.assert_allclose(got.cpu().numpy(), want, rtol=0, atol=1e-10)


@pytest.mark.parametrize("case", ["n2_40x48x3", "n1_64x64x1", "n1_60x60x3"])
def test_golden_cases(cuda_device, case):
    images, outputs = load()[case]
    for lmd in outputs:
        _parity(images, lmd, cuda_device)


@pytest.mark.parametrize("N,H,W,C,seed", [(1, 40, 48, 3, 11), (3, 48, 40, 3, 12), (1, 30, 50, 1, 13),
                                          (3, 30, 50, 3, 14), (1, 2, 2048, 3, 15), (1, 2, 2048, 1, 16)])
def test_rectangular_sizes(cuda_device, N, H, W, C, seed):
    from tests.golden.make_golden_l0 import case_images
    _parity(case_images(N, H, W, C, seed), 0.05, cuda_device)


def test_strided_float64_input(cuda_device):
    from dss_b200.ops import l0_smooth
    from tests.golden.make_golden_l0 import case_images
    images = case_images(2, 40, 48, 3, 21)
    want, margins = l0_oracle.l0_smooth(images, 0.05)
    assert margins.min() >= 1e-8
    # (N, C, H, W) storage seen as (N, H, W, C)
    planar = torch.from_numpy(np.ascontiguousarray(images.transpose(0, 3, 1, 2))).to(cuda_device)
    got = l0_smooth(planar.permute(0, 2, 3, 1), 0.05)
    np.testing.assert_allclose(got.cpu().numpy(), want, rtol=0, atol=1e-10)


def test_full_size_renders(cuda_device):
    from dss_b200.ops import SplatParams, l0_smooth, make_shading, render_points, shared_cloud_splats
    from dss_b200.core.lighting import DirectionalLights
    from dss_b200.core.camera import camera_matrices
    from dss_b200.utils.io import read_ply
    from tests.util import GOLDEN_DIR, random_cameras
    d = read_ply(os.path.join(GOLDEN_DIR, "ply", "bunny-8000.ply"))
    pts = torch.from_numpy(d["points"])
    pts = (pts - pts.mean(0)) / (pts - pts.mean(0)).norm(dim=1).max()
    pts, nrm = pts.to(cuda_device), torch.from_numpy(d["normals"]).to(cuda_device)
    N, S = 8, 512
    proj, view = (m.to(cuda_device) for m in camera_matrices(random_cameras(N, seed=3)))
    lights = DirectionalLights(ambient_color=((0.6, 0.6, 0.6),), diffuse_color=((0.4, 0.4, 0.4),),
                               specular_color=((0.0, 0.0, 0.0),), direction=((0.3, 1.0, 0.5),)).to(cuda_device)
    h, frames = shared_cloud_splats(pts, N, True, False)
    prm = SplatParams(image_size=S, points_per_pixel=5, cutoff_threshold=1.0, clip_pts_grad=0.05, znear=0.1)
    with torch.no_grad():
        rgb = render_points(pts, torch.nn.functional.normalize(nrm, dim=-1), torch.ones_like(pts), proj, view, h, prm,
                            shading=make_shading(lights, view), deterministic=True, frames=frames).image[..., :3]
    rgb = rgb.contiguous()
    got = l0_smooth(rgb, 0.05)
    assert got.dtype == torch.float32
    want, _ = l0_oracle.l0_smooth(rgb.cpu().numpy().astype(np.float64), 0.05)
    assert float(rgb.std()) > 0.05
    np.testing.assert_allclose(got.cpu().numpy(), want, rtol=0, atol=1e-6)


def test_zero_lambda_is_the_identity(cuda_device):
    from dss_b200.ops import l0_smooth
    rng = np.random.default_rng(4)
    images = rng.random((2, 48, 40, 3))
    got = l0_smooth(torch.from_numpy(images).to(cuda_device), 0.0)
    np.testing.assert_allclose(got.cpu().numpy(), images, rtol=0, atol=1e-12)


@pytest.mark.parametrize("shape,dtype,where,exc", [
    ((1, 49, 48, 3), torch.float32, "cuda", ValueError),
    ((1, 2, 4096, 3), torch.float32, "cuda", ValueError),
    ((1, 40, 48, 2), torch.float32, "cuda", ValueError),
    ((1, 40, 48, 3), torch.int32, "cuda", TypeError),
    ((40, 48, 3), torch.float32, "cuda", ValueError),
    ((1, 40, 48, 3), torch.float32, "cpu", RuntimeError),
])
def test_refusals(cuda_device, shape, dtype, where, exc):
    from dss_b200 import _lib
    from dss_b200.ops import l0_smooth
    x = torch.zeros(shape, dtype=dtype, device=cuda_device if where == "cuda" else "cpu")
    _lib.ctx(cuda_device)
    before = _lib.launch_count(cuda_device)
    with pytest.raises(exc):
        l0_smooth(x)
    assert _lib.launch_count(cuda_device) == before


def test_deterministic_and_graph_capturable(cuda_device):
    from dss_b200.ops import l0_smooth
    from tests.golden.make_golden_l0 import case_images
    x = torch.from_numpy(case_images(3, 60, 64, 3, 31)).float().to(cuda_device)
    a, b = l0_smooth(x, 0.05), l0_smooth(x, 0.05)
    assert torch.equal(a, b)
    s = torch.cuda.Stream(cuda_device)
    s.wait_stream(torch.cuda.current_stream(cuda_device))
    with torch.cuda.stream(s):
        l0_smooth(x, 0.05)      # warm-up on the capture stream
    torch.cuda.current_stream(cuda_device).wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        c = l0_smooth(x, 0.05)
    g.replay()
    torch.cuda.synchronize(cuda_device)
    assert torch.equal(a, c)
