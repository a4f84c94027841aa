"""CPU tests of the device-resident training views: the conversion rule the gather kernel meets, the store's choice of
uint8 or float32, the host-side index check, and the new C symbol."""
from fractions import Fraction

import numpy as np
import pytest
import torch

from dss_b200 import _lib
from dss_b200.utils import dataset
from dss_b200.utils.dataset import MVRData


def test_numpy_float32_division_by_255_is_correctly_rounded():
    # the kernel computes __fdiv_rn(u, 255.f); load_all_images computes numpy's float32 u / 255.0
    got = np.arange(256, dtype=np.float32) / 255.0
    assert got.dtype == np.float32
    for k in range(256):
        exact = Fraction(k, 255)
        q = got[k]
        below, above = np.nextafter(q, np.float32(-1)), np.nextafter(q, np.float32(2))
        err = abs(Fraction(float(q)) - exact)
        assert err < abs(Fraction(float(below)) - exact) and err < abs(Fraction(float(above)) - exact), k


def _data_dict(tmp_path, V):
    cams = np.tile(np.eye(4, dtype=np.float32), (V, 1, 1))
    cams[:, 3, 2] = 2.5
    path = tmp_path / "data_dict.npz"
    np.savez(path, camera_mat=cams)
    return str(path)


def _views(tmp_path, V=3, H=5, W=7, seed=0):
    g = np.random.default_rng(seed)
    k = g.integers(0, 256, size=(V, 3, H, W)).astype(np.float32)
    images = [torch.from_numpy(k[i] / np.float32(255.0)) for i in range(V)]
    masks = [torch.from_numpy((g.random((1, H, W)) < 0.5).astype(np.float32)) for _ in range(V)]
    return _data_dict(tmp_path, V), images, masks


def test_8bit_views_get_a_uint8_store(tmp_path):
    path, images, masks = _views(tmp_path)
    views = MVRData(path, images=images, masks=masks).device_views("cpu")
    assert views.store.dtype == torch.uint8 and tuple(views.store.shape) == (3, 5, 7, 4)
    for i in range(3):
        k = views.store[i].numpy()
        np.testing.assert_array_equal((k[..., :3].astype(np.float32) / 255.0).transpose(2, 0, 1), images[i].numpy())
        np.testing.assert_array_equal(k[..., 3], masks[i][0].numpy())
    assert views.nbytes == 3 * 5 * 7 * 4 + 2 * 3 * 16 * 4
    assert views.light_cls is None and views.lights(torch.zeros(1, dtype=torch.int64)) is None


@pytest.mark.parametrize("change", ["one_ulp_up", "one_ulp_down", "fractional_mask", "mask_two", "negative_zero",
                                    "nan"])
def test_other_views_keep_their_float32_bits(tmp_path, change):
    path, images, masks = _views(tmp_path)
    img, m = images[1].numpy(), masks[2].numpy()
    if change == "one_ulp_up":
        img[0, 1, 2] = np.nextafter(img[0, 1, 2], np.float32(2))
    elif change == "one_ulp_down":
        img[2, 4, 6] = np.nextafter(np.float32(1.0), np.float32(0))
    elif change == "fractional_mask":
        m[0, 0, 3] = 0.25
    elif change == "mask_two":
        m[0, 2, 2] = 2.0
    elif change == "negative_zero":
        img[1, 0, 0] = -0.0
    else:
        img[1, 3, 3] = np.nan
    views = MVRData(path, images=images, masks=masks).device_views("cpu")
    assert views.store.dtype == torch.float32
    for i in range(3):
        s = views.store[i].numpy()
        assert np.array_equal(s[..., :3].transpose(2, 0, 1).view(np.uint32), images[i].numpy().view(np.uint32))
        assert np.array_equal(s[..., 3].view(np.uint32), masks[i][0].numpy().view(np.uint32))


def test_a_data_directory_gets_a_uint8_store(tmp_path):
    from PIL import Image
    V, H, W = 2, 6, 4
    g = np.random.default_rng(1)
    for d in ("image", "mask"):
        (tmp_path / d).mkdir()
    for i in range(V):
        Image.fromarray(g.integers(0, 256, size=(H, W, 3)).astype(np.uint8)).save(tmp_path / "image" / ("%d.png" % i))
        # any non-zero grey level is inside the mask
        Image.fromarray(g.integers(0, 3, size=(H, W)).astype(np.uint8) * 100).save(tmp_path / "mask" / ("%d.png" % i))
    _data_dict(tmp_path, V)
    data = MVRData(str(tmp_path))
    views = data.device_views("cpu")
    assert views.store.dtype == torch.uint8
    for i in range(V):
        rgb = np.asarray(Image.open(tmp_path / "image" / ("%d.png" % i)))
        np.testing.assert_array_equal(views.store[i, ..., :3].numpy(), rgb)
        np.testing.assert_array_equal(views.store[i, ..., 3].numpy(), data.masks[i][0].numpy())


def test_images_of_another_dtype_are_refused(tmp_path):
    path, images, masks = _views(tmp_path)
    images[0] = images[0].double()
    with pytest.raises(TypeError, match="float32"):
        MVRData(path, images=images, masks=masks).device_views("cpu")


def test_host_indices_are_checked_before_any_upload(tmp_path, monkeypatch):
    path, images, masks = _views(tmp_path, V=4)
    views = MVRData(path, images=images, masks=masks).device_views("cpu")
    assert views.check([0, 3, -1, -4, np.int64(2)]) == [0, 3, 3, 0, 2]
    made = []
    real = torch.tensor
    monkeypatch.setattr(dataset.torch, "tensor", lambda *a, **k: made.append(a) or real(*a, **k))
    for bad in ([0, 4], [-5], [1.5], [2, 100]):
        with pytest.raises(IndexError):
            views.batch(bad)
        with pytest.raises(IndexError):
            views.upload(bad)
    assert made == []
    idx = views.upload([3, 1, 3])
    assert idx.dtype == torch.int64 and idx.tolist() == [3, 1, 3] and len(made) == 1


def test_the_gather_symbol_is_exported():
    assert "dss_gather_views" in _lib.EXPORTED_SYMBOLS
    assert hasattr(_lib.load(), "dss_gather_views")
