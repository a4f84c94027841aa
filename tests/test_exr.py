"""CPU: the OpenEXR reader and writer of dss_b200.utils.io: round trips at every supported compression and pixel type,
the fixtures OpenCV's codec wrote (tests/golden/make_golden_exr.py), and the refusals."""
import os
import struct

import numpy as np
import pytest

from dss_b200.utils.io import read_exr, write_exr
from tests.golden.make_golden_exr import fixture_values

EXR_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "exr")


@pytest.mark.parametrize("compression", ["NONE", "RLE", "ZIPS", "ZIP"])
@pytest.mark.parametrize("pixel_type", ["FLOAT", "HALF"])
@pytest.mark.parametrize("shape", [(1, 1), (37, 23), (16, 5)])
def test_round_trip(tmp_path, compression, pixel_type, shape):
    rng = np.random.default_rng(0)
    a = (rng.random(shape) * 10).astype(np.float32)
    a[: shape[0] // 2, : shape[1] // 2] = 100.0                 # runs for RLE, a zfar-like background
    if a.size > 3:
        a.flat[:3] = [np.inf, -0.0, 1e-3]
    path = str(tmp_path / "d.exr")
    write_exr(path, a, compression, pixel_type)
    want = a if pixel_type == "FLOAT" else a.astype(np.float16).astype(np.float32)
    got = read_exr(path)
    assert got.dtype == np.float32 and got.shape == shape
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_default_is_float_zip_y(tmp_path):
    path = str(tmp_path / "d.exr")
    write_exr(path, fixture_values())
    blob = open(path, "rb").read()
    assert b"channels\0chlist\0" in blob and b"Y\0" + struct.pack("<i", 2) in blob
    i = blob.index(b"compression\0compression\0") + len(b"compression\0compression\0") + 4
    assert blob[i] == 3                                          # ZIP
    assert np.array_equal(read_exr(path), fixture_values())


@pytest.mark.parametrize("name", sorted(f for f in os.listdir(EXR_DIR) if not f.startswith("piz")))
def test_reads_opencv_fixtures(name):
    want = fixture_values()
    if "_half_" in name:
        want = want.astype(np.float16).astype(np.float32)
    assert np.array_equal(read_exr(os.path.join(EXR_DIR, name)), want)


def test_refuses_piz_naming_it():
    with pytest.raises(ValueError, match="PIZ compression is not read"):
        read_exr(os.path.join(EXR_DIR, "piz_float_1.exr"))


def test_refuses_other_files(tmp_path):
    p = tmp_path / "x.exr"
    p.write_bytes(b"\x89PNG\r\n\x1a\n" + b"\0" * 16)
    with pytest.raises(ValueError, match="not an OpenEXR file"):
        read_exr(str(p))
    blob = bytearray(open(os.path.join(EXR_DIR, "none_float_1.exr"), "rb").read())
    blob[4:8] = struct.pack("<i", 2 | 0x200)                     # tiled
    p.write_bytes(bytes(blob))
    with pytest.raises(ValueError, match="single-part scanline"):
        read_exr(str(p))
    with pytest.raises(ValueError, match="PIZ"):
        write_exr(str(p), np.zeros((2, 2)), "PIZ")
    with pytest.raises(ValueError):
        write_exr(str(p), np.zeros((2, 2, 3)))
