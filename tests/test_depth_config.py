"""CPU: the dense-depth configuration keys, the data's depth maps (MVRData(load_dense_depth=True)) and their refusals."""
import os

import numpy as np
import pytest
import torch

from dss_b200.training.config import DEFAULTS, check_depth, load_config, step_settings
from dss_b200.utils.dataset import MVRData
from dss_b200.utils.io import write_exr


def test_defaults_and_keys(tmp_path):
    assert DEFAULTS["data"]["load_dense_depth"] is False and DEFAULTS["data"]["depth_folder"] == "depth"
    assert DEFAULTS["data"]["depth_extension"] == "exr" and DEFAULTS["training"]["lambda_dr_depth"] == 0.0
    p = tmp_path / "c.yml"
    p.write_text("data: {load_dense_depth: true, depth_folder: dd, depth_extension: exr}\n"
                 "training: {lambda_dr_depth: 0.5}\n")
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("error")                          # every key is one the loop reads
        cfg = load_config(str(p))
    assert step_settings(cfg)["lambda_dr_depth"] == 0.5
    check_depth(cfg, True)


@pytest.mark.parametrize("lam,depth,has,msg", [
    (1.0, True, False, "needs dense depth maps"), (-1.0, False, False, "lambda_dr_depth must be"),
    (float("inf"), True, True, "lambda_dr_depth must be"), ("1", True, True, "lambda_dr_depth must be"),
    (0.0, "yes", False, "load_dense_depth must be")])
def test_refusals(lam, depth, has, msg):
    cfg = {"data": dict(DEFAULTS["data"], load_dense_depth=depth), "training": {"lambda_dr_depth": lam}}
    with pytest.raises(ValueError, match=msg):
        check_depth(cfg, has)


def _data_dir(tmp_path, V=3, H=6, depth_sizes=None, n_depth=None):
    d = tmp_path / "data"
    os.makedirs(d / "depth", exist_ok=True)
    np.savez(d / "data_dict.npz", camera_mat=np.tile(np.eye(4, dtype=np.float32), (V, 1, 1)))
    sizes = depth_sizes or [(H, H)] * (V if n_depth is None else n_depth)
    maps = []
    for i, s in enumerate(sizes):
        m = np.full(s, 1.0 + i, np.float32)
        write_exr(str(d / "depth" / ("%06d.exr" % i)), m)
        maps.append(m)
    (d / "depth" / "notes.txt").write_text("not a depth map")
    images = [torch.zeros(3, H, H) for _ in range(V)]
    masks = [torch.ones(1, H, H) for _ in range(V)]
    return str(d), images, masks, maps


def test_reads_the_depth_folder(tmp_path):
    d, images, masks, maps = _data_dir(tmp_path)
    data = MVRData(d, images=images, masks=masks, load_dense_depth=True)
    assert [os.path.basename(f) for f in data.depth_files] == ["%06d.exr" % i for i in range(3)]
    for i in range(3):
        assert data[i]["img.depth"].shape == (1, 6, 6) and np.array_equal(data[i]["img.depth"][0], maps[i])
    assert "img.depth" not in MVRData(d, images=images, masks=masks)[0]


def test_refuses_a_wrong_count_or_size(tmp_path):
    d, images, masks, _ = _data_dir(tmp_path, n_depth=2)
    with pytest.raises(ValueError, match="invalid number of dense depth maps"):
        MVRData(d, images=images, masks=masks, load_dense_depth=True)
    d, images, masks, _ = _data_dir(tmp_path / "b", depth_sizes=[(6, 6), (6, 5), (6, 6)])
    with pytest.raises(ValueError, match="depth map 1 has size"):
        MVRData(d, images=images, masks=masks, load_dense_depth=True)
    with pytest.raises(ValueError, match="does not exist"):
        MVRData(d, images=images, masks=masks, load_dense_depth=True, depth_folder="nope")
