"""GPU: the training loop (python -m dss_b200.training.train) end to end on a dataset generated from the torus of
tests/test_mesh_data.py: a run with validation and model selection, exact resume mid-epoch, the time-limit exit and the
scheduler reaching the step."""
import os
import subprocess
import sys

import pytest
import torch
import yaml

from dss_b200.ops import chamfer_distance
from dss_b200.utils.io import read_ply, save_obj
from tests.test_mesh_data import torus

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def data_dir(cuda_device, tmp_path_factory):
    from dss_b200.utils.create_mvr_data import main
    tmp = tmp_path_factory.mktemp("loop_data")
    verts, faces = torus()
    mesh = tmp / "torus.obj"
    save_obj(str(mesh), verts.numpy(), faces.numpy())
    return main(["--points", str(mesh), "--output", str(tmp / "data"), "--num_cameras", "16", "--image-size", "128",
                 "--tri_color_light", "--point_lights", "--seed", "3"])[0]


def write_config(path, data_dir, out_dir, **training):
    """configs/dss.yml at 128^2 with 2000 points and batch 4"""
    cfg = {"name": "torus", "data": {"data_dir": data_dir},
           "model": {"model_kwargs": {"n_points_per_cloud": 2000, "learn_colors": False, "learn_points": True,
                                      "learn_normals": True}},
           "renderer": {"is_neural_texture": False,
                        "raster_params": {"Vrk_invariant": True, "Vrk_isotropic": False, "clip_pts_grad": 0.05,
                                          "cutoff_threshold": 1.0, "depth_merging_threshold": 0.05, "image_size": 128,
                                          "points_per_pixel": 5, "radii_backward_scaler": 5}},
           "training": dict({"out_dir": str(out_dir), "batch_size": 4, "print_every": 10, "checkpoint_every": 400,
                             "validate_every": 100, "lambda_dr_proj": 0.01, "lambda_dr_repel": 0.0,
                             "steps_dss_backward_radii": 200, "scheduler_milestones": [500, 800]}, **training)}
    with open(path, "w") as f:
        yaml.safe_dump(cfg, f)
    return str(path)


def run_cli(config, *args):
    env = dict(os.environ)
    env["PYTHONPATH"] = ROOT + os.pathsep + env.get("PYTHONPATH", "")
    r = subprocess.run([sys.executable, "-m", "dss_b200.training.train", "--config", config, *args], cwd=ROOT, env=env,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1200)
    return r.returncode, r.stdout


def test_loop_trains_and_selects_a_model(data_dir, tmp_path):
    from dss_b200.training.train import ground_truth_cloud, initial_cloud
    from dss_b200.utils.dataset import MVRData
    cfg = write_config(tmp_path / "c.yml", data_dir, tmp_path / "out")
    code, log = run_cli(cfg, "--max-it", "300")
    assert code == 0, log
    out = tmp_path / "out" / "torus"
    with open(out / "metrics.jsonl") as f:
        lines = f.read().splitlines()
    assert len(lines) == 300 // 10
    assert (out / "config.yaml").exists() and (out / "train.log").exists() and (out / "model.pt").exists()
    best = torch.load(out / "model_best.pt", map_location="cpu", weights_only=False)
    ply = read_ply(str(out / "val" / "best.ply"))
    assert ply["points"].shape == (2000, 3) and ply["normals"].shape == (2000, 3)
    assert torch.equal(torch.from_numpy(ply["points"]), best["model"]["points"][0])
    # the initial cloud's chamfer distance to the same ground truth
    d = torch.device("cuda:0")
    gt = ground_truth_cloud(MVRData(data_dir), data_dir, 8000, d)
    p0, n0, _ = initial_cloud(2000, 0, d)
    init = float(chamfer_distance(gt[0][None], p0[None], x_normals=gt[1][None], y_normals=n0[None])[0])
    print("chamfer_point: initial %.5f, best %.5f (%.3fx) at it %d" % (init, best["loss_val_best"],
                                                                       best["loss_val_best"] / init, best["it"]))
    assert best["loss_val_best"] <= 0.5 * init


def test_resume_is_exact(data_dir, tmp_path):
    a = write_config(tmp_path / "a.yml", data_dir, tmp_path / "a")
    b = write_config(tmp_path / "b.yml", data_dir, tmp_path / "b")
    code, log = run_cli(a, "--max-it", "240")
    assert code == 0, log
    code, log = run_cli(b, "--max-it", "130")        # 16 views, batch 4: 4 iterations per epoch, 130 is mid-epoch
    assert code == 0, log
    mid = torch.load(tmp_path / "b" / "torus" / "model.pt", map_location="cpu", weights_only=False)
    assert mid["it"] == 129 and mid["epoch_pos"] % 16 != 0
    code, log = run_cli(b, "--max-it", "240")
    assert code == 0, log
    assert "resumed" in log
    ca = torch.load(tmp_path / "a" / "torus" / "model.pt", map_location="cpu", weights_only=False)
    cb = torch.load(tmp_path / "b" / "torus" / "model.pt", map_location="cpu", weights_only=False)
    assert ca["it"] == cb["it"] == 239 and ca["epoch_it"] == cb["epoch_it"]
    for k in ("points", "normals", "colors"):
        assert torch.equal(ca["model"][k], cb["model"][k]), k
    sa, sb = ca["optimizer"]["state"], cb["optimizer"]["state"]
    assert sa.keys() == sb.keys()
    for i in sa:
        for k in sa[i]:
            assert torch.equal(torch.as_tensor(sa[i][k]), torch.as_tensor(sb[i][k])), (i, k)
    assert ca["lr_scheduler"] == cb["lr_scheduler"] and ca["schedule"] == cb["schedule"]
    assert torch.equal(ca["sampler"], cb["sampler"]) and ca["epoch_order"] == cb["epoch_order"]


def test_exit_after_zero(data_dir, tmp_path):
    cfg = write_config(tmp_path / "c.yml", data_dir, tmp_path / "out")
    code, log = run_cli(cfg, "--exit-after", "0")
    assert code == 3, log
    ck = torch.load(tmp_path / "out" / "torus" / "model.pt", map_location="cpu", weights_only=False)
    assert ck["it"] == 0 and ck["model"]["points"].shape == (1, 2000, 3)
    assert ck["model"]["points_activation"].shape == (1, 2000) and bool(ck["model"]["points_activation"].all())


def test_schedule_reaches_the_step(data_dir, tmp_path):
    from dss_b200.training.config import load_config
    from dss_b200.training.train import Trainer
    cfg = load_config(write_config(tmp_path / "c.yml", data_dir, tmp_path / "out", steps_dss_backward_radii=50,
                                   validate_every=0))
    t = Trainer(cfg)
    assert t.run(exit_after=-1, max_it=121) == 0
    assert t.it == 120
    assert t.step.params.radii_backward_scaler == 5 * 0.99 ** 2
    assert t.step._captured[0] == tuple(t.step.params)       # the replay ran with it
