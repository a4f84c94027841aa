"""CPU: the training loop's configuration (load_config over the restated defaults, the mapping to the step), its
schedules against the reference's formulas written out here, its initial cloud's icosphere, and the cosine rule the
chamfer kernel restates."""
import bisect
import copy
import warnings

import pytest
import torch
import torch.nn.functional as F

from dss_b200.training.config import DEFAULTS, check_config, load_config, splat_params, step_settings
from dss_b200.training.train import compound_lambda_proj, make_lr_scheduler, make_optimizer, radii_backward_scaler
from dss_b200.utils.create_mvr_data import ico_sphere


def write(path, text):
    path.write_text(text)
    return str(path)


# ---- load_config ------------------------------------------------------------------------------------------------------

def test_inherit_chain_and_recursive_override(tmp_path):
    base = write(tmp_path / "base.yml", "name: base\ntraining:\n  batch_size: 4\n  print_every: 7\n"
                                        "renderer:\n  raster_params:\n    image_size: 128\n    points_per_pixel: 8\n")
    child = write(tmp_path / "child.yml", "inherit_from: %s\nname: child\ntraining:\n  batch_size: 2\n"
                                          "renderer:\n  raster_params:\n    points_per_pixel: 3\n" % base)
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        cfg = load_config(child)
    assert cfg["name"] == "child"
    assert cfg["training"]["batch_size"] == 2 and cfg["training"]["print_every"] == 7     # child over base
    rp = cfg["renderer"]["raster_params"]
    assert rp["image_size"] == 128 and rp["points_per_pixel"] == 3                          # merged, not replaced
    assert rp["cutoff_threshold"] == DEFAULTS["renderer"]["raster_params"]["cutoff_threshold"]   # defaults below


def test_defaults_for_absent_keys(tmp_path):
    cfg = load_config(write(tmp_path / "empty.yml", "name: x\n"))
    # configs/default.yaml values, and the Trainer's keyword defaults
    assert cfg["training"]["scheduler_milestones"] == [500, 800] and cfg["training"]["scheduler_gamma"] == 0.5
    assert cfg["training"]["lambda_dr_proj"] == 0.1 and cfg["training"]["lambda_dr_repel"] == 0.1
    assert cfg["training"]["model_selection_metric"] == "chamfer_point"
    assert cfg["training"]["model_selection_mode"] == "minimize"
    assert cfg["training"]["resume_from"] == "model.pt" and cfg["training"]["validate_every"] == 500
    assert cfg["training"]["n_eval_points"] == 8000 and cfg["training"]["steps_dss_backward_radii"] == 100
    assert cfg["model"]["model_kwargs"]["n_points_per_cloud"] == 8000
    assert cfg["renderer"]["raster_params"]["Vrk_isotropic"] is False
    assert cfg["renderer"]["raster_params"]["radii_backward_scaler"] == 5
    # the defaults are not shared between calls
    cfg["training"]["batch_size"] = 99
    assert load_config(write(tmp_path / "e2.yml", "name: y\n"))["training"]["batch_size"] == 1


def test_unknown_keys_warn_once(tmp_path):
    path = write(tmp_path / "c.yml", "training:\n  visualize_every: 100\n  debug_every: 100\n  batch_sise: 3\n"
                                     "  learning_rate: 0.1\ngeneration:\n  resolution: 64\n"
                                     "renderer:\n  raster_params:\n    bin_size: 0\n    max_points_per_bin: 100\n")
    with pytest.warns(UserWarning) as rec:
        load_config(path)
    assert len(rec) == 1
    msg = str(rec[0].message)
    for key in ("training.visualize_every", "training.debug_every", "training.batch_sise", "generation"):
        assert key in msg
    for key in ("learning_rate", "bin_size", "max_points_per_bin"):     # accepted: no effect in the reference either
        assert key not in msg


def test_dss_yml_settings(tmp_path):
    # configs/dss.yml's training-relevant entries
    path = write(tmp_path / "dss.yml", """
name: dss_proj
model:
  model_kwargs: {n_points_per_cloud: 5000, learn_colors: false, learn_points: true, learn_normals: true}
renderer:
  is_neural_texture: false
  raster_params: {Vrk_invariant: true, Vrk_isotropic: false, clip_pts_grad: 0.05, cutoff_threshold: 1.0,
                  depth_merging_threshold: 0.05, image_size: 512, points_per_pixel: 5, radii_backward_scaler: 5}
training: {batch_size: 8, lambda_dr_proj: 0.01, lambda_dr_repel: 0.0, steps_dss_backward_radii: 200,
           gamma_dss_backward_radii: 0.9, limit_dss_backward_radii: 2}
""")
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        cfg = load_config(path)
    prm = splat_params(cfg, znear=0.1, zfar=100.0)
    assert (prm.image_size, prm.points_per_pixel, prm.cutoff_threshold, prm.radii_backward_scaler) == (512, 5, 1.0, 5.0)
    assert (prm.clip_pts_grad, prm.backface_culling, prm.znear, prm.zfar) == (0.05, False, pytest.approx(0.1), 100.0)
    s = step_settings(cfg)
    assert s["Vrk_invariant"] is True and s["Vrk_isotropic"] is False
    assert s["lambda_dr_proj"] == 0.01 and s["lambda_dr_repel"] == 0.0 and s["learn"] == ("points", "normals")


def test_refusals(tmp_path):
    cfg = load_config(write(tmp_path / "n.yml", "renderer:\n  is_neural_texture: true\n"))
    with pytest.raises(NotImplementedError, match="NeuralTexture"):
        check_config(cfg, (512, 512), True)
    cfg = load_config(write(tmp_path / "ok.yml", "name: ok\n"))
    check_config(cfg, (512, 512), True)
    with pytest.raises(ValueError, match="image_size"):
        check_config(cfg, (128, 128), True)
    with pytest.raises(ValueError, match="lights"):
        check_config(cfg, (512, 512), False)


# ---- schedules -------------------------------------------------------------------------------------------------------

def reference_radii(init, steps, it):
    # TrainerScheduler(init, steps, limit_dss_backward_radii=1.0), gamma_dss_backward_radii left at 0.99
    gamma = 0.99 ** (it // steps)
    return max(init * gamma, 1.0)


@pytest.mark.parametrize("it", [0, 99, 100, 1000, 100 * 200])
def test_radii_backward_scaler(it):
    assert radii_backward_scaler(5.0, 100, it) == reference_radii(5.0, 100, it)
    assert radii_backward_scaler(5.0, 100, 0) == 5.0 and radii_backward_scaler(5.0, 100, 99) == 5.0
    assert radii_backward_scaler(5.0, 100, 100) == 5.0 * 0.99
    assert radii_backward_scaler(5.0, 100, 100 * 200) == 1.0           # 5 * 0.99^200 < 1: the limit
    assert radii_backward_scaler(5.0, -1, it) == 5.0                    # off


def test_compounding_lambda_proj():
    class T:
        lambda_dr_proj = 0.01
    t, lam = T(), 0.01
    for it in range(60):
        # scheduler.py:50-53 with steps_proj 10, gamma_proj 5, limit 1.0
        i = it // 10
        t.lambda_dr_proj = min(t.lambda_dr_proj * 5 ** i, 1.0)
        lam = compound_lambda_proj(lam, 10, 5, it)
        assert lam == t.lambda_dr_proj
    assert compound_lambda_proj(0.25, 10, 5, 25) == 1.0
    assert compound_lambda_proj(0.01, 10, 5, 9) == 0.01 and compound_lambda_proj(0.01, -1, 5, 99) == 0.01


def test_multistep_lr_per_epoch():
    cfg = copy.deepcopy(DEFAULTS)
    cfg["training"]["scheduler_milestones"], cfg["training"]["scheduler_gamma"] = [3, 5], 0.5
    t = {k: torch.zeros(4, 3, requires_grad=k != "colours") for k in ("points", "normals", "colours")}
    opt = make_optimizer(t)
    assert [g["lr"] for g in opt.param_groups] == [0.01, 0.01]
    assert all(g["betas"] == (0.5, 0.9) for g in opt.param_groups)
    assert opt.param_groups[0]["params"][0] is t["normals"] and opt.param_groups[1]["params"][0] is t["points"]
    sched = make_lr_scheduler(opt, cfg)
    for epoch in range(8):
        want = 0.01 * 0.5 ** bisect.bisect_right([3, 5], epoch)
        assert opt.param_groups[0]["lr"] == pytest.approx(want, rel=1e-15)
        opt.step()
        sched.step()
    t["colours"].requires_grad_(True)
    assert [g["lr"] for g in make_optimizer(t).param_groups] == [0.01, 0.01, 1.0]


# ---- initial cloud: the icosphere --------------------------------------------------------------------------------------

@pytest.mark.parametrize("level", [0, 1, 4])
def test_ico_sphere(level):
    verts, faces = ico_sphere(level)
    V, Fc = 10 * 4 ** level + 2, 20 * 4 ** level
    assert verts.shape == (V, 3) and faces.shape == (Fc, 3) and verts.dtype == torch.float32
    assert (verts.double().norm(dim=1) - 1).abs().max() < 1e-6
    edges = {tuple(sorted(e)) for f in faces.tolist() for e in ((f[0], f[1]), (f[1], f[2]), (f[2], f[0]))}
    assert V - len(edges) + Fc == 2
    v = verts.double()
    n = torch.cross(v[faces[:, 1]] - v[faces[:, 0]], v[faces[:, 2]] - v[faces[:, 0]], dim=1)
    assert ((n * v[faces].mean(1)).sum(1) > 0).all()                     # counter-clockwise seen from outside
    assert len(set(map(tuple, faces.sort(1).values.tolist()))) == Fc      # no face twice
    if level == 4:
        assert (V, Fc) == (2562, 5120)


# ---- the chamfer kernel's cosine: torch's cosine_similarity(eps=1e-6) ---------------------------------------------------

def test_cosine_rule_is_torch():
    g = torch.Generator().manual_seed(0)
    a = torch.randn(2000, 3, generator=g, dtype=torch.float64)
    b = torch.randn(2000, 3, generator=g, dtype=torch.float64)
    a[:5] *= 1e-9                                                         # below eps: clamped norms
    b[5:10] = 0.0
    na = a.norm(dim=1, keepdim=True).clamp_min(1e-6)
    nb = b.norm(dim=1, keepdim=True).clamp_min(1e-6)
    rule = ((a / na) * (b / nb)).sum(1)
    assert torch.allclose(rule, F.cosine_similarity(a, b, dim=1, eps=1e-6), rtol=0, atol=1e-15)
