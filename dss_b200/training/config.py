"""YAML configuration of the training loop: the reference's ``load_config`` rules (config.py:15-78) over a restated copy
of the ``configs/default.yaml`` values the loop reads, and the mapping from a configuration to the step's settings.

``load_config(path)`` reads ``path``; when it names ``inherit_from``, that file is loaded first (recursively) as its
base, otherwise the defaults below are; then the file's entries update the base recursively (a nested dict merges, any
other value replaces).  Keys the loop does not implement get one warning that lists them."""
import copy
import warnings

import yaml

__all__ = ["DEFAULTS", "load_config", "update_recursive", "check_config", "step_settings", "splat_params"]

# The configs/default.yaml values the loop reads, plus the reference Trainer's keyword defaults it passes on
# (trainer.py:73-80: n_eval_points, steps_dss_backward_radii) and what is this loop's own (seed, backup_every 0: off).
DEFAULTS = {
    "name": "demo",
    "data": {"type": "MVR", "data_dir": "example_data", "data_dict": "data_dict.npz", "img_folder": "image",
             "mask_folder": "mask", "img_extension": "png", "mask_extension": "png", "n_imgs": None,
             "resolution": [512, 512]},
    "renderer": {
        "is_neural_texture": False,
        "lighting": "from_data",
        "raster_params": {"backface_culling": False, "Vrk_invariant": False, "Vrk_isotropic": False,
                          "bin_size": None, "clip_pts_grad": 0.05, "cutoff_threshold": 0.5,
                          "depth_merging_threshold": 0.05, "image_size": 512, "max_points_per_bin": None,
                          "points_per_pixel": 5, "radii_backward_scaler": 5, "antialiasing_sigma": 1.0},
    },
    "model": {"type": "point",
              "model_kwargs": {"learn_points": True, "learn_normals": True, "learn_colors": False,
                               "n_points_per_cloud": 8000}},
    "training": {
        "out_dir": "exp", "seed": 0,
        "lambda_dr_rgb": 1.0, "lambda_dr_silhouette": 1.0, "lambda_dr_proj": 0.1, "lambda_dr_repel": 0.1,
        "batch_size": 1, "print_every": 10, "checkpoint_every": 500, "validate_every": 500, "backup_every": 0,
        "scheduler_milestones": [500, 800], "scheduler_gamma": 0.5, "logfile": "train.log",
        "resume_from": "model.pt", "model_selection_metric": "chamfer_point", "model_selection_mode": "minimize",
        "n_eval_points": 8000, "steps_dss_backward_radii": 100, "steps_proj": -1, "gamma_proj": 5,
    },
}

# Keys of the reference's configurations that change nothing in its point-model training with data lights (the
# renderer classes it instantiates are the ones this loop runs, `learning_rate` is overridden by the per-group rates,
# the data-loader and visualisation details have no counterpart here, and TrainerScheduler is given neither
# gamma_dss_backward_radii nor limit_dss_backward_radii, trainer.py:118-123): accepted without a warning.
_NO_EFFECT = {
    "type", "test",
    "data.img_extension_input", "data.depth_folder", "data.img_with_camera", "data.img_with_mask",
    "renderer.renderer_type", "renderer.raster_type", "renderer.compositor_type", "renderer.composite_params",
    "training.batch_size_val", "training.n_workers", "training.patch_size", "training.learning_rate",
    "training.overwrite_visualization", "training.n_debug_points", "training.point_file", "training.n_training_points",
    "training.gamma_dss_backward_radii", "training.limit_dss_backward_radii",
}


def update_recursive(dict1, dict2):
    """config.py:64-78: every entry of dict2 into dict1; nested dicts merge, other values replace."""
    for k, v in dict2.items():
        if isinstance(v, dict):
            if not isinstance(dict1.get(k), dict):
                dict1[k] = {}
            update_recursive(dict1[k], v)
        else:
            dict1[k] = v


def _read(path):
    with open(path, "r") as f:
        cfg = yaml.safe_load(f)
    return {} if cfg is None else cfg


def _load(path, default_path):
    special = _read(path)
    inherit_from = special.get("inherit_from")
    if inherit_from is not None:
        cfg = _load(inherit_from, default_path)
    elif default_path is not None:
        cfg = copy.deepcopy(DEFAULTS)
        update_recursive(cfg, _read(default_path))
    else:
        cfg = copy.deepcopy(DEFAULTS)
    update_recursive(cfg, special)
    return cfg


def _unknown(cfg, ref, prefix=""):
    out = []
    for k, v in cfg.items():
        name = prefix + str(k)
        if name in _NO_EFFECT or name == "inherit_from":
            continue
        if k not in ref:
            out.append(name)
        elif isinstance(v, dict) and isinstance(ref[k], dict):
            out += _unknown(v, ref[k], name + ".")
    return out


def load_config(path, default_path=None):
    """The configuration of ``path`` over its ``inherit_from`` chain, over ``default_path`` (a YAML file) or, without
    one, :data:`DEFAULTS`.  A plain nested dict.  Keys the loop does not read (``training.visualize_every``,
    ``training.debug_every``, the ``generation`` block, misspelt keys ...) are kept and named in one warning."""
    cfg = _load(path, default_path)
    unknown = _unknown(cfg, DEFAULTS)
    if unknown:
        warnings.warn("the training loop does not implement these configuration keys, they are ignored: %s"
                      % ", ".join(unknown), stacklevel=2)
    return cfg


def check_config(cfg, resolution, has_lights):
    """Refuse what the loop cannot train: a neural texture, lighting other than the data's, an image size other than
    the data's ``resolution`` (H, W), data without per-image lights."""
    r = cfg["renderer"]
    if r.get("is_neural_texture", False):
        raise NotImplementedError("renderer.is_neural_texture: true is not supported (NeuralTexture is out of scope); "
                                  "the loop shades with the data's lights")
    if r.get("lighting", "from_data") != "from_data":
        raise NotImplementedError("renderer.lighting must be 'from_data', got %r" % r.get("lighting"))
    S = int(r["raster_params"]["image_size"])
    if resolution is None or tuple(resolution) != (S, S):
        raise ValueError("renderer.raster_params.image_size %d does not match the data's image resolution %s"
                         % (S, None if resolution is None else tuple(resolution)))
    if not has_lights:
        raise ValueError("the data directory has no lights_%d entries: the loop shades with the data's lights")


SELECTION_METRICS = ("chamfer_point", "chamfer_normal", "p2f_avg")


def selection_metric(cfg):
    """``training.model_selection_metric`` if the loop can select by it: the chamfer distances of the reference's
    trainer, or ``p2f_avg``, the mean distance of the cloud's points to ``<data_dir>/mesh.obj``."""
    metric = cfg["training"]["model_selection_metric"]
    if metric not in SELECTION_METRICS:
        raise NotImplementedError("model_selection_metric %r: the loop selects by one of %s"
                                  % (metric, ", ".join(SELECTION_METRICS)))
    return metric


def splat_params(cfg, znear, zfar):
    """``SplatParams`` of ``renderer.raster_params`` (``bin_size`` / ``max_points_per_bin`` are accepted and ignored, as
    ``PointsRasterizationSettings`` ignores them) with the data cameras' depth range."""
    from ..core.rasterizer import PointsRasterizationSettings, _splat_params
    rp = cfg["renderer"]["raster_params"]
    rs = PointsRasterizationSettings(**{k: v for k, v in rp.items() if k in PointsRasterizationSettings.__slots__})
    return _splat_params(rs, None, {"znear": znear, "zfar": zfar})


def step_settings(cfg):
    """The ``TrainStep`` keyword settings of a configuration: the splat shape flags, the lambdas and what is learnt."""
    rp, tr, mk = cfg["renderer"]["raster_params"], cfg["training"], cfg["model"]["model_kwargs"]
    learn = tuple(name for name, key in (("points", "learn_points"), ("normals", "learn_normals"),
                                         ("colours", "learn_colors")) if mk.get(key, False))
    return {"Vrk_invariant": bool(rp["Vrk_invariant"]), "Vrk_isotropic": bool(rp["Vrk_isotropic"]),
            "lambda_dr_rgb": float(tr["lambda_dr_rgb"]), "lambda_dr_silhouette": float(tr["lambda_dr_silhouette"]),
            "lambda_dr_proj": float(tr["lambda_dr_proj"]), "lambda_dr_repel": float(tr["lambda_dr_repel"]),
            "learn": learn}
