"""YAML configuration of the training loop: the reference's ``load_config`` rules (config.py:15-78) over a restated copy
of the ``configs/default.yaml`` values the loop reads, and the mapping from a configuration to the step's settings.

``load_config(path)`` reads ``path``; when it names ``inherit_from``, that file is loaded first (recursively) as its
base, otherwise the defaults below are; then the file's entries update the base recursively (a nested dict merges, any
other value replaces).  Keys the loop does not implement get one warning that lists them."""
import copy
import warnings

import yaml

__all__ = ["DEFAULTS", "load_config", "update_recursive", "check_config", "check_growth", "check_pruning", "check_cameras", "check_depth",
           "cloud_size", "check_cloud_size", "GROW_K", "step_settings", "splat_params", "EVAL_SAMPLINGS", "SELECTION_METRICS",
           "IMAGE_METRICS", "selection_metric"]

EVAL_SAMPLINGS = ("uniform", "poisson_disk")

# The configs/default.yaml values the loop reads, plus the reference Trainer's keyword defaults it passes on
# (trainer.py:73-80: n_eval_points, steps_dss_backward_radii) and what is this loop's own (seed, backup_every 0: off,
# eval_sampling: how the validation's ground truth is drawn from the data's mesh, see train.ground_truth_cloud).
DEFAULTS = {
    "name": "demo",
    "data": {"type": "MVR", "data_dir": "example_data", "data_dict": "data_dict.npz", "img_folder": "image",
             "mask_folder": "mask", "img_extension": "png", "mask_extension": "png", "n_imgs": None,
             "resolution": [512, 512], "load_dense_depth": False, "depth_folder": "depth", "depth_extension": "exr"},
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
                               "n_points_per_cloud": 8000, "learn_cameras": False}},
    "training": {
        "out_dir": "exp", "seed": 0,
        "lambda_dr_rgb": 1.0, "lambda_dr_silhouette": 1.0, "lambda_dr_proj": 0.1, "lambda_dr_repel": 0.1,
        "batch_size": 1, "print_every": 10, "checkpoint_every": 500, "validate_every": 500, "backup_every": 0,
        "scheduler_milestones": [500, 800], "scheduler_gamma": 0.5, "logfile": "train.log",
        "resume_from": "model.pt", "model_selection_metric": "chamfer_point", "model_selection_mode": "minimize",
        "n_eval_points": 8000, "steps_dss_backward_radii": 100, "steps_proj": -1, "gamma_proj": 5,
        "eval_sampling": "uniform",
        "grow_milestones": [], "grow_points": [],
        "prune_milestones": [], "prune_min_views": 1, "prune_max_outside": 0,
        "lr_cameras": 1e-4, "cameras_from_it": 300,
        "lambda_dr_depth": 0.0,
    },
}

# the neighbourhood size of the loop's growth events (ops.upsample_points' default): a cloud that grows needs more
# than GROW_K and at least 10 points, so a prune never leaves GROW_K or fewer
GROW_K = 16

# Keys of the reference's configurations that change nothing in its point-model training with data lights (the
# renderer classes it instantiates are the ones this loop runs, `learning_rate` is overridden by the per-group rates,
# the data-loader and visualisation details have no counterpart here, and TrainerScheduler is given neither
# gamma_dss_backward_radii nor limit_dss_backward_radii, trainer.py:118-123): accepted without a warning.
_NO_EFFECT = {
    "type", "test",
    "data.img_extension_input", "data.img_with_camera", "data.img_with_mask",
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


def check_config(cfg, resolution, has_lights, has_depth=False):
    """Refuse what the loop cannot train: a neural texture, lighting other than the data's, an image size other than
    the data's ``resolution`` (H, W), data without per-image lights, a depth term without depth maps
    (``has_depth``)."""
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
    check_growth(cfg)
    check_pruning(cfg)
    check_cameras(cfg)
    check_depth(cfg, has_depth)


def check_depth(cfg, has_depth):
    """Refuse depth settings the loop cannot follow: ``training.lambda_dr_depth`` must be a finite number >= 0,
    ``data.load_dense_depth`` a bool, and a lambda > 0 needs the data's depth maps (``has_depth``)."""
    lam, on = cfg["training"].get("lambda_dr_depth", 0.0), cfg["data"].get("load_dense_depth", False)
    if isinstance(lam, bool) or not isinstance(lam, (int, float)) or not 0 <= lam < float("inf"):
        raise ValueError("training.lambda_dr_depth must be a number >= 0, got %r" % (lam,))
    if not isinstance(on, bool):
        raise ValueError("data.load_dense_depth must be true or false, got %r" % (on,))
    if lam > 0 and not has_depth:
        raise ValueError("training.lambda_dr_depth %g needs dense depth maps: set data.load_dense_depth: true with the "
                         "maps in <data_dir>/%s" % (lam, cfg["data"].get("depth_folder", "depth")))


def _is_int(x):
    return isinstance(x, int) and not isinstance(x, bool)


def check_growth(cfg):
    """Refuse a growth schedule the loop cannot follow: ``training.grow_milestones`` (the iterations at whose start the
    cloud grows) and ``training.grow_points`` (its size from that iteration on) must be lists of one length, the
    milestones strictly increasing integers >= 1, the sizes strictly increasing integers above
    ``model.model_kwargs.n_points_per_cloud``, and that initial cloud one ``ops.upsample_points`` can grow with k =
    :data:`GROW_K` (more than k and at least 10 points)."""
    from ..ops import upsample_schedule
    tr = cfg["training"]
    ms, ns = tr.get("grow_milestones", []), tr.get("grow_points", [])
    if not isinstance(ms, (list, tuple)) or not isinstance(ns, (list, tuple)):
        raise ValueError("training.grow_milestones and training.grow_points must be lists, got %r and %r" % (ms, ns))
    if len(ms) != len(ns):
        raise ValueError("training.grow_milestones has %d entries and training.grow_points %d: they must pair up"
                         % (len(ms), len(ns)))
    if not ms:
        return
    if not all(_is_int(m) for m in ms) or ms[0] < 1 or any(b <= a for a, b in zip(ms, ms[1:])):
        raise ValueError("training.grow_milestones must be strictly increasing integers >= 1, got %r" % (list(ms),))
    n0 = cfg["model"]["model_kwargs"]["n_points_per_cloud"]
    if not all(_is_int(n) for n in ns) or any(b <= a for a, b in zip(ns, ns[1:])):
        raise ValueError("training.grow_points must be strictly increasing integers, got %r" % (list(ns),))
    if ns[0] <= n0:
        raise ValueError("training.grow_points must start above model.model_kwargs.n_points_per_cloud (%d), got %r"
                         % (n0, list(ns)))
    try:
        upsample_schedule([n0], [ns[0]], GROW_K)
    except ValueError as e:
        raise ValueError("training.grow_points: the initial cloud of n_points_per_cloud = %d points cannot grow (%s)"
                         % (n0, e)) from None


def check_pruning(cfg):
    """Refuse a pruning schedule the loop cannot follow: ``training.prune_milestones`` (the iterations at whose start
    the cloud is pruned) must be a list of strictly increasing integers >= 1, ``training.prune_min_views`` (keep a point
    seen in at least this many views; 0: no such test) an integer >= 0, ``training.prune_max_outside`` (keep a point
    over background in at most this many views; None: no such test) an integer >= 0 or None, and milestones need one
    of the two tests on."""
    tr = cfg["training"]
    ms = tr.get("prune_milestones", [])
    k, j = tr.get("prune_min_views", 1), tr.get("prune_max_outside", 0)
    if not isinstance(ms, (list, tuple)) or not all(_is_int(m) for m in ms) or (ms and ms[0] < 1) \
            or any(b <= a for a, b in zip(ms, ms[1:])):
        raise ValueError("training.prune_milestones must be a list of strictly increasing integers >= 1, got %r" % (ms,))
    if not _is_int(k) or k < 0:
        raise ValueError("training.prune_min_views must be an integer >= 0 (0: no such test), got %r" % (k,))
    if j is not None and (not _is_int(j) or j < 0):
        raise ValueError("training.prune_max_outside must be an integer >= 0 or null (no such test), got %r" % (j,))
    if ms and k == 0 and j is None:
        raise ValueError("training.prune_milestones is set, but prune_min_views 0 and prune_max_outside null turn both "
                         "of its tests off")


def check_cameras(cfg):
    """Refuse camera refinement settings the loop cannot follow: ``model.model_kwargs.learn_cameras`` must be a bool,
    ``training.lr_cameras`` (the Adam learning rate of the pose corrections) a finite number > 0 and
    ``training.cameras_from_it`` (the first iteration whose step learns them) an integer >= 0."""
    tr = cfg["training"]
    on = cfg["model"]["model_kwargs"].get("learn_cameras", False)
    lr, start = tr.get("lr_cameras", 1e-4), tr.get("cameras_from_it", 300)
    if not isinstance(on, bool):
        raise ValueError("model.model_kwargs.learn_cameras must be true or false, got %r" % (on,))
    if isinstance(lr, bool) or not isinstance(lr, (int, float)) or not 0 < lr < float("inf"):
        raise ValueError("training.lr_cameras must be a number > 0, got %r" % (lr,))
    if not _is_int(start) or start < 0:
        raise ValueError("training.cameras_from_it must be an integer >= 0, got %r" % (start,))


def cloud_size(cfg, it):
    """The cloud's size during (and after) iteration ``it`` under the growth schedule: the ``grow_points`` entry of the
    last milestone <= ``it``, or ``n_points_per_cloud`` before the first (``it`` = -1: the initial cloud)."""
    tr = cfg["training"]
    n = int(cfg["model"]["model_kwargs"]["n_points_per_cloud"])
    for m, size in zip(tr.get("grow_milestones", []), tr.get("grow_points", [])):
        if int(m) <= it:
            n = int(size)
    return n


def check_cloud_size(cfg, it, n_points):
    """Refuse a checkpoint of ``n_points`` points saved after iteration ``it`` that the growth and pruning schedules
    cannot give there (say, a schedule or ``n_points_per_cloud`` was edited since).  Without either schedule the
    checkpoint's cloud is taken at whatever size it has, as it always was.  With pruning, where the last event at or
    before ``it`` is a prune (a growth on the same iteration comes after it), the size may be anything from
    ``GROW_K + 1`` to :func:`cloud_size`'s, or that size itself (a prune that removed nothing or would have left too
    few); everywhere else it must be :func:`cloud_size`'s."""
    tr = cfg["training"]
    if not tr.get("grow_milestones") and not tr.get("prune_milestones"):
        return
    want = cloud_size(cfg, it)
    n = int(n_points)
    last_prune = max((int(m) for m in tr.get("prune_milestones", []) if int(m) <= it), default=None)
    last_grow = max((int(m) for m in tr.get("grow_milestones", []) if int(m) <= it), default=None)
    pruned = last_prune is not None and (last_grow is None or last_prune > last_grow)
    if n == want or (pruned and GROW_K < n < want):
        return
    raise ValueError("the checkpoint holds %d points after it=%d, but model.model_kwargs.n_points_per_cloud with "
                     "training.grow_milestones / grow_points%s gives %s there: the configuration changed since it "
                     "was written" % (n, it, " and prune_milestones" if tr.get("prune_milestones") else "",
                                      "%d to %d" % (GROW_K + 1, want) if pruned else want))


IMAGE_METRICS = ("iou", "psnr")
SELECTION_METRICS = ("chamfer_point", "chamfer_normal", "p2f_avg") + IMAGE_METRICS


def selection_metric(cfg):
    """``training.model_selection_metric`` if the loop can select by it: the chamfer distances of the reference's
    trainer, ``p2f_avg``, the mean distance of the cloud's points to ``<data_dir>/mesh.obj``, or the image-space
    ``iou`` / ``psnr`` of its ``evaluate_2d`` (:data:`IMAGE_METRICS`, both errors: minimize them)."""
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
            "lambda_dr_depth": float(tr.get("lambda_dr_depth", 0.0)), "learn": learn}
