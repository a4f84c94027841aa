"""The training loop: the reference's ``train_mvr.py`` with its ``Trainer`` (train_mvr.py:66-230, DSS/training/
trainer.py:73-238) on :class:`GraphedTrainStep`, from a data directory to a trained cloud.

    python -m dss_b200.training.train --config CFG.yml [--exit-after S] [--max-it N]
    torchrun --nproc-per-node G -m dss_b200.training.train --config CFG.yml [...] [--dist-backend nccl|gloo]

- data: ``MVRData(data.data_dir)``, which is also the validation set.  Every epoch draws ``len(data)`` view indices
  with replacement from uniform weights (``WeightedSubsetRandomSampler``: ``torch.multinomial`` on the loop's own
  generator) and cuts them into batches of ``training.batch_size`` views, the last partial batch dropped.  Every view's
  image, mask, cameras and lights (the per-image ``lights_%d`` entries) are uploaded once, at start, into a
  ``DeviceViews`` store (``MVRData.device_views``: 4 bytes per pixel for 8-bit data); the captured step gathers each
  batch from it (``GraphedTrainStep.from_views``), so an iteration uploads nothing but its (B,) view indices.
- model: ``model.model_kwargs.n_points_per_cloud`` area-weighted samples of ``ico_sphere(4)`` scaled by 0.5 with their
  face normals and albedo ones (config.py:177-183), drawn from ``training.seed``.
- optimizer: Adam, betas (0.5, 0.9), one group per learnt tensor: normals lr 0.01, points lr 0.01, colours lr 1.0
  (train_mvr.py:83-95); ``MultiStepLR(scheduler_milestones, scheduler_gamma)`` stepped after every epoch.
- before every step the reference Trainer's ``TrainerScheduler`` (scheduler.py:36-53 with the arguments of
  trainer.py:114-123): see :func:`radii_backward_scaler` and :func:`compound_lambda_proj`.
- every ``print_every`` iterations the losses go to ``<out>/<logfile>`` and one JSON line to ``<out>/metrics.jsonl``
  (the loop's only host synchronisations besides validation); every ``validate_every`` (it > 0) the chamfer distances
  of the ground-truth cloud against the current one (trainer.py:144-171; ``training.eval_sampling: poisson_disk`` draws
  it as the reference does, see :func:`ground_truth_cloud`), and on improvement of
  ``training.model_selection_metric`` ``model_best.pt`` and ``val/best.ply``.  With the metric ``p2f_avg`` the loop
  reads ``<data_dir>/mesh.obj`` once (it must exist) and every validation adds ``p2f_avg`` / ``p2f_std``, the mean and
  population standard deviation of the exact distances of the cloud's points to that mesh.  With ``iou`` or ``psnr``
  the validation is the reference's ``evaluate_2d`` instead (see :meth:`Trainer.evaluate`): it needs only the images,
  masks, cameras and lights, so data without a ground-truth cloud (``points`` / ``normals``) or mesh trains;
  ``model.pt`` every ``checkpoint_every``, ``model_%d.pt`` every ``backup_every``.
- growth (``training.grow_milestones`` / ``grow_points``, empty by default): at the start of iteration
  ``grow_milestones[i]``, before the schedules and the batch, the cloud grows to ``grow_points[i]`` points
  (:meth:`Trainer.grow`): its rows and their Adam moments stay, the new rows and their moments come from one
  ``upsample_points`` call, and the step is built anew with Adam and ``MultiStepLR`` continuing from their state.
  A checkpoint holds the cloud at its size; a resumed run grows at the milestones still ahead, and refuses a
  checkpoint whose size is not the one the schedule gives at its ``it``.
- pruning (``training.prune_milestones``, empty by default, with ``prune_min_views`` 1 and ``prune_max_outside`` 0):
  at the start of iteration ``prune_milestones[i]``, before a growth on the same iteration, the cloud keeps the points
  seen in at least ``prune_min_views`` views and over background in at most ``prune_max_outside`` (:meth:`Trainer.prune`,
  from ``ops.point_coverage`` over every view); the kept rows and their Adam moments stay in order and the step is
  built anew as after a growth.  A cloud with nothing to remove, or that would keep ``GROW_K`` points or fewer, is left
  as it is.  A checkpoint saved after a prune may hold any size from ``GROW_K + 1`` to the schedule's.
- camera refinement (``model.model_kwargs.learn_cameras``, off by default): one pose correction per view
  (``ops.pose_cameras``), learnt from iteration ``training.cameras_from_it`` on (before it the step is built without
  them, as when refinement is off, and at it the step is built anew with them) by one more Adam group, betas (0.5, 0.9)
  and ``training.lr_cameras``, stepped by the same ``MultiStepLR``.  Growth and pruning leave the poses and their Adam
  moments as they are.  Validation and pruning see the refined cameras (``DeviceViews.with_poses``), the log line adds
  the mean and maximum correction angle (degrees) and translation, and checkpoints hold ``"cameras": {"poses"}``; a
  checkpoint without them resumes at zero poses with a fresh Adam group.
- ``training.resume_from`` (in ``<out>``) is loaded when it exists, and the run continues where it stopped, mid-epoch
  included: a resumed run computes what an uninterrupted one does.  (The reference starts a new epoch.)
- ``--exit-after S`` saves ``model.pt`` and exits with status 3 once S seconds have passed (checked after every
  iteration; a negative S never exits); ``--max-it N`` saves ``model.pt`` and exits 0 after iteration N - 1.

Several GPUs (``WORLD_SIZE`` > 1 in the environment, as torchrun sets it with ``RANK``, ``LOCAL_RANK``,
``LOCAL_WORLD_SIZE``, ``MASTER_ADDR`` and ``MASTER_PORT``; ranks started by hand with the same variables work alike):
every rank joins the group through ``init_method="env://"`` and runs the view-sharded step, an eager
``TrainStep(..., grad_sync=GradSync())`` (``dss_b200.parallel``).  Without ``WORLD_SIZE``, or with 1, the loop above
runs unchanged.
- devices: ``--dist-backend nccl`` (the default) puts rank r on ``cuda:LOCAL_RANK`` and refuses, on every rank before
  joining the group, a ``LOCAL_WORLD_SIZE`` larger than the number of visible GPUs; ``gloo`` puts it on
  ``cuda:(LOCAL_RANK % device_count)``, for G ranks sharing one GPU.  The group has a timeout of
  :data:`DIST_TIMEOUT`, so a rank that dies turns the others' next collective into an error, and every exit destroys it.
- ``training.batch_size`` is the batch of one iteration over ALL the ranks, so G ranks solve the problem one GPU
  solves with the same config, to the summation order of the render gradients and the image-loss sums.  Every rank draws
  the same epoch order from ``training.seed`` and takes the same batch; :func:`deal_batch` deals its views by
  ``assign_views`` over costs from the host camera matrices, and each rank gathers its own from its copy of the device
  views (``DeviceViews.batch``; every rank holds them all, as the views dealt to a rank change from batch to batch; a
  rank dealt none runs the step's zero-view path).  Every rank keeps its own Adam, ``MultiStepLR`` and schedules: their
  gradients are the same bits, so the replicas stay the same and no parameters are broadcast.
- rank 0 alone writes the log, ``metrics.jsonl``, ``config.yaml``, the checkpoints and ``val/best.ply``, loads the
  ground truth and validates; the other ranks print only errors.  The checks that can fail on the data or the config
  run on every rank before the first collective, so a bad configuration fails every rank with the one-GPU message.
- before every iteration that may write a checkpoint (``checkpoint_every``, ``backup_every``, ``validate_every``, the
  time limit and the end) the ranks check that their points, normals and colours are the same bits
  (``parallel.check_replicas``) and all raise if not; rank 0 logs "Replica check".
- ``--exit-after``: the ranks agree on leaving after an iteration with one host all-reduce over a gloo group
  (``parallel.agree_any``; no device synchronisation), and all exit with status 3 after rank 0 saved ``model.pt``: no
  rank returns before rank 0's save is done, on any normal exit (one more host all-reduce).  torchrun reports a
  worker's non-zero exit as a failure of the job and stops the other workers; the status 3 is that of every rank's
  process.  Every checkpoint is written to ``<name>.tmp`` and moved over ``<name>``, so a killed writer leaves the
  previous checkpoint whole.
- every rank loads ``training.resume_from``; the checkpoint does not depend on G, so a run resumes on another number
  of GPUs (mid-epoch included), and on the same number continues bit for bit.
- every rank grows its replica at a milestone with the same deterministic call, builds a new eager step, and the
  ranks check right after it that their points, normals, colours and Adam moments are the same bits.  A prune covers
  views ``rank, rank + G, ...`` on each rank and sums the int32 counts over the ranks (exact, in any order), so every
  rank keeps the same points, and the same check follows.
"""
import argparse
import errno
import json
import math
import os
import sys
import time
from datetime import timedelta

import numpy as np
import torch
import torch.distributed as dist
import torch.nn.functional as F
import yaml

from ..core.cloud import PointClouds3D
from ..ops import chamfer_distance, evaluate_2d, point_coverage, upsample_points
from ..parallel import GradSync, agree_any, assign_views, check_replicas, view_costs_from_cameras
from ..utils.create_mvr_data import ico_sphere, sample_points_from_mesh
from ..utils.dataset import MVRData
from ..utils.evaluate import p2f_stats
from ..utils.io import read_mesh, save_ply
from .config import (EVAL_SAMPLINGS, GROW_K, IMAGE_METRICS, check_cloud_size, check_config, load_config,
                     selection_metric, splat_params, step_settings)
from .step import GraphedTrainStep, TrainStep

__all__ = ["radii_backward_scaler", "compound_lambda_proj", "initial_cloud", "make_optimizer", "make_lr_scheduler",
           "ground_truth_cloud", "check_ground_truth", "load_data", "dist_env", "rank_device", "deal_batch", "Trainer",
           "pose_stats", "main"]

EXIT_TIME_LIMIT = 3        # train_mvr.py:221-227
CAMERA_GROUP = "cameras"   # the name of the pose corrections' Adam group
EVAL_SEED = 0              # the fixed draw of the ground-truth samples
# a collective waits this long for the other ranks before it fails: longer than rank 0's validation of a large cloud,
# while the others wait at their next collective
DIST_TIMEOUT = timedelta(minutes=15)


def radii_backward_scaler(init, steps, it):
    """TrainerScheduler.step's ``radii_backward_scaler`` as the reference's Trainer configures it (trainer.py:118-123:
    gamma left at its default 0.99, limit 1.0; the YAML's ``gamma_dss_backward_radii`` / ``limit_dss_backward_radii``
    never reach it): ``max(init 0.99^(it // steps), 1.0)``, or ``init`` unchanged when ``steps <= 0``."""
    if steps <= 0:
        return init
    return max(init * 0.99 ** (it // steps), 1.0)


def compound_lambda_proj(lam, steps_proj, gamma_proj, it, limit=1.0):
    """TrainerScheduler.step's projection weight (scheduler.py:50-53), applied to the CURRENT value before every step,
    so it compounds: ``min(lam gamma_proj^(it // steps_proj), limit)``; unchanged when ``steps_proj <= 0``."""
    if steps_proj <= 0:
        return lam
    return min(lam * gamma_proj ** (it // steps_proj), limit)


def initial_cloud(n_points, seed=0, device="cuda"):
    """The reference's initial cloud (config.py:177-183): ``n_points`` area-weighted samples of ``ico_sphere(4)``
    scaled by 0.5, their face normals and albedo ones, drawn from a generator seeded with ``seed``.  (P,3) float32 x 3."""
    dev = torch.device(device)
    verts, faces = ico_sphere(4)
    g = torch.Generator(device=dev).manual_seed(int(seed))
    points, normals = sample_points_from_mesh((verts * 0.5).to(dev), faces.to(dev), int(n_points), generator=g)
    return points.contiguous(), normals.contiguous(), torch.ones_like(points)


def make_optimizer(tensors, poses=None, lr_cameras=None):
    """train_mvr.py:83-95: Adam, betas (0.5, 0.9), groups in the reference's order for the tensors that require grad:
    normals lr 0.01, points lr 0.01, colours lr 1.0.  ``tensors``: {"points", "normals", "colours"}.  ``poses``: the
    (V,6) camera corrections, one more group last, named ``"cameras"``, with lr ``lr_cameras``."""
    groups = [{"params": [tensors[name]], "lr": lr, "betas": (0.5, 0.9)}
              for name, lr in (("normals", 0.01), ("points", 0.01), ("colours", 1.0)) if tensors[name].requires_grad]
    if not groups:
        raise ValueError("nothing to learn: model.model_kwargs sets every learn_* false")
    if poses is not None:
        groups.append({"params": [poses], "lr": float(lr_cameras), "betas": (0.5, 0.9), "name": CAMERA_GROUP})
    return torch.optim.Adam(groups, lr=0.01, betas=(0.5, 0.9))


def pose_stats(poses):
    """(4,) float32 on the poses' device: the mean and maximum rotation angle (degrees) and translation norm of the
    (V,6) corrections"""
    with torch.no_grad():
        ang, tr = torch.rad2deg(poses[:, :3].norm(dim=1)), poses[:, 3:].norm(dim=1)
        return torch.stack([ang.mean(), ang.amax(), tr.mean(), tr.amax()]).double()


def make_lr_scheduler(optimizer, cfg):
    """train_mvr.py:128-130: MultiStepLR over epochs, stepped once after every epoch."""
    tr = cfg["training"]
    return torch.optim.lr_scheduler.MultiStepLR(optimizer, list(tr["scheduler_milestones"]),
                                                gamma=float(tr["scheduler_gamma"]))


def ground_truth_cloud(data, data_dir, n_eval_points, device, sampling="uniform"):
    """(points, normals) the validation measures against: the stored cloud when ``n_eval_points`` <= 0 or equals its
    size; otherwise, with ``sampling`` "uniform", ``n_eval_points`` area-weighted samples of ``<data_dir>/mesh.obj``
    drawn once from a fixed seed, and with "poisson_disk" the reference's ``get_pointclouds(num_points=n_eval_points)``:
    geodesic Poisson-disk samples of that mesh (:meth:`MVRData.get_pointclouds`).  Only those compare with the
    reference's own chamfer values."""
    check_ground_truth(data, data_dir, n_eval_points, sampling)
    stored = data.get_pointclouds()
    n = int(n_eval_points)
    if n <= 0 or n == stored.points_packed().shape[0]:
        return stored.points_packed().to(device), stored.normals_packed().to(device)
    if sampling == "poisson_disk":
        pc = data.get_pointclouds(num_points=n)
        return pc.points_packed().to(device), pc.normals_packed().to(device)
    verts, faces = read_mesh(os.path.join(data_dir, "mesh.obj"))
    g = torch.Generator(device=device).manual_seed(EVAL_SEED)
    return sample_points_from_mesh(torch.from_numpy(verts).float().to(device), torch.from_numpy(faces).long().to(device),
                                   n, generator=g)


def check_ground_truth(data, data_dir, n_eval_points, sampling="uniform"):
    """the errors :func:`ground_truth_cloud` would raise on these arguments, without loading or sampling anything: an
    unknown ``sampling``, and a missing ``<data_dir>/mesh.obj`` when the samples are drawn from it.  (Every rank of a
    sharded run checks this at start, while only rank 0 loads the ground truth.)"""
    if sampling not in EVAL_SAMPLINGS:
        raise ValueError("training.eval_sampling must be one of %s, got %r" % (", ".join(EVAL_SAMPLINGS), sampling))
    n = int(n_eval_points)
    if n <= 0 or n == len(data.data_dict["points"]):
        return
    if sampling == "poisson_disk":
        data.sampled_mesh(n)
        return
    mesh = os.path.join(data_dir, "mesh.obj")
    if not os.path.isfile(mesh):
        raise FileNotFoundError(errno.ENOENT, os.strerror(errno.ENOENT), mesh)      # what reading it would raise


def load_data(cfg):
    """the configuration's ``MVRData`` (its ``data`` block), which must have images and masks"""
    dc = cfg["data"]
    data = MVRData(dc["data_dir"], data_dict=dc["data_dict"], n_imgs=dc["n_imgs"], img_folder=dc["img_folder"],
                   mask_folder=dc["mask_folder"], img_extension=dc["img_extension"], mask_extension=dc["mask_extension"],
                   load_dense_depth=bool(dc.get("load_dense_depth", False)), depth_folder=dc.get("depth_folder", "depth"),
                   depth_extension=dc.get("depth_extension", "exr"))
    if data.images is None or data.masks is None:
        raise ValueError("%s has no images and masks" % dc["data_dir"])
    return data


def dist_env(environ=None):
    """``{"rank", "world", "local_rank", "local_world"}`` from the variables torchrun sets (``RANK``, ``WORLD_SIZE``,
    ``LOCAL_RANK``, ``LOCAL_WORLD_SIZE``; the local ones default to the global), or None when ``WORLD_SIZE`` is unset or
    1: the single-GPU loop."""
    env = os.environ if environ is None else environ
    world = int(env.get("WORLD_SIZE", "1") or 1)
    if world <= 1:
        return None
    rank = int(env["RANK"])
    return {"rank": rank, "world": world, "local_rank": int(env.get("LOCAL_RANK", rank)),
            "local_world": int(env.get("LOCAL_WORLD_SIZE", world))}


def rank_device(backend, local_rank, local_world, n_gpus):
    """The device of a rank: ``cuda:local_rank`` over nccl, which needs a GPU per local rank (a RuntimeError
    otherwise, raised before the rank joins the group, so that every rank fails alike and none waits);
    ``cuda:(local_rank % n_gpus)`` over gloo, so that several ranks can share a GPU."""
    if n_gpus < 1:
        raise RuntimeError("the training loop needs a CUDA device (sm_90a); rank %d sees none" % local_rank)
    if backend == "nccl":
        if local_world > n_gpus:
            raise RuntimeError("--dist-backend nccl runs one rank per GPU, but %d local ranks share %d visible GPU%s; "
                               "start at most %d, or use --dist-backend gloo to share GPUs"
                               % (local_world, n_gpus, "" if n_gpus == 1 else "s", n_gpus))
        return torch.device("cuda", local_rank)
    if backend == "gloo":
        return torch.device("cuda", local_rank % n_gpus)
    raise ValueError("--dist-backend must be nccl or gloo, got %r" % (backend,))


def deal_batch(camera_mat, idx, world):
    """The views of batch ``idx`` (indices into the data, repeats allowed) dealt to ``world`` ranks:
    ``assign_views(view_costs_from_cameras(camera_mat[idx]), world)``, a list per rank of the data indices it renders.
    Every position of ``idx`` goes to exactly one rank; a rank gets none when ``len(idx) < world``.  ``camera_mat``: the
    data's (V,4,4) host world-to-view matrices, so dealing needs no device round trip, and every rank deals alike."""
    idx = [int(i) for i in idx]
    mats = torch.from_numpy(np.asarray(camera_mat, dtype=np.float32)[np.asarray(idx, dtype=np.int64)].reshape(-1, 4, 4))
    return [[idx[j] for j in part] for part in assign_views(view_costs_from_cameras(mats).tolist(), world)]


class _Log:
    """lines to ``<out>/<logfile>`` (and stdout), JSON records to ``<out>/metrics.jsonl``; ``quiet``: neither (the
    ranks other than 0)"""

    def __init__(self, out_dir, logfile, quiet=False):
        self.quiet = quiet
        if not quiet:
            self.text = open(os.path.join(out_dir, logfile), "a")
            self.metrics = open(os.path.join(out_dir, "metrics.jsonl"), "a")

    def info(self, msg):
        if self.quiet:
            return
        line = "%s %s" % (time.strftime("%Y-%m-%d %H:%M:%S"), msg)
        print(line, flush=True)
        self.text.write(line + "\n")
        self.text.flush()

    def record(self, rec):
        if self.quiet:
            return
        self.metrics.write(json.dumps(rec) + "\n")
        self.metrics.flush()

    def close(self):
        if not self.quiet:
            self.text.close()
            self.metrics.close()


class Trainer:
    """The loop's state and one iteration at a time (see the module docstring).  ``Trainer(cfg).run(exit_after,
    max_it)`` returns the process exit status.  ``grad_sync``: a ``GradSync`` of world size G > 1 makes this rank one
    of G that shard every batch's views (the process group initialised, ``device`` this rank's GPU)."""

    def __init__(self, cfg, device="cuda", grad_sync=None):
        self.cfg = cfg
        self.dev = torch.device(device)
        self.sync = grad_sync if grad_sync is not None and grad_sync.world_size > 1 else None
        self.world = 1 if self.sync is None else self.sync.world_size
        self.rank = 0 if self.sync is None else dist.get_rank(self.sync.group)
        self.lead = self.rank == 0
        self.host_group = None          # the gloo group of the exit agreement, made by run() when it needs one
        self._checked_it = None         # the iteration the replica guard last ran at
        tr, dc = cfg["training"], cfg["data"]
        self.out_dir = os.path.join(str(tr["out_dir"]), str(cfg["name"]))
        self.val_dir = os.path.join(self.out_dir, "val")
        if self.lead:
            os.makedirs(self.val_dir, exist_ok=True)
        self.log = _Log(self.out_dir, tr["logfile"], quiet=not self.lead)
        # ---- data: every view's image, mask, cameras and lights on the device, uploaded once
        self.data = load_data(cfg)
        V = len(self.data)
        self.views = self.data.device_views(self.dev)
        self.log.info("Views on the device: %d of %dx%d, %s store, %.1f MB"
                      % (V, self.views.H, self.views.W, str(self.views.store.dtype).replace("torch.", ""),
                         self.views.nbytes / 1e6))
        check_config(cfg, self.data.resolution, self.views.light_cls is not None, self.views.depth is not None)
        self.metric = selection_metric(cfg)
        self.mesh = None
        if self.metric == "p2f_avg":
            mesh_path = os.path.join(dc["data_dir"], "mesh.obj")
            if not os.path.isfile(mesh_path):
                raise ValueError("model_selection_metric p2f_avg measures against %s, which does not exist" % mesh_path)
            if self.lead:
                verts, faces = read_mesh(mesh_path)
                self.mesh = (torch.from_numpy(verts).float().to(self.dev), torch.from_numpy(faces).to(self.dev))
        cams = self.data.get_cameras()
        self.params = splat_params(cfg, cams.znear, cams.zfar)
        self.settings = step_settings(cfg)
        self.batch_size = int(tr["batch_size"])
        if V // self.batch_size < 1:
            raise ValueError("batch_size %d is larger than the %d views: an epoch would have no batch"
                             % (self.batch_size, V))
        self.gt = None
        if self.metric not in IMAGE_METRICS:
            missing = [k for k in ("points", "normals") if k not in self.data.data_dict]
            if missing:
                raise ValueError("model_selection_metric %s measures against the data's cloud, but %s has no %s; "
                                 "select by iou or psnr to train without one"
                                 % (self.metric, os.path.join(dc["data_dir"], dc["data_dict"]), " / ".join(missing)))
            check_ground_truth(self.data, dc["data_dir"], tr["n_eval_points"], tr.get("eval_sampling", "uniform"))
        if self.metric not in IMAGE_METRICS and self.lead:
            self.gt = ground_truth_cloud(self.data, dc["data_dir"], tr["n_eval_points"], self.dev,
                                         tr.get("eval_sampling", "uniform"))
        # ---- state: fresh, then whatever the checkpoint holds
        self.gen = torch.Generator().manual_seed(int(tr["seed"]))
        self.epoch_it, self.it, self.order, self.pos = -1, -1, None, 0
        self.sign = {"minimize": -1, "maximize": 1}.get(tr["model_selection_mode"])
        if self.sign is None:
            raise ValueError("model_selection_mode must be either maximize or minimize.")
        self.best = -self.sign * math.inf
        self.radii_init = self.params.radii_backward_scaler
        self.lambda_dr_proj = self.settings["lambda_dr_proj"]
        self.learn_cameras = bool(cfg["model"]["model_kwargs"].get("learn_cameras", False))
        self.lr_cameras, self.cameras_from_it = float(tr.get("lr_cameras", 1e-4)), int(tr.get("cameras_from_it", 300))
        if self.learn_cameras:
            self.views.check_rigid()
        self.poses = None
        ckpt_path = os.path.join(self.out_dir, str(tr["resume_from"]))
        # loaded to the host: the optimizer moves its state to the parameters' device, the sampler state stays there
        ckpt = torch.load(ckpt_path, map_location="cpu", weights_only=False) if os.path.exists(ckpt_path) else None
        if ckpt is None:
            points, normals, colours = initial_cloud(cfg["model"]["model_kwargs"]["n_points_per_cloud"], tr["seed"],
                                                     self.dev)
        else:
            points, normals, colours = (ckpt["model"][k][0].to(self.dev) for k in ("points", "normals", "colors"))
            self.epoch_it, self.it, self.best = int(ckpt["epoch_it"]), int(ckpt["it"]), float(ckpt["loss_val_best"])
            self.gen.set_state(ckpt["sampler"])
            self.order, self.pos = ckpt["epoch_order"], int(ckpt["epoch_pos"])
            self.lambda_dr_proj = float(ckpt["schedule"]["lambda_dr_proj"])
            self.params = self.params._replace(radii_backward_scaler=float(ckpt["schedule"]["radii_backward_scaler"]))
            check_cloud_size(cfg, self.it, points.shape[0])
            self.log.info("resumed from %s at it=%d, epoch %d" % (ckpt_path, self.it, self.epoch_it))
        state = None if ckpt is None else (ckpt["optimizer"], ckpt["lr_scheduler"])
        has_poses = ckpt is not None and "cameras" in ckpt
        if ckpt is not None and not self.learn_cameras and any(
                g.get("name") == CAMERA_GROUP for g in ckpt["optimizer"]["param_groups"]):
            raise ValueError("the checkpoint %s learnt camera poses: resume it with model.model_kwargs.learn_cameras: "
                             "true" % ckpt_path)
        poses = None
        if self.learn_cameras:
            poses = torch.zeros((V, 6), dtype=torch.float32, device=self.dev)
            if has_poses:
                p = ckpt["cameras"]["poses"]
                if tuple(p.shape) != (V, 6):
                    raise ValueError("the checkpoint %s holds camera poses of shape %s, but the data has %d views"
                                     % (ckpt_path, tuple(p.shape), V))
                poses = p.to(self.dev, torch.float32)
            elif state is not None:
                # a checkpoint without poses: they start at zero with a fresh Adam group, appended after the cloud's
                state = (dict(state[0], param_groups=list(state[0]["param_groups"]) + [None]),
                         dict(state[1], base_lrs=list(state[1]["base_lrs"]) + [self.lr_cameras],
                              _last_lr=list(state[1]["_last_lr"]) + [self.lr_cameras]))
                self.log.info("the checkpoint holds no camera poses: they start at zero")
        # the growth schedule: {iteration: the cloud's size from its start on}
        self.grow_at = {int(m): int(n) for m, n in zip(tr.get("grow_milestones", []), tr.get("grow_points", []))}
        self.prune_at = set(int(m) for m in tr.get("prune_milestones", []))
        self.prune_min_views, self.prune_max_outside = int(tr.get("prune_min_views", 1)), tr.get("prune_max_outside", 0)
        if self.prune_at and self.prune_min_views > V:
            raise ValueError("training.prune_min_views %d is above the data's %d views: a prune would remove every point"
                             % (self.prune_min_views, V))
        if self.lead:
            with open(os.path.join(self.out_dir, "config.yaml"), "w") as f:
                yaml.safe_dump(cfg, f, sort_keys=False)
        self._build(points, normals, colours, poses, self._cameras_due(self.it + 1), state)

    # ---- pieces ------------------------------------------------------------------------------------------------------
    def _cameras_due(self, it):
        """whether the step of iteration ``it`` learns the camera poses"""
        return self.learn_cameras and it >= self.cameras_from_it

    def _build(self, points, normals, colours, poses=None, cameras=False, state=None):
        """the step on this cloud, its Adam and ``MultiStepLR``; ``poses``: the (V,6) camera corrections when they are
        learnt, and ``cameras`` whether this step learns them (the step then holds the leaf, otherwise the trainer
        does, so that the Adam group stays); ``state``: (optimizer, lr scheduler) state dicts to continue from (a
        checkpoint's, or those of an event), where a pose group of None stands for a fresh one"""
        s = dict(self.settings)
        learn, s["lambda_dr_proj"] = s.pop("learn"), self.lambda_dr_proj
        if cameras:
            s["poses"] = poses
        if self.sync is None:
            # captured on any batch of the right shape: the capture's warm-up steps leave the cloud unchanged, and every
            # iteration loads its own view indices first (the sharded step is eager)
            self.step = GraphedTrainStep.from_views(points, normals, colours, self.params, self.views,
                                                    list(range(self.batch_size)), learn=learn, **s)
        else:
            self.step = TrainStep(points, normals, colours, self.params, learn=learn, grad_sync=self.sync,
                                  views=self.views if cameras else None, **s)
        self.poses = self.step.poses if cameras else (
            None if poses is None else poses.detach().clone().requires_grad_(True))
        self.opt = make_optimizer({"points": self.step.points, "normals": self.step.normals,
                                   "colours": self.step.colours}, self.poses, self.lr_cameras)
        self.lr_sched = make_lr_scheduler(self.opt, self.cfg)
        if state is not None:
            groups = state[0]["param_groups"]
            if groups and groups[-1] is None:
                fresh = self.opt.state_dict()["param_groups"][-1]
                state = (dict(state[0], param_groups=groups[:-1] + [fresh]), state[1])
            self.opt.load_state_dict(state[0])
            self.lr_sched.load_state_dict(state[1])

    def _cloud_state(self):
        """the cloud's (points, normals, colours), detached, Adam's state dict, and the (state index, moment) keys of
        the moments of every learnt tensor of the cloud (not of the camera poses, which no cloud event changes)"""
        s, sd = self.step, self.opt.state_dict()
        cloud = {i for g in sd["param_groups"] if g.get("name") != CAMERA_GROUP for i in g["params"]}
        keys = [(i, k) for i in sorted(sd["state"]) if i in cloud for k in ("exp_avg", "exp_avg_sq")]
        return (s.points.detach(), s.normals.detach(), s.colours.detach()), sd, keys

    def _rebuild(self, points, normals, colours, sd, moments):
        """the step built anew on a changed cloud, after an event: Adam continues from ``sd`` with the moments
        ``moments`` ({(state index, moment): rows}), and ``MultiStepLR`` from its state: step counts, betas and the
        current learning rates"""
        state = {i: dict(st) for i, st in sd["state"].items()}
        for (i, k), m in moments.items():
            state[i][k] = m
        sched = self.lr_sched.state_dict()
        poses = None if self.poses is None else self.poses.detach()
        self.step = self.opt = self.lr_sched = None     # the old step and its graph go first
        self._build(points, normals, colours, poses, self._cameras_due(self.it), (dict(sd, state=state), sched))

    def start_cameras(self):
        """the step built anew with the camera poses learnt (at ``cameras_from_it``): the cloud, the poses and Adam's
        state as they are"""
        (points, normals, colours), sd, _ = self._cloud_state()
        self._rebuild(points, normals, colours, sd, {})
        self.log.info("Learning the camera poses from it=%d" % self.it)

    def views_now(self):
        """the data's device views with the current camera corrections (the views themselves when none are learnt)"""
        return self.views if self.poses is None else self.views.with_poses(self.poses)

    def grow(self, n):
        """The growth event: the cloud grows from P to ``n`` points, at the start of a milestone's iteration.  The P
        rows of the points, normals and colours and of Adam's moments stay as they are; the new rows are those of one
        ``upsample_points(points, n, k=GROW_K)`` call that is given the unit normals and, as features, the colours and
        the moments of every learnt tensor side by side, so that a child's moments follow the ``(f_q + 2 f_p) / 3``
        rule of its colour (a child with zero moments would take a first step of about 1.6 lr in every coordinate:
        Adam's step count, and with it the bias correction, is shared by the whole tensor).  The step is built anew on
        the grown cloud (the old one and its graph dropped first), and Adam and ``MultiStepLR`` continue from the old
        ones' state: step counts, betas and the current learning rates.  Deterministic, so replicas stay replicas."""
        t0 = time.perf_counter()
        (points, normals, colours), sd, keys = self._cloud_state()
        P = points.shape[0]
        moments = [sd["state"][i][k] for i, k in keys]
        up = upsample_points(points, n, k=GROW_K, normals=F.normalize(normals, dim=-1),
                             features=torch.cat([colours] + moments, 1))
        grown = lambda rows, new: torch.cat([rows, new[P:]])
        cols = torch.split(up.features, 3, 1)
        self._rebuild(grown(points, up.points), grown(normals, up.normals), grown(colours, cols[0]), sd,
                      {key: grown(m, col) for key, m, col in zip(keys, moments, cols[1:])})
        torch.cuda.synchronize(self.dev)
        self.log.info("Grew the cloud at it=%d: %d -> %d points (%.1f ms: upsample and new step)"
                      % (self.it, P, n, 1e3 * (time.perf_counter() - t0)))

    def prune(self):
        """The prune event, at the start of a milestone's iteration (before a growth on the same one): the view coverage
        of the cloud (:func:`~dss_b200.ops.point_coverage` over all the data's views, ``batch_size`` at a time, with the
        step's current splat settings; on G ranks each covers views ``rank, rank + G, ...`` and the int32 counts are
        summed over the ranks, exactly), and the points kept where ``seen >= prune_min_views`` and ``outside <=
        prune_max_outside`` (a test off: 0, null).  The kept rows of the points, normals, colours and Adam's moments stay
        in their order, and the step is built anew as after a growth.  The cloud is left as it is when every point
        passes, or when GROW_K or fewer would remain (so that a later growth can run)."""
        t0 = time.perf_counter()
        (points, normals, colours), sd, keys = self._cloud_state()
        P, st = points.shape[0], self.step
        cov = point_coverage(points, normals, self.views_now(), self.params, self.batch_size,
                             range(self.rank, len(self.views), self.world), st.Vrk_invariant, st.Vrk_isotropic,
                             st.frnn_radius)
        st = None
        if self.sync is not None:
            for c in cov:
                dist.all_reduce(c, op=dist.ReduceOp.SUM, group=self.sync.group)
        k, j = self.prune_min_views, self.prune_max_outside
        few = cov.seen < k
        over = cov.outside > j if j is not None else torch.zeros_like(few)
        keep = ~(few | over)
        n, n_few, n_over = torch.stack([keep.sum(), few.sum(), over.sum()]).tolist()
        why = ", ".join(([] if k == 0 else ["%d seen in fewer than %d views" % (n_few, k)])
                        + ([] if j is None else ["%d outside the masks in more than %d views" % (n_over, j)]))
        if n == P or n <= GROW_K:
            self.log.info("Kept the cloud at it=%d: %s (%s)" % (
                self.it, "every point passes" if n == P else "pruning would leave %d points, %d or fewer" % (n, GROW_K),
                why))
            return
        idx = keep.nonzero()[:, 0]
        rows = lambda t: t.index_select(0, idx)
        self._rebuild(rows(points), rows(normals), rows(colours), sd,
                      {(i, m): rows(sd["state"][i][m]) for i, m in keys})
        torch.cuda.synchronize(self.dev)
        self.log.info("Pruned the cloud at it=%d: %d -> %d points (%s; %.1f ms)"
                      % (self.it, P, n, why, 1e3 * (time.perf_counter() - t0)))

    def _schedule(self):
        """TrainerScheduler.step (trainer.py:227) before the step; a changed setting makes the next replay capture"""
        tr = self.cfg["training"]
        r = radii_backward_scaler(self.radii_init, int(tr["steps_dss_backward_radii"]), self.it)
        if r != self.params.radii_backward_scaler:
            self.log.info("Updated radii_backward_scaler: %s -> %s" % (self.params.radii_backward_scaler, r))
            self.params = self.params._replace(radii_backward_scaler=r)
        self.lambda_dr_proj = compound_lambda_proj(self.lambda_dr_proj, int(tr["steps_proj"]), float(tr["gamma_proj"]),
                                                   self.it)
        self.step.params, self.step.lambda_dr_proj = self.params, self.lambda_dr_proj

    def cloud(self):
        """the current cloud with unit normals (PointModel.get_point_clouds)"""
        return self.step.points.detach(), F.normalize(self.step.normals.detach(), dim=-1)

    def evaluate(self):
        """trainer.py:144-171: chamfer distances of the ground truth (x) against the current cloud (y); selecting by
        p2f_avg, also the mean and population standard deviation of the points' distances to the data's mesh.
        Selecting by iou or psnr, instead the image-space metrics of ``Trainer.evaluate_2d`` (trainer.py:173-212,
        581-586): every view rendered at resolution // 4 (train_mvr.py:135) with the step's shading and splat flags,
        ``batch_size`` views at a time, scored by :func:`~dss_b200.ops.evaluate_2d`."""
        if self.metric in IMAGE_METRICS:
            st = self.step
            ev = evaluate_2d(st.points, st.normals, st.colours, self.views_now(), self.params,
                             max(1, self.data.resolution[0] // 4), self.batch_size, st.Vrk_invariant, st.Vrk_isotropic,
                             st.frnn_radius, st.shininess)
            return {"iou": float(ev["iou"]), "psnr": float(ev["psnr"])}
        points, normals = self.cloud()
        with torch.no_grad():
            cd_p, cd_n = chamfer_distance(PointClouds3D([self.gt[0]], [self.gt[1]]), PointClouds3D([points], [normals]))
        ev = {"chamfer_point": float(cd_p), "chamfer_normal": float(cd_n)}
        if self.mesh is not None:
            _, ev["p2f_avg"], ev["p2f_std"] = p2f_stats(points, self.mesh)
        return ev

    def _validate(self, metric):
        """validation and model selection (rank 0): the log line, and on improvement ``model_best.pt`` and
        ``val/best.ply``"""
        ev = self.evaluate()
        self.log.info("Validation metric (%s): %.4g  (%s)" % (metric, ev[metric], json.dumps(ev)))
        if self.sign * (ev[metric] - self.best) > 0:
            self.best = ev[metric]
            self.log.info("New best model (loss %.4g)" % self.best)
            self.save("model_best.pt")
            points, normals = self.cloud()
            save_ply(os.path.join(self.val_dir, "best.ply"), points.cpu().numpy(), normals=normals.cpu().numpy())

    def save(self, name):
        """``<out>/name``, replaced whole (rank 0 alone writes; the other ranks return)"""
        if not self.lead:
            return
        s = self.step
        P0 = s.points.shape[0]
        # written next to the target and moved over it: a process killed mid-write leaves the previous file whole
        path = os.path.join(self.out_dir, name)
        tmp = path + ".tmp"
        torch.save({
            "model": {"points": s.points.detach()[None].clone(), "normals": s.normals.detach()[None].clone(),
                      "colors": s.colours.detach()[None].clone(),
                      "points_activation": torch.ones((1, P0), dtype=torch.bool, device=self.dev)},
            "optimizer": self.opt.state_dict(), "lr_scheduler": self.lr_sched.state_dict(),
            "epoch_it": self.epoch_it, "it": self.it, "loss_val_best": self.best,
            "schedule": {"radii_backward_scaler": self.params.radii_backward_scaler,
                         "lambda_dr_proj": self.lambda_dr_proj},
            "sampler": self.gen.get_state(), "epoch_order": list(self.order), "epoch_pos": self.pos,
            **({} if self.poses is None else {"cameras": {"poses": self.poses.detach().clone()}}),
        }, tmp)
        os.replace(tmp, path)

    def check_replicas(self, event=False):
        """the replica guard of a sharded run, before an iteration's checkpoints: every rank raises unless the ranks'
        points, normals and colours are the same bits (one all-reduce, one host synchronisation).  Once per
        iteration; nothing on one GPU.  ``event``: the check right after a growth event, before the iteration's step,
        which also covers Adam's moments and leaves the guard of the iteration's checkpoints to run."""
        if self.sync is None or (not event and self._checked_it == self.it):
            return
        s = self.step
        named = [("points", s.points), ("normals", s.normals), ("colours", s.colours)]
        if self.poses is not None:
            named.append(("camera poses", self.poses))
        if event:
            named += [("Adam's %s of the %s" % (k, n), self.opt.state[t][k]) for n, t in named
                      if t in self.opt.state for k in ("exp_avg", "exp_avg_sq")]
        check_replicas(named, self.sync.group)
        if not event:
            self._checked_it = self.it
        self.log.info("Replica check: the %d ranks hold the same points, normals%s and colours%s"
                      % (self.world, ", camera poses" if self.poses is not None else "",
                         " and Adam moments" if event else ""))

    def _out_of_time(self, exit_after, t0):
        """whether to leave after this iteration; a sharded run's ranks agree (any rank's clock decides for all)"""
        if exit_after is None or exit_after < 0:
            return False
        over = time.time() - t0 >= exit_after
        if self.sync is None:
            return over
        return agree_any(over, self._host_group())

    def _host_group(self):
        """the gloo group of the host-side agreements, made on first use (by every rank at the same point)"""
        if self.host_group is None:
            self.host_group = dist.new_group(backend="gloo", timeout=DIST_TIMEOUT)
        return self.host_group

    def _leave_together(self):
        """on a sharded run's exit, after rank 0's last save: no rank returns before rank 0 has written, since a
        launcher that sees one worker exit non-zero (torchrun, on the time limit's status 3) stops the others"""
        if self.sync is not None:
            agree_any(False, self._host_group())

    # ---- the loop ----------------------------------------------------------------------------------------------------
    def run(self, exit_after=600.0, max_it=None):
        tr = self.cfg["training"]
        print_every, checkpoint_every = int(tr["print_every"]), int(tr["checkpoint_every"])
        backup_every, validate_every = int(tr["backup_every"]), int(tr["validate_every"])
        metric = self.metric
        V, bs = len(self.data), self.batch_size
        t0 = t0b = time.time()
        try:
            while max_it is None or self.it + 1 < max_it:
                if self.order is None or self.pos + bs > len(self.order):
                    if self.order is not None:
                        self.lr_sched.step()          # the end of an epoch (train_mvr.py:229-230)
                    self.epoch_it += 1
                    self.order = torch.multinomial(torch.ones(V, dtype=torch.float64), V, True,
                                                   generator=self.gen).tolist()
                    self.pos = 0
                idx = self.order[self.pos:self.pos + bs]
                self.pos += bs
                self.it += 1
                if self.it in self.prune_at:
                    self.prune()                      # first: a growth on the same iteration seeds no strays
                if self.it in self.grow_at:
                    self.grow(self.grow_at[self.it])
                if self.learn_cameras and self.step.poses is None and self._cameras_due(self.it):
                    self.start_cameras()
                if self.it in self.prune_at or self.it in self.grow_at:
                    self.check_replicas(event=True)
                self._schedule()
                if self.sync is None:
                    self.step.load_views(idx)
                    if self.step.stale():
                        self.step.capture()
                    loss = self.step.replay()
                else:
                    mine = self.views.upload(deal_batch(self.data.camera_mat, idx, self.world)[self.rank])
                    loss = self.step(*self.views.batch_at(mine), idx=mine if self.step.poses is not None else None,
                                     depth=self.views.depth_at(mine) if self.step.lambda_dr_depth > 0 else None)
                self.opt.step()
                it = self.it
                if self.lead and print_every > 0 and it % print_every == 0:
                    names = list(loss) + ([] if self.poses is None else
                                          ["cam_rot_mean", "cam_rot_max", "cam_trans_mean", "cam_trans_max"])
                    cam = [] if self.poses is None else list(pose_stats(self.poses))
                    vals = dict(zip(names, torch.stack([v.double() for v in loss.values()] + cam).tolist()))
                    self.log.info("[Epoch %02d] it=%03d, loss=%.4f, time=%.4f " % (self.epoch_it, it, vals["loss"],
                                                                                   time.time() - t0b)
                                  + " ".join("%s=%.4g" % kv for kv in vals.items() if kv[0] != "loss"))
                    self.log.record(dict(it=it, epoch=self.epoch_it, time=time.time() - t0, **vals))
                    t0b = time.time()
                if it > 0 and checkpoint_every > 0 and it % checkpoint_every == 0:
                    self.check_replicas()
                    self.log.info("Saving checkpoint")
                    self.save("model.pt")
                if it > 0 and backup_every > 0 and it % backup_every == 0:
                    self.check_replicas()
                    self.log.info("Backup checkpoint")
                    self.save("model_%d.pt" % it)
                if it > 0 and validate_every > 0 and it % validate_every == 0:
                    self.check_replicas()             # before rank 0 may write model_best.pt
                    if self.lead:
                        self._validate(metric)
                if self._out_of_time(exit_after, t0):
                    self.check_replicas()
                    self.log.info("Time limit reached. Exiting.")
                    self.save("model.pt")
                    self._leave_together()
                    return EXIT_TIME_LIMIT
            self.check_replicas()
            self.save("model.pt")
            self._leave_together()
            return 0
        finally:
            self.log.close()


def main(argv=None):
    p = argparse.ArgumentParser(description="Train a point cloud from a multi-view data directory (train_mvr.py).")
    p.add_argument("--config", required=True, help="YAML configuration (inherit_from chains over the defaults)")
    p.add_argument("--exit-after", type=float, default=600,
                   help="save model.pt and exit with status 3 after this many seconds (negative: never)")
    p.add_argument("--max-it", type=int, default=None, help="save model.pt and exit 0 after this many iterations")
    p.add_argument("--dist-backend", choices=("nccl", "gloo"), default="nccl",
                   help="under torchrun (WORLD_SIZE > 1): nccl, one GPU per rank, or gloo, ranks sharing GPUs")
    args = p.parse_args(argv)
    env = dist_env()
    if env is None:
        if not torch.cuda.is_available():
            raise RuntimeError("the training loop needs a CUDA device (sm_90a)")
        cfg = load_config(args.config)
        return Trainer(cfg).run(exit_after=args.exit_after, max_it=args.max_it)
    # refused here, before the group is joined, a bad device count fails every rank at once
    dev = rank_device(args.dist_backend, env["local_rank"], env["local_world"], torch.cuda.device_count())
    cfg = load_config(args.config)
    torch.cuda.set_device(dev)
    dist.init_process_group(args.dist_backend, init_method="env://", rank=env["rank"], world_size=env["world"],
                            timeout=DIST_TIMEOUT)
    try:
        return Trainer(cfg, dev, grad_sync=GradSync()).run(exit_after=args.exit_after, max_it=args.max_it)
    finally:
        dist.destroy_process_group()


if __name__ == "__main__":
    sys.exit(main())
