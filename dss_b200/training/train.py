"""The training loop: the reference's ``train_mvr.py`` with its ``Trainer`` (train_mvr.py:66-230, DSS/training/
trainer.py:73-238) on :class:`GraphedTrainStep`, from a data directory to a trained cloud.

    python -m dss_b200.training.train --config CFG.yml [--exit-after S] [--max-it N]

- data: ``MVRData(data.data_dir)``, which is also the validation set.  Every epoch draws ``len(data)`` view indices
  with replacement from uniform weights (``WeightedSubsetRandomSampler``: ``torch.multinomial`` on the loop's own
  generator) and cuts them into batches of ``training.batch_size`` views, the last partial batch dropped.  A batch is
  staged in pinned memory (``MVRData.pinned_batch``) and uploaded without blocking; its lights are the per-image
  ``lights_%d`` entries.
- model: ``model.model_kwargs.n_points_per_cloud`` area-weighted samples of ``ico_sphere(4)`` scaled by 0.5 with their
  face normals and albedo ones (config.py:177-183), drawn from ``training.seed``.
- optimizer: Adam, betas (0.5, 0.9), one group per learnt tensor: normals lr 0.01, points lr 0.01, colours lr 1.0
  (train_mvr.py:83-95); ``MultiStepLR(scheduler_milestones, scheduler_gamma)`` stepped after every epoch.
- before every step the reference Trainer's ``TrainerScheduler`` (scheduler.py:36-53 with the arguments of
  trainer.py:114-123): see :func:`radii_backward_scaler` and :func:`compound_lambda_proj`.
- every ``print_every`` iterations the losses go to ``<out>/<logfile>`` and one JSON line to ``<out>/metrics.jsonl``
  (the loop's only host synchronisations besides validation); every ``validate_every`` (it > 0) the chamfer distances
  of the ground-truth cloud against the current one (trainer.py:144-171), and on improvement of
  ``training.model_selection_metric`` ``model_best.pt`` and ``val/best.ply``.  With the metric ``p2f_avg`` the loop
  reads ``<data_dir>/mesh.obj`` once (it must exist) and every validation adds ``p2f_avg`` / ``p2f_std``, the mean and
  population standard deviation of the exact distances of the cloud's points to that mesh; ``model.pt`` every ``checkpoint_every``, ``model_%d.pt`` every ``backup_every``.
- ``training.resume_from`` (in ``<out>``) is loaded when it exists, and the run continues where it stopped, mid-epoch
  included: a resumed run computes what an uninterrupted one does.  (The reference starts a new epoch.)
- ``--exit-after S`` saves ``model.pt`` and exits with status 3 once S seconds have passed (checked after every
  iteration; a negative S never exits); ``--max-it N`` saves ``model.pt`` and exits 0 after iteration N - 1.
"""
import argparse
import json
import math
import os
import sys
import time

import torch
import torch.nn.functional as F
import yaml

from ..core.camera import camera_matrices
from ..core.cloud import PointClouds3D
from ..core.lighting import DirectionalLights, PointLights
from ..ops import chamfer_distance
from ..utils.create_mvr_data import ico_sphere, sample_points_from_mesh
from ..utils.dataset import MVRData
from ..utils.evaluate import p2f_stats
from ..utils.io import read_mesh, save_ply
from .config import check_config, load_config, selection_metric, splat_params, step_settings
from .step import GraphedTrainStep

__all__ = ["radii_backward_scaler", "compound_lambda_proj", "initial_cloud", "make_optimizer", "make_lr_scheduler",
           "ground_truth_cloud", "Trainer", "main"]

EXIT_TIME_LIMIT = 3        # train_mvr.py:221-227
EVAL_SEED = 0              # the fixed draw of the ground-truth samples


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


def make_optimizer(tensors):
    """train_mvr.py:83-95: Adam, betas (0.5, 0.9), groups in the reference's order for the tensors that require grad:
    normals lr 0.01, points lr 0.01, colours lr 1.0.  ``tensors``: {"points", "normals", "colours"}."""
    groups = [{"params": [tensors[name]], "lr": lr, "betas": (0.5, 0.9)}
              for name, lr in (("normals", 0.01), ("points", 0.01), ("colours", 1.0)) if tensors[name].requires_grad]
    if not groups:
        raise ValueError("nothing to learn: model.model_kwargs sets every learn_* false")
    return torch.optim.Adam(groups, lr=0.01, betas=(0.5, 0.9))


def make_lr_scheduler(optimizer, cfg):
    """train_mvr.py:128-130: MultiStepLR over epochs, stepped once after every epoch."""
    tr = cfg["training"]
    return torch.optim.lr_scheduler.MultiStepLR(optimizer, list(tr["scheduler_milestones"]),
                                                gamma=float(tr["scheduler_gamma"]))


def ground_truth_cloud(data, data_dir, n_eval_points, device):
    """(points, normals) the validation measures against: the stored cloud when ``n_eval_points`` <= 0 or equals its
    size, otherwise ``n_eval_points`` area-weighted samples of ``<data_dir>/mesh.obj`` drawn once from a fixed seed.
    (The reference samples the mesh with pymeshlab's Poisson-disk sampling, so absolute values differ from its own.)"""
    stored = data.get_pointclouds()
    n = int(n_eval_points)
    if n <= 0 or n == stored.points_packed().shape[0]:
        return stored.points_packed().to(device), stored.normals_packed().to(device)
    verts, faces = read_mesh(os.path.join(data_dir, "mesh.obj"))
    g = torch.Generator(device=device).manual_seed(EVAL_SEED)
    return sample_points_from_mesh(torch.from_numpy(verts).float().to(device), torch.from_numpy(faces).long().to(device),
                                   n, generator=g)


class _Log:
    """lines to ``<out>/<logfile>`` (and stdout), JSON records to ``<out>/metrics.jsonl``"""

    def __init__(self, out_dir, logfile):
        self.text = open(os.path.join(out_dir, logfile), "a")
        self.metrics = open(os.path.join(out_dir, "metrics.jsonl"), "a")

    def info(self, msg):
        line = "%s %s" % (time.strftime("%Y-%m-%d %H:%M:%S"), msg)
        print(line, flush=True)
        self.text.write(line + "\n")
        self.text.flush()

    def record(self, rec):
        self.metrics.write(json.dumps(rec) + "\n")
        self.metrics.flush()

    def close(self):
        self.text.close()
        self.metrics.close()


class Trainer:
    """The loop's state and one iteration at a time (see the module docstring).  ``Trainer(cfg).run(exit_after,
    max_it)`` returns the process exit status."""

    def __init__(self, cfg, device="cuda"):
        self.cfg = cfg
        self.dev = torch.device(device)
        tr, dc = cfg["training"], cfg["data"]
        self.out_dir = os.path.join(str(tr["out_dir"]), str(cfg["name"]))
        self.val_dir = os.path.join(self.out_dir, "val")
        os.makedirs(self.val_dir, exist_ok=True)
        self.log = _Log(self.out_dir, tr["logfile"])
        # ---- data: images in host memory, cameras and lights of every view on the device
        self.data = MVRData(dc["data_dir"], data_dict=dc["data_dict"], n_imgs=dc["n_imgs"], img_folder=dc["img_folder"],
                            mask_folder=dc["mask_folder"], img_extension=dc["img_extension"],
                            mask_extension=dc["mask_extension"])
        if self.data.images is None or self.data.masks is None:
            raise ValueError("%s has no images and masks" % dc["data_dir"])
        V = len(self.data)
        lights = [self.data[i].get("lights") for i in range(V)]
        check_config(cfg, self.data.resolution, all(l is not None for l in lights))
        self.mesh = None
        if selection_metric(cfg) == "p2f_avg":
            mesh_path = os.path.join(dc["data_dir"], "mesh.obj")
            if not os.path.isfile(mesh_path):
                raise ValueError("model_selection_metric p2f_avg measures against %s, which does not exist" % mesh_path)
            verts, faces = read_mesh(mesh_path)
            self.mesh = (torch.from_numpy(verts).float().to(self.dev), torch.from_numpy(faces).to(self.dev))
        kind = str(self.data.data_dict["lights_type"]) if "lights_type" in self.data.data_dict else ""
        self.light_cls = PointLights if "PointLights" in kind else DirectionalLights
        vec = "location" if self.light_cls is PointLights else "direction"
        self.light_props = {k: torch.stack([torch.as_tensor(l[src]) for l in lights]).to(self.dev)
                            for k, src in (("ambient_color", "ambient_color"), ("diffuse_color", "diffuse_color"),
                                           ("specular_color", "specular_color"), (vec, vec))}
        cams = self.data.get_cameras()
        proj, _ = camera_matrices(cams)
        self.proj_all = proj.to(self.dev)
        self.params = splat_params(cfg, cams.znear, cams.zfar)
        self.settings = step_settings(cfg)
        self.batch_size = int(tr["batch_size"])
        if V // self.batch_size < 1:
            raise ValueError("batch_size %d is larger than the %d views: an epoch would have no batch"
                             % (self.batch_size, V))
        self.gt = ground_truth_cloud(self.data, dc["data_dir"], tr["n_eval_points"], self.dev)
        # ---- state: fresh, then whatever the checkpoint holds
        self.gen = torch.Generator().manual_seed(int(tr["seed"]))
        self.epoch_it, self.it, self.order, self.pos = -1, -1, None, 0
        self.sign = {"minimize": -1, "maximize": 1}.get(tr["model_selection_mode"])
        if self.sign is None:
            raise ValueError("model_selection_mode must be either maximize or minimize.")
        self.best = -self.sign * math.inf
        self.radii_init = self.params.radii_backward_scaler
        self.lambda_dr_proj = self.settings["lambda_dr_proj"]
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
            self.log.info("resumed from %s at it=%d, epoch %d" % (ckpt_path, self.it, self.epoch_it))
        with open(os.path.join(self.out_dir, "config.yaml"), "w") as f:
            yaml.safe_dump(cfg, f, sort_keys=False)
        # the step is captured on any batch of the right shape: the capture's warm-up steps leave the cloud unchanged,
        # and every iteration loads its own batch first
        self._build(points, normals, colours, self._batch(list(range(self.batch_size))), ckpt)

    # ---- pieces ------------------------------------------------------------------------------------------------------
    def _batch(self, idx):
        """the views ``idx`` on the device, uploaded from pinned memory without blocking"""
        b = self.data.pinned_batch(idx)
        idx_dev = torch.tensor(idx, dtype=torch.int64).pin_memory().to(self.dev, non_blocking=True)
        img = b["img.rgb"].to(self.dev, non_blocking=True).permute(0, 2, 3, 1)
        mask = b["img.mask"].to(self.dev, non_blocking=True)[:, 0]
        view = b["camera_mat"].to(self.dev, non_blocking=True)
        proj = self.proj_all.index_select(0, idx_dev)
        lights = self.light_cls(**{k: v.index_select(0, idx_dev) for k, v in self.light_props.items()},
                                device=self.dev)
        return img, mask, proj, view, lights

    def _build(self, points, normals, colours, batch, ckpt):
        s = dict(self.settings)
        learn, s["lambda_dr_proj"] = s.pop("learn"), self.lambda_dr_proj
        self.step = GraphedTrainStep(points, normals, colours, self.params, *batch, learn=learn, **s)
        self.opt = make_optimizer({"points": self.step.points, "normals": self.step.normals,
                                   "colours": self.step.colours})
        self.lr_sched = make_lr_scheduler(self.opt, self.cfg)
        if ckpt is not None:
            self.opt.load_state_dict(ckpt["optimizer"])
            self.lr_sched.load_state_dict(ckpt["lr_scheduler"])

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
        p2f_avg, also the mean and population standard deviation of the points' distances to the data's mesh"""
        points, normals = self.cloud()
        with torch.no_grad():
            cd_p, cd_n = chamfer_distance(PointClouds3D([self.gt[0]], [self.gt[1]]), PointClouds3D([points], [normals]))
        ev = {"chamfer_point": float(cd_p), "chamfer_normal": float(cd_n)}
        if self.mesh is not None:
            _, ev["p2f_avg"], ev["p2f_std"] = p2f_stats(points, self.mesh)
        return ev

    def save(self, name):
        s = self.step
        P0 = s.points.shape[0]
        torch.save({
            "model": {"points": s.points.detach()[None].clone(), "normals": s.normals.detach()[None].clone(),
                      "colors": s.colours.detach()[None].clone(),
                      "points_activation": torch.ones((1, P0), dtype=torch.bool, device=self.dev)},
            "optimizer": self.opt.state_dict(), "lr_scheduler": self.lr_sched.state_dict(),
            "epoch_it": self.epoch_it, "it": self.it, "loss_val_best": self.best,
            "schedule": {"radii_backward_scaler": self.params.radii_backward_scaler,
                         "lambda_dr_proj": self.lambda_dr_proj},
            "sampler": self.gen.get_state(), "epoch_order": list(self.order), "epoch_pos": self.pos,
        }, os.path.join(self.out_dir, name))

    # ---- the loop ----------------------------------------------------------------------------------------------------
    def run(self, exit_after=600.0, max_it=None):
        tr = self.cfg["training"]
        print_every, checkpoint_every = int(tr["print_every"]), int(tr["checkpoint_every"])
        backup_every, validate_every = int(tr["backup_every"]), int(tr["validate_every"])
        metric = tr["model_selection_metric"]
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
                self._schedule()
                self.step.load(*self._batch(idx))
                if self.step.stale():
                    self.step.capture()
                loss = self.step.replay()
                self.opt.step()
                it = self.it
                if print_every > 0 and it % print_every == 0:
                    vals = {k: float(v) for k, v in loss.items()}
                    self.log.info("[Epoch %02d] it=%03d, loss=%.4f, time=%.4f " % (self.epoch_it, it, vals["loss"],
                                                                                   time.time() - t0b)
                                  + " ".join("%s=%.4g" % kv for kv in vals.items() if kv[0] != "loss"))
                    self.log.record(dict(it=it, epoch=self.epoch_it, time=time.time() - t0, **vals))
                    t0b = time.time()
                if it > 0 and checkpoint_every > 0 and it % checkpoint_every == 0:
                    self.log.info("Saving checkpoint")
                    self.save("model.pt")
                if it > 0 and backup_every > 0 and it % backup_every == 0:
                    self.log.info("Backup checkpoint")
                    self.save("model_%d.pt" % it)
                if it > 0 and validate_every > 0 and it % validate_every == 0:
                    ev = self.evaluate()
                    self.log.info("Validation metric (%s): %.4g  (%s)" % (metric, ev[metric], json.dumps(ev)))
                    if self.sign * (ev[metric] - self.best) > 0:
                        self.best = ev[metric]
                        self.log.info("New best model (loss %.4g)" % self.best)
                        self.save("model_best.pt")
                        points, normals = self.cloud()
                        save_ply(os.path.join(self.val_dir, "best.ply"), points.cpu().numpy(),
                                 normals=normals.cpu().numpy())
                if exit_after is not None and exit_after >= 0 and time.time() - t0 >= exit_after:
                    self.log.info("Time limit reached. Exiting.")
                    self.save("model.pt")
                    return EXIT_TIME_LIMIT
            self.save("model.pt")
            return 0
        finally:
            self.log.close()


def main(argv=None):
    p = argparse.ArgumentParser(description="Train a point cloud from a multi-view data directory (train_mvr.py).")
    p.add_argument("--config", required=True, help="YAML configuration (inherit_from chains over the defaults)")
    p.add_argument("--exit-after", type=float, default=600,
                   help="save model.pt and exit with status 3 after this many seconds (negative: never)")
    p.add_argument("--max-it", type=int, default=None, help="save model.pt and exit 0 after this many iterations")
    args = p.parse_args(argv)
    if not torch.cuda.is_available():
        raise RuntimeError("the training loop needs a CUDA device (sm_90a)")
    cfg = load_config(args.config)
    return Trainer(cfg).run(exit_after=args.exit_after, max_it=args.max_it)


if __name__ == "__main__":
    sys.exit(main())
