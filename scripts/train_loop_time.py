"""Time the training loop's pieces: ops.chamfer_distance (csrc/chamfer.cu) at 8000 ground-truth points against 5 000,
100 000 and 1 000 000 model points with normals, next to a torch brute force (torch.cdist in chunks on the GPU), and the
loop of dss_b200.training.train at configs/dss.yml's settings (512^2 views) at each size of ``--points`` / ``--batch``
(by default 5 000 points with 8 views per batch, and 1 000 000 with 64), next to three arms on the same batches, in the
same process, each over ``--loop-its`` iterations:

  replay    -- bare GraphedTrainStep.replay() of a batch already loaded;
  staged    -- MVRData.pinned_batch, the non-blocking upload, load() and replay(): the loop before its views were
               resident on the device;
  resident  -- load_views() and replay() of the loop's own step (GraphedTrainStep.from_views): what the loop does.

    python scripts/train_loop_time.py [--iters 20] [--loop-its 200] [--points 5000 1000000] [--batch 8 64]
                                      [--ranks G] [--no-chamfer] [--out results.json]

CUDA events around each chamfer call, median after warm-up.  The arms are host wall-clock rates between two device
synchronisations.  The loop's rate is taken between two of its own logged records (each ends in a host
synchronisation), after the capture and a warm-up.  ``--ranks G`` > 1 runs the loop as G NCCL ranks, one process and
one GPU each, started with torchrun's variables (the view-sharded eager step; no arms), and reports rank 0's rate; a G
larger than the number of visible GPUs is refused.  The data has max(64, batch) views.  Prints one JSON line with the
card name and its power limit."""
import argparse
import json
import os
import shutil
import signal
import socket
import subprocess
import sys
import tempfile
import time

import torch
import torch.nn.functional as F
import yaml

from timing import card, median_ms
from dss_b200.ops import chamfer_distance


def torch_chamfer(x, y, xn, yn, budget=1 << 28):
    """pytorch3d's chamfer_distance (mean, mean) for one cloud each, as chunked torch.cdist on the device"""
    def one_way(q, p, qn, pn):
        chunk = max(1, budget // p.shape[0])
        d, c = [], []
        for s in range(0, q.shape[0], chunk):
            m, a = (torch.cdist(q[s:s + chunk], p) ** 2).min(1)
            d.append(m)
            c.append(1 - F.cosine_similarity(qn[s:s + chunk], pn[a], dim=1, eps=1e-6).abs())
        return torch.cat(d).mean(), torch.cat(c).mean()
    dx, cx = one_way(x, y, xn, yn)
    dy, cy = one_way(y, x, yn, xn)
    return dx + dy, cx + cy


def chamfer_times(dev, warmup, iters):
    g = torch.Generator().manual_seed(0)
    gt = F.normalize(torch.randn(8000, 3, generator=g), dim=1).to(dev)
    gtn = gt.clone()
    out = {}
    for P in (5000, 100000, 1000000):
        y = (F.normalize(torch.randn(P, 3, generator=g), dim=1) * 0.9 + 0.01 * torch.randn(P, 3, generator=g)).to(dev)
        yn = F.normalize(torch.randn(P, 3, generator=g), dim=1).to(dev)
        ours = chamfer_distance(gt[None], y[None], x_normals=gtn[None], y_normals=yn[None])
        ref = torch_chamfer(gt, y, gtn, yn)
        out["chamfer_ms_8000x%d" % P] = median_ms(
            lambda: chamfer_distance(gt[None], y[None], x_normals=gtn[None], y_normals=yn[None]), warmup, iters)
        out["torch_cdist_ms_8000x%d" % P] = median_ms(lambda: torch_chamfer(gt, y, gtn, yn), 1, max(3, iters // 4))
        out["rel_diff_8000x%d" % P] = [float((ours[k] - ref[k]).abs() / ref[k].abs()) for k in (0, 1)]
    return out


def _run_ranks(cfg_path, ranks, max_it, tmp, timeout=3600):
    """the loop as ``ranks`` NCCL ranks, one GPU each, as torchrun starts them, each in its own session with its
    output in a file under ``tmp``.  When a rank fails or the time runs out every rank still running is killed, so
    none is left waiting at a collective; raises then."""
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    procs, logs = [], []
    for r in range(ranks):
        env = dict(os.environ, RANK=str(r), LOCAL_RANK=str(r), WORLD_SIZE=str(ranks), LOCAL_WORLD_SIZE=str(ranks),
                   MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        env["PYTHONPATH"] = root + os.pathsep + env.get("PYTHONPATH", "")
        logs.append(open(os.path.join(tmp, "rank%d.log" % r), "w+"))
        procs.append(subprocess.Popen([sys.executable, "-m", "dss_b200.training.train", "--config", cfg_path,
                                       "--exit-after", "-1", "--max-it", str(max_it), "--dist-backend", "nccl"],
                                      cwd=root, env=env, stdout=logs[-1], stderr=subprocess.STDOUT,
                                      start_new_session=True))
    deadline = time.time() + timeout
    try:
        while any(p.poll() is None for p in procs):
            if any(p.poll() not in (None, 0) for p in procs) or time.time() > deadline:
                break
            time.sleep(0.2)
    finally:
        for p in procs:
            if p.poll() is None:
                os.killpg(p.pid, signal.SIGKILL)
                p.wait()
    for r, (p, log) in enumerate(zip(procs, logs)):
        log.seek(0)
        out = log.read()
        log.close()
        if p.returncode != 0:
            raise RuntimeError("rank %d exited with %d:\n%s" % (r, p.returncode, out))


def loop_times(dev, loop_its, tmp, points=5000, batch=8, ranks=1):
    from dss_b200.training.config import load_config
    from dss_b200.training.train import Trainer
    from dss_b200.utils.create_mvr_data import main as create
    from dss_b200.utils.io import save_obj
    from tests.test_mesh_data import torus
    verts, faces = torus(nu=192, nv=96)
    save_obj(os.path.join(tmp, "torus.obj"), verts.numpy(), faces.numpy())
    n_views = max(64, batch)
    data_dir = create(["--points", os.path.join(tmp, "torus.obj"), "--output", os.path.join(tmp, "data"),
                       "--num_cameras", str(n_views), "--image-size", "512", "--tri_color_light", "--point_lights"])[0]
    cfg_path = os.path.join(tmp, "dss.yml")
    warm = 40
    with open(cfg_path, "w") as f:
        yaml.safe_dump({
            "name": "time", "data": {"data_dir": data_dir},
            "model": {"model_kwargs": {"n_points_per_cloud": points, "learn_colors": False}},
            "renderer": {"raster_params": {"Vrk_invariant": True, "Vrk_isotropic": False, "clip_pts_grad": 0.05,
                                           "cutoff_threshold": 1.0, "depth_merging_threshold": 0.05,
                                           "image_size": 512, "points_per_pixel": 5, "radii_backward_scaler": 5}},
            "training": {"out_dir": os.path.join(tmp, "out"), "batch_size": batch, "lambda_dr_proj": 0.01,
                         "lambda_dr_repel": 0.0, "steps_dss_backward_radii": 200, "print_every": warm,
                         "validate_every": 0, "checkpoint_every": 0}}, f)
    cfg = load_config(cfg_path)
    t = None
    if ranks == 1:
        t = Trainer(cfg)
        t.run(exit_after=-1, max_it=warm + loop_its + 1)
    else:
        _run_ranks(cfg_path, ranks, warm + loop_its + 1, tmp)
    with open(os.path.join(cfg["training"]["out_dir"], "time", "metrics.jsonl")) as f:
        recs = [json.loads(line) for line in f]
    first = next(r for r in recs if r["it"] >= warm)
    last = recs[-1]
    res = {"ranks": ranks, "loop_points": points, "loop_batch": batch,
           "loop_it_per_s": (last["it"] - first["it"]) / (last["time"] - first["time"]),
           "loop_its_timed": last["it"] - first["it"]}
    if t is None:
        return res
    res.update(arm_rates(t, n_views, batch, loop_its))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ev = t.evaluate()
    res["validation_ms_%d_vs_8000" % points] = (time.perf_counter() - t0) * 1e3
    res["chamfer_point_at_end"] = ev["chamfer_point"]
    return res


def staged_batch(data, dev, proj_all, light_props, idx):
    """the views ``idx`` as the loop staged them before they were resident: pinned, uploaded without blocking"""
    b = data.pinned_batch(idx)
    idx_dev = torch.tensor(idx, dtype=torch.int64).pin_memory().to(dev, non_blocking=True)
    img = b["img.rgb"].to(dev, non_blocking=True).permute(0, 2, 3, 1)
    mask = b["img.mask"].to(dev, non_blocking=True)[:, 0]
    view = b["camera_mat"].to(dev, non_blocking=True)
    light_cls, props = light_props
    lights = light_cls(**{k: v.index_select(0, idx_dev) for k, v in props.items()}, device=dev)
    return img, mask, proj_all.index_select(0, idx_dev), view, lights


def arm_rates(t, n_views, batch, loop_its):
    """it/s of the three arms on the same batches (the loop's last epoch order, cut into batches)"""
    from dss_b200.core.camera import camera_matrices
    from dss_b200.training.step import GraphedTrainStep
    dev, data, resident = t.dev, t.data, t.step
    proj_all = camera_matrices(data.get_cameras())[0].to(dev)
    light_props = data.light_props(dev)
    batches = [t.order[i:i + batch] for i in range(0, n_views - batch + 1, batch)]
    stage = lambda idx: staged_batch(data, dev, proj_all, light_props, idx)
    s = dict(t.settings)
    learn, s["lambda_dr_proj"] = s.pop("learn"), t.lambda_dr_proj
    staged = GraphedTrainStep(resident.points.detach(), resident.normals.detach(), resident.colours.detach(), t.params,
                              *stage(batches[0]), learn=learn, **s)
    arms = {
        "replay": lambda idx: staged.replay(),
        "staged": lambda idx: (staged.load(*stage(idx)), staged.replay()),
        "resident": lambda idx: (resident.load_views(idx), resident.replay()),
    }
    out = {}
    for name, fn in arms.items():
        for idx in batches[:3]:
            fn(idx)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(loop_its):
            fn(batches[i % len(batches)])
        torch.cuda.synchronize()
        out["%s_it_per_s" % name] = loop_its / (time.perf_counter() - t0)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--loop-its", type=int, default=200)
    ap.add_argument("--points", type=int, nargs="+", default=[5000, 1000000], help="the loop's cloud sizes")
    ap.add_argument("--batch", type=int, nargs="+", default=[8, 64],
                    help="the loop's views per batch (over all the ranks), one per --points")
    ap.add_argument("--ranks", type=int, default=1, help="run the loop as this many NCCL ranks, one GPU each")
    ap.add_argument("--no-chamfer", action="store_true", help="time the loop alone")
    ap.add_argument("--out", default=None)
    opt = ap.parse_args()
    have = torch.cuda.device_count()
    if opt.ranks < 1 or opt.ranks > have:
        raise SystemExit("--ranks %d: the loop runs one rank per GPU and %d GPU%s visible"
                         % (opt.ranks, have, " is" if have == 1 else "s are"))
    if len(opt.points) != len(opt.batch):
        raise SystemExit("--points and --batch take one value per loop size")
    dev = torch.device("cuda:0")
    res = {} if opt.no_chamfer else chamfer_times(dev, opt.warmup, opt.iters)
    res["loops"] = []
    for points, batch in zip(opt.points, opt.batch):
        tmp = tempfile.mkdtemp(prefix="dss_loop_time_")
        try:
            res["loops"].append(loop_times(dev, opt.loop_its, tmp, points, batch, opt.ranks))
        finally:
            shutil.rmtree(tmp, ignore_errors=True)
        torch.cuda.empty_cache()
    gpu = card()
    res["card"], res["power_limit"] = gpu["name"], gpu["power_limit"]
    print(json.dumps(res))
    if opt.out:
        with open(opt.out, "w") as f:
            json.dump(res, f)


if __name__ == "__main__":
    main()
