"""Time of one view-sharded training step: ``TrainStep(..., grad_sync=GradSync())`` at G = 1, 2, 4 and 8 ranks, one
process and one GPU per rank over NCCL, at configs/dss.yml's settings (512², K = 5, Vrk_invariant, lambda_dr_proj =
0.01, learning points and normals) on the sphere of bench.py's scene, by default P0 = 1 000 000 points and 64 views
dealt by ``assign_views``.  G = 1 is the single-GPU step over all the views.  A G larger than the number of visible
GPUs is reported as not measured.

Each rank warms up, then times every step with CUDA events (host included: the step is eager); rank 0 reports the
median and range of its samples.  The collectives make every rank wait for the slowest, so rank 0's time is the step's.

    python scripts/train_step_sharded_time.py [--points 1000000] [--views 64] [--steps 20] [--warmup 3] [--gpus 1,2,4,8]
"""
import argparse
import os
import socket
import subprocess
import sys

import torch

from timing import card, events_ms, spread


def worker(a):
    import torch.distributed as dist
    from dss_b200.core.lighting import DirectionalLights
    from dss_b200.ops import SplatParams, render_points
    from dss_b200.parallel import GradSync, assign_views, view_costs_from_cameras
    from dss_b200.training.step import TrainStep
    from tests.util import scene

    rank, G = a.rank, a.world
    dev = torch.device("cuda", rank)
    torch.cuda.set_device(dev)
    if G > 1:
        dist.init_process_group("nccl", init_method="tcp://127.0.0.1:%d" % a.port, rank=rank, world_size=G)
    N, S, P0 = a.views, 512, a.points
    prm = SplatParams(image_size=S, points_per_pixel=5, cutoff_threshold=1.0, depth_merging_threshold=0.05,
                      radii_backward_scaler=5.0, clip_pts_grad=0.05, znear=0.1)
    pts, nrm, col, proj, view, _ = scene(P0, N, seed=0)
    pts, nrm, col, proj, view = (t.to(dev) for t in (pts, nrm, col, proj, view))
    g = torch.Generator().manual_seed(P0)
    rows = [0.2 * torch.rand(N, 1, 3, generator=g), 0.5 * torch.rand(N, 1, 3, generator=g),
            0.1 * torch.rand(N, 1, 3, generator=g), torch.randn(N, 1, 3, generator=g)]
    mine = assign_views(view_costs_from_cameras(view).tolist(), G)[rank]
    idx = torch.tensor(mine, dtype=torch.long, device=dev)
    with torch.no_grad():
        tgt = render_points(pts + 0.01 * torch.randn(3, generator=g).to(dev), nrm, col.flip(1), proj[idx], view[idx],
                            torch.full((len(mine),), 3e-4, device=dev), prm).image
    img = tgt[..., :3].contiguous()
    mask = (tgt[..., 3] > 0).float()
    lights = DirectionalLights(ambient_color=rows[0][mine], diffuse_color=rows[1][mine], specular_color=rows[2][mine],
                               direction=rows[3][mine], device=dev)
    step = TrainStep(pts, nrm, col, prm, grad_sync=GradSync() if G > 1 else None)
    batch = (img, mask, proj[idx], view[idx], lights)
    for _ in range(a.warmup):
        step(*batch)
    torch.cuda.synchronize()
    ms = [events_ms(lambda: step(*batch), 1) for _ in range(a.steps)]
    if rank == 0:
        print("RESULT %d %.3f %.3f %.3f %d" % (G, *spread(ms), len(mine)))
    if G > 1:
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=1000000)
    ap.add_argument("--views", type=int, default=64)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--gpus", default="1,2,4,8")
    ap.add_argument("--rank", type=int, default=-1)
    ap.add_argument("--world", type=int, default=1)
    ap.add_argument("--port", type=int, default=0)
    a = ap.parse_args()
    if a.rank >= 0:
        return worker(a)
    if not torch.cuda.is_available():
        sys.exit("train_step_sharded_time.py needs a CUDA device")
    have = torch.cuda.device_count()
    gpu = card()
    print("gpus: %d visible (%s, %s)" % (have, gpu["name"], gpu["power_limit"]))
    print("P0 = %d, %d views of 512^2, K = 5" % (a.points, a.views))
    for G in (int(x) for x in a.gpus.split(",")):
        if G > have:
            print("  G = %d: not measured (%d GPU%s visible)" % (G, have, "" if have == 1 else "s"))
            continue
        s = socket.socket()
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
        s.close()
        cmd = [sys.executable, os.path.abspath(__file__), "--points", str(a.points), "--views", str(a.views),
               "--steps", str(a.steps), "--warmup", str(a.warmup), "--world", str(G), "--port", str(port)]
        procs = [subprocess.Popen(cmd + ["--rank", str(r)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
                 for r in range(G)]
        try:
            outs = [p.communicate(timeout=1800)[0] for p in procs]
        finally:
            for p in procs:
                if p.poll() is None:
                    p.kill()
                    p.wait()
        line = [l for l in outs[0].splitlines() if l.startswith("RESULT")]
        if any(p.returncode for p in procs) or not line:
            print("  G = %d: failed\n%s" % (G, "\n".join(o[-2000:] for o in outs)))
            continue
        _, g, med, lo, hi, nv = line[0].split()
        print("  G = %s: %s ms/step median (%s-%s), %s views on rank 0" % (g, med, lo, hi, nv))


if __name__ == "__main__":
    main()
