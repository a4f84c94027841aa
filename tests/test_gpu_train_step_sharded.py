"""GPU tests of the view-sharded training step: ``TrainStep(..., grad_sync=GradSync())`` on 2 ranks, each with the
views ``assign_views`` deals it, against one ``TrainStep`` over all the views, on the bunny at configs/dss.yml's
settings (512², K = 5).  The ranks are 2 worker processes on one GPU over gloo, and, where two GPUs exist, on two GPUs
over NCCL.

What must hold, and why:
  - exact: ``visibility`` and ``inmask`` (ORs of bytes), the render of each view, the regularisers (replicated on the
    same cloud and filters) and the RGB part of the image-loss gradient that each rank feeds the render backward (its
    coefficient has M, an integer count, summed over the ranks).  The alpha part's IoU coefficients come from the
    per-view fp64 sums I_n, U_n, whose block partition follows the number of views a call holds, so an alpha entry may
    round to the neighbouring float: at most 1 ulp.
  - close: the image-loss scalars within a few float32 ulps (the same fp64 sums, added in another order); d points and
    d normals within 1e-5 of the largest gradient (the render gradients are summed over the views in another order).
  - the same bits on every rank: loss, filters, leaves and gradients after ``step()``, and the parameters after 10
    Adam steps.
"""
import os
import socket
import subprocess
import sys
import tempfile

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ADAM_LR = 1e-4
ADAM_STEPS = 10
# Adam's first steps move a component by about lr * sign(g), whatever |g| is; a component whose gradient is within
# rounding of zero could take the other sign in the sharded sum and so differ by 2 lr after one step.  Elsewhere the
# trajectories differ by the rounding of the gradients (1e-7 of the largest): 6e-8 after 10 steps at lr 1e-4 on an H100.
# The bound, 2 lr, allows one such flipped step and fails on a systematic difference.
ADAM_TOL = 2 * ADAM_LR

pytestmark = pytest.mark.gpu

_WORKER = r'''
import os, sys, torch, torch.distributed as dist
sys.path.insert(0, %(root)r)
rank, backend, out_dir, port = int(sys.argv[1]), sys.argv[2], sys.argv[3], int(sys.argv[4])
dev = torch.device("cuda", rank if backend == "nccl" else 0)
torch.cuda.set_device(dev)
dist.init_process_group(backend, init_method="tcp://127.0.0.1:%%d" %% port, rank=rank, world_size=2)
import dss_b200.training.step as step_mod
from dss_b200 import _lib
from dss_b200.core.lighting import DirectionalLights
from dss_b200.ops import SplatParams, render_points
from dss_b200.parallel import GradSync, assign_views, view_costs_from_cameras
from dss_b200.training.step import TrainStep
from dss_b200.utils.io import read_ply
from tests.util import GOLDEN_DIR, camera_matrices, random_cameras

# the gradient of the image that each step feeds the render backward
seen = []
_render = step_mod.render_points
def hooked(*a, **k):
    out = _render(*a, **k)
    out.image.register_hook(lambda g: seen.append(g.detach().clone()))
    return out
step_mod.render_points = hooked

ply = read_ply(os.path.join(GOLDEN_DIR, "ply", "bunny-8000.ply"))
pts = torch.as_tensor(ply["points"], dtype=torch.float32)
pts = (pts - pts.mean(0)) / (pts - pts.mean(0)).norm(dim=1).max() * 0.6
nrm = torch.nn.functional.normalize(torch.as_tensor(ply["normals"], dtype=torch.float32), dim=1)
col = torch.rand(pts.shape, generator=torch.Generator().manual_seed(3))
pts, nrm, col = pts.to(dev), nrm.to(dev), col.to(dev)
S = 512
prm = SplatParams(image_size=S, points_per_pixel=5, cutoff_threshold=1.0, depth_merging_threshold=0.05,
                  radii_backward_scaler=5.0, clip_pts_grad=0.05, znear=0.1)
F32 = torch.finfo(torch.float32).eps


def make_batch(N, seed, per_view, mask_kind):
    proj, view = (m.to(dev) for m in camera_matrices(random_cameras(N, seed, dist=(1.6, 2.2))))
    g = torch.Generator().manual_seed(seed)
    B = N if per_view else 1
    rows = [0.2 * torch.rand(B, 1, 3, generator=g), 0.5 * torch.rand(B, 1, 3, generator=g),
            0.1 * torch.rand(B, 1, 3, generator=g), torch.randn(B, 1, 3, generator=g)]
    with torch.no_grad():
        tgt = render_points(pts + 0.01 * torch.randn(3, generator=g).to(dev), nrm, col.flip(1), proj, view,
                            torch.full((N,), 1e-3, device=dev), prm).image
    img = tgt[..., :3].contiguous()
    mask = {"f32": (tgt[..., 3] > 0).float(), "u8": (tgt[..., 3] > 0).to(torch.uint8) * 255}[mask_kind]

    def lights(views):
        sel = (lambda t: t[list(views)]) if per_view else (lambda t: t)
        a, d, s, r = (sel(t) for t in rows)
        return DirectionalLights(ambient_color=a, diffuse_color=d, specular_color=s, direction=r, device=dev)
    return img, mask, proj, view, lights


def views_of(batch, views):
    img, mask, proj, view, lights = batch
    idx = torch.tensor(views, dtype=torch.long, device=dev)
    return img[idx], mask[idx], proj[idx], view[idx], lights(views)


def deal(proj, view):
    return assign_views(view_costs_from_cameras(view).tolist(), 2)[rank]


saved = {}
report = []
def case(name, N, seed, lam_repel=0.0, per_view=False, mask_kind="f32"):
    batch = make_batch(N, seed, per_view, mask_kind)
    mine = deal(batch[2], batch[3])
    kw = dict(lambda_dr_repel=lam_repel)
    seen.clear()
    single = TrainStep(pts, nrm, col, prm, **kw)
    single(*views_of(batch, range(N)))
    g_single = seen[-1]
    seen.clear()
    sharded = TrainStep(pts, nrm, col, prm, grad_sync=GradSync(), **kw)
    sharded(*views_of(batch, mine))
    torch.cuda.synchronize()
    assert torch.equal(sharded.visibility, single.visibility), name
    assert torch.equal(sharded.inmask, single.inmask), name
    assert single.inmask.any(), name
    alpha_diff = 0
    if mine:
        idx = torch.tensor(mine, dtype=torch.long, device=dev)
        assert torch.equal(sharded.image, single.image[idx]), name
        g, gs = seen[-1], g_single[idx]
        assert torch.equal(g[..., :3], gs[..., :3]), name
        a, b = g[..., 3], gs[..., 3]
        ulp = (torch.nextafter(b.abs(), torch.full_like(b, float("inf"))) - b.abs())
        assert ((a - b).abs() <= ulp).all(), (name, float((a - b).abs().max()))
        alpha_diff = int((a != b).sum())
    else:
        assert seen == [] and sharded.image.shape == (0, S, S, 4)
    for k, v in single.loss.items():
        w, got = float(v), float(sharded.loss[k])
        tol = 0.0 if k in ("loss_dr_proj", "loss_dr_repel") else 4 * F32 * abs(w)
        assert abs(got - w) <= tol, (name, k, got, w)
    worst = []
    for got, want in ((sharded.points.grad, single.points.grad), (sharded.normals.grad, single.normals.grad)):
        scale = float(want.abs().max())
        err = float((got - want).abs().max())
        assert scale > 0 and err <= 1e-5 * scale, (name, err, scale)
        worst.append(err / scale)
    assert sharded.colours.grad is None
    report.append("%%s: views %%s, alpha gradient entries 1 ulp apart: %%d, d points / d normals: %%.2e / %%.2e of the "
                  "largest" %% (name, mine, alpha_diff, worst[0], worst[1]))
    saved[name] = {"loss": torch.stack([v.float() for v in sharded.loss.values()]).cpu(),
                   "vis": sharded.visibility.cpu(), "inm": sharded.inmask.cpu(),
                   "points": sharded.points.detach().cpu(), "normals": sharded.normals.detach().cpu(),
                   "gp": sharded.points.grad.cpu(), "gn": sharded.normals.grad.cpu()}
    return batch, mine


batch, mine = case("N=8", 8, 11)
case("N=5", 5, 12)
case("N=1", 1, 13)
case("repel", 8, 14, lam_repel=0.05)
case("per-view lights", 8, 15, per_view=True)
case("uint8 mask", 8, 16, mask_kind="u8")

# launches: the sharded step adds the image loss's finish and the gated filter pass to the step on the same views
local = TrainStep(pts, nrm, col, prm)
sharded = TrainStep(pts, nrm, col, prm, grad_sync=GradSync())
counts = []
for st in (local, sharded, local, sharded):
    st(*views_of(batch, mine))
    torch.cuda.synchronize()
    n0 = _lib.launch_count(dev)
    st(*views_of(batch, mine))
    torch.cuda.synchronize()
    counts.append(_lib.launch_count(dev) - n0)
assert counts[0] == counts[2] and counts[1] == counts[3] and counts[1] - counts[0] == 2, counts
report.append("library launches per step on %%d views: %%d on one GPU, %%d sharded" %% (len(mine), counts[0], counts[1]))

# a short training run: 10 Adam steps, sharded against one GPU
def train(sync, views):
    st = TrainStep(pts, nrm, col, prm, grad_sync=sync)
    opt = torch.optim.Adam([st.points, st.normals], lr=%(lr)r)
    for _ in range(%(steps)d):
        opt.zero_grad(set_to_none=True)
        st(*views_of(batch, views))
        opt.step()
    torch.cuda.synchronize()
    return st.points.detach(), st.normals.detach()

p1, n1 = train(None, list(range(8)))
p2, n2 = train(GradSync(), mine)
dev_p, dev_n = float((p2 - p1).abs().max()), float((n2 - n1).abs().max())
assert dev_p <= %(tol)r and dev_n <= %(tol)r, (dev_p, dev_n)
report.append("after %(steps)d Adam steps at lr %(lr)g: |points - one GPU| <= %%.3e, |normals - one GPU| <= %%.3e"
              %% (dev_p, dev_n))
saved["adam"] = {"points": p2.cpu(), "normals": n2.cpu()}
torch.save(saved, os.path.join(out_dir, "rank%%d.pt" %% rank))
dist.destroy_process_group()
print("\n".join(report))
print("rank", rank, "ok")
'''


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _run_workers(backend):
    with tempfile.TemporaryDirectory() as d:
        w = os.path.join(d, "worker.py")
        with open(w, "w") as f:
            f.write(_WORKER % {"root": ROOT, "lr": ADAM_LR, "steps": ADAM_STEPS, "tol": ADAM_TOL})
        env = dict(os.environ, PYTHONPATH=ROOT)
        port = _free_port()
        procs = [subprocess.Popen([sys.executable, w, str(r), backend, d, str(port)], stdout=subprocess.PIPE,
                                  stderr=subprocess.STDOUT, text=True, cwd=ROOT, env=env) for r in range(2)]
        try:
            outs = [p.communicate(timeout=900)[0] for p in procs]
        finally:
            for p in procs:
                if p.poll() is None:
                    p.kill()
                    p.wait()
        for r, (p, o) in enumerate(zip(procs, outs)):
            assert p.returncode == 0 and "rank %d ok" % r in o, o
        print(outs[0])
        saved = [torch.load(os.path.join(d, "rank%d.pt" % r)) for r in range(2)]
    # the same bits on every rank
    assert saved[0].keys() == saved[1].keys()
    for name in saved[0]:
        for k, t in saved[0][name].items():
            assert torch.equal(t, saved[1][name][k]), (name, k)


def test_sharded_train_step_on_two_gloo_ranks(cuda_device):
    _run_workers("gloo")


def test_sharded_train_step_on_two_gpus_over_nccl(cuda_device):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    _run_workers("nccl")


def test_grad_sync_of_world_size_one_gives_the_single_gpu_step(cuda_device):
    from dss_b200.ops import SplatParams
    from dss_b200.parallel import GradSync
    from dss_b200.training.step import GraphedTrainStep, TrainStep
    from tests.test_gpu_train_step import batch
    from tests.util import scene
    d = cuda_device
    P0, N, S = 20000, 4, 128
    pts, nrm, col, _, _, _ = scene(P0, N, seed=61)
    pts, nrm, col = pts.to(d), nrm.to(d), col.to(d)
    prm = SplatParams(image_size=S, points_per_pixel=5, znear=0.1, clip_pts_grad=0.05, radii_backward_scaler=5.0)
    b = batch(N, S, d, seed=62)
    sync = GradSync()
    assert sync.world_size == 1
    res = []
    for s in (None, sync):
        st = TrainStep(pts, nrm, col, prm, lambda_dr_repel=0.05, grad_sync=s)
        st(*b)
        torch.cuda.synchronize()
        res.append(st)
    a, c = res
    for k in a.loss:
        assert torch.equal(a.loss[k], c.loss[k]), k
    assert torch.equal(a.image, c.image) and torch.equal(a.visibility, c.visibility)
    assert torch.equal(a.inmask, c.inmask)
    # float atomics in the colour scatter feed the shading's position and normal gradients: two runs of one step agree
    # to their order, not to the bit
    torch.testing.assert_close(c.points.grad, a.points.grad, rtol=1e-4, atol=1e-9)
    torch.testing.assert_close(c.normals.grad, a.normals.grad, rtol=1e-4, atol=1e-9)
    assert sync.calls == 0 and sync.bytes_reduced == 0
    # the graphed step takes a world size of one as well
    GraphedTrainStep(pts, nrm, col, prm, *b, grad_sync=sync)
