"""GPU: the dense depth of the splat blend (render_points(..., depth=True)) and the fused depth loss.

What must hold:
  - D equals the float64 restatement (tests/depth_oracle.py) on the render's own idx / weights / records, within float32
    rounding of a k-order sum, for shared, packed and anisotropic clouds and S = 1;
  - its gradient is the z-buffer gradient g_D w_k of every listed slot: positions, view / proj and pose gradients
    against float64 (tests/util.render_backward_f64, the view-depth sum p_h g_z, tests/pose_oracle.pose_map) within
    1e-5 of the largest, on shared, packed, anisotropic and S = 1 renders; an empty view gets zeros;
  - the depth backward gives the same bits twice and from a CUDA graph replay; with depth=False every output and
    gradient keeps its bits;
  - the fused loss equals the torch body in float64, including M = 0, non-finite and out-of-range ground truth, and the
    2-rank sharded loss equals the one-GPU loss."""
import os
import sys

import numpy as np
import pytest
import torch

from dss_b200.ops import SplatParams, local_frames, pose_cameras, render_points
from dss_b200.training.losses import depth_loss, depth_loss_torch
from tests import depth_oracle as O
from tests.util import packed_offsets, render_backward_f64_of, scene

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _case(kind, S=48, P0=1500, N=3):
    pts, nrm, col, proj, view, _ = scene(P0, N, seed=4)
    prm = SplatParams(image_size=S, points_per_pixel=5, znear=0.1, clip_pts_grad=-1.0)
    kw = dict(h=torch.full((N,), 3e-4, device=DEV))
    cols = col.repeat(N, 1).to(DEV)
    first = num = None
    if kind == "packed":
        first, num = packed_offsets(N, P0)
        num = num.clone()
        num[1] = 0                                            # an empty view
        pts, nrm = pts.repeat(N, 1), nrm.repeat(N, 1)
        first, num = first.to(DEV), num.to(DEV)
    if kind == "aniso":
        kw = dict(h=None, frames=local_frames(pts.to(DEV)))
    return pts.to(DEV), nrm.to(DEV), cols, proj.to(DEV), view.to(DEV), prm, kw, first, num


def _render(kind, S=48, requires=(), **extra):
    pts, nrm, cols, proj, view, prm, kw, first, num = _case(kind, S)
    p = pts.clone().requires_grad_(True)
    pr, vw = proj.clone().requires_grad_("cams" in requires), view.clone().requires_grad_("cams" in requires)
    out = render_points(p, nrm, cols, pr, vw, kw.pop("h"), prm, first, num, shared_cloud=kind != "packed",
                        return_fragments=True, **kw, **extra)
    return out, p, pr, vw, prm, first, num


@pytest.mark.parametrize("kind,S", [("shared", 48), ("packed", 48), ("aniso", 48), ("shared", 1)])
def test_depth_map_against_the_oracle(cuda_device, kind, S):
    out, *_ = _render(kind, S, depth=True)
    idx, w, z = (t.cpu().numpy() for t in (out.idx, out.weights, out.records[:, 2]))
    want = O.depth_map(idx, w, z)
    D = out.depth.detach().cpu().numpy().astype(np.float64)
    # float32 rounding of a k-order sum of K products
    bound = 4 * 5 * np.finfo(np.float32).eps * (np.abs(w) * np.abs(z[np.maximum(idx, 0)])).sum(-1) + 1e-30
    assert (np.abs(D - want) <= bound).all()
    assert (D[idx[..., 0] < 0] == 0).all()


def _view_grad_f64(ref, pts, N, first, num):
    """d L / d view (N,4,4) float64 from the reference's clipped NDC gradients: only column 2 (the view depth),
    grad_view[n][r][2] = sum over view n's slots of p_h[r] g_z"""
    shared = first is None
    P0 = pts.shape[0]
    fi = np.arange(N) * P0 if shared else first.cpu().numpy()
    nu = np.full(N, P0) if shared else num.cpu().numpy()
    pts = pts.detach().cpu().numpy().astype(np.float64)
    gv = np.zeros((N, 4, 4))
    for n in range(N):
        f, m = int(fi[n]), int(nu[n])
        p = pts[:m] if shared else pts[f:f + m]
        ph = np.concatenate([p, np.ones((m, 1))], 1)
        gv[n, :, 2] = ph.T @ ref["ndc"][f:f + m, 2]
    return gv


@pytest.mark.parametrize("kind,S", [("shared", 48), ("packed", 48), ("aniso", 48), ("shared", 1)])
def test_gradients_against_float64(cuda_device, kind, S):
    out, p, pr, vw, prm, first, num = _render(kind, S, requires=("cams",), depth=True)
    g = torch.randn(out.depth.shape, generator=torch.Generator().manual_seed(1)).to(DEV)
    (out.depth * g).sum().backward()
    # the depth gradient is a z-buffer gradient g_D w_k on every slot, summed in float64 by the reference
    gz = (g[..., None] * out.weights).detach()
    ref = render_backward_f64_of(out, p.detach(), pr.detach(), vw.detach(), prm, torch.zeros_like(out.image), gz,
                                 first, num)
    got = p.grad.cpu().numpy().astype(np.float64)
    scale = np.abs(ref["world"]).max()
    assert scale > 0 or S == 1
    assert np.abs(got - ref["world"]).max() <= 1e-5 * scale
    if kind == "packed":                                       # view 1 is empty: its rows and its cameras get zeros
        f, n = int(first[1]), int(first[2])
        assert (got[f:n] == 0).all()
        assert (vw.grad[1] == 0).all()
    # the depth moves the view depth only: proj (screen x, y) receives nothing, view only its depth column
    gv = _view_grad_f64(ref, p, out.depth.shape[0], first, num)
    assert pr.grad.abs().max() == 0 and vw.grad[:, :, [0, 1, 3]].abs().max() == 0
    got_v = vw.grad.cpu().numpy().astype(np.float64)
    assert np.abs(got_v - gv).max() <= 1e-5 * np.abs(gv).max()
    assert np.abs(gv).max() > 0 or S == 1


def test_pose_gradient_against_float64(cuda_device):
    from tests.pose_oracle import pose_map
    pts, nrm, cols, proj, view, prm, kw, _, _ = _case("shared")
    idx = torch.tensor([0, 2, 1], device=DEV)
    poses = (torch.randn(3, 6, generator=torch.Generator().manual_seed(5)) * 1e-3).to(DEV).requires_grad_(True)
    v, pr = pose_cameras(poses, idx, view, proj)
    out = render_points(pts, nrm, cols, pr, v, kw["h"], prm, return_fragments=True, depth=True)
    g = torch.randn(out.idx.shape[:3], generator=torch.Generator().manual_seed(3)).to(DEV)
    (out.depth * g).sum().backward()
    gz = (g[..., None] * out.weights).detach()
    ref = render_backward_f64_of(out, pts, pr.detach(), v.detach(), prm, torch.zeros_like(out.image), gz)
    gv = torch.from_numpy(_view_grad_f64(ref, pts, 3, None, None))
    p64 = poses.detach().cpu().double().requires_grad_(True)
    v64, pr64 = pose_map(p64, idx.cpu(), view.cpu(), proj.cpu())
    want, = torch.autograd.grad([v64, pr64], p64, [gv, torch.zeros_like(pr64)])
    assert want.abs().max() > 0
    assert (poses.grad.cpu().double() - want).abs().max() <= 1e-5 * want.abs().max()


def test_depth_backward_is_deterministic_and_replays(cuda_device):
    pts, nrm, cols, proj, view, prm, kw, _, _ = _case("shared")
    g = torch.randn(3, 48, 48, generator=torch.Generator().manual_seed(4)).to(DEV)
    p = pts.clone().requires_grad_(True)

    def run():
        p.grad = None
        out = render_points(p, nrm, cols, proj, view, kw["h"], prm, depth=True)
        (out.depth * g).sum().backward()
        return out.depth.detach().clone(), p.grad.clone()

    d1, g1 = run()
    d2, g2 = run()
    assert torch.equal(d1, d2) and torch.equal(g1, g2)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            run()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        p.grad = None
        out = render_points(p, nrm, cols, proj, view, kw["h"], prm, depth=True)
        (out.depth * g).sum().backward()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out.depth, d1) and torch.equal(p.grad, g1)


@pytest.mark.parametrize("kind", ["shared", "packed", "aniso"])
def test_depth_false_keeps_every_bit(cuda_device, kind):
    res = []
    for extra in ({}, {"depth": False}, {"depth": True}):
        out, p, pr, vw, *_ = _render(kind, requires=("cams",), **extra)
        g = torch.randn(out.image.shape, generator=torch.Generator().manual_seed(6)).to(DEV)
        out.image.backward(g)
        res.append((out, p.grad, pr.grad, vw.grad))
    # packed rows no view range covers hold no records (their memory is not written)
    first, num = _case(kind)[7:]
    rows = torch.ones(res[0][0].records.shape[0], dtype=torch.bool, device=DEV)
    if first is not None:
        rows[:] = False
        for f, m in zip(first.tolist(), num.tolist()):
            rows[f:f + m] = True
    for other in res[1:]:
        for name in ("image", "idx", "weights", "visible", "zbuf", "qvalue"):
            assert torch.equal(getattr(res[0][0], name), getattr(other[0], name)), name
        for name in ("records", "scaler"):
            assert torch.equal(getattr(res[0][0], name)[rows], getattr(other[0], name)[rows]), name
        for x, y in zip(res[0][1:], other[1:]):
            assert torch.equal(x, y)
    assert res[0][0].depth is None and res[1][0].depth is None


def _loss_inputs(N=3, S=40, seed=0, mask_dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    depth = torch.rand(N, S, S, generator=g) * 4 + 1
    gt = depth + torch.randn(N, S, S, generator=g) * 0.3
    gt[0, 0, :3] = torch.tensor([float("nan"), float("inf"), -float("inf")])
    gt[0, 1, :4] = torch.tensor([0.5, 10.0, 0.1, 50.0])
    gt[1, 2, 2] = depth[1, 2, 2]
    rgba = torch.rand(N, S, S, 4, generator=g)
    rgba[..., 3] = (rgba[..., 3] > 0.2).float()
    mask = torch.rand(N, S, S, generator=g) > 0.2
    return depth, rgba, gt, mask.to(mask_dtype)


@pytest.mark.parametrize("mask_dtype", [torch.float32, torch.uint8, torch.bool])
def test_fused_loss_against_the_torch_body(cuda_device, mask_dtype):
    depth, rgba, gt, mask = _loss_inputs(mask_dtype=mask_dtype)
    for m in (mask, torch.zeros_like(mask)):                  # M = 0 as well
        d = depth.to(DEV).requires_grad_(True)
        loss = depth_loss(d, rgba.to(DEV), gt.to(DEV), m.to(DEV), 0.7, 0.5, 10.0)
        loss.backward()
        d64 = depth.double().requires_grad_(True)
        ref = depth_loss_torch(d64, rgba.double(), gt.double(), m, 0.7, 0.5, 10.0)
        if ref.requires_grad:
            ref.backward()
        assert abs(float(loss.detach()) - float(ref.detach())) <= 1e-6 * max(1.0, abs(float(ref.detach())))
        want = d64.grad if d64.grad is not None else torch.zeros_like(d64)
        assert torch.allclose(d.grad.cpu().double(), want, rtol=1e-6, atol=1e-9)
    # two runs: the same bits
    a = [depth_loss(depth.to(DEV), rgba.to(DEV), gt.to(DEV), mask.to(DEV), 0.7, 0.5, 10.0) for _ in range(2)]
    assert torch.equal(a[0], a[1])


_WORKER = r"""
import os, sys, torch, torch.distributed as dist
sys.path.insert(0, os.environ["ROOT"])
from dss_b200.training.losses import depth_loss
from tests.test_gpu_depth import _loss_inputs
rank = int(os.environ["RANK"])
dist.init_process_group("gloo", rank=rank, world_size=2)
dev = torch.device("cuda:0")
depth, rgba, gt, mask = (t.to(dev) for t in _loss_inputs())
mine = [0, 1, 2] if rank == 0 else []                     # rank 1 holds no views
sel = lambda t: t[mine] if mine else t[:0]
d = sel(depth).clone().requires_grad_(True)
loss = depth_loss(d, sel(rgba), sel(gt), sel(mask), 0.7, 0.5, 10.0, group=dist.group.WORLD)
loss.backward()
one = depth.clone().requires_grad_(True)
ref = depth_loss(one, rgba, gt, mask, 0.7, 0.5, 10.0)
ref.backward()
assert torch.equal(loss, ref), (float(loss), float(ref))
if mine:
    assert torch.equal(d.grad, one.grad)
# split 2 / 1
mine = [0, 2] if rank == 0 else [1]
d = depth[mine].clone().requires_grad_(True)
loss = depth_loss(d, rgba[mine], gt[mine], mask[mine], 0.7, 0.5, 10.0, group=dist.group.WORLD)
loss.backward()
assert abs(float(loss) - float(ref)) <= 1e-6 * float(ref)
assert torch.equal(d.grad, one.grad[mine])
dist.destroy_process_group()
print("ok", rank)
"""


def test_sharded_loss_matches_one_gpu(cuda_device, tmp_path):
    import subprocess
    from tests.test_gpu_train_step_sharded import _free_port
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    script = tmp_path / "w.py"
    script.write_text(_WORKER)
    port = str(_free_port())
    procs = [subprocess.Popen([sys.executable, str(script)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                              env=dict(os.environ, ROOT=root, RANK=str(r), WORLD_SIZE="2", MASTER_ADDR="127.0.0.1",
                                       MASTER_PORT=port, PYTHONPATH=root))
             for r in range(2)]
    outs = [p.communicate(timeout=600)[0] for p in procs]
    assert [p.returncode for p in procs] == [0, 0], outs
