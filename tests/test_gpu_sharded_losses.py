"""GPU tests of the view-sharded image loss and point filters, the kernels a rank of a view-sharded training step runs:
`dss_image_loss_partial`, `dss_image_loss_finish` and `dss_image_loss_backward` on a summed total row
(csrc/image_loss.cu), and `dss_point_filters_gated` (csrc/point_filter.cu).

One process plays every rank, as the C contract allows: each shard of consecutive views runs `partial` (an empty
shard contributes a zero row), the total rows are summed in float64 in rank order, `finish` forms the scalars from the
sum, and each shard runs `backward` on its own view rows with the summed row in place of its own.  The result is
checked two ways:
  - against the float64 torch body over all the views, within the per-element bounds of tests/test_gpu_image_loss.py;
  - against the unsharded fused call over all the views: the RGB gradient bit for bit (its weight divides by M, an
    integer count, the same summed or not), alpha within 1 ulp and the scalars within 1 ulp (the per-view sums I_n,
    U_n and the total row are fp64 sums over another block partition, added in another order).
The point filters: the shards' visibility ORed into a gate, the gated calls' inmask ORed over the shards, equal the
ungated call over all the views bit for bit; and the gate alone decides visibility.

Last, one 2-rank gloo run on one GPU ties the Python route with a group (`image_loss(..., group=...)`,
`point_filters(out, mask, group)`, `point_filters_no_views`) to the kernels checked above, bit for bit.

Every check runs twice on the same inputs and asserts that both runs give the same bits.
"""
import ctypes as C
import os
import socket
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

from dss_b200 import _lib
from dss_b200.ops import SplatParams, render_points
from dss_b200.training.losses import _image_loss_args
from tests.test_gpu_image_loss import KEYS, bits, check, random_case, ulp32, upstream
from tests.test_gpu_train_step import make_mask, render_cloud, special_records, torch_filters
from tests.test_point_filter import filters_np
from tests.util import scene

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(autouse=True)
def _cuda(cuda_device):
    return cuda_device


def bounds(splits):
    """shard sizes -> [(first view, end view)] of consecutive views"""
    ends = np.cumsum(splits)
    return [(int(e - s), int(e)) for s, e in zip(splits, ends)]


def same_bits(a, b):
    return all(torch.equal(bits(x), bits(y)) for x, y in zip(a, b))


# ---- 1. the image loss, ranks simulated in one process ----------------------------------------------------------------
def image_inputs(N, H, W, seed, dev, mask="frac", gt="contig", m0=(), u0=()):
    """random_case with the mask as `mask` ("frac": float with fractional values, "f32": float 0/1, "u8": bytes 0..7,
    "bool"), the GT RGB as a permuted (N,3,H,W) view (`gt="perm"`), no pixel where both masks are non-zero in the views
    `m0` (M = 0 there) and mask and alpha both zero in the views `u0` (U_n = 0)"""
    rgba, img, m = random_case(N, H, W, seed, dev, fractional=mask == "frac")
    if mask == "u8":
        g = torch.Generator().manual_seed(seed + 1)
        m = ((m != 0) * torch.randint(1, 8, m.shape, generator=g).to(dev)).to(torch.uint8)
    elif mask == "bool":
        m = m != 0
    for n in m0:
        rgba[n, ..., 3] = torch.where(m[n] != 0, 0.0, rgba[n, ..., 3])
    for n in u0:
        m[n] = 0
        rgba[n, ..., 3] = 0.0
    if gt == "perm":
        img = img.permute(0, 3, 1, 2).contiguous().permute(0, 2, 3, 1)
        assert not img.is_contiguous()
    return rgba, img, m


def _scalars(dev):
    return [torch.empty((), dtype=torch.float32, device=dev) for _ in KEYS]


def sharded(rgba, img, mask, splits, lr, ls, ups):
    """the loss over all the views as len(splits) ranks compute it, rank k holding the next splits[k] views ->
    (the three scalars, the (N,H,W,4) gradient assembled from the ranks' slices)"""
    (N, H, W), dev = rgba.shape[:3], rgba.device
    assert sum(splits) == N
    shards = []
    row = torch.zeros(5, dtype=torch.float64, device=dev)
    for a, b in bounds(splits):
        totals = torch.zeros((b - a + 1, 5), dtype=torch.float64, device=dev)     # an empty shard: a zero row
        if b > a:
            _lib.call("dss_image_loss_partial", dev, *_image_loss_args(rgba[a:b], img[a:b], mask[a:b], lr, ls), totals)
        shards.append((a, b, totals))
        row = row + totals[b - a]                                                # float64, in rank order
    losses = _scalars(dev)
    _lib.call("dss_image_loss_finish", dev, row, H, W, float(lr), float(ls), *losses)
    grad = torch.full_like(rgba, float("nan"))                                   # every entry must be written
    for a, b, totals in shards:
        if b > a:
            totals[b - a] = row
            _lib.call("dss_image_loss_backward", dev, *_image_loss_args(rgba[a:b], img[a:b], mask[a:b], lr, ls),
                      totals, *ups, grad[a:b])
    return losses, grad


def unsharded(rgba, img, mask, lr, ls, ups):
    """dss_image_loss_forward / _backward over all the views"""
    dev = rgba.device
    args = _image_loss_args(rgba, img, mask, lr, ls)
    totals = torch.empty((rgba.shape[0] + 1, 5), dtype=torch.float64, device=dev)
    losses = _scalars(dev)
    _lib.call("dss_image_loss_forward", dev, *args, totals, *losses)
    grad = torch.full_like(rgba, float("nan"))
    _lib.call("dss_image_loss_backward", dev, *args, totals, *ups, grad)
    return losses, grad


def within_ulp(got, want):
    """NaN at the same places, elsewhere |got - want| <= 1 ulp of want"""
    nan = torch.isnan(want)
    if not torch.equal(torch.isnan(got), nan):
        return False
    g, w = got.double()[~nan], want.double()[~nan]
    return bool(((g - w).abs() <= ulp32(w)).all())


def check_sharded(name, rgba, img, mask, splits, lr=1.0, ls=1.0, seed=0, nan_ok=False):
    ups = upstream(seed, rgba.device)
    assert len({float(u) for u in ups}) == 3 and 1.0 not in {float(u) for u in ups}
    (losses, grad), again = sharded(rgba, img, mask, splits, lr, ls, ups), sharded(rgba, img, mask, splits, lr, ls, ups)
    assert same_bits(losses, again[0]) and torch.equal(bits(grad), bits(again[1])), name
    (w_losses, w_grad), again = unsharded(rgba, img, mask, lr, ls, ups), unsharded(rgba, img, mask, lr, ls, ups)
    assert same_bits(w_losses, again[0]) and torch.equal(bits(w_grad), bits(again[1])), name
    # against float64 over all the views
    check(name, losses, grad, rgba, img, mask, lr, ls, ups, nan_ok)
    # against the unsharded call
    assert torch.equal(bits(grad[..., :3]), bits(w_grad[..., :3])), name
    assert within_ulp(grad[..., 3], w_grad[..., 3]), name
    for k, got, want in zip(KEYS, losses, w_losses):
        assert within_ulp(got, want), (name, k, float(got), float(want))
    return losses, grad


# (id, N, H, W, splits, image_inputs options).  The forward gives each view min(ceil(4 SMs / N), ceil(HW / 256)) blocks
# (il_blocks): at 300 x 200 on an H100's 132 SMs, 235 in a shard of one view, 76 in one of seven, 66 over all eight.
SPLIT_CASES = [
    ("1+7 views at 300x200", 8, 300, 200, [1, 7], {}),
    ("7+1 views at 300x200, uint8 mask", 8, 300, 200, [7, 1], {"mask": "u8"}),
    ("2+0+4, an empty shard", 6, 128, 96, [2, 0, 4], {"mask": "f32"}),
    ("all views on one of 4 shards, bool mask, permuted gt", 5, 64, 80, [0, 0, 5, 0], {"mask": "bool", "gt": "perm"}),
    ("1+2+3+4 at 7x513, permuted gt", 10, 7, 513, [1, 2, 3, 4], {"gt": "perm"}),
    ("3+1 at 17x40, uint8 mask, permuted gt", 4, 17, 40, [3, 1], {"mask": "u8", "gt": "perm"}),
    ("1x1 images", 3, 1, 1, [1, 0, 2], {}),
    ("1x1 images, bool mask", 4, 1, 1, [0, 4, 0], {"mask": "bool"}),
    # the finish's view loop (256 threads) wraps in the 270-view shard and in the unsharded call
    ("300 views over 3 shards", 300, 16, 16, [270, 29, 1], {"mask": "u8"}),
]


@pytest.mark.parametrize("name,N,H,W,splits,opts", SPLIT_CASES, ids=[c[0] for c in SPLIT_CASES])
def test_sharded_image_loss_matches_float64_and_the_unsharded_call(name, N, H, W, splits, opts, cuda_device):
    rgba, img, mask = image_inputs(N, H, W, N + H + W, cuda_device, **opts)
    check_sharded(name, rgba, img, mask, splits, seed=N + W)
    check_sharded(name, rgba, img, mask, splits, 0.7, 2.5, seed=N + W + 1)


@pytest.mark.parametrize("where", ["one shard", "every shard"])
def test_rgb_term_is_zero_where_M_is_zero(where, cuda_device):
    """M = 0 summed over the shards: the RGB term is +0 and so is its gradient (no 0 / 0); M = 0 on one shard only:
    that shard's views get no RGB gradient, but its weight is the summed M, not the shard's"""
    N, splits = 6, [3, 0, 3]
    m0 = range(3, 6) if where == "one shard" else range(N)
    rgba, img, mask = image_inputs(N, 48, 48, 31, cuda_device, m0=m0)
    losses, grad = check_sharded(where, rgba, img, mask, splits, seed=31)
    zero = torch.zeros((), device=cuda_device)
    assert torch.equal(bits(grad[3:, ..., :3]), bits(torch.zeros_like(grad[3:, ..., :3])))
    if where == "every shard":
        assert torch.equal(bits(losses[1]), bits(zero))
        assert torch.equal(bits(grad[..., :3]), bits(torch.zeros_like(grad[..., :3])))
        assert torch.equal(bits(losses[0]), bits(losses[2]))
    else:
        assert float(losses[1]) > 0 and grad[:3, ..., :3].any()


def test_views_with_U_zero(cuda_device):
    """mask and alpha both zero in a view (U_n = 0, eps_denom's clamp): alone on its shard and next to others; its
    gradient is +0 and every other view's is that of the float64 body"""
    N, splits, u0 = 5, [1, 4], (0, 2)
    rgba, img, mask = image_inputs(N, 40, 40, 41, cuda_device, u0=u0)
    _, grad = check_sharded("U = 0", rgba, img, mask, splits, seed=41)
    for n in u0:
        assert torch.equal(bits(grad[n]), bits(torch.zeros_like(grad[n]))), n
    assert grad[1].any() and grad[3].any()


@pytest.mark.parametrize("lr,ls", [(0.0, 1.5), (-1.0, 0.8), (1.5, 0.0), (0.7, -2.0), (0.0, -1.0)])
def test_absent_terms_read_nothing(lr, ls, cuda_device):
    """a term whose lambda is not > 0 is +0 with a +0 gradient, on every shard; without the RGB term the GT RGB is not
    read (it is all NaN here), without the silhouette term a NaN alpha inside mask_pred reaches nothing"""
    N, splits = 5, [2, 0, 3]
    rgba, img, mask = image_inputs(N, 32, 24, 51, cuda_device)
    if lr <= 0:
        img = torch.full_like(img, float("nan"))
    if ls <= 0:
        for n, y, x in ((0, 3, 4), (3, 5, 6), (4, 7, 7)):     # NaN.bool() is true: inside mask_pred
            mask[n, y, x] = 1.0
            rgba[n, y, x, 3] = float("nan")
    losses, grad = check_sharded("lambda %g, %g" % (lr, ls), rgba, img, mask, splits, lr, ls, seed=51)
    assert all(bool(torch.isfinite(x)) for x in losses) and torch.isfinite(grad).all()
    zero = torch.zeros((), device=cuda_device)
    for absent, k, ch in ((lr <= 0, 1, slice(0, 3)), (ls <= 0, 2, slice(3, 4))):
        if absent:
            assert torch.equal(bits(losses[k]), bits(zero))
            assert torch.equal(bits(grad[..., ch]), bits(torch.zeros_like(grad[..., ch])))
        else:
            assert float(losses[k]) > 0 and grad[..., ch].any()


def test_nan_in_prediction_on_one_shard(cuda_device):
    """NaN in the RGBA of one shard's views: the NaN pattern of the float64 body (NaN inside mask_pred reaches the
    losses; a NaN alpha makes its view's alpha gradient NaN; a NaN rgb has sign 0), the other shard's gradient finite"""
    N, splits = 6, [2, 4]
    rgba, img, mask = image_inputs(N, 24, 24, 61, cuda_device)
    mask[2, 1, 1] = 1.0
    rgba[2, 1, 1, 3] = 0.5
    rgba[2, 1, 1, 0] = float("nan")
    mask[3, 2, 3] = 1.0
    rgba[3, 2, 3, 3] = float("nan")            # inside the GT mask: counts in M
    mask[5, 9, 9] = 1.0
    rgba[5, 9, 9, 1] = float("nan")
    rgba[5, 9, 9, 3] = 0.0                     # outside mask_pred: the NaN rgb is never read
    losses, grad = check_sharded("nan", rgba, img, mask, splits, seed=61, nan_ok=True)
    assert all(torch.isnan(x) for x in losses)
    assert torch.isnan(grad[3, ..., 3]).all() and torch.isfinite(grad[..., :3]).all()
    assert torch.isfinite(grad[:2]).all() and torch.isfinite(grad[[2, 4, 5]]).all()


# ---- 2. the gated point filters ----------------------------------------------------------------------------------------
def filters(records, visible, mask, N, P0, gate=None, out=None):
    """dss_point_filters (gate None) or dss_point_filters_gated on N views of P0 points -> (visibility, inmask) uint8.
    The outputs start as 0xAB, so an entry the kernel leaves unwritten shows."""
    dev = records.device
    m = mask[:, 0] if mask.dim() == 4 else mask
    vis, inm = out if out is not None else (torch.full((P0,), 0xAB, dtype=torch.uint8, device=dev) for _ in range(2))
    head = (records, visible, 1, N, P0, m, int(m.dtype != torch.float32), (C.c_int64 * 3)(*m.stride()), m.shape[1],
            m.shape[2])
    if gate is None:
        _lib.call("dss_point_filters", dev, *head, vis, inm)
    else:
        _lib.call("dss_point_filters_gated", dev, *head, gate, vis, inm)
    return vis, inm


def shard_of(records, visible, mask, N, P0, a, b):
    return records.view(N, P0, 8)[a:b].reshape(-1, 8), visible.view(N, P0)[a:b].reshape(-1), mask[a:b], b - a, P0


def seven_mask(layout, N, H, W, seed, dev):
    """a byte mask of 0 and 7, contiguous or transposed"""
    m = make_mask("bool", "contig", N, H, W, seed, dev).to(torch.uint8) * 7
    if layout == "perm":
        m = m.transpose(1, 2).contiguous().transpose(1, 2)
    return m


def filter_checks(records, visible, mask, N, P0, splits, bad):
    """every check of the gated filters on one set of records -> their outputs, for the determinism check"""
    dev = records.device
    u8 = lambda t: t.to(torch.uint8)
    whole = filters(records, visible, mask, N, P0)
    want_vis, want_inm = torch_filters(records, visible, mask)
    assert torch.equal(whole[0], u8(want_vis)) and torch.equal(whole[1], u8(want_inm))
    assert visible.any() and whole[1].any()

    # shard ORs equal the whole: the shards' visibility ORed into the gate, the gated inmask ORed over the shards
    gate = torch.zeros(P0, dtype=torch.uint8, device=dev)          # an empty shard's contribution
    own = []
    for a, b in bounds(splits):
        if b > a:
            own.append(filters(*shard_of(records, visible, mask, N, P0, a, b))[0])
            gate |= own[-1]
    inmask = torch.zeros(P0, dtype=torch.uint8, device=dev)
    for a, b in bounds(splits):
        if b > a:
            vis, inm = filters(*shard_of(records, visible, mask, N, P0, a, b), gate=gate)
            assert torch.equal(vis, gate)
            inmask |= inm
    assert torch.equal(gate, whole[0]) and torch.equal(inmask, whole[1])
    if len(own) > 1:      # the gate is wider than a shard's own visibility
        assert any((gate != o).any() for o in own)

    # the gate decides alone: an all-zero gate over visible points ...
    zero = filters(records, visible, mask, N, P0, gate=torch.zeros(P0, dtype=torch.uint8, device=dev))
    assert not zero[0].any() and not zero[1].any()
    # ... and an all-one gate over points visible nowhere: the inmask of the masks alone
    nowhere = torch.zeros_like(visible)
    ones = filters(records, nowhere, mask, N, P0, gate=torch.ones(P0, dtype=torch.uint8, device=dev))
    everywhere = filters(records, torch.ones_like(visible), mask, N, P0)
    assert torch.equal(ones[0], torch.ones_like(ones[0])) and torch.equal(ones[1], everywhere[1])
    assert not ones[1][bad].any()                                  # non-finite positions are outside every mask
    m = mask.reshape(N, *mask.shape[-2:])
    H, W = m.shape[1:]
    if H & (H - 1) == 0 and W & (W - 1) == 0:
        # at power-of-two sizes the unnormalisation's product is exact, so the kernel's contracted multiply-add rounds
        # as the restatement's two float32 steps do
        xy = records.view(N, P0, 8)[..., :2].cpu().numpy()
        _, np_inm, _ = filters_np(xy, np.ones((N, P0), bool), m.cpu().numpy())
        assert np.array_equal(ones[1].cpu().numpy(), np_inm.astype(np.uint8))

    # a gate that differs from the call's own visibility, with values other than 1; the gate and the visibility output
    # one buffer, as ops.point_filters passes them
    g = torch.Generator().manual_seed(P0)
    gate = torch.tensor([0, 1, 5], dtype=torch.uint8)[torch.randint(0, 3, (P0,), generator=g)].to(dev)
    separate = filters(records, visible, mask, N, P0, gate=gate)
    alias = gate.clone()
    aliased = filters(records, visible, mask, N, P0, gate=alias,
                      out=(alias, torch.full((P0,), 0xAB, dtype=torch.uint8, device=dev)))
    assert torch.equal(separate[0], u8(gate != 0)) and torch.equal(separate[1], u8(gate != 0) & ones[1])
    assert torch.equal(aliased[0], separate[0]) and torch.equal(aliased[1], separate[1])
    return [*whole, gate, inmask, *zero, *ones, *separate, *aliased]


# (id, N views, P0, mask kind, layout, H, W, splits)
FILTER_CASES = [
    ("8 views, float 64x128", 8, 5003, "f32", "contig", 64, 128, [3, 0, 1, 4]),
    ("8 views, bytes of 7 transposed 48x80", 8, 5003, "u8x7", "perm", 48, 80, [1, 7]),
    ("8 views, bytes of 7 32x32", 8, 2049, "u8x7", "contig", 32, 32, [0, 5, 3]),
    ("3 views, bool (N,1,H,W) 64x64", 3, 1025, "bool", "n1hw", 64, 64, [1, 1, 1, 0]),
    ("3 views, bytes transposed 16x64", 3, 700, "u8", "perm", 16, 64, [2, 1]),
    ("1 view", 1, 257, "f32", "perm", 32, 16, [0, 1]),
]


@pytest.mark.parametrize("name,N,P0,kind,layout,H,W,splits", FILTER_CASES, ids=[c[0] for c in FILTER_CASES])
def test_gated_point_filters(name, N, P0, kind, layout, H, W, splits, cuda_device):
    d = cuda_device
    assert sum(splits) == N and P0 % 256
    out, _, _ = render_cloud(P0, N, 64, d, seed=N + P0)
    mask = seven_mask(layout, N, H, W, N + H, d) if kind == "u8x7" else make_mask(kind, layout, N, H, W, N + H, d)
    if layout == "perm":
        assert not mask.is_contiguous()
    special, bad = special_records(out, N, P0, (H, W), seed=P0)
    for o, b in ((out, torch.zeros(0, dtype=torch.long, device=d)), (special, bad)):
        first = filter_checks(o.records, o.visible, mask, N, P0, splits, b)
        again = filter_checks(o.records, o.visible, mask, N, P0, splits, b)
        assert all(torch.equal(x, y) for x, y in zip(first, again)), name


# ---- 3. the Python route with a process group: 2 gloo ranks on one GPU -------------------------------------------------
GROUP_SPLITS = {"rank 0 without views": [0, 5], "M = 0 on rank 1": [3, 2]}
GROUP_LAMBDAS = (0.7, 1.3)
GROUP_P0 = 2003


def group_image_inputs(dev):
    """5 views; views 3 and 4 have M = 0"""
    rgba, img, mask = image_inputs(5, 24, 40, 71, dev, mask="u8", gt="perm", m0=(3, 4))
    return rgba, img, mask, upstream(71, dev)


def group_render(dev, views):
    """the render of `views` of a shared cloud of GROUP_P0 points, and the masks of the filters"""
    pts, nrm, col, proj, view, _ = scene(GROUP_P0, 5, seed=72)
    idx = torch.tensor(views, dtype=torch.long)
    prm = SplatParams(image_size=64, znear=0.1, clip_pts_grad=0.05)
    with torch.no_grad():
        out = render_points(pts.to(dev), nrm.to(dev), col.to(dev), proj[idx].to(dev), view[idx].to(dev),
                            torch.full((len(views),), 3e-4, device=dev), prm)
    return out, make_mask("f32", "perm", 5, 48, 80, seed=73, dev=dev)[idx.to(dev)]


_WORKER = r'''
import sys, torch, torch.distributed as dist
sys.path.insert(0, %(root)r)
rank, out_dir, port = int(sys.argv[1]), sys.argv[2], int(sys.argv[3])
dev = torch.device("cuda", 0)
torch.cuda.set_device(dev)
dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%%d" %% port, rank=rank, world_size=2)
from dss_b200.ops import point_filters, point_filters_no_views
from dss_b200.training.losses import image_loss
from tests.test_gpu_sharded_losses import (GROUP_LAMBDAS, GROUP_P0, GROUP_SPLITS, KEYS, bounds, group_image_inputs,
                                           group_render)
group = dist.group.WORLD
saved = {}
for name, splits in GROUP_SPLITS.items():
    rgba, img, mask, ups = group_image_inputs(dev)
    a, b = bounds(splits)[rank]
    x = rgba[a:b].clone().requires_grad_(True)
    loss = image_loss(x, img[a:b], mask[a:b], *GROUP_LAMBDAS, group=group)
    torch.autograd.backward([loss[k] for k in KEYS], ups)
    if b > a:
        vis, inm = point_filters(*group_render(dev, list(range(a, b))), group)
    else:
        vis, inm = point_filters_no_views(GROUP_P0, dev, group)
    torch.cuda.synchronize()
    saved[name] = {"losses": torch.stack([loss[k].detach() for k in KEYS]).cpu(),
                   "grad": None if x.grad is None else x.grad.cpu(), "vis": vis.cpu(), "inm": inm.cpu()}
torch.save(saved, "%%s/rank%%d.pt" %% (out_dir, rank))
dist.destroy_process_group()
print("rank", rank, "ok")
'''


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def test_image_loss_and_point_filters_with_a_group_of_two_gloo_ranks(cuda_device):
    """each rank's losses and filters are the same bits, equal to the one-process simulation of section 1 and to the
    ungated filters of all the views; each rank's RGBA gradient is its slice of section 1's, bit for bit"""
    d = cuda_device
    with tempfile.TemporaryDirectory() as tmp:
        w = os.path.join(tmp, "worker.py")
        with open(w, "w") as f:
            f.write(_WORKER % {"root": ROOT})
        env = dict(os.environ, PYTHONPATH=ROOT)
        port = _free_port()
        procs = [subprocess.Popen([sys.executable, w, str(r), tmp, str(port)], stdout=subprocess.PIPE,
                                  stderr=subprocess.STDOUT, text=True, cwd=ROOT, env=env) for r in range(2)]
        try:
            outs = [p.communicate(timeout=300)[0] for p in procs]
        finally:
            for p in procs:
                if p.poll() is None:
                    p.kill()
                    p.wait()
        for r, (p, o) in enumerate(zip(procs, outs)):
            assert p.returncode == 0 and "rank %d ok" % r in o, o
        saved = [torch.load(os.path.join(tmp, "rank%d.pt" % r)) for r in range(2)]

    rgba, img, mask, ups = group_image_inputs(d)
    assert not (mask[3:].bool() & rgba[3:, ..., 3].bool()).any() and (mask[:3].bool() & rgba[:3, ..., 3].bool()).any()
    out, fmask = group_render(d, list(range(5)))
    want_vis, want_inm = filters(out.records, out.visible, fmask, 5, GROUP_P0)
    assert want_inm.any()
    for name, splits in GROUP_SPLITS.items():
        r0, r1 = (s[name] for s in saved)
        for k in ("losses", "vis", "inm"):
            assert torch.equal(r0[k].view(torch.uint8), r1[k].view(torch.uint8)), (name, k)
        losses, grad = sharded(rgba, img, mask, splits, *GROUP_LAMBDAS, ups)
        assert torch.equal(bits(r0["losses"]), bits(torch.stack(losses).cpu())), name
        for r, (a, b) in enumerate(bounds(splits)):
            got = saved[r][name]["grad"]
            if b > a:
                assert torch.equal(bits(got), bits(grad[a:b].cpu())), (name, r)
            else:
                assert got is None or got.numel() == 0, (name, r)
        assert torch.equal(r0["vis"].to(torch.uint8), want_vis.cpu()), name
        assert torch.equal(r0["inm"].to(torch.uint8), want_inm.cpu()), name
