"""GPU: the training views resident on the device.  The gather kernel (csrc/views.cu) against the values
MVRData.load_all_images / load_all_masks give; DeviceViews against the staged pinned_batch upload; the graphed step
built from_views against the staged step, bit for bit; no host synchronisation in a resident iteration; the loop
against a replay of the same batches through the staged public pieces; and evaluate_2d on the store."""
import numpy as np
import pytest
import torch

from dss_b200.core.camera import camera_matrices
from dss_b200.core.lighting import pack_lights
from dss_b200.ops import evaluate_2d, gather_views, image_metrics
from dss_b200.training.step import GraphedTrainStep
from dss_b200.utils.dataset import MVRData
from tests.test_gpu_train_loop import data_dir, write_config  # noqa: F401  (data_dir: a fixture)

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


_INT = {torch.float32: torch.int32, torch.float64: torch.int64}


def bits(t):
    t = t.detach().cpu().contiguous()
    return t.view(_INT[t.dtype]) if t.dtype in _INT else t


def same(a, b):
    assert a.dtype == b.dtype and a.shape == b.shape, (a.dtype, b.dtype, a.shape, b.shape)
    assert torch.equal(bits(a), bits(b))


# ---- the gather ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S", [1, 7, 128, 513])
@pytest.mark.parametrize("V", [1, 16])
def test_gather_gives_the_loaded_bits(S, V):
    g = np.random.default_rng(S * 100 + V)
    # every byte value in every channel, the rest random
    k = g.integers(0, 256, size=(V, S, S, 4)).astype(np.uint8)
    flat = k.reshape(-1, 4)
    n = min(256, flat.shape[0])
    for c in range(4):
        flat[:n, c] = np.roll(np.arange(256, dtype=np.uint8), 37 * c)[:n]
    store = torch.from_numpy(k).to(DEV)
    rgb_ref = k[..., :3].astype(np.float32) / 255.0                        # load_all_images
    mask_ref = k[..., 3].astype(bool).astype(np.float32)                   # load_all_masks
    for idx in ([0], list(range(V)), [V - 1, 0, V - 1, V // 2, 0, 0], []):
        idx_dev = torch.tensor(idx, dtype=torch.int64, device=DEV)
        img = torch.full((len(idx), S, S, 3), float("nan"), device=DEV)
        mask = torch.full((len(idx), S, S), float("nan"), device=DEV)
        gather_views(store, idx_dev, img, mask)
        same(img, torch.from_numpy(rgb_ref[idx]))
        same(mask, torch.from_numpy(mask_ref[idx]))


@pytest.mark.parametrize("S", [7, 128])
def test_gather_of_a_float32_store_copies_the_bits(S):
    g = torch.Generator().manual_seed(S)
    store = torch.randn(5, S, S, 4, generator=g)
    store[0, 0, 0] = torch.tensor([float("nan"), -0.0, float("inf"), 0.3])
    store[1, -1, -1, 3] = 1e-40                                              # a denormal
    idx = [4, 0, 1, 4]
    img, mask = gather_views(store.to(DEV), torch.tensor(idx, device=DEV),
                             torch.empty(4, S, S, 3, device=DEV), torch.empty(4, S, S, device=DEV))
    same(img, store[idx][..., :3].contiguous())
    same(mask, store[idx][..., 3].contiguous())


def test_gather_into_outputs_off_16_byte_alignment():
    # a 4-pixel-multiple view whose outputs start 4 bytes into their buffers: the scalar route
    k = torch.randint(0, 256, (3, 8, 8, 4), dtype=torch.uint8, generator=torch.Generator().manual_seed(5))
    buf_i, buf_m = torch.empty(2 * 64 * 3 + 1, device=DEV), torch.empty(2 * 64 + 1, device=DEV)
    img, mask = buf_i[1:].view(2, 8, 8, 3), buf_m[1:].view(2, 8, 8)
    gather_views(k.to(DEV), torch.tensor([2, 0], device=DEV), img, mask)
    ref = k[[2, 0]].numpy()
    same(img, torch.from_numpy(ref[..., :3].astype(np.float32) / 255.0))
    same(mask, torch.from_numpy(ref[..., 3].astype(bool).astype(np.float32)))


# ---- the store against the staged upload -------------------------------------------------------------------------
def staged(data, idx):
    """the views idx as the loop uploaded them from pinned memory before the views were resident"""
    b = data.pinned_batch(idx)
    idx_dev = torch.tensor(idx, dtype=torch.int64).pin_memory().to(DEV, non_blocking=True)
    img = b["img.rgb"].to(DEV, non_blocking=True).permute(0, 2, 3, 1)
    mask = b["img.mask"].to(DEV, non_blocking=True)[:, 0]
    view = b["camera_mat"].to(DEV, non_blocking=True)
    proj = camera_matrices(data.get_cameras())[0].to(DEV).index_select(0, idx_dev)
    cls, props = data.light_props(DEV)
    lights = cls(**{k: v.index_select(0, idx_dev) for k, v in props.items()}, device=DEV)
    return img, mask, proj, view, lights


@pytest.mark.parametrize("idx", [[5], [3, 0, 15, 3, 7, 7, 1, 12]])
def test_store_equals_the_staged_upload(data_dir, idx):  # noqa: F811
    data = MVRData(data_dir)
    views = data.device_views(DEV)
    assert views.store.dtype == torch.uint8 and len(views) == 16
    a, b = views.batch(idx), staged(data, idx)
    for x, y in zip(a[:4], b[:4]):
        same(x, y.contiguous())
    ra, aa, ka = pack_lights(a[4])
    rb, ab, kb = pack_lights(b[4])
    assert ka == kb
    same(ra, rb)
    same(aa, ab)
    # the shared form at batch 1, as the staged path hands it to the step
    assert ra.dim() == (2 if len(idx) == 1 else 3)


# ---- the graphed step ---------------------------------------------------------------------------------------------
def step_args(data_dir, tmp_path):  # noqa: F811
    """the data, the loop's splat settings at tests/test_gpu_train_loop.py's configuration, and its initial cloud"""
    from dss_b200.training.config import load_config, splat_params
    from dss_b200.training.train import initial_cloud
    data = MVRData(data_dir)
    cams = data.get_cameras()
    cfg = load_config(write_config(tmp_path / "c.yml", data_dir, tmp_path / "out"))
    return data, splat_params(cfg, cams.znear, cams.zfar), initial_cloud(2000, 0, DEV)


@pytest.mark.parametrize("B", [1, 8])
@pytest.mark.parametrize("splats", ["Vrk_invariant", "anisotropic"])
def test_step_from_views_equals_the_staged_step(data_dir, tmp_path, B, splats):  # noqa: F811
    data, params, (p, n, c) = step_args(data_dir, tmp_path)
    flags = dict(Vrk_invariant=True, Vrk_isotropic=False) if splats == "Vrk_invariant" else \
        dict(Vrk_invariant=False, Vrk_isotropic=False)
    g = torch.Generator().manual_seed(B)
    batches = [torch.randint(0, 16, (B,), generator=g).tolist() for _ in range(4)]
    batches.insert(2, batches[0])                                           # a repeated batch
    views = data.device_views(DEV)
    a = GraphedTrainStep.from_views(p, n, c, params, views, batches[0], **flags)
    b = GraphedTrainStep(p, n, c, params, *staged(data, batches[0]), **flags)
    with pytest.raises(RuntimeError, match="load_views"):
        a.load(*staged(data, batches[0]))
    with pytest.raises(RuntimeError, match="from_views"):
        b.load_views(batches[0])
    with pytest.raises(ValueError, match="views"):
        a.load_views(batches[0] + [0])
    for idx in batches:
        a.load_views(idx)
        b.load(*staged(data, idx))
        la, lb = a.replay(), b.replay()
        assert la.keys() == lb.keys()
        for k in la:
            same(la[k], lb[k])
        for x, y in ((a.image, b.image), (a.visibility, b.visibility), (a.inmask, b.inmask),
                     (a.img, b.img.contiguous()), (a.mask_img, b.mask_img), (a.proj, b.proj), (a.view, b.view),
                     (a.lights, b.lights), (a.ambient, b.ambient)):
            same(x, y)
        for x, y in zip((a.points, a.normals, a.colours), (b.points, b.normals, b.colours)):
            assert (x.grad is None) == (y.grad is None)
            if x.grad is not None:
                same(x.grad, y.grad)
        # the same Adam-like move on both clouds, so that the batches meet different clouds
        for s in (a, b):
            s.points.data.add_(s.points.grad, alpha=-1e-3)


def test_resident_iteration_makes_no_host_synchronisation(data_dir, tmp_path):  # noqa: F811
    data, params, (p, n, c) = step_args(data_dir, tmp_path)
    step = GraphedTrainStep.from_views(p, n, c, params, data.device_views(DEV), [0, 1, 2, 3], Vrk_invariant=True,
                                       Vrk_isotropic=False)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for idx in ([4, 5, 6, 7], [7, 7, 0, 15]):
            step.load_views(idx)
            step.replay()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert torch.isfinite(step.loss["loss"]).item()


# ---- the loop -----------------------------------------------------------------------------------------------------
def test_loop_equals_the_staged_replay(data_dir, tmp_path):  # noqa: F811
    from dss_b200.training.config import load_config, splat_params, step_settings
    from dss_b200.training.train import Trainer, initial_cloud, make_lr_scheduler, make_optimizer
    cfg = load_config(write_config(tmp_path / "c.yml", data_dir, tmp_path / "out", print_every=0,
                                   validate_every=0, checkpoint_every=0, steps_dss_backward_radii=1000))
    n_it = 30
    assert Trainer(cfg).run(exit_after=-1, max_it=n_it) == 0
    ck = torch.load(tmp_path / "out" / "torus" / "model.pt", map_location="cpu", weights_only=False)
    assert ck["it"] == n_it - 1
    # the same iterations through the public pieces, staged
    tr = cfg["training"]
    data = MVRData(data_dir)
    V, bs = len(data), int(tr["batch_size"])
    cams = data.get_cameras()
    s = step_settings(cfg)
    learn = s.pop("learn")
    points, normals, colours = initial_cloud(cfg["model"]["model_kwargs"]["n_points_per_cloud"], tr["seed"], DEV)
    step = GraphedTrainStep(points, normals, colours, splat_params(cfg, cams.znear, cams.zfar),
                            *staged(data, list(range(bs))), learn=learn, **s)
    opt = make_optimizer({"points": step.points, "normals": step.normals, "colours": step.colours})
    sched = make_lr_scheduler(opt, cfg)
    gen = torch.Generator().manual_seed(int(tr["seed"]))
    order, pos = None, 0
    for _ in range(n_it):
        if order is None or pos + bs > len(order):
            if order is not None:
                sched.step()
            order, pos = torch.multinomial(torch.ones(V, dtype=torch.float64), V, True, generator=gen).tolist(), 0
        step.load(*staged(data, order[pos:pos + bs]))
        pos += bs
        if step.stale():
            step.capture()
        step.replay()
        opt.step()
    assert ck["epoch_order"] == order and ck["epoch_pos"] == pos
    for key, t in (("points", step.points), ("normals", step.normals), ("colors", step.colours)):
        same(ck["model"][key][0], t.detach())
    sa, sb = ck["optimizer"]["state"], opt.state_dict()["state"]
    assert sa.keys() == sb.keys()
    for i in sa:
        for k in sa[i]:
            same(torch.as_tensor(sa[i][k]), torch.as_tensor(sb[i][k]))


# ---- validation ---------------------------------------------------------------------------------------------------
def test_evaluate_2d_reads_the_store(data_dir, tmp_path):  # noqa: F811
    data, params, (p, n, c) = step_args(data_dir, tmp_path)
    flags = (True, False, 0.2, 64.0)
    a = evaluate_2d(p, n, c, data.device_views(DEV), params, 32, 5, *flags)
    b = evaluate_2d(p, n, c, data, params, 32, 5, *flags)
    for k in ("iou", "psnr", "per_view"):
        same(a[k], b[k])


def test_evaluate_2d_of_float_views_equals_the_stacked_upload(data_dir, tmp_path):  # noqa: F811
    base, params, (p, n, c) = step_args(data_dir, tmp_path)
    g = torch.Generator().manual_seed(9)
    # non-8-bit images and fractional masks: a float32 store
    images = [(im + 1e-3 * torch.rand(im.shape, generator=g)).clamp(0, 1) for im in base.images]
    masks = [torch.rand(m.shape, generator=g) for m in base.masks]
    data = MVRData(data_dir, images=images, masks=masks)
    assert data.device_views(DEV).store.dtype == torch.float32
    from dss_b200.ops import render_data_views
    ev = evaluate_2d(p, n, c, data, params, 128, 4, True, False)
    rows = []
    for i in range(0, len(data), 4):
        views = list(range(i, min(i + 4, len(data))))
        image = render_data_views(p, n, c, data, params, views, True, False)
        rgb = torch.stack([images[v] for v in views]).to(DEV).permute(0, 2, 3, 1)
        mask = torch.stack([masks[v] for v in views]).to(DEV)
        rows.append(image_metrics(image, rgb, mask).per_view)
    same(ev["per_view"], torch.cat(rows))
