"""GPU: dss_image_metrics against tests/image_metrics_oracle.py and torch's CUDA F.interpolate, its determinism and
capture, and the image-space validation through the training loop (model selection by iou / psnr, data without a
ground-truth cloud, the loop's values against image_metrics) and the ``generate --images`` export."""
import json
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from dss_b200.ops import evaluate_2d, image_metrics, render_data_views
from tests import image_metrics_oracle as im
from tests.test_gpu_train_loop import ROOT, data_dir, run_cli, write_config  # noqa: F401 (data_dir: a fixture)

pytestmark = pytest.mark.gpu


def inputs(V, H, W, s, mask_kind="float", permuted=False, seed=0, empty=()):
    g = torch.Generator().manual_seed(seed)
    pred = torch.rand(V, s, s, 4, generator=g) * 1.2 - 0.1                    # unclamped, as renders may be
    rgb = torch.rand(V, 3, H, W, generator=g)
    gt = rgb.permute(0, 2, 3, 1) if permuted else rgb.permute(0, 2, 3, 1).contiguous()
    m = torch.rand(V, H, W, generator=g)
    mask = {"float": m, "bool": m > 0.5, "uint8": (m > 0.5).to(torch.uint8)}[mask_kind]
    for n in empty:
        pred[n, ..., 3] = 0
        mask[n] = 0
    return pred, gt, mask


CASES = [(1, 64, 64, 64), (1, 64, 64, 16), (130, 64, 64, 16), (3, 100, 100, 37), (2, 64, 64, 96), (130, 40, 40, 40),
         (2, 48, 30, 12)]


@pytest.mark.parametrize("mask_kind", ["float", "bool", "uint8"])
@pytest.mark.parametrize("V,H,W,s", CASES)
def test_kernel_equals_the_oracle(cuda_device, V, H, W, s, mask_kind):
    pred, gt, mask = inputs(V, H, W, s, mask_kind, permuted=V % 2 == 0, seed=V + H + s, empty=(0,) if V > 2 else ())
    out = image_metrics(pred.to(cuda_device), gt.to(cuda_device), mask.to(cuda_device))
    ref, iou, psnr = im.image_metrics(pred.numpy(), gt.numpy(), mask.float().numpy())
    got = out.per_view.cpu().numpy()
    assert got.shape == (V, 5)
    # the sums: I and U within 1e-6 relative (an empty view's are exactly 0), E likewise
    np.testing.assert_allclose(got[:, :3], ref[:, :3], rtol=1e-6, atol=0)
    np.testing.assert_allclose(got[:, 3], ref[:, 3], rtol=0, atol=1e-6)
    np.testing.assert_allclose(got[:, 4], ref[:, 4], rtol=1e-6, atol=0)
    if V > 2:
        assert got[0, 0] == 0 and got[0, 1] == 0 and got[0, 3] == 1.0
    assert abs(float(out.iou) - got[:, 3].mean()) < 1e-12 and abs(float(out.psnr) - got[:, 4].mean()) < 1e-12 * psnr
    assert abs(float(out.iou) - iou) < 1e-6 and abs(float(out.psnr) - psnr) < 1e-6 * psnr


def test_same_size_reads_the_ground_truth_unchanged(cuda_device):
    """at s == H the resize returns the input: with alpha = 1 and a zero render, I_n = sum m and E_n = sum g^2, both
    summed from the stored values"""
    V, S = 4, 48
    _, gt, mask = inputs(V, S, S, S, permuted=True, seed=7)
    pred = torch.zeros(V, S, S, 4)
    pred[..., 3] = 1
    out = image_metrics(pred.to(cuda_device), gt.to(cuda_device), mask.to(cuda_device)).per_view.cpu()
    ref_I = mask.double().sum((1, 2))
    ref_E = (gt.double() ** 2).sum((1, 2, 3))
    torch.testing.assert_close(out[:, 0], ref_I, rtol=1e-14, atol=0)
    torch.testing.assert_close(out[:, 2], ref_E, rtol=1e-14, atol=0)


@pytest.mark.parametrize("H,W,s", [(20, 20, 8), (7, 7, 2), (37, 23, 11), (12, 12, 18), (5, 5, 5)])
def test_resized_mask_matches_torch_cuda(cuda_device, H, W, s):
    """one view per output pixel, its alpha one there and zero elsewhere: I_n is the resized mask at that pixel, which
    equals torch's CUDA F.interpolate to 1e-6 (the mask and the RGB share the resize)"""
    g = torch.Generator().manual_seed(H * W + s)
    m = torch.rand(H, W, generator=g, dtype=torch.float32).to(cuda_device)
    V = s * s
    pred = torch.zeros(V, s * s, 4, device=cuda_device)
    pred[torch.arange(V), torch.arange(V), 3] = 1
    gt = torch.zeros(1, H, W, 3, device=cuda_device).expand(V, H, W, 3)
    out = image_metrics(pred.view(V, s, s, 4), gt, m.expand(V, H, W))
    ref = F.interpolate(m[None, None], size=(s, s), mode="bilinear", align_corners=False).reshape(-1)
    torch.testing.assert_close(out.per_view[:, 0].float(), ref, rtol=0, atol=1e-6)
    if s == H:
        assert torch.equal(out.per_view[:, 0].float(), m.reshape(-1))


def test_bitwise_repeatable_and_capturable(cuda_device):
    pred, gt, mask = (t.to(cuda_device) for t in inputs(130, 128, 128, 32, "uint8", permuted=True, seed=3))
    a, b = image_metrics(pred, gt, mask), image_metrics(pred, gt, mask)
    assert torch.equal(a.per_view, b.per_view) and torch.equal(a.iou, b.iou) and torch.equal(a.psnr, b.psnr)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        image_metrics(pred, gt, mask)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        c = image_metrics(pred, gt, mask)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(c.per_view, a.per_view) and torch.equal(c.iou, a.iou) and torch.equal(c.psnr, a.psnr)


def test_rejects_bad_inputs(cuda_device):
    pred, gt, mask = (t.to(cuda_device) for t in inputs(2, 16, 16, 8))
    with pytest.raises(RuntimeError):
        image_metrics(pred[..., :3], gt, mask)
    with pytest.raises(RuntimeError):
        image_metrics(pred, gt[:1], mask)
    with pytest.raises(TypeError):
        image_metrics(pred, gt.double(), mask)
    with pytest.raises(TypeError):
        image_metrics(pred, gt, mask.double())
    with pytest.raises(RuntimeError):
        image_metrics(pred, gt, mask[:, :8])


# ---- the training loop and the export --------------------------------------------------------------------------------

def _config(tmp_path, data, name, **training):
    return write_config(tmp_path / (name + ".yml"), data, tmp_path / name, **training)


def test_loop_selects_by_iou_and_leaves_training_unchanged(data_dir, tmp_path):
    a = _config(tmp_path, data_dir, "iou", model_selection_metric="iou", validate_every=50)
    b = _config(tmp_path, data_dir, "cd", model_selection_metric="chamfer_point", validate_every=50)
    code, log = run_cli(a, "--max-it", "160")
    assert code == 0, log
    assert "Validation metric (iou)" in log and '"psnr"' in log
    code, log_b = run_cli(b, "--max-it", "160")
    assert code == 0, log_b
    out = tmp_path / "iou" / "torus"
    assert (out / "model_best.pt").exists() and (out / "val" / "best.ply").exists()
    best = torch.load(out / "model_best.pt", map_location="cpu", weights_only=False)
    assert 0.0 <= best["loss_val_best"] <= 1.0
    ca = torch.load(out / "model.pt", map_location="cpu", weights_only=False)
    cb = torch.load(tmp_path / "cd" / "torus" / "model.pt", map_location="cpu", weights_only=False)
    assert ca["it"] == cb["it"] == 159
    for k in ("points", "normals", "colors"):
        assert torch.equal(ca["model"][k], cb["model"][k]), k      # validation does not perturb training
    # the export of the selected model: min(vis_n_outputs, V) renders and the metrics report
    env = dict(os.environ)
    env["PYTHONPATH"] = ROOT + os.pathsep + env.get("PYTHONPATH", "")
    r = subprocess.run([sys.executable, "-m", "dss_b200.utils.generate", "--config", a, "--depth", "6", "--images"],
                       cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0, r.stdout
    gen = out / "generation"
    pngs = sorted(os.listdir(gen / "images"))
    assert pngs == ["%04d.png" % i for i in range(16)]          # vis_n_outputs 30 > 16 views
    from PIL import Image
    assert np.asarray(Image.open(gen / "images" / pngs[0])).shape == (128, 128, 4)
    with open(gen / "image_metrics.json") as f:
        rep = json.load(f)
    assert rep["views"] == 16 and [m["image_size"] for m in rep["metrics"]] == [32, 128]
    for m in rep["metrics"]:
        assert len(m["per_view"]["iou"]) == 16 and 0 <= m["iou"] <= 1 and m["psnr"] > 0
        db = [-10 * np.log10(p / 3) for p in m["per_view"]["psnr"]]
        np.testing.assert_allclose(m["per_view"]["psnr_db"], db, rtol=1e-12)
        assert abs(m["psnr_db"] - np.mean(db)) < 1e-9


def test_data_without_a_cloud_trains_under_iou_only(data_dir, tmp_path):
    from dss_b200.training.config import load_config
    from dss_b200.training.train import Trainer
    bare = tmp_path / "bare"
    shutil.copytree(data_dir, bare)
    d = dict(np.load(bare / "data_dict.npz", allow_pickle=True))
    del d["points"], d["normals"]
    np.savez(bare / "data_dict.npz", **d)
    if (bare / "mesh.obj").exists():
        os.remove(bare / "mesh.obj")
    t = Trainer(load_config(_config(tmp_path, str(bare), "bare", model_selection_metric="iou", validate_every=20)))
    assert t.run(exit_after=-1, max_it=21) == 0
    assert (tmp_path / "bare" / "torus" / "model_best.pt").exists()
    with pytest.raises(ValueError, match="points"):
        Trainer(load_config(_config(tmp_path, str(bare), "bare_cd", model_selection_metric="chamfer_point")))


def test_metrics_rank_the_data_cloud_above_the_initial_sphere(data_dir, tmp_path):
    from dss_b200.training.config import load_config
    from dss_b200.training.train import Trainer, initial_cloud
    from dss_b200.utils.dataset import MVRData
    dev = torch.device("cuda:0")
    t = Trainer(load_config(_config(tmp_path, data_dir, "m", model_selection_metric="psnr")))
    st, s = t.step, t.data.resolution[0] // 4
    flags = (st.Vrk_invariant, st.Vrk_isotropic, st.frnn_radius, st.shininess)
    # the loop's values equal image_metrics on the same renders of all the views at once (up to the fp64 order of
    # the mean over the views)
    ev = t.evaluate()
    image = render_data_views(st.points, st.normals, st.colours, t.data, t.params._replace(image_size=s),
                              range(len(t.data)), *flags)
    b = t.data.pinned_batch(list(range(len(t.data))))
    ref = image_metrics(image, b["img.rgb"].to(dev).permute(0, 2, 3, 1), b["img.mask"].to(dev))
    assert abs(ev["iou"] - float(ref.iou)) <= 1e-12 * abs(float(ref.iou))
    assert abs(ev["psnr"] - float(ref.psnr)) <= 1e-12 * abs(float(ref.psnr))
    # the data's own cloud scores lower errors than the initial ico-sphere
    pc = MVRData(data_dir).get_pointclouds()
    pts, nrm = pc.points_packed().to(dev), pc.normals_packed().to(dev)
    gt = evaluate_2d(pts, nrm, torch.ones_like(pts), t.data, t.params, s, 4, *flags)
    p0, n0, c0 = initial_cloud(2000, 0, dev)
    init = evaluate_2d(p0, n0, c0, t.data, t.params, s, 4, *flags)
    print("iou: data cloud %.4f, initial %.4f; psnr: %.5f, %.5f" % (float(gt["iou"]), float(init["iou"]),
                                                                    float(gt["psnr"]), float(init["psnr"])))
    assert float(gt["iou"]) < float(init["iou"]) and float(gt["psnr"]) < float(init["psnr"])
    assert abs(float(init["iou"]) - ev["iou"]) < 1e-12                     # the loop starts from that sphere
