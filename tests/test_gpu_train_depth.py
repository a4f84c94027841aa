"""GPU: dense depth supervision in the training step and the loop (training.lambda_dr_depth, data.load_dense_depth), on
the torus data of tests/test_gpu_train_loop.py, whose create_mvr_data run now writes depth/%06d.exr.

What must hold:
  - create_mvr_data's depth maps are render_mesh's z-buffer with zfar on the background, bit for bit;
  - at lambda_dr_depth = 0 the step reads no depth (the same bits with and without depth maps); with it > 0 the graphed step (which gathers the batch's
    depth inside the capture) equals the eager one and reports loss_dr_depth;
  - the loop trains with the term, resumes exactly mid-epoch, and runs on 2 ranks, also with a rank dealt no views,
    whose collectives must pair with the other rank's (its first iteration matches one GPU's)."""
import os

import numpy as np
import pytest
import torch
import yaml

from dss_b200.training.step import GraphedTrainStep, TrainStep
from dss_b200.utils.dataset import MVRData
from dss_b200.utils.io import read_exr
from tests.test_gpu_train_loop import data_dir, run_cli, write_config  # noqa: F401
from tests.test_gpu_train_loop_sharded import F32, LOSS_ULPS, _records, run_ranks

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
FLAGS = dict(Vrk_invariant=True, Vrk_isotropic=False, lambda_dr_proj=0.01)


def test_depth_maps_are_the_mesh_zbuf(data_dir):  # noqa: F811
    from dss_b200.core.camera import camera_matrices
    from dss_b200.ops import render_mesh
    from dss_b200.utils.io import read_mesh
    data = MVRData(data_dir, load_dense_depth=True)
    cams = data.get_cameras()
    proj, view = camera_matrices(cams)
    verts, faces = read_mesh(os.path.join(data_dir, "mesh.obj"))
    r = render_mesh(torch.from_numpy(verts).to(DEV), torch.from_numpy(faces).to(DEV), proj.to(DEV), view.to(DEV), 128)
    want = torch.where(r.pix_to_face >= 0, r.zbuf, torch.tensor(cams.zfar, dtype=torch.float32, device=DEV)).cpu()
    files = sorted(os.listdir(os.path.join(data_dir, "depth")))
    assert files == ["%06d.exr" % i for i in range(16)]
    got = torch.from_numpy(np.stack([read_exr(os.path.join(data_dir, "depth", f)) for f in files]))
    assert torch.equal(got.view(torch.int32), want.view(torch.int32))
    assert torch.equal(torch.from_numpy(np.stack([d[0] for d in (data[i]["img.depth"] for i in range(16))])), got)
    assert (got < cams.zfar).any() and (got == cams.zfar).any()


def _step_args(data_dir, tmp_path):
    from dss_b200.training.config import load_config, splat_params
    from dss_b200.training.train import initial_cloud
    data = MVRData(data_dir, load_dense_depth=True)
    cams = data.get_cameras()
    cfg = load_config(write_config(tmp_path / "c.yml", data_dir, tmp_path / "out"))
    return data, splat_params(cfg, cams.znear, cams.zfar), initial_cloud(2000, 0, DEV)


def test_lambda_zero_reads_no_depth(data_dir, tmp_path):  # noqa: F811
    # at lambda 0 the depth maps the views hold change nothing: the step on views without them gives the same bits
    # (that this is the step of before is what the unchanged tests of test_gpu_train_step.py show)
    data, params, (p, n, c) = _step_args(data_dir, tmp_path)
    with_depth, without = data.device_views(DEV), MVRData(data_dir).device_views(DEV)
    assert with_depth.depth is not None and without.depth is None
    idx = [3, 9, 3, 12]
    a = GraphedTrainStep.from_views(p, n, c, params, with_depth, idx, lambda_dr_depth=0.0, **FLAGS)
    b = GraphedTrainStep.from_views(p, n, c, params, without, idx, **FLAGS)
    assert a.depth is None
    for batch in (idx, [0, 15, 15, 7]):
        for s in (a, b):
            s.load_views(batch)
            s.replay()
        assert a.loss.keys() == b.loss.keys() and "loss_dr_depth" not in a.loss
        for k in a.loss:
            assert torch.equal(a.loss[k], b.loss[k]), k
        for name in ("image", "visibility", "inmask"):
            assert torch.equal(getattr(a, name), getattr(b, name)), name
        for name in ("points", "normals"):
            assert torch.equal(getattr(a, name).grad, getattr(b, name).grad), name


def test_depth_step_graphed_equals_eager(data_dir, tmp_path):  # noqa: F811
    data, params, (p, n, c) = _step_args(data_dir, tmp_path)
    views = data.device_views(DEV)
    assert views.depth is not None and views.depth.shape == (16, 128, 128)
    idx = [3, 9, 3, 12]
    graphed = GraphedTrainStep.from_views(p, n, c, params, views, idx, lambda_dr_depth=0.5, **FLAGS)
    plain = TrainStep(p, n, c, params, **FLAGS)
    eager = TrainStep(p, n, c, params, lambda_dr_depth=0.5, **FLAGS)
    with pytest.raises(RuntimeError, match="depth"):
        eager(*views.batch(idx))
    for batch in (idx, [0, 15, 15, 7]):
        graphed.load_views(batch)
        graphed.replay()
        dev_idx = views.upload(batch)
        eager(*views.batch(batch), depth=views.depth_at(dev_idx))
        plain(*views.batch(batch))
        for k in eager.loss:
            assert torch.equal(graphed.loss[k], eager.loss[k]), k
        assert float(eager.loss["loss_dr_depth"]) > 0
        assert torch.equal(eager.loss["loss"], plain.loss["loss"] + eager.loss["loss_dr_depth"])
        for name in ("points", "normals"):
            assert torch.equal(getattr(graphed, name).grad, getattr(eager, name).grad), name
        assert not torch.equal(eager.points.grad, plain.points.grad)


def _depth_config(path, data_dir, out_dir, **training):  # noqa: F811
    cfg_path = write_config(path, data_dir, out_dir, lambda_dr_depth=1.0, **training)
    with open(cfg_path) as f:
        cfg = yaml.safe_load(f)
    cfg["data"]["load_dense_depth"] = True
    with open(cfg_path, "w") as f:
        yaml.safe_dump(cfg, f)
    return cfg_path


def _load(path):
    return torch.load(path, map_location="cpu", weights_only=False)


def test_loop_trains_and_resumes_exactly(data_dir, tmp_path):  # noqa: F811
    # the schedule of tests/test_gpu_train_loop.py::test_resume_is_exact, with the depth term
    a = _depth_config(tmp_path / "a.yml", data_dir, tmp_path / "a")
    b = _depth_config(tmp_path / "b.yml", data_dir, tmp_path / "b")
    code, log = run_cli(a, "--max-it", "240")
    assert code == 0, log
    assert "loss_dr_depth" in log
    with open(os.path.join(tmp_path / "a" / "torus", "metrics.jsonl")) as f:
        import json
        recs = [json.loads(line) for line in f]
    assert recs[-1]["loss_dr_depth"] < recs[0]["loss_dr_depth"]
    code, log = run_cli(b, "--max-it", "130")                # 4 iterations per epoch: 130 is mid-epoch
    assert code == 0, log
    code, log = run_cli(b, "--max-it", "240")
    assert code == 0 and "resumed" in log, log
    ca, cb = _load(tmp_path / "a" / "torus" / "model.pt"), _load(tmp_path / "b" / "torus" / "model.pt")
    assert ca["it"] == cb["it"] == 239
    for k in ("points", "normals", "colors"):
        assert torch.equal(ca["model"][k], cb["model"][k]), k


def test_loop_refuses_depth_without_maps(data_dir, tmp_path):  # noqa: F811
    cfg = write_config(tmp_path / "c.yml", data_dir, tmp_path / "c", lambda_dr_depth=1.0)
    code, log = run_cli(cfg, "--max-it", "2")
    assert code != 0 and "load_dense_depth" in log, log


def test_loop_on_two_ranks(data_dir, tmp_path):  # noqa: F811
    cfg = _depth_config(tmp_path / "c.yml", data_dir, tmp_path / "c", validate_every=0)
    codes, outs, _ = run_ranks(cfg, "--max-it", "30")
    assert codes == [0, 0], outs
    assert "loss_dr_depth" in outs[0]


def test_rank_without_views(data_dir, tmp_path):  # noqa: F811
    # batch 1 on 2 ranks: rank 1 is dealt no view at every iteration and runs the step's zero-view path, whose depth
    # loss all-reduce must come where the other rank's does
    one = _depth_config(tmp_path / "one.yml", data_dir, tmp_path / "one", batch_size=1, print_every=1, validate_every=0)
    two = _depth_config(tmp_path / "two.yml", data_dir, tmp_path / "two", batch_size=1, print_every=1, validate_every=0)
    code, log = run_cli(one, "--max-it", "1")
    assert code == 0, log
    codes, outs, _ = run_ranks(two, "--max-it", "10", timeout=300)
    assert codes == [0, 0], outs
    r1, recs = _records(tmp_path / "one" / "torus"), _records(tmp_path / "two" / "torus")
    assert [r["it"] for r in recs] == list(range(10))
    assert r1[0]["loss_dr_depth"] > 0
    for k in ("loss", "loss_dr_rgb", "loss_dr_silhouette", "loss_dr_depth"):
        assert abs(recs[0][k] - r1[0][k]) <= LOSS_ULPS * F32 * abs(r1[0][k]), (k, recs[0][k], r1[0][k])
    ck = _load(tmp_path / "two" / "torus" / "model.pt")
    assert ck["it"] == 9 and bool(torch.isfinite(ck["model"]["points"]).all())
