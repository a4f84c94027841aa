"""GPU: camera refinement in the training step and the loop (model.model_kwargs.learn_cameras), on the torus data of
tests/test_gpu_train_loop.py with perturbed cameras (create_mvr_data --camera-noise 1 0.01).

What must hold:
  - the step: at zero poses its loss, image, filters and cloud gradients are those of the step without poses, bit for
    bit; the graphed step equals the eager one, poses' gradient included; a resident iteration makes no host
    synchronisation;
  - the loop runs through cameras_from_it, a prune and a growth, and the poses and their Adam moments keep their bits
    across both events;
  - a mid-epoch resume is bit-exact for the cloud, the poses and Adam's state; a checkpoint without poses resumes at
    zero poses; a checkpoint of another view count is refused;
  - the iou validation is evaluate_2d's on the data with the refined cameras, and generate --images writes them;
  - on 2 ranks the pose gradient is the one-GPU step's, with a view repeated across the ranks and a rank without views,
    and after 10 Adam steps every rank holds the same poses; the loop's replica check covers them."""
import os
import re
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

from dss_b200.training.step import GraphedTrainStep, TrainStep
from dss_b200.utils.dataset import MVRData
from dss_b200.utils.io import save_obj
from tests.test_gpu_train_loop import ROOT, write_config
from tests.test_gpu_train_step_sharded import _free_port
from tests.test_mesh_data import torus

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


@pytest.fixture(scope="module")
def noisy_dir(cuda_device, tmp_path_factory):
    from dss_b200.utils.create_mvr_data import main
    tmp = tmp_path_factory.mktemp("noisy_data")
    verts, faces = torus()
    save_obj(str(tmp / "torus.obj"), verts.numpy(), faces.numpy())
    return main(["--points", str(tmp / "torus.obj"), "--output", str(tmp / "data"), "--num_cameras", "16",
                 "--image-size", "128", "--tri_color_light", "--point_lights", "--seed", "3",
                 "--camera-noise", "1", "0.01"])[0]


def step_args(data_dir, tmp_path):
    from dss_b200.training.config import load_config, splat_params
    from dss_b200.training.train import initial_cloud
    data = MVRData(data_dir)
    cams = data.get_cameras()
    cfg = load_config(write_config(tmp_path / "c.yml", data_dir, tmp_path / "out"))
    return data, splat_params(cfg, cams.znear, cams.zfar), initial_cloud(2000, 0, DEV)


FLAGS = dict(Vrk_invariant=True, Vrk_isotropic=False, lambda_dr_proj=0.01)


def test_zero_poses_give_todays_step(noisy_dir, tmp_path):
    data, params, (p, n, c) = step_args(noisy_dir, tmp_path)
    views = data.device_views(DEV)
    idx = [3, 9, 3, 12]
    plain = GraphedTrainStep.from_views(p, n, c, params, views, idx, **FLAGS)
    posed = GraphedTrainStep.from_views(p, n, c, params, views, idx, poses=torch.zeros(16, 6, device=DEV), **FLAGS)
    eager = TrainStep(p, n, c, params, poses=torch.zeros(16, 6, device=DEV), views=views, **FLAGS)
    for batch in (idx, [0, 15, 15, 7]):
        for s in (plain, posed):
            s.load_views(batch)
            s.replay()
        eager(*views.batch(batch), idx=views.upload(batch))
        for k in plain.loss:
            assert torch.equal(plain.loss[k], posed.loss[k]) and torch.equal(plain.loss[k], eager.loss[k]), k
        for name in ("image", "visibility", "inmask"):
            assert torch.equal(getattr(plain, name), getattr(posed, name)), name
            assert torch.equal(getattr(plain, name), getattr(eager, name)), name
        for name in ("points", "normals"):
            assert torch.equal(getattr(plain, name).grad, getattr(posed, name).grad), name
            assert torch.equal(getattr(plain, name).grad, getattr(eager, name).grad), name
        assert posed.settings() != plain.settings()
        assert torch.equal(posed.poses.grad, eager.poses.grad)
        g = posed.poses.grad
        rows = torch.zeros(16, dtype=torch.bool)
        rows[batch] = True
        assert (g[~rows.to(DEV)] == 0).all() and (g[rows.to(DEV)].abs().sum(1) > 0).all()


def test_resident_iteration_with_poses_makes_no_host_synchronisation(noisy_dir, tmp_path):
    data, params, (p, n, c) = step_args(noisy_dir, tmp_path)
    step = GraphedTrainStep.from_views(p, n, c, params, data.device_views(DEV), [0, 1, 2, 3],
                                       poses=torch.zeros(16, 6, device=DEV), **FLAGS)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for idx in ([4, 5, 6, 7], [7, 7, 0, 15]):
            step.load_views(idx)
            step.replay()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert torch.isfinite(step.poses.grad).all()


def test_a_step_without_the_batch_views_is_refused(noisy_dir, tmp_path):
    data, params, (p, n, c) = step_args(noisy_dir, tmp_path)
    views = data.device_views(DEV)
    eager = TrainStep(p, n, c, params, poses=torch.zeros(16, 6, device=DEV), views=views, **FLAGS)
    with pytest.raises(RuntimeError, match="takes the batch's views"):
        eager(*views.batch([0, 1]))
    with pytest.raises(ValueError, match="pass views=DeviceViews"):
        TrainStep(p, n, c, params, poses=torch.zeros(16, 6, device=DEV), **FLAGS)
    with pytest.raises(RuntimeError, match=r"poses must be a float32 \(16, 6\)"):
        TrainStep(p, n, c, params, poses=torch.zeros(15, 6, device=DEV), views=views, **FLAGS)


# ---- the loop -----------------------------------------------------------------------------------------------------
def trainer(noisy_dir, tmp_path, out="out", learn=True, **training):
    from dss_b200.training.config import load_config
    from dss_b200.training.train import Trainer
    path = write_config(tmp_path / (out + ".yml"), noisy_dir, tmp_path / out, **training)
    cfg = load_config(path)
    cfg["model"]["model_kwargs"]["learn_cameras"] = learn
    return Trainer(cfg)


def pose_state(t):
    st = t.opt.state.get(t.poses, {})
    return [t.poses.detach().clone()] + [st[k].clone() for k in ("exp_avg", "exp_avg_sq") if k in st]


def same(a, b):
    return len(a) == len(b) and all(torch.equal(x, y) for x, y in zip(a, b))


def test_loop_keeps_the_poses_through_events(noisy_dir, tmp_path):
    t = trainer(noisy_dir, tmp_path, cameras_from_it=6, grow_milestones=[14], grow_points=[3000],
                prune_milestones=[14], validate_every=0, lr_cameras=1e-3)
    seen = {}
    for name in ("grow", "prune"):
        fn = getattr(t, name)

        def spy(*a, _fn=fn, _name=name):
            before = pose_state(t)
            _fn(*a)
            seen[_name] = (before, pose_state(t))
        setattr(t, name, spy)
    assert t.run(exit_after=-1, max_it=20) == 0
    assert t.step.points.shape[0] == 3000 or "Pruned" in open(tmp_path / "out" / "torus" / "train.log").read()
    for name in ("grow", "prune"):
        before, after = seen[name]
        assert len(before) == 3 and same(before, after), name
    assert t.poses.abs().sum() > 0
    log = open(tmp_path / "out" / "torus" / "train.log").read()
    assert "Learning the camera poses from it=6" in log and "cam_rot_max=" in log


def test_resume_is_exact_with_poses(noisy_dir, tmp_path):
    kw = dict(cameras_from_it=3, validate_every=0, checkpoint_every=0)
    a = trainer(noisy_dir, tmp_path, "a", **kw)
    assert a.run(exit_after=-1, max_it=30) == 0
    b = trainer(noisy_dir, tmp_path, "b", **kw)
    assert b.run(exit_after=-1, max_it=18) == 0             # 16 views, batch 4: mid-epoch
    b = trainer(noisy_dir, tmp_path, "b", **kw)
    assert b.it == 17 and b.run(exit_after=-1, max_it=30) == 0
    ca, cb = (torch.load(tmp_path / x / "torus" / "model.pt", map_location="cpu", weights_only=False) for x in "ab")
    for k in ("points", "normals", "colors"):
        assert torch.equal(ca["model"][k], cb["model"][k]), k
    assert torch.equal(ca["cameras"]["poses"], cb["cameras"]["poses"])
    sa, sb = ca["optimizer"]["state"], cb["optimizer"]["state"]
    assert sa.keys() == sb.keys()
    for i in sa:
        for k in sa[i]:
            assert torch.equal(sa[i][k], sb[i][k]), (i, k)


def test_checkpoint_without_poses_resumes_and_wrong_views_are_refused(noisy_dir, tmp_path):
    t = trainer(noisy_dir, tmp_path, learn=False, validate_every=0, checkpoint_every=0)
    assert t.run(exit_after=-1, max_it=6) == 0
    path = tmp_path / "out" / "torus" / "model.pt"
    ck = torch.load(path, map_location="cpu", weights_only=False)
    assert "cameras" not in ck
    t = trainer(noisy_dir, tmp_path, cameras_from_it=0, validate_every=0, checkpoint_every=0)
    assert torch.equal(t.poses, torch.zeros(16, 6, device=DEV))
    assert t.opt.param_groups[-1]["name"] == "cameras" and t.opt.param_groups[-1]["lr"] == t.lr_cameras
    assert t.run(exit_after=-1, max_it=10) == 0 and t.poses.abs().sum() > 0
    ck = torch.load(path, map_location="cpu", weights_only=False)
    ck["cameras"]["poses"] = torch.zeros(17, 6)
    torch.save(ck, path)
    with pytest.raises(ValueError, match="camera poses of shape \\(17, 6\\), but the data has 16 views"):
        trainer(noisy_dir, tmp_path, cameras_from_it=0)
    ck["cameras"]["poses"] = torch.zeros(16, 6)
    torch.save(ck, path)
    with pytest.raises(ValueError, match="learnt camera poses"):
        trainer(noisy_dir, tmp_path, learn=False)


def test_validation_and_generate_see_the_refined_cameras(noisy_dir, tmp_path):
    from dss_b200.ops import evaluate_2d
    from dss_b200.training.config import load_config
    from dss_b200.utils.generate import generate
    t = trainer(noisy_dir, tmp_path, cameras_from_it=0, validate_every=0, model_selection_metric="iou",
                lr_cameras=3e-3)
    assert t.run(exit_after=-1, max_it=12) == 0
    ev = t.evaluate()
    refined = t.views.with_poses(t.poses).camera_mat.cpu().numpy()
    data = MVRData(noisy_dir)
    data.camera_mat = refined.copy()
    st = t.step
    ref = evaluate_2d(st.points, st.normals, st.colours, data, t.params, 32, 4, st.Vrk_invariant, st.Vrk_isotropic,
                      st.frnn_radius, st.shininess)
    # the same cameras; their projections differ by the rounding of two ways of composing them
    assert abs(ev["iou"] - float(ref["iou"])) <= 2e-3 and abs(ev["psnr"] - float(ref["psnr"])) <= 2e-3 * ev["psnr"]
    cfg = load_config(str(tmp_path / "out.yml"))
    cfg["model"]["model_kwargs"]["learn_cameras"] = True
    cfg["generation"] = {"vis_n_outputs": 2}
    generate(cfg, depth=6, model=str(tmp_path / "out" / "torus" / "model.pt"), images=True)
    saved = np.load(tmp_path / "out" / "torus" / "generation" / "cameras.npz")["camera_mat"]
    assert saved.dtype == np.float32 and np.array_equal(saved, refined)


# ---- two ranks ----------------------------------------------------------------------------------------------------
_WORKER = r'''
import os, sys, torch, torch.distributed as dist
sys.path.insert(0, %(root)r)
rank, out_dir, port, data_dir = int(sys.argv[1]), sys.argv[2], int(sys.argv[3]), sys.argv[4]
dev = torch.device("cuda", 0)
torch.cuda.set_device(dev)
dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%%d" %% port, rank=rank, world_size=2)
from dss_b200.parallel import GradSync, check_replicas
from dss_b200.training.step import TrainStep
from dss_b200.training.train import initial_cloud
from dss_b200.utils.dataset import MVRData
from dss_b200.ops import SplatParams
data = MVRData(data_dir)
views = data.device_views(dev)
cams = data.get_cameras()
prm = SplatParams(image_size=128, points_per_pixel=5, cutoff_threshold=1.0, clip_pts_grad=0.05,
                  znear=float(cams.znear), zfar=float(cams.zfar))
p, n, c = initial_cloud(2000, 0, dev)
kw = dict(Vrk_invariant=True, Vrk_isotropic=False, lambda_dr_proj=0.01)
poses = torch.zeros(16, 6, device=dev)
poses[:, :3] = 0.003
out = {}
for name, parts in (("split", [[5, 2, 9], [5, 11]]), ("empty", [[5, 2, 9, 5, 11], []])):
    one = TrainStep(p, n, c, prm, poses=poses, views=views, **kw)
    full = [i for part in parts for i in part]
    one(*views.batch(full), idx=views.upload(full))
    sharded = TrainStep(p, n, c, prm, poses=poses, views=views, grad_sync=GradSync(), **kw)
    mine = views.upload(parts[rank])
    sharded(*views.batch_at(mine), idx=mine)
    ref, got = one.poses.grad, sharded.poses.grad
    err = float((got - ref).abs().max()) / float(ref.abs().max())
    print("rank %%d %%s: pose gradient error %%.3g of the largest" %% (rank, name, err))
    assert err <= 1e-6, err
    out[name] = got.cpu()
# 10 Adam steps on the sharded step: the same pose bits on every rank
step = TrainStep(p, n, c, prm, poses=poses, views=views, grad_sync=GradSync(), **kw)
opt = torch.optim.Adam([step.points, step.normals, step.poses], lr=1e-4, betas=(0.5, 0.9))
batches = [[[1, 2], [3]], [[4], [4, 0]], [[7, 8, 9], []]] * 4
for b in batches[:10]:
    mine = views.upload(b[rank])
    step(*views.batch_at(mine), idx=mine)
    opt.step()
check_replicas([("camera poses", step.poses)])
out["poses"] = step.poses.detach().cpu()
torch.save(out, os.path.join(out_dir, "rank%%d.pt" %% rank))
print("rank %%d ok" %% rank)
dist.destroy_process_group()
'''


def test_sharded_pose_gradient_and_replicas(noisy_dir):
    with tempfile.TemporaryDirectory() as d:
        w = os.path.join(d, "worker.py")
        with open(w, "w") as f:
            f.write(_WORKER % {"root": ROOT})
        env = dict(os.environ, PYTHONPATH=ROOT)
        port = _free_port()
        procs = [subprocess.Popen([sys.executable, w, str(r), d, str(port), noisy_dir], stdout=subprocess.PIPE,
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
        saved = [torch.load(os.path.join(d, "rank%d.pt" % r)) for r in range(2)]
    for k in saved[0]:
        assert torch.equal(saved[0][k], saved[1][k]), k


def test_sharded_loop_checks_the_poses(noisy_dir, tmp_path):
    from tests.test_gpu_train_loop_sharded import run_ranks
    path = write_config(tmp_path / "c.yml", noisy_dir, tmp_path / "out", validate_every=0, checkpoint_every=6)
    import yaml
    with open(path) as f:
        cfg = yaml.safe_load(f)
    cfg["model"]["model_kwargs"]["learn_cameras"] = True
    cfg["training"]["cameras_from_it"] = 2
    with open(path, "w") as f:
        yaml.safe_dump(cfg, f)
    codes, outs, _ = run_ranks(str(path), "--max-it", "8")
    assert codes == [0, 0], outs
    log = open(tmp_path / "out" / "torus" / "train.log").read()
    assert re.search(r"Replica check: the 2 ranks hold the same points, normals, camera poses and colours", log), log
    ck = torch.load(tmp_path / "out" / "torus" / "model.pt", map_location="cpu", weights_only=False)
    assert ck["cameras"]["poses"].abs().sum() > 0
