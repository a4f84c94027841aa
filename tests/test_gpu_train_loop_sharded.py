"""GPU: the training loop on several ranks (python -m dss_b200.training.train under torchrun's environment), on the
torus data and configuration of tests/test_gpu_train_loop.py.  Two ranks share one H100 over gloo, as the sharded
step's tests do; where two GPUs are visible the first two tests run again over NCCL, one GPU per rank.

What must hold, and why:
  - the first iteration against the one-GPU loop: the same batch, dealt over the ranks, gives the loss within a few
    float32 ulps (the image-loss sums are added in another order; the regularisers run replicated on the same cloud and
    filters: the same bits), and after one Adam step the points and normals within 2 lr (one flipped step at a gradient
    within rounding of zero, the argument of ADAM_TOL in tests/test_gpu_train_step_sharded.py), equal to rounding
    elsewhere;
  - the quality bar of the one-GPU loop, rank 0 alone writing, the replica guard running;
  - resume: bit for bit on the same number of ranks, and across 1 and 2 ranks the counters, epoch order and sampler
    continue;
  - a rank dealt no views (batch 1 on 2 ranks) trains along, with the one-GPU loss at it = 0;
  - the time limit and a refused configuration end every rank, and no process is left; under torchrun, which stops
    the other workers on the first non-zero exit, the time limit's model.pt is whole.
The ranks are started with torchrun's variables and a free localhost port, each in its own session, and every session
is killed on a timeout."""
import json
import os
import re
import shutil
import signal
import socket
import subprocess
import sys

import pytest
import torch

from dss_b200.ops import chamfer_distance
from tests.test_gpu_train_loop import data_dir, run_cli, write_config  # noqa: F401  (data_dir: a fixture)

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LR = 0.01                      # the Adam lr of points and normals (make_optimizer)
LOSS_ULPS = 4                  # the sharded step's bound on the image-loss scalars
ROUNDING = 1e-6                # a few float32 ulps at the torus's coordinates
TIMEOUT = 900
F32 = torch.finfo(torch.float32).eps


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _communicate(procs, timeout):
    """outputs of ``procs`` (each the leader of its own session); on a timeout every session is killed"""
    try:
        return [p.communicate(timeout=timeout)[0] for p in procs]
    finally:
        for p in procs:
            if p.poll() is None:
                os.killpg(p.pid, signal.SIGKILL)
                p.wait()


def _env(**extra):
    env = dict(os.environ, **extra)
    env["PYTHONPATH"] = ROOT + os.pathsep + env.get("PYTHONPATH", "")
    return env


def run_ranks(configs, *args, backend="gloo", timeout=TIMEOUT):
    """the loop on 2 ranks, started as torchrun starts them; ``configs``: one path, or one per rank.  Returns the exit
    codes, the outputs and the processes."""
    if isinstance(configs, str):
        configs = [configs, configs]
    G, port = len(configs), _free_port()
    procs = [subprocess.Popen([sys.executable, "-m", "dss_b200.training.train", "--config", configs[r], *args,
                               "--dist-backend", backend],
                              cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                              start_new_session=True,
                              env=_env(RANK=str(r), LOCAL_RANK=str(r), WORLD_SIZE=str(G), LOCAL_WORLD_SIZE=str(G),
                                       MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port)))
             for r in range(G)]
    outs = _communicate(procs, timeout)
    return [p.returncode for p in procs], outs, procs


def _load(path):
    return torch.load(path, map_location="cpu", weights_only=False)


def _records(out):
    with open(os.path.join(out, "metrics.jsonl")) as f:
        return [json.loads(line) for line in f]


def _need(backend):
    if backend == "nccl" and torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")


def test_pinned_batch_of_no_views(data_dir):  # noqa: F811
    from dss_b200.utils.dataset import MVRData
    data = MVRData(data_dir)
    full, empty = data.pinned_batch([3, 1]), data.pinned_batch([])
    assert full.keys() == empty.keys() == {"camera_mat", "img.rgb", "img.mask"}
    for k in full:
        assert empty[k].shape == (0,) + full[k].shape[1:] and empty[k].dtype == full[k].dtype, k
    assert torch.equal(full["camera_mat"], torch.from_numpy(data.camera_mat[[3, 1]]))


@pytest.mark.parametrize("backend", ["gloo", "nccl"])
def test_first_iteration_matches_one_gpu(data_dir, tmp_path, backend):  # noqa: F811
    _need(backend)
    one = write_config(tmp_path / "one.yml", data_dir, tmp_path / "one")
    two = write_config(tmp_path / "two.yml", data_dir, tmp_path / "two")
    code, log = run_cli(one, "--max-it", "1")
    assert code == 0, log
    codes, outs, _ = run_ranks(two, "--max-it", "1", backend=backend)
    assert codes == [0, 0], outs
    r1, r2 = _records(tmp_path / "one" / "torus")[0], _records(tmp_path / "two" / "torus")[0]
    assert r1["it"] == r2["it"] == 0
    ulps = {}
    for k in ("loss", "loss_dr_rgb", "loss_dr_silhouette", "loss_dr_proj", "loss_dr_repel"):
        ulps[k] = abs(r2[k] - r1[k]) / (F32 * abs(r1[k])) if r1[k] else abs(r2[k])
        assert ulps[k] <= (0 if k in ("loss_dr_proj", "loss_dr_repel") else LOSS_ULPS), (k, r1[k], r2[k])
    c1, c2 = _load(tmp_path / "one" / "torus" / "model.pt"), _load(tmp_path / "two" / "torus" / "model.pt")
    assert c1["it"] == c2["it"] == 0 and c1["epoch_order"] == c2["epoch_order"]
    report = []
    for k in ("points", "normals"):
        d = (c2["model"][k] - c1["model"][k]).abs()
        flipped = int((d > ROUNDING).sum())
        assert float(d.max()) <= 2 * LR, (k, float(d.max()))
        assert flipped <= d.numel() // 100, (k, flipped)
        report.append("%s: max |diff| %.3e, %d of %d entries beyond rounding" % (k, float(d.max()), flipped, d.numel()))
    assert torch.equal(c1["model"]["colors"], c2["model"]["colors"])
    print("%s, loss ulps %s; %s" % (backend, {k: round(v, 2) for k, v in ulps.items()}, "; ".join(report)))


@pytest.mark.parametrize("backend", ["gloo", "nccl"])
def test_loop_trains_on_two_ranks(data_dir, tmp_path, backend):  # noqa: F811
    from dss_b200.training.train import ground_truth_cloud, initial_cloud
    from dss_b200.utils.dataset import MVRData
    _need(backend)
    # rank 1 reads a configuration that differs only in the output directory: whatever it wrote would land there
    c0 = write_config(tmp_path / "c0.yml", data_dir, tmp_path / "out")
    c1 = write_config(tmp_path / "c1.yml", data_dir, tmp_path / "rank1")
    codes, outs, _ = run_ranks([c0, c1], "--max-it", "300", backend=backend)
    assert codes == [0, 0], outs
    assert not (tmp_path / "rank1").exists() and "[Epoch" not in outs[1], outs[1]
    out = tmp_path / "out" / "torus"
    assert len(_records(out)) == 300 // 10
    assert sorted(os.listdir(out)) == ["config.yaml", "metrics.jsonl", "model.pt", "model_best.pt", "train.log", "val"]
    assert os.listdir(out / "val") == ["best.ply"]
    with open(out / "train.log") as f:
        log = f.read()
    # before the validations at it = 100, 200 (model_best.pt may follow) and the final model.pt
    assert log.count("Replica check: the 2 ranks hold the same points, normals and colours") == 3, log
    best = _load(out / "model_best.pt")
    d = torch.device("cuda:0")
    gt = ground_truth_cloud(MVRData(data_dir), data_dir, 8000, d)
    p0, n0, _ = initial_cloud(2000, 0, d)
    init = float(chamfer_distance(gt[0][None], p0[None], x_normals=gt[1][None], y_normals=n0[None])[0])
    print("%s chamfer_point: initial %.5f, best %.5f (%.3fx) at it %d" % (
        backend, init, best["loss_val_best"], best["loss_val_best"] / init, best["it"]))
    assert best["loss_val_best"] <= 0.5 * init


def test_resume_on_two_ranks_is_exact(data_dir, tmp_path):  # noqa: F811
    a = write_config(tmp_path / "a.yml", data_dir, tmp_path / "a")
    b = write_config(tmp_path / "b.yml", data_dir, tmp_path / "b")
    codes, outs, _ = run_ranks(a, "--max-it", "100")
    assert codes == [0, 0], outs
    codes, outs, _ = run_ranks(b, "--max-it", "50")        # 4 iterations per epoch: 50 is mid-epoch
    assert codes == [0, 0], outs
    mid = _load(tmp_path / "b" / "torus" / "model.pt")
    assert mid["it"] == 49 and mid["epoch_pos"] % 16 != 0
    codes, outs, _ = run_ranks(b, "--max-it", "100")
    assert codes == [0, 0], outs
    assert "resumed" in outs[0]
    ca, cb = _load(tmp_path / "a" / "torus" / "model.pt"), _load(tmp_path / "b" / "torus" / "model.pt")
    assert ca["it"] == cb["it"] == 99 and ca["epoch_it"] == cb["epoch_it"]
    for k in ("points", "normals", "colors"):
        assert torch.equal(ca["model"][k], cb["model"][k]), k
    sa, sb = ca["optimizer"]["state"], cb["optimizer"]["state"]
    assert sa.keys() == sb.keys()
    for i in sa:
        for k in sa[i]:
            assert torch.equal(torch.as_tensor(sa[i][k]), torch.as_tensor(sb[i][k])), (i, k)
    assert ca["lr_scheduler"] == cb["lr_scheduler"] and ca["schedule"] == cb["schedule"]
    assert torch.equal(ca["sampler"], cb["sampler"]) and ca["epoch_order"] == cb["epoch_order"]


def test_resume_across_rank_counts(data_dir, tmp_path):  # noqa: F811
    two_one = write_config(tmp_path / "a.yml", data_dir, tmp_path / "a")
    one_two = write_config(tmp_path / "b.yml", data_dir, tmp_path / "b")
    codes, outs, _ = run_ranks(two_one, "--max-it", "50")
    assert codes == [0, 0], outs
    code, log = run_cli(one_two, "--max-it", "50")
    assert code == 0, log
    code, log = run_cli(two_one, "--max-it", "80")
    assert code == 0 and "resumed" in log, log
    codes, outs, _ = run_ranks(one_two, "--max-it", "80")
    assert codes == [0, 0] and "resumed" in outs[0], outs
    ca, cb = _load(tmp_path / "a" / "torus" / "model.pt"), _load(tmp_path / "b" / "torus" / "model.pt")
    assert ca["it"] == cb["it"] == 79 and ca["epoch_it"] == cb["epoch_it"] == 79 // 4
    assert torch.equal(ca["sampler"], cb["sampler"]) and ca["epoch_order"] == cb["epoch_order"]
    assert ca["epoch_pos"] == cb["epoch_pos"] and ca["lr_scheduler"] == cb["lr_scheduler"]
    assert ca["schedule"] == cb["schedule"]
    for c in (ca, cb):
        for k in ("exp_avg", "exp_avg_sq"):
            assert all(bool(torch.isfinite(s[k]).all()) for s in c["optimizer"]["state"].values())
        assert all(s["step"] == 80 for s in c["optimizer"]["state"].values())
    for log in (tmp_path / "a" / "torus" / "metrics.jsonl", tmp_path / "b" / "torus" / "metrics.jsonl"):
        assert [r["it"] for r in _records(log.parent)] == list(range(0, 80, 10))


def test_rank_without_views(data_dir, tmp_path):  # noqa: F811
    # batch 1 on 2 ranks: rank 1 is dealt no view at every iteration and runs the step's zero-view path
    one = write_config(tmp_path / "one.yml", data_dir, tmp_path / "one", batch_size=1, print_every=1)
    two = write_config(tmp_path / "two.yml", data_dir, tmp_path / "two", batch_size=1, print_every=1)
    code, log = run_cli(one, "--max-it", "1")
    assert code == 0, log
    codes, outs, _ = run_ranks(two, "--max-it", "10")
    assert codes == [0, 0], outs
    r1, recs = _records(tmp_path / "one" / "torus"), _records(tmp_path / "two" / "torus")
    assert [r["it"] for r in recs] == list(range(10))
    for k in ("loss", "loss_dr_rgb", "loss_dr_silhouette"):
        assert abs(recs[0][k] - r1[0][k]) <= LOSS_ULPS * F32 * abs(r1[0][k]), (k, recs[0][k], r1[0][k])
    ck = _load(tmp_path / "two" / "torus" / "model.pt")
    assert ck["it"] == 9 and bool(torch.isfinite(ck["model"]["points"]).all())
    assert "Replica check" in outs[0]


def _gone(procs):
    for p in procs:
        try:
            os.killpg(p.pid, 0)
        except ProcessLookupError:
            continue
        return False
    return True


def test_exit_after_zero_on_two_ranks(data_dir, tmp_path):  # noqa: F811
    cfg = write_config(tmp_path / "c.yml", data_dir, tmp_path / "out")
    codes, outs, procs = run_ranks(cfg, "--exit-after", "0")
    assert codes == [3, 3], outs
    ck = _load(tmp_path / "out" / "torus" / "model.pt")
    assert ck["it"] == 0 and ck["model"]["points"].shape == (1, 2000, 3)
    assert _gone(procs)


@pytest.mark.parametrize("refusal", ["batch_size", "mesh"])
def test_refused_configuration_fails_every_rank(data_dir, tmp_path, refusal):  # noqa: F811
    if refusal == "batch_size":
        cfg = write_config(tmp_path / "c.yml", data_dir, tmp_path / "out", batch_size=17)
        msg = "batch_size 17 is larger than the 16 views: an epoch would have no batch"
    else:
        # the validation's 8000 samples are drawn from mesh.obj, which only rank 0 reads; every rank checks it exists
        bare = tmp_path / "bare"
        shutil.copytree(data_dir, bare)
        os.remove(bare / "mesh.obj")
        cfg = write_config(tmp_path / "c.yml", str(bare), tmp_path / "out")
        msg = "No such file or directory: '%s'" % (bare / "mesh.obj")
    codes, outs, procs = run_ranks(cfg, "--max-it", "5", timeout=180)
    assert all(c != 0 for c in codes), outs
    assert all(msg in o for o in outs), outs
    code, log = run_cli(cfg, "--max-it", "5")
    assert code != 0 and msg in log, log
    assert _gone(procs)


def test_torchrun_launch(data_dir, tmp_path):  # noqa: F811
    cfg = write_config(tmp_path / "c.yml", data_dir, tmp_path / "out")
    p = subprocess.Popen([sys.executable, "-m", "torch.distributed.run", "--standalone", "--nproc-per-node", "2",
                          "-m", "dss_b200.training.train", "--config", cfg, "--dist-backend", "gloo", "--max-it", "20"],
                         cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                         start_new_session=True, env=_env())
    out = _communicate([p], TIMEOUT)[0]
    assert p.returncode == 0, out
    assert _load(tmp_path / "out" / "torus" / "model.pt")["it"] == 19
    assert _gone([p])


def test_torchrun_time_limit_saves_before_any_rank_leaves(data_dir, tmp_path):  # noqa: F811
    # torchrun stops the other workers on the first non-zero exit: rank 1's status 3 must not cut rank 0's save short
    cfg = write_config(tmp_path / "c.yml", data_dir, tmp_path / "out")
    p = subprocess.Popen([sys.executable, "-m", "torch.distributed.run", "--standalone", "--nproc-per-node", "2",
                          "-m", "dss_b200.training.train", "--config", cfg, "--dist-backend", "gloo",
                          "--exit-after", "0"],
                         cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                         start_new_session=True, env=_env())
    out = _communicate([p], TIMEOUT)[0]
    assert p.returncode != 0, out                     # torchrun reports the workers' status 3 as a failure
    assert re.search(r"exitcode\s*:\s*3\b", out), out
    run_dir = tmp_path / "out" / "torus"
    ck = _load(run_dir / "model.pt")
    assert ck["it"] == 0 and ck["model"]["points"].shape == (1, 2000, 3)
    assert not [f for f in os.listdir(run_dir) if f.endswith(".tmp")]
    assert _gone([p])
