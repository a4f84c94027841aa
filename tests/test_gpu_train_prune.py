"""GPU: pruning the cloud during training (training.prune_milestones, prune_min_views, prune_max_outside), on the torus
data and configuration of tests/test_gpu_train_loop.py and the rank launcher of tests/test_gpu_train_loop_sharded.py.

What must hold:
  - the event: the kept rows and their Adam moments are the rows before it at an independently recomputed ``keep``
    (the coverage oracle on the views' renders and masks), in order; Adam's step counts and learning rates and the LR
    scheduler go on; planted strays go; a prune that would leave GROW_K or fewer points, or remove none, leaves the
    cloud and its step as they are;
  - a run that prunes and grows trains to the quality bar of the fixed-size loop and saves at its final size;
  - a run stopped before a milestone and resumed prunes there and ends with the bits of an uninterrupted run, on one
    GPU and on two ranks; across 1 and 2 ranks it resumes and continues; two ranks keep the points one GPU keeps."""
import re
import shutil

import numpy as np
import pytest
import torch

from dss_b200.ops import _data_view_renderer
from dss_b200.training.config import GROW_K
from tests.test_gpu_point_coverage import oracle
from tests.test_gpu_train_grow import MOMENTS, _same_checkpoints, _snapshot
from tests.test_gpu_train_loop import data_dir, run_cli, write_config  # noqa: F401  (data_dir: a fixture)
from tests.test_gpu_train_loop_sharded import LR, _load, _records, run_ranks

pytestmark = pytest.mark.gpu

# above the torus (radius 0.85, height 0.25): over background in some view of any camera ring around it
STRAYS = [[0, 0.8, 0], [0, -0.8, 0], [0, 0.55, 0], [0.2, 0.7, -0.2], [-0.2, -0.7, 0.2]]
PRUNED = re.compile(r"Pruned the cloud at it=(\d+): (\d+) -> (\d+) points")


def _keep_oracle(t, points, normals, min_views, max_outside):
    """keep of the cloud (points, normals as stored) from the coverage oracle on the trainer's renders of every view,
    one at a time, against the views' masks"""
    st, views = t.step, t.views
    render = _data_view_renderer(points, normals, torch.ones_like(points), views, st.Vrk_invariant, st.Vrk_isotropic,
                                 st.frnn_radius, st.shininess)
    seen = outside = 0
    for v in range(len(views)):
        _, mask = views.gather(views.upload([v]))
        s, o = oracle(render(t.params, [v]), mask, 1)
        seen, outside = seen + s, outside + o
    return (seen >= min_views) & ((outside <= max_outside) if max_outside is not None else True)


def _trainer(data_dir, tmp_path, **training):  # noqa: F811
    from dss_b200.training.config import load_config
    from dss_b200.training.train import Trainer
    cfg = load_config(write_config(tmp_path / "c.yml", data_dir, tmp_path / "out", validate_every=0, **training))
    return Trainer(cfg)


def _log(tmp_path):
    with open(tmp_path / "out" / "torus" / "train.log") as f:
        return f.read()


def test_prune_event_is_exact(data_dir, tmp_path):  # noqa: F811
    M = 22                            # 16 views, batch 4: the milestone is mid-epoch, past one LR-scheduler step
    t = _trainer(data_dir, tmp_path, scheduler_milestones=[2, 4], prune_milestones=[M])
    seen = {}
    prune = t.prune

    def spy():
        assert t.it == M
        with torch.no_grad():         # plant strays among the trained points (the step is rebuilt by the event)
            t.step.points[:len(STRAYS)] = torch.tensor(STRAYS, device=t.dev)
        before = _snapshot(t)
        c = before["cloud"]
        keep = _keep_oracle(t, c["points"], c["normals"], 1, 0)
        prune()
        seen.update(before=before, keep=keep, after=_snapshot(t), leaves=(t.step.points, t.step.normals), opt=t.opt)

    t.prune = spy
    assert t.run(exit_after=-1, max_it=M + 1) == 0
    before, after, keep = seen["before"], seen["after"], seen["keep"]
    P, n = 2000, int(keep.sum())
    assert not keep[:len(STRAYS)].any() and GROW_K < n < P
    idx = torch.from_numpy(np.nonzero(keep)[0]).to(t.dev)
    for k in ("points", "normals", "colours"):
        assert torch.equal(after["cloud"][k], before["cloud"][k][idx]), k
    for mb, ma in zip(before["moments"], after["moments"]):
        for k in MOMENTS:
            assert torch.equal(ma[k], mb[k][idx]), k
    assert [float(s) for s in after["steps"]] == [float(s) for s in before["steps"]] == [M] * 2
    assert after["groups"] == before["groups"]
    assert [g["lr"] for g in before["groups"]] == [LR * 0.5 ** 2] * 2
    assert after["sched"] == before["sched"]
    opt, leaves = seen["opt"], seen["leaves"]
    assert all(float(opt.state[p]["step"]) == M + 1 for p in leaves)
    assert t.step.points.shape == (n, 3)
    log = _log(tmp_path)
    assert "Pruned the cloud at it=%d: %d -> %d points" % (M, P, n) in log, log
    print([line for line in log.splitlines() if "Pruned" in line])


@pytest.mark.parametrize("case", ["too_few", "none_removed"])
def test_prune_that_changes_nothing(data_dir, tmp_path, case):  # noqa: F811
    M = 6
    th = dict(prune_min_views=1, prune_max_outside=0) if case == "too_few" else \
        dict(prune_min_views=0, prune_max_outside=16)
    t = _trainer(data_dir, tmp_path, prune_milestones=[M], **th)
    seen = {}
    prune = t.prune

    def spy():
        if case == "too_few":        # all but GROW_K points past zfar: seen in no view
            with torch.no_grad():
                t.step.points[GROW_K:] = 1e3
        seen["before"], seen["step"] = _snapshot(t), t.step
        prune()
        seen["after"], seen["same_step"] = _snapshot(t), t.step is seen["step"]

    t.prune = spy
    assert t.run(exit_after=-1, max_it=M + 1) == 0
    assert seen["same_step"]
    for k in ("points", "normals", "colours"):
        assert torch.equal(seen["after"]["cloud"][k], seen["before"]["cloud"][k]), k
    log = _log(tmp_path)
    want = "pruning would leave" if case == "too_few" else "every point passes"
    assert "Kept the cloud at it=%d: %s" % (M, want) in log, log
    assert t.step.points.shape == (2000, 3)


def test_loop_prunes_grows_and_trains(data_dir, tmp_path):  # noqa: F811
    from dss_b200.training.train import ground_truth_cloud, initial_cloud
    from dss_b200.ops import chamfer_distance
    from dss_b200.utils.dataset import MVRData
    cfg = write_config(tmp_path / "c.yml", data_dir, tmp_path / "out", grow_milestones=[100, 200],
                       grow_points=[4000, 8000], prune_milestones=[100, 200], validate_every=250)
    code, log = run_cli(cfg, "--max-it", "501")
    assert code == 0, log
    print("\n".join(line for line in log.splitlines()
                    if any(w in line for w in ("Validation", "Grew", "Pruned", "Kept"))))
    events = [line for line in log.splitlines() if "Pruned" in line or "Kept the cloud" in line or "Grew" in line]
    assert len(events) == 4 and "at it=100" in events[0] and "Grew the cloud at it=100" in events[1], events
    assert "at it=200" in events[2] and "Grew the cloud at it=200" in events[3] and "-> 8000 points" in events[3]
    out = tmp_path / "out" / "torus"
    ck, best = _load(out / "model.pt"), _load(out / "model_best.pt")
    assert ck["it"] == 500 and ck["model"]["points"].shape == (1, 8000, 3)
    assert ck["model"]["points_activation"].shape == (1, 8000)
    d = torch.device("cuda:0")
    gt = ground_truth_cloud(MVRData(data_dir), data_dir, 8000, d)
    p0, n0, _ = initial_cloud(2000, 0, d)
    init = float(chamfer_distance(gt[0][None], p0[None], x_normals=gt[1][None], y_normals=n0[None])[0])
    print("chamfer_point: initial %.5f, best %.5f (%.3fx) at it %d" % (init, best["loss_val_best"],
                                                                       best["loss_val_best"] / init, best["it"]))
    assert best["loss_val_best"] <= 0.5 * init


def test_resume_across_a_prune_milestone_is_exact(data_dir, tmp_path):  # noqa: F811
    prune = dict(prune_milestones=[150])
    a = write_config(tmp_path / "a.yml", data_dir, tmp_path / "a", **prune)
    b = write_config(tmp_path / "b.yml", data_dir, tmp_path / "b", **prune)
    code, log = run_cli(a, "--max-it", "240")
    assert code == 0 and "at it=150" in log, log
    event = [line.split(" ", 2)[2] for line in log.splitlines() if "at it=150" in line][0].split(" (")[0]
    print(event)
    code, log = run_cli(b, "--max-it", "130")
    assert code == 0 and "at it=150" not in log, log
    code, log = run_cli(b, "--max-it", "240")
    assert code == 0 and "resumed" in log and event in log, log
    ca, cb = _load(tmp_path / "a" / "torus" / "model.pt"), _load(tmp_path / "b" / "torus" / "model.pt")
    _same_checkpoints(ca, cb, 239)
    ra = {r["it"]: r for r in _records(tmp_path / "a" / "torus")}
    rb = {r["it"]: r for r in _records(tmp_path / "b" / "torus")}
    for it in range(150, 240, 10):
        assert {k: v for k, v in ra[it].items() if k != "time"} == {k: v for k, v in rb[it].items() if k != "time"}


def test_two_ranks_keep_what_one_gpu_keeps(data_dir, tmp_path):  # noqa: F811
    # both resume from one checkpoint written just before the milestone: the same cloud gives the same keep
    M = 20
    prune = dict(prune_milestones=[M], print_every=M, prune_min_views=2, prune_max_outside=1)
    one = write_config(tmp_path / "one.yml", data_dir, tmp_path / "one", **prune)
    two = write_config(tmp_path / "two.yml", data_dir, tmp_path / "two", **prune)
    code, log = run_cli(one, "--max-it", str(M))
    assert code == 0, log
    (tmp_path / "two" / "torus").mkdir(parents=True)
    shutil.copy(tmp_path / "one" / "torus" / "model.pt", tmp_path / "two" / "torus" / "model.pt")
    code, log = run_cli(one, "--max-it", str(M + 1))
    assert code == 0, log
    codes, outs, _ = run_ranks(two, "--max-it", str(M + 1))
    assert codes == [0, 0], outs
    e1, e2 = PRUNED.findall(log), PRUNED.findall(outs[0])
    assert len(e1) == 1 and e1 == e2, (log, outs[0])
    assert "Replica check: the 2 ranks hold the same points, normals and colours and Adam moments" in outs[0], outs[0]
    c1, c2 = _load(tmp_path / "one" / "torus" / "model.pt"), _load(tmp_path / "two" / "torus" / "model.pt")
    n = int(e1[0][2])
    assert c1["model"]["points"].shape == c2["model"]["points"].shape == (1, n, 3)
    assert torch.equal(c1["model"]["colors"], c2["model"]["colors"])
    for k in ("points", "normals"):
        assert float((c2["model"][k] - c1["model"][k]).abs().max()) <= 2 * LR, k


def test_resume_across_rank_counts_and_a_prune_milestone(data_dir, tmp_path):  # noqa: F811
    prune = dict(prune_milestones=[60], prune_min_views=2)
    two_one = write_config(tmp_path / "a.yml", data_dir, tmp_path / "a", **prune)
    one_two = write_config(tmp_path / "b.yml", data_dir, tmp_path / "b", **prune)
    codes, outs, _ = run_ranks(two_one, "--max-it", "50")
    assert codes == [0, 0], outs
    code, log = run_cli(one_two, "--max-it", "50")
    assert code == 0, log
    code, log = run_cli(two_one, "--max-it", "80")
    assert code == 0 and "resumed" in log and "at it=60" in log, log
    codes, outs, _ = run_ranks(one_two, "--max-it", "80")
    assert codes == [0, 0] and "resumed" in outs[0] and "at it=60" in outs[0], outs
    ca, cb = _load(tmp_path / "a" / "torus" / "model.pt"), _load(tmp_path / "b" / "torus" / "model.pt")
    assert ca["it"] == cb["it"] == 79 and ca["epoch_it"] == cb["epoch_it"] == 79 // 4
    assert ca["lr_scheduler"] == cb["lr_scheduler"] and ca["schedule"] == cb["schedule"]
    for c in (ca, cb):
        P = c["model"]["points"].shape[1]
        assert 16 < P <= 2000
        for s in c["optimizer"]["state"].values():
            assert s["step"] == 80
            for k in MOMENTS:
                assert s[k].shape == (P, 3) and bool(torch.isfinite(s[k]).all())


def test_resume_on_two_ranks_across_a_prune_milestone_is_exact(data_dir, tmp_path):  # noqa: F811
    prune = dict(prune_milestones=[70], prune_min_views=2)
    a = write_config(tmp_path / "a.yml", data_dir, tmp_path / "a", **prune)
    b = write_config(tmp_path / "b.yml", data_dir, tmp_path / "b", **prune)
    codes, outs, _ = run_ranks(a, "--max-it", "100")
    assert codes == [0, 0], outs
    codes, outs, _ = run_ranks(b, "--max-it", "50")
    assert codes == [0, 0], outs
    codes, outs, _ = run_ranks(b, "--max-it", "100")
    assert codes == [0, 0] and "resumed" in outs[0] and "at it=70" in outs[0], outs
    _same_checkpoints(_load(tmp_path / "a" / "torus" / "model.pt"), _load(tmp_path / "b" / "torus" / "model.pt"), 99)
