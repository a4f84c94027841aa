"""GPU: growing the cloud during training (training.grow_milestones / grow_points), on the torus data and configuration
of tests/test_gpu_train_loop.py and the rank launcher of tests/test_gpu_train_loop_sharded.py.

What must hold:
  - the event: the rows the cloud had and their Adam moments stay the same bits, the new rows are those of a direct
    upsample_points call on the same inputs, and Adam's step counts and learning rates and the LR scheduler go on;
  - a run that grows 2000 -> 4000 -> 8000 trains to the quality bar of the fixed-size loop and saves the grown cloud;
  - a run stopped before a milestone and resumed grows there and ends with the bits of an uninterrupted run, on one GPU
    and on two ranks; across 1 and 2 ranks it ends at the grown size with its counters continuing;
  - on two ranks the replicas agree after the event, and the first iteration after it matches one GPU's within the
    tolerance of the sharded loop's first iteration."""
import torch
import torch.nn.functional as F
import pytest

from dss_b200.ops import chamfer_distance, upsample_points
from dss_b200.utils.io import read_ply
from tests.test_gpu_train_loop import data_dir, run_cli, write_config  # noqa: F401  (data_dir: a fixture)
from tests.test_gpu_train_loop_sharded import F32, LOSS_ULPS, LR, ROUNDING, _load, _records, run_ranks

pytestmark = pytest.mark.gpu

MOMENTS = ("exp_avg", "exp_avg_sq")


def _snapshot(t):
    """the trainer's cloud, Adam state (per group, in group order) and LR scheduler state, copied"""
    s, opt = t.step, t.opt
    params = [g["params"][0] for g in opt.param_groups]
    return {"cloud": {k: getattr(s, k).detach().clone() for k in ("points", "normals", "colours")},
            "moments": [{k: opt.state[p][k].clone() for k in MOMENTS} for p in params],
            "steps": [opt.state[p]["step"].clone() for p in params],
            "groups": [{k: v for k, v in g.items() if k != "params"} for g in opt.param_groups],
            "sched": t.lr_sched.state_dict()}


def test_growth_event_is_exact(data_dir, tmp_path):  # noqa: F811
    from dss_b200.training.config import load_config
    from dss_b200.training.train import Trainer
    M, N = 22, 3500                   # 16 views, batch 4: the milestone is mid-epoch, past one LR-scheduler step
    cfg = load_config(write_config(tmp_path / "c.yml", data_dir, tmp_path / "out", validate_every=0,
                                   scheduler_milestones=[2, 4], grow_milestones=[M], grow_points=[N]))
    t = Trainer(cfg)
    seen = {}
    grow = t.grow

    def spy(n):
        assert t.it == M and n == N
        before = _snapshot(t)
        c = before["cloud"]
        feats = torch.cat([c["colours"]] + [m[k] for m in before["moments"] for k in MOMENTS], 1)
        ref = upsample_points(c["points"], n, k=16, normals=F.normalize(c["normals"], dim=-1), features=feats)
        grow(n)
        seen.update(before=before, ref=ref, after=_snapshot(t),
                    leaves=(t.step.points, t.step.normals, t.step.colours), opt=t.opt)

    t.grow = spy
    assert t.run(exit_after=-1, max_it=M + 1) == 0
    before, after, ref = seen["before"], seen["after"], seen["ref"]
    P = before["cloud"]["points"].shape[0]
    assert P == 2000 and ref.points.shape[0] == N
    # the rows the cloud had, bit for bit; the new ones, the direct call's
    new = {"points": ref.points, "normals": ref.normals, "colours": ref.features[:, :3]}
    for k in ("points", "normals", "colours"):
        a = after["cloud"][k]
        assert a.shape == (N, 3) and a.dtype == torch.float32, k
        assert torch.equal(a[:P], before["cloud"][k]), k
        assert torch.equal(a[P:], new[k][P:]), k
    # the stored normals are not unit and are not renormalised; the children's are
    assert not torch.allclose(before["cloud"]["normals"].norm(dim=1), torch.ones(P, device=a.device))
    assert torch.allclose(after["cloud"]["normals"][P:].norm(dim=1), torch.ones(N - P, device=a.device), atol=1e-6)
    col = 3
    for g, (mb, ma) in enumerate(zip(before["moments"], after["moments"])):
        for k in MOMENTS:
            assert ma[k].shape == (N, 3), (g, k)
            assert torch.equal(ma[k][:P], mb[k]), (g, k)
            assert torch.equal(ma[k][P:], ref.features[P:, col:col + 3]), (g, k)
            col += 3
    assert col == ref.features.shape[1]
    # Adam's step counts, betas and (already decayed) learning rates, and the LR scheduler, go on
    assert [float(s) for s in after["steps"]] == [float(s) for s in before["steps"]] == [M] * len(before["steps"])
    assert after["groups"] == before["groups"]
    assert [g["lr"] for g in before["groups"]] == [LR * 0.5 ** 2] * 2     # two epochs past both LR milestones
    assert after["sched"] == before["sched"]
    # the new optimizer updates the new step's leaves, and the iteration at the milestone trained them
    opt, leaves = seen["opt"], seen["leaves"]
    params = [g["params"][0] for g in opt.param_groups]
    assert len(params) == 2 and params[0] is leaves[1] and params[1] is leaves[0]      # normals, points
    assert t.step.points is leaves[0] and not torch.equal(t.step.points.detach(), after["cloud"]["points"])
    assert all(float(opt.state[p]["step"]) == M + 1 for p in leaves[:2])
    with open(tmp_path / "out" / "torus" / "train.log") as f:
        log = f.read()
    assert "Grew the cloud at it=%d: 2000 -> %d points" % (M, N) in log


def test_loop_grows_and_trains(data_dir, tmp_path):  # noqa: F811
    from dss_b200.training.config import load_config
    from dss_b200.training.train import ground_truth_cloud, initial_cloud
    from dss_b200.utils.dataset import MVRData
    from dss_b200.utils.generate import generate, load_cloud
    # validated on the grown cloud alone, at 250 and 500: the chamfer distance of a freshly grown cloud is worse than
    # that of the cloud it grew from (the new points sit next to the sparsest points, often strays; DESIGN.md §3)
    cfg = write_config(tmp_path / "c.yml", data_dir, tmp_path / "out", grow_milestones=[100, 200],
                       grow_points=[4000, 8000], validate_every=250)
    code, log = run_cli(cfg, "--max-it", "501")
    assert code == 0, log
    assert "Grew the cloud at it=100: 2000 -> 4000 points" in log
    assert "Grew the cloud at it=200: 4000 -> 8000 points" in log
    print("\n".join(line for line in log.splitlines() if "Validation" in line or "Grew" in line))
    out = tmp_path / "out" / "torus"
    ck, best = _load(out / "model.pt"), _load(out / "model_best.pt")
    assert ck["it"] == 500 and ck["model"]["points"].shape == (1, 8000, 3)
    assert ck["model"]["points_activation"].shape == (1, 8000)
    ply = read_ply(str(out / "val" / "best.ply"))
    assert ply["points"].shape == (8000, 3) and ply["normals"].shape == (8000, 3)
    assert torch.equal(torch.from_numpy(ply["points"]), best["model"]["points"][0])
    d = torch.device("cuda:0")
    gt = ground_truth_cloud(MVRData(data_dir), data_dir, 8000, d)
    p0, n0, _ = initial_cloud(2000, 0, d)
    init = float(chamfer_distance(gt[0][None], p0[None], x_normals=gt[1][None], y_normals=n0[None])[0])
    print("chamfer_point: initial %.5f, best %.5f (%.3fx) at it %d" % (init, best["loss_val_best"],
                                                                       best["loss_val_best"] / init, best["it"]))
    assert best["loss_val_best"] <= 0.5 * init
    # the export reads the grown checkpoint
    points, normals, _ = load_cloud(str(out / "model_best.pt"), d)
    assert points.shape == (8000, 3)
    _, _, n, mesh = generate(load_config(cfg), depth=6)
    assert n == 8000 and mesh.faces.shape[0] > 0


def _same_checkpoints(ca, cb, it):
    """test_resume_is_exact's comparison: every field the same"""
    assert ca["it"] == cb["it"] == it and ca["epoch_it"] == cb["epoch_it"]
    for k in ("points", "normals", "colors", "points_activation"):
        assert torch.equal(ca["model"][k], cb["model"][k]), k
    sa, sb = ca["optimizer"]["state"], cb["optimizer"]["state"]
    assert sa.keys() == sb.keys()
    for i in sa:
        assert sa[i].keys() == sb[i].keys()
        for k in sa[i]:
            assert torch.equal(torch.as_tensor(sa[i][k]), torch.as_tensor(sb[i][k])), (i, k)
    assert ca["optimizer"]["param_groups"] == cb["optimizer"]["param_groups"]
    assert ca["lr_scheduler"] == cb["lr_scheduler"] and ca["schedule"] == cb["schedule"]
    assert ca["loss_val_best"] == cb["loss_val_best"]
    assert torch.equal(ca["sampler"], cb["sampler"]) and ca["epoch_order"] == cb["epoch_order"]
    assert ca["epoch_pos"] == cb["epoch_pos"]


def test_resume_across_a_milestone_is_exact(data_dir, tmp_path):  # noqa: F811
    grow = dict(grow_milestones=[150], grow_points=[4000])
    a = write_config(tmp_path / "a.yml", data_dir, tmp_path / "a", **grow)
    b = write_config(tmp_path / "b.yml", data_dir, tmp_path / "b", **grow)
    code, log = run_cli(a, "--max-it", "240")
    assert code == 0 and "Grew the cloud at it=150: 2000 -> 4000 points" in log, log
    code, log = run_cli(b, "--max-it", "130")
    assert code == 0 and "Grew" not in log, log
    mid = _load(tmp_path / "b" / "torus" / "model.pt")
    assert mid["it"] == 129 and mid["model"]["points"].shape == (1, 2000, 3)
    code, log = run_cli(b, "--max-it", "240")
    assert code == 0 and "resumed" in log and "Grew the cloud at it=150: 2000 -> 4000 points" in log, log
    ca, cb = _load(tmp_path / "a" / "torus" / "model.pt"), _load(tmp_path / "b" / "torus" / "model.pt")
    assert ca["model"]["points"].shape == (1, 4000, 3)
    _same_checkpoints(ca, cb, 239)
    # the records of the iterations after the milestone are the same bits too
    ra = {r["it"]: r for r in _records(tmp_path / "a" / "torus")}
    rb = {r["it"]: r for r in _records(tmp_path / "b" / "torus")}
    for it in range(150, 240, 10):
        assert {k: v for k, v in ra[it].items() if k != "time"} == {k: v for k, v in rb[it].items() if k != "time"}


def test_resume_with_another_schedule_is_refused(data_dir, tmp_path):  # noqa: F811
    a = write_config(tmp_path / "a.yml", data_dir, tmp_path / "a", grow_milestones=[20], grow_points=[3000])
    code, log = run_cli(a, "--max-it", "30")
    assert code == 0, log
    edited = write_config(tmp_path / "a.yml", data_dir, tmp_path / "a", grow_milestones=[40], grow_points=[3000])
    code, log = run_cli(edited, "--max-it", "50")
    assert code != 0
    assert "the checkpoint holds 3000 points after it=29, but" in log and "gives 2000 there" in log, log


def test_two_ranks_grow_as_one_gpu(data_dir, tmp_path):  # noqa: F811
    # both resume from one checkpoint written just before the milestone: the same cloud and Adam state grow alike
    import shutil
    M = 20
    grow = dict(grow_milestones=[M], grow_points=[4000], print_every=M)
    one = write_config(tmp_path / "one.yml", data_dir, tmp_path / "one", **grow)
    two = write_config(tmp_path / "two.yml", data_dir, tmp_path / "two", **grow)
    code, log = run_cli(one, "--max-it", str(M))
    assert code == 0, log
    (tmp_path / "two" / "torus").mkdir(parents=True)
    shutil.copy(tmp_path / "one" / "torus" / "model.pt", tmp_path / "two" / "torus" / "model.pt")
    code, log = run_cli(one, "--max-it", str(M + 1))
    assert code == 0 and "Grew the cloud at it=%d: 2000 -> 4000 points" % M in log, log
    codes, outs, _ = run_ranks(two, "--max-it", str(M + 1))
    assert codes == [0, 0], outs
    assert "Grew the cloud at it=%d: 2000 -> 4000 points" % M in outs[0], outs[0]
    assert "Replica check: the 2 ranks hold the same points, normals and colours and Adam moments" in outs[0], outs[0]
    r1 = {r["it"]: r for r in _records(tmp_path / "one" / "torus")}[M]
    r2 = {r["it"]: r for r in _records(tmp_path / "two" / "torus")}[M]
    for k in ("loss", "loss_dr_rgb", "loss_dr_silhouette", "loss_dr_proj", "loss_dr_repel"):
        ulps = abs(r2[k] - r1[k]) / (F32 * abs(r1[k])) if r1[k] else abs(r2[k])
        assert ulps <= (0 if k in ("loss_dr_proj", "loss_dr_repel") else LOSS_ULPS), (k, r1[k], r2[k])
    c1, c2 = _load(tmp_path / "one" / "torus" / "model.pt"), _load(tmp_path / "two" / "torus" / "model.pt")
    assert c1["it"] == c2["it"] == M and c1["model"]["points"].shape == c2["model"]["points"].shape == (1, 4000, 3)
    for k in ("points", "normals"):
        d = (c2["model"][k] - c1["model"][k]).abs()
        assert float(d.max()) <= 2 * LR, (k, float(d.max()))
        assert int((d > ROUNDING).sum()) <= d.numel() // 100, k
    assert torch.equal(c1["model"]["colors"], c2["model"]["colors"])


def test_resume_across_rank_counts_and_a_milestone(data_dir, tmp_path):  # noqa: F811
    grow = dict(grow_milestones=[60], grow_points=[4000])
    two_one = write_config(tmp_path / "a.yml", data_dir, tmp_path / "a", **grow)
    one_two = write_config(tmp_path / "b.yml", data_dir, tmp_path / "b", **grow)
    codes, outs, _ = run_ranks(two_one, "--max-it", "50")
    assert codes == [0, 0], outs
    code, log = run_cli(one_two, "--max-it", "50")
    assert code == 0, log
    code, log = run_cli(two_one, "--max-it", "80")
    assert code == 0 and "resumed" in log and "Grew the cloud at it=60" in log, log
    codes, outs, _ = run_ranks(one_two, "--max-it", "80")
    assert codes == [0, 0] and "resumed" in outs[0] and "Grew the cloud at it=60" in outs[0], outs
    ca, cb = _load(tmp_path / "a" / "torus" / "model.pt"), _load(tmp_path / "b" / "torus" / "model.pt")
    assert ca["it"] == cb["it"] == 79 and ca["epoch_it"] == cb["epoch_it"] == 79 // 4
    assert torch.equal(ca["sampler"], cb["sampler"]) and ca["epoch_order"] == cb["epoch_order"]
    assert ca["epoch_pos"] == cb["epoch_pos"] and ca["lr_scheduler"] == cb["lr_scheduler"]
    assert ca["schedule"] == cb["schedule"]
    for c in (ca, cb):
        for k in ("points", "normals", "colors"):
            assert c["model"][k].shape == (1, 4000, 3), k
        for s in c["optimizer"]["state"].values():
            assert s["step"] == 80
            for k in MOMENTS:
                assert s[k].shape == (4000, 3) and bool(torch.isfinite(s[k]).all())
    for run in ("a", "b"):
        assert [r["it"] for r in _records(tmp_path / run / "torus")] == list(range(0, 80, 10))


def test_resume_on_two_ranks_across_a_milestone_is_exact(data_dir, tmp_path):  # noqa: F811
    grow = dict(grow_milestones=[70], grow_points=[4000])
    a = write_config(tmp_path / "a.yml", data_dir, tmp_path / "a", **grow)
    b = write_config(tmp_path / "b.yml", data_dir, tmp_path / "b", **grow)
    codes, outs, _ = run_ranks(a, "--max-it", "100")
    assert codes == [0, 0], outs
    codes, outs, _ = run_ranks(b, "--max-it", "50")
    assert codes == [0, 0], outs
    codes, outs, _ = run_ranks(b, "--max-it", "100")
    assert codes == [0, 0] and "resumed" in outs[0] and "Grew the cloud at it=70: 2000 -> 4000" in outs[0], outs
    ca, cb = _load(tmp_path / "a" / "torus" / "model.pt"), _load(tmp_path / "b" / "torus" / "model.pt")
    assert ca["model"]["points"].shape == (1, 4000, 3)
    _same_checkpoints(ca, cb, 99)
