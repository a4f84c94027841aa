"""CPU: the host side of dss_b200.utils.evaluate -- the jet ramp, the .xyz files, pairing predictions with their ground
truth, evaluation.csv -- and the training loop's model-selection metrics."""
import csv
import os

import numpy as np
import pytest

from dss_b200.utils.evaluate import (FIELDS, evaluation_rows, jet, pair_files, read_points, read_xyz, summary_line,
                                     write_evaluation_csv, write_p2f_xyz)


def test_jet_knots_and_clip():
    vmax = 0.003
    # matplotlib's jet knots (position, value) per channel; linear halfway between two knots
    knots = [[(0.0, 0.0), (0.35, 0.0), (0.66, 1.0), (0.89, 1.0), (1.0, 0.5)],
             [(0.0, 0.0), (0.125, 0.0), (0.375, 1.0), (0.64, 1.0), (0.91, 0.0), (1.0, 0.0)],
             [(0.0, 0.5), (0.11, 1.0), (0.34, 1.0), (0.65, 0.0), (1.0, 0.0)]]
    for ch, ks in enumerate(knots):
        for (p0, v0), (p1, v1) in zip(ks, ks[1:]):
            assert jet([p0 * vmax])[0, ch] == pytest.approx(v0, abs=1e-12), (ch, p0)
            assert jet([(p0 + p1) / 2 * vmax])[0, ch] == pytest.approx((v0 + v1) / 2, abs=1e-12), (ch, p0, p1)
    assert np.allclose(jet([0.5 * vmax])[0], [(0.5 - 0.35) / 0.31, 1.0, (0.65 - 0.5) / 0.31], atol=1e-12)
    # clipped at vmax and at 0, non-finite values as 0
    assert np.array_equal(jet([vmax, 1.0, 1e30]), np.tile([[0.5, 0, 0]], (3, 1)))
    assert np.array_equal(jet([-1.0, np.nan, np.inf]), np.tile([[0, 0, 0.5]], (3, 1)))


def test_xyz_round_trip(tmp_path):
    g = np.random.default_rng(0)
    pts = g.standard_normal((50, 3)).astype(np.float32) * np.float32(1e3)
    d = g.random(50) ** 3
    d[3] = np.nan
    write_p2f_xyz(str(tmp_path / "a.xyz"), pts, d)
    a = read_xyz(str(tmp_path / "a.xyz"))
    assert a.shape == (50, 4)
    assert np.array_equal(a[:, :3].astype(np.float32), pts)
    assert np.array_equal(a[:, 3], d, equal_nan=True)
    assert np.array_equal(read_points(str(tmp_path / "a.xyz")), pts)
    (tmp_path / "empty.xyz").write_text("")
    assert read_xyz(str(tmp_path / "empty.xyz")).shape == (0, 4)


def touch(path):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    open(path, "w").close()
    return str(path)


def test_pairing(tmp_path):
    pred = tmp_path / "pred"
    a, b = touch(pred / "a.ply"), touch(pred / "sub" / "b.ply")
    touch(pred / "a_cdF.ply")            # outputs of an earlier run are not predictions
    touch(pred / "a_cdB.ply")
    touch(pred / "c.xyz")
    gt_file = touch(tmp_path / "gt.ply")
    assert pair_files(gt_file, str(pred), "*.ply") == [(gt_file, a), (gt_file, b)]
    gt_a, gt_b = touch(tmp_path / "gts" / "a.ply"), touch(tmp_path / "gts" / "deep" / "b.xyz")
    touch(tmp_path / "gts" / "z.ply")
    assert pair_files(str(tmp_path / "gts"), str(pred), "*.ply") == [(gt_a, a), (gt_b, b)]
    assert pair_files(str(tmp_path / "gts"), str(pred), "*.xyz") == []     # c has no ground truth
    with pytest.raises(FileNotFoundError):
        pair_files(str(tmp_path / "missing"), str(pred), "*.ply")


def test_evaluation_csv(tmp_path):
    pairs = [{"name": "a.ply", "cd_forward_mean": 0.5, "cd_backward_mean": 0.25, "hausdorff": 2.0,
              "p2f": np.array([1.0, 3.0, np.nan])},
             {"name": "b.ply", "cd_forward_mean": 0.125, "cd_backward_mean": 1.0, "hausdorff": 4.0,
              "p2f": np.zeros(0)},        # an empty p2f file keeps its row
             {"name": "c.ply", "cd_forward_mean": 1.0, "cd_backward_mean": 2.0, "hausdorff": 6.0, "p2f": None},
             {"name": "d.ply", "cd_forward_mean": 0.0, "cd_backward_mean": 0.0, "hausdorff": 0.0,
              "p2f": np.array([5.0])}]
    rows, final = evaluation_rows(pairs)
    assert [r["name"] for r in rows] == ["a.ply", "b.ply", "c.ply", "d.ply"]
    assert float(rows[0]["CD"]) == 0.75 and float(rows[0]["hausdorff"]) == 2.0
    assert float(rows[0]["p2f avg"]) == 2.0 and float(rows[0]["p2f std"]) == 1.0
    assert rows[1]["p2f avg"] == rows[1]["p2f std"] == "-" and rows[2]["p2f avg"] == "-"
    assert float(rows[3]["p2f avg"]) == 5.0 and float(rows[3]["p2f std"]) == 0.0
    assert all(r["nuc_%d" % k] == "-" for r in rows + [final] for k in range(7))
    assert final["name"] == "-"
    assert float(final["CD"]) == (0.5 + 0.125 + 1.0) / 4 + (0.25 + 1.0 + 2.0) / 4
    assert float(final["hausdorff"]) == 3.0
    allp = np.array([1.0, 3.0, 5.0])          # every pair's distances together, NaN ignored
    assert float(final["p2f avg"]) == 3.0 and float(final["p2f std"]) == pytest.approx(np.std(allp), rel=1e-15)
    write_evaluation_csv(str(tmp_path / "evaluation.csv"), rows, final)
    with open(tmp_path / "evaluation.csv") as f:
        back = list(csv.DictReader(f))
    assert list(back[0].keys()) == FIELDS and len(back) == 5
    assert back == rows + [final]
    line = summary_line("pred", final)
    assert line.startswith("pred ") and len(line.split("|")) == 4
    assert summary_line("x", evaluation_rows(pairs[2:3])[1]).count("|") == 1     # no p2f: CD and hausdorff only


def test_selection_metrics():
    from dss_b200.training.config import DEFAULTS, selection_metric
    import copy
    cfg = copy.deepcopy(DEFAULTS)
    for m in ("chamfer_point", "chamfer_normal", "p2f_avg"):
        cfg["training"]["model_selection_metric"] = m
        assert selection_metric(cfg) == m
    for m in ("p2f_std", "CD", "loss"):
        cfg["training"]["model_selection_metric"] = m
        with pytest.raises(NotImplementedError):
            selection_metric(cfg)
