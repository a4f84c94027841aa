"""Score predicted point clouds against the ground truth: the reference's scripts/evaluatePointClouds.py.

    python -m dss_b200.utils.evaluate --gt GT --pred DIR [DIR ...] --name PATTERN [--mesh MESH]

Per prediction (the files matching ``DIR/**/PATTERN``, ``.ply`` or ``.xyz``) and its ground truth (``--gt`` a file:
that file for every prediction; a directory: the file with the prediction's basename):

- ``cd_forward`` / ``cd_backward``: the squared distance of every predicted point to its nearest ground-truth point,
  and of every ground-truth point to its nearest prediction (K = 1 of the device K-NN, raw coordinates);
  ``CD = mean(cd_forward) + mean(cd_backward)``, ``hausdorff = max(cd_forward) + max(cd_backward)`` -- the reference's
  definition: a sum of the two maxima of SQUARED distances, not the Hausdorff distance;
- ``p2f``: with ``--mesh``, the exact distance of every predicted point to the mesh (:func:`point_mesh_distance`),
  written to ``<pred>_point2mesh_distance.xyz`` as ``x y z d`` lines; without it, that file is read if it exists (the
  reference read the output of an external program from it).  ``p2f avg`` / ``p2f std`` are its NaN-ignoring mean and
  population standard deviation.
- ``<pred>_cdF.ply`` / ``<pred>_cdB.ply``: the predicted and the ground-truth points coloured by a jet ramp of
  ``cd_forward`` / ``cd_backward`` clipped at 0.003.

Every prediction directory gets an ``evaluation.csv`` (in the directory of its first prediction, as in the reference):
``name, CD, hausdorff, p2f avg, p2f std, nuc_0..nuc_6``, one row per pair and a final row with the mean ``CD`` and
``hausdorff`` over the pairs and ``p2f`` over all the pairs' distances together; missing values and the NUC columns
(not computed) are ``-``.  Unlike the reference, a pair whose p2f file is empty keeps its row and its place in the means,
and files this tool writes are never taken as predictions.
"""
import argparse
import csv
import glob
import os
import sys
from typing import NamedTuple, Optional

import numpy as np
import torch

from ..frnn_grid import knn_points_packed
from ..ops import point_mesh_distance
from .io import read_mesh, read_ply, save_ply

__all__ = ["CloudScores", "evaluate_cloud", "p2f_stats", "jet", "read_points", "read_xyz", "write_p2f_xyz", "pair_files",
           "evaluation_rows", "write_evaluation_csv", "summary_line", "main"]

FIELDS = ["name", "CD", "hausdorff", "p2f avg", "p2f std"] + ["nuc_%d" % d for d in range(7)]
CD_COLOUR_MAX = 0.003
OUTPUT_SUFFIXES = ("_cdF.ply", "_cdB.ply", "_point2mesh_distance.xyz")

# matplotlib's "jet" (its _jet_data): (position, value) knots of each channel, linear in between
_JET = (((0.0, 0.0), (0.35, 0.0), (0.66, 1.0), (0.89, 1.0), (1.0, 0.5)),
        ((0.0, 0.0), (0.125, 0.0), (0.375, 1.0), (0.64, 1.0), (0.91, 0.0), (1.0, 0.0)),
        ((0.0, 0.5), (0.11, 1.0), (0.34, 1.0), (0.65, 0.0), (1.0, 0.0)))


class CloudScores(NamedTuple):
    cd_forward: torch.Tensor          # (P,) float32 squared distance of each prediction to the ground truth, NaN: none
    cd_backward: torch.Tensor         # (G,) float32 the same from each ground-truth point to the predictions
    cd_forward_mean: float
    cd_backward_mean: float
    CD: float
    hausdorff: float
    p2f: Optional[torch.Tensor]       # (P,) float64 distance of each prediction to the mesh, or None without one
    p2f_avg: Optional[float]
    p2f_std: Optional[float]


def jet(values, vmax=CD_COLOUR_MAX):
    """(N,) values -> (N,3) float64 rgb in [0, 1]: the jet ramp of clip(values / vmax, 0, 1), linear between
    matplotlib's knots (matplotlib samples it at 256 levels).  Non-finite values take the colour of 0."""
    v = np.asarray(values, dtype=np.float64)
    t = np.clip(np.where(np.isfinite(v), v, 0.0) / vmax, 0.0, 1.0)
    return np.stack([np.interp(t, [k[0] for k in ch], [k[1] for k in ch]) for ch in _JET], -1)


def read_xyz(path):
    """whitespace-separated text, one point per line -> (N, columns) float64; (0, 4) for an empty file"""
    with open(path) as f:
        rows = [line.split() for line in f if line.strip()]
    if not rows:
        return np.zeros((0, 4))
    return np.asarray(rows, dtype=np.float64)


def read_points(path):
    """(N,3) float32 points of a ``.ply`` (its vertices) or ``.xyz`` file (the first three columns)"""
    if path.lower().endswith(".ply"):
        return read_ply(path)["points"]
    a = read_xyz(path)
    return np.ascontiguousarray(a[:, :3], dtype=np.float32)


def write_p2f_xyz(path, points, dists):
    """``x y z d`` lines: points (N,3) float32 (9 significant digits, exact), dists (N,) float64 (17, exact)"""
    points, dists = np.asarray(points, dtype=np.float32), np.asarray(dists, dtype=np.float64)
    with open(path, "w") as f:
        for p, d in zip(points, dists):
            f.write("%.9g %.9g %.9g %.17g\n" % (p[0], p[1], p[2], d))


def _strip_ext(path):
    return os.path.splitext(os.path.basename(path))[0]


def pair_files(gt, pred_dir, pattern):
    """[(gt path, prediction path)] of one prediction directory: the predictions are the files matching
    ``pred_dir/**/pattern`` (sorted; this tool's own outputs excluded); a ``gt`` file goes with each of them, a ``gt``
    directory gives each prediction the ground truth of the same basename (``.ply`` or ``.xyz``; a prediction without
    one is left out)."""
    preds = sorted(p for p in glob.glob(os.path.join(pred_dir, "**", pattern), recursive=True)
                   if os.path.isfile(p) and not p.endswith(OUTPUT_SUFFIXES))
    if os.path.isfile(gt):
        return [(gt, p) for p in preds]
    if not os.path.isdir(gt):
        raise FileNotFoundError("--gt %s is neither a file nor a directory" % gt)
    by_name = {}
    for ext in ("ply", "xyz"):
        for g in sorted(glob.glob(os.path.join(gt, "**", "*." + ext), recursive=True)):
            by_name.setdefault(_strip_ext(g), g)
    return [(by_name[_strip_ext(p)], p) for p in preds if _strip_ext(p) in by_name]


def _fmt(x):
    return "-" if x is None else repr(float(x))


def evaluation_rows(pairs):
    """The CSV rows of one prediction directory.  ``pairs``: one dict per pair {name, cd_forward_mean,
    cd_backward_mean, hausdorff, p2f (1-D distances, possibly empty) or None}.  Returns (rows, final) as dicts over
    :data:`FIELDS` with string values; ``final`` holds the mean CD and hausdorff over the pairs and p2f over all the
    distances together (the reference's final row)."""
    rows, all_p2f = [], []
    n = len(pairs)
    sum_f = sum_b = sum_h = 0.0
    for pr in pairs:
        row = dict.fromkeys(FIELDS, "-")
        row["name"] = pr["name"]
        row["CD"] = _fmt(pr["cd_forward_mean"] + pr["cd_backward_mean"])
        row["hausdorff"] = _fmt(pr["hausdorff"])
        sum_f, sum_b, sum_h = sum_f + pr["cd_forward_mean"], sum_b + pr["cd_backward_mean"], sum_h + pr["hausdorff"]
        d = pr.get("p2f")
        if d is not None and len(d):
            d = np.asarray(d, dtype=np.float64)
            row["p2f avg"], row["p2f std"] = _fmt(np.nanmean(d)), _fmt(np.nanstd(d))
            all_p2f.append(d)
        rows.append(row)
    final = dict.fromkeys(FIELDS, "-")
    if n:
        final["CD"] = _fmt(sum_f / n + sum_b / n)
        final["hausdorff"] = _fmt(sum_h / n)
    if all_p2f:
        d = np.concatenate(all_p2f)
        final["p2f avg"], final["p2f std"] = _fmt(np.nanmean(d)), _fmt(np.nanstd(d))
    return rows, final


def write_evaluation_csv(path, rows, final):
    with open(path, "w", newline="") as f:
        w = csv.DictWriter(f, fieldnames=FIELDS)
        w.writeheader()
        for r in rows + [final]:
            w.writerow(r)


def summary_header():
    return "{:60s} ".format("name") + "|".join("{:>15s}".format(d) for d in FIELDS[1:])


def summary_line(tag, final):
    """the reference's one line per directory: the tag, then the final row's values that are present"""
    vals = [float(final[k]) for k in ("CD", "hausdorff", "p2f avg", "p2f std") if final[k] != "-"]
    return "{:60s} ".format(tag) + "|".join("{:>15.8f}".format(v) for v in vals)


def _nn_sq(queries, points):
    """squared distance of every query row to its nearest point (K = 1), NaN where there is none"""
    dev = queries.device
    one = torch.zeros(1, dtype=torch.int64, device=dev)
    d, _ = knn_points_packed(points, one, torch.tensor([points.shape[0]], device=dev), 1, queries=queries,
                             query_first_idx=one, query_num=torch.tensor([queries.shape[0]], device=dev),
                             return_idx=False)
    d = d[:, 0]
    return torch.where(d < 0, torch.full_like(d, float("nan")), d)


def evaluate_cloud(pred, gt_points, mesh=None):
    """The reference's scores of one predicted cloud (see the module docstring) -> :class:`CloudScores`.  ``pred``
    (P,3) and ``gt_points`` (G,3) float32 CUDA tensors; ``mesh``: (verts (V,3), faces (F,3)) on the same device, or
    None.  Means, maxima and the p2f statistics are reduced on the device in float64 (NaN rows propagate into CD and
    hausdorff, as numpy's mean and max do; the p2f statistics ignore them)."""
    pred, gt_points = pred.detach().float().contiguous(), gt_points.detach().float().contiguous()
    fwd, bwd = _nn_sq(pred, gt_points), _nn_sq(gt_points, pred)
    f64, b64 = fwd.double(), bwd.double()
    mf, mb = f64.mean(), b64.mean()
    stats = torch.stack([mf, mb, mf + mb, f64.max() + b64.max()]).tolist()
    p2f, avg, std = p2f_stats(pred, mesh) if mesh is not None else (None, None, None)
    return CloudScores(fwd, bwd, stats[0], stats[1], stats[2], stats[3], p2f, avg, std)


def p2f_stats(points, mesh):
    """(p2f (P,) float64 device tensor, nanmean, population nanstd) of the distances of ``points`` (P,3) to ``mesh``
    (verts (V,3), faces (F,3)), reduced on the device in float64"""
    p2f = point_mesh_distance(points.detach().float(), mesh[0].detach().float(), mesh[1]).sq_dists.double().sqrt()
    v = p2f[~torch.isnan(p2f)]
    m = v.mean()
    avg, std = torch.stack([m, ((v - m) ** 2).mean().sqrt()]).tolist()
    return p2f, avg, std


def _evaluate_dir(gt, pred_dir, pattern, mesh, device):
    pairs = pair_files(gt, pred_dir, pattern)
    if not pairs:
        print("{:60s} no predictions matching {} (with a ground truth)".format(os.path.basename(pred_dir), pattern))
        return None
    results = []
    for gt_path, pred_path in pairs:
        gt_pts = torch.from_numpy(read_points(gt_path)).to(device)
        pred_pts = torch.from_numpy(read_points(pred_path)).to(device)
        s = evaluate_cloud(pred_pts, gt_pts, mesh)
        stem = pred_path[:-4]
        for pts, d, suffix in ((pred_pts, s.cd_forward, "_cdF.ply"), (gt_pts, s.cd_backward, "_cdB.ply")):
            save_ply(stem + suffix, pts.cpu().numpy(), colors=jet(d.cpu().numpy()))
        p2f_path = stem + "_point2mesh_distance.xyz"
        if s.p2f is not None:
            write_p2f_xyz(p2f_path, pred_pts.cpu().numpy(), s.p2f.cpu().numpy())
            p2f = s.p2f.cpu().numpy()
        elif os.path.isfile(p2f_path):
            p2f = read_xyz(p2f_path)[:, 3]
        else:
            p2f = None
        results.append({"name": os.path.basename(pred_path), "cd_forward_mean": s.cd_forward_mean,
                        "cd_backward_mean": s.cd_backward_mean, "hausdorff": s.hausdorff, "p2f": p2f})
    rows, final = evaluation_rows(results)
    out_dir = os.path.dirname(pairs[0][1])
    write_evaluation_csv(os.path.join(out_dir, "evaluation.csv"), rows, final)
    print(summary_line(os.path.basename(out_dir), final))
    return rows, final


def main(argv=None):
    ap = argparse.ArgumentParser(description="Score point clouds against a ground truth (evaluatePointClouds.py).")
    ap.add_argument("--gt", required=True, help="ground-truth file, or a directory of them (paired by basename)")
    ap.add_argument("--pred", nargs="+", required=True, help="directories of predictions")
    ap.add_argument("--name", required=True, help="file name pattern of the predictions, e.g. '*.ply'")
    ap.add_argument("--mesh", default=None, help="ground-truth mesh: compute the point-to-surface distances")
    opt = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise RuntimeError("the evaluation needs a CUDA device (sm_90a)")
    device = torch.device("cuda", torch.cuda.current_device())
    mesh = None
    if opt.mesh:
        v, f = read_mesh(opt.mesh)
        mesh = (torch.from_numpy(np.ascontiguousarray(v, dtype=np.float32)).to(device),
                torch.from_numpy(np.ascontiguousarray(f)).to(device))
    print(summary_header())
    for d in opt.pred:
        _evaluate_dir(opt.gt, d, opt.name, mesh, device)
    return 0


if __name__ == "__main__":
    sys.exit(main())
