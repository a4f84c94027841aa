"""Remove outliers from a point cloud, upsample it and project it onto its surface: the reference's
``remove_outliers``, ``upsample``, ``denoise_normals`` and ``project_to_latent_surface`` (DSS/core/cloud.py:363-378,
555-632, 515-553, 442-513) on a file.

    python -m dss_b200.utils.resample IN OUT [--remove-outliers [--tolerance 0.05] [--outlier-k 16]]
                                             [--upsample N [--k 16]]
                                             [--denoise-normals] [--project [--project-k 31]]

Reads IN (``.ply`` vertices, with their normals and colours when present, or ``.xyz``, the first three columns), drops
with ``--remove-outliers`` the points whose ``--outlier-k`` neighbourhood is not planar
(:func:`dss_b200.ops.outlier_ratio`), then with ``--upsample`` grows the cloud to N points
(:func:`dss_b200.ops.upsample_points`), carrying normals and colours to the new points, then with
``--denoise-normals`` smooths the normals (:func:`dss_b200.ops.denoise_normals`; the smoothed ones are written), then
with ``--project`` moves every point onto the RIMLS surface of the cloud (:func:`dss_b200.ops.project_to_surface`), and
writes OUT, a binary PLY.  The input points come first in OUT, in their order (less the removed ones).  Both last
steps need normals: for a cloud without them, ``python -m dss_b200.utils.normals`` estimates them first."""
import argparse
import sys

import numpy as np
import torch

__all__ = ["resample_file", "main"]


def resample_file(src, dst, remove_outliers=False, tolerance=0.05, outlier_k=16, upsample=None, k=16, project=False,
                  project_k=31, denoise=False):
    """``src`` -> ``dst`` as the command line does it; returns (input points, points after outlier removal, points
    written)"""
    from ..ops import denoise_normals, outlier_ratio, project_to_surface, upsample_points
    from .evaluate import read_xyz
    from .io import read_ply, save_ply
    if src.lower().endswith(".ply"):
        d = read_ply(src)
        pts, nrm, col = d["points"], d["normals"], d["colors"]
    else:
        pts, nrm, col = np.ascontiguousarray(read_xyz(src)[:, :3], dtype=np.float32), None, None
    if (project or denoise) and nrm is None:
        raise ValueError("%s has no normals, which --project and --denoise-normals need: estimate them first with "
                         "python -m dss_b200.utils.normals" % src)
    dev = torch.device("cuda")
    to = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(dev)
    p, n, c = to(pts), to(nrm), to(col)
    n_in = p.shape[0]
    if remove_outliers:
        keep = outlier_ratio(p, outlier_k, tolerance).keep
        p, n, c = p[keep], None if n is None else n[keep], None if c is None else c[keep]
    n_kept = p.shape[0]
    if upsample is not None:
        up = upsample_points(p, upsample, k, n, c)
        p, n, c = up.points, up.normals, up.features
    if denoise:
        n = denoise_normals(p, n)
    if project:
        p = project_to_surface(p, n, project_k).points
    arr = lambda t: None if t is None else t.cpu().numpy()
    save_ply(dst, arr(p), colors=arr(c), normals=arr(n))
    return n_in, n_kept, p.shape[0]


def main(argv=None):
    p = argparse.ArgumentParser(description="Remove outliers from a point cloud, upsample it, denoise its normals and/or "
                                            "project it onto its surface (the reference's remove_outliers, upsample, "
                                            "denoise_normals and project_to_latent_surface).")
    p.add_argument("input", help="point cloud: .ply (vertices, normals and colours carried) or .xyz (x y z per line)")
    p.add_argument("output", help="PLY file of the result")
    p.add_argument("--remove-outliers", action="store_true",
                   help="drop the points whose neighbourhood is not planar (applied before upsampling)")
    p.add_argument("--tolerance", type=float, default=0.05,
                   help="keep a point when l0 / (l0 + l1 + l2) of its neighbourhood is below this")
    p.add_argument("--outlier-k", type=int, default=16, help="neighbourhood of the outlier test, 3 .. 32")
    p.add_argument("--upsample", type=int, default=None, metavar="N", help="grow the cloud to N points")
    p.add_argument("--k", type=int, default=16, help="neighbourhood of the upsampling, 3 .. 31")
    p.add_argument("--project", action="store_true",
                   help="move every point onto the RIMLS surface of the cloud (last); needs normals")
    p.add_argument("--project-k", type=int, default=31, help="neighbourhood of the projection, 3 .. 31")
    p.add_argument("--denoise-normals", action="store_true",
                   help="smooth the normals (after upsampling, before projecting) and write the smoothed ones")
    args = p.parse_args(argv)
    if not torch.cuda.is_available():
        raise RuntimeError("resampling needs a CUDA device (sm_90a)")
    n_in, n_kept, n_out = resample_file(args.input, args.output, args.remove_outliers, args.tolerance, args.outlier_k,
                                        args.upsample, args.k, args.project, args.project_k, args.denoise_normals)
    msg = "%s: %d points in" % (args.output, n_in)
    if args.remove_outliers:
        msg += ", %d outliers removed" % (n_in - n_kept)
    if args.upsample is not None:
        msg += ", %d added" % (n_out - n_kept)
    if args.denoise_normals:
        msg += ", normals denoised"
    if args.project:
        msg += ", projected"
    print(msg + ", %d written" % n_out)
    return 0


if __name__ == "__main__":
    sys.exit(main())
