"""Estimate and orient the normals of a point cloud: meshlab's "Compute normals for point sets" (K neighbours, no
smoothing, no viewpoint), the step of the reference's scripts/poisson_sampling_pca.mlx that gives its evaluation clouds
their normals.

    python -m dss_b200.utils.normals IN OUT [--k 20] [--no-orient] [--mesh MESH] [--depth 8]

Reads the points of IN (``.ply`` vertices or ``.xyz``, the first three columns; any normals IN carries are ignored),
computes :func:`dss_b200.ops.estimate_normals` on the device and writes OUT, a binary PLY of the points and their
normals.  With ``--mesh`` it also writes the screened Poisson surface of the result at ``--depth`` (``.obj`` or
``.ply`` by MESH's extension).  Orientation is consistent within a connected component of the k-NN graph only, so the
number of components is printed when there is more than one."""
import argparse
import sys

import torch

__all__ = ["estimate_file", "main"]


def estimate_file(src, dst, k=20, orient=True, mesh=None, depth=8):
    """``src`` -> ``dst`` as the command line does it; returns (the PointNormals on the device, the number of
    components (0 without ``orient``), the PoissonMesh or None)"""
    from ..ops import estimate_normals, poisson_reconstruction
    from .evaluate import read_points
    from .io import save_obj, save_ply
    pts = torch.from_numpy(read_points(src)).cuda()
    est = estimate_normals(pts, k=k, orient=orient)
    save_ply(dst, pts.cpu().numpy(), normals=est.normals.cpu().numpy())
    roots = est.root[est.root >= 0]
    components = int(torch.unique(roots).numel()) if orient else 0
    rec = None
    if mesh is not None:
        rec = poisson_reconstruction(pts, est.normals, depth=depth)
        v, f = rec.verts.cpu().numpy(), rec.faces.cpu().numpy()
        if mesh.lower().endswith(".obj"):
            save_obj(mesh, v, f)
        else:
            save_ply(mesh, v, faces=f)
    return est, components, rec


def main(argv=None):
    p = argparse.ArgumentParser(description="Estimate and orient point normals (meshlab's Compute normals for point "
                                            "sets) and optionally mesh the result.")
    p.add_argument("input", help="point cloud: .ply (vertices) or .xyz (x y z per line); its normals are ignored")
    p.add_argument("output", help="PLY file of the points and their estimated normals")
    p.add_argument("--k", type=int, default=20, help="neighbourhood size, 3 .. 32 (meshlab's K)")
    p.add_argument("--no-orient", action="store_true",
                   help="skip the spanning-tree orientation: each normal's largest component is positive")
    p.add_argument("--mesh", default=None, help="also write the screened Poisson surface of the result here")
    p.add_argument("--depth", type=int, default=8, help="octree depth of the reconstruction: a 2^depth grid (2 .. 9)")
    args = p.parse_args(argv)
    if not torch.cuda.is_available():
        raise RuntimeError("normal estimation needs a CUDA device (sm_90a)")
    est, components, rec = estimate_file(args.input, args.output, args.k, not args.no_orient, args.mesh, args.depth)
    invalid = int((~torch.isfinite(est.normals).all(1)).sum())
    print("%s: %d points%s" % (args.output, est.normals.shape[0],
                                ", %d without a normal (non-finite or too few neighbours)" % invalid if invalid else ""))
    if components > 1:
        print("%d connected components: the orientation is consistent within each one only" % components)
    if rec is not None:
        print("%s: %d vertices, %d faces" % (args.mesh, rec.verts.shape[0], rec.faces.shape[0]))
    return 0


if __name__ == "__main__":
    sys.exit(main())
