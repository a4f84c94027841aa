"""Mint K-NN golden vectors from the REFERENCE's own ground truth, FRNNBruteForceCPU (external/FRNN/frnn/csrc/
bruteforce/bruteforce_cpu.cpp), compiled into oracle/_ref/dss_ref_frnn_cpu.  Run in the build container:

    python -m tests.golden.make_golden_knn

Inputs: the reference's example clouds (normalised like create_mvr_data_from_mesh.py:122-126) and seeded random
clouds, with the query the splat-size rule makes (K = 7, r = 0.2: DSS/core/rasterizer.py:313-326) and a radius small
enough to leave some neighbour lists short."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import build_ref                                   # noqa: E402
from tests.golden.make_golden import read_ply_xyz_normals     # noqa: E402


def main():
    ref = build_ref.ref_frnn_cpu()
    assert ref is not None, "needs /root/reference (or a prebuilt oracle/_ref/dss_ref_frnn_cpu)"
    clouds = {}
    for name, limit in (("teapot_normal_dense", 2500), ("bunny-8000", 2500), ("sphere_2k", 2000)):
        path = "/root/reference/example_data/pointclouds/%s.ply" % name
        if os.path.exists(path):
            clouds[name.replace("-", "_")] = read_ply_xyz_normals(path, limit)[0]
    rng = np.random.default_rng(7)
    clouds["random_cube"] = rng.uniform(-0.5, 0.5, (1500, 3)).astype(np.float32)
    dup = rng.uniform(-0.5, 0.5, (600, 3)).astype(np.float32)
    clouds["random_with_duplicates"] = np.concatenate([dup, dup[:200], dup[:50]]).astype(np.float32)   # exact ties
    out = {}
    for name, xyz in clouds.items():
        p = torch.from_numpy(xyz)[None]
        n = torch.tensor([xyz.shape[0]], dtype=torch.int64)
        for tag, K, r in (("k7_r0.2", 7, 0.2), ("k12_r0.05", 12, 0.05)):
            idxs, dists = ref.frnn_bf_cpu(p, p, n, n, K, r)
            out["%s__%s__dists" % (name, tag)] = dists[0].numpy()
            out["%s__%s__idxs" % (name, tag)] = idxs[0].numpy().astype(np.int32)
        out["%s__points" % name] = xyz
    # the edge families of tests/test_gpu_knn_edges.py, small, as padded batches: "edge_<family>__{points (N,P,3),
    # lengths (N,), K, r, dists (N,P,K), idxs (N,P,K)}"
    for name, (pts, lens, K, r) in edge_families().items():
        idxs, dists = ref.frnn_bf_cpu(torch.from_numpy(pts), torch.from_numpy(pts), torch.from_numpy(lens),
                                      torch.from_numpy(lens), K, r)
        key = "edge_" + name
        out[key + "__points"], out[key + "__lengths"] = pts, lens
        out[key + "__K"], out[key + "__r"] = np.int64(K), np.float32(r)
        out[key + "__dists"], out[key + "__idxs"] = dists.numpy(), idxs.numpy().astype(np.int32)
    np.savez_compressed(os.path.join(HERE, "knn_frnn_bruteforce.npz"), **out)
    print("wrote knn_frnn_bruteforce.npz:", sorted(clouds), sorted(edge_families()))


def edge_families():
    """name -> (points (N,P,3) f32 padded, lengths (N,) i64, K, r > 0): seeded small instances of the GPU edge
    families -- duplicates beyond K, pairs exactly at r (dyadic) and one ulp inside, a shuffled integer lattice whose
    equal distances straddle the K-th slot, NaN / inf rows, the long line of the ring bound, a ragged batch"""
    from tests.util import knn_long_line
    f32 = np.float32
    rng = np.random.default_rng(17)
    fam = {}

    def one(p, K, r):
        p = np.ascontiguousarray(p, f32)
        return p[None], np.array([len(p)], np.int64), K, r

    base = rng.uniform(-0.5, 0.5, (40, 3)).astype(f32)
    dup = np.concatenate([base, np.repeat(base[:3], 12, axis=0)])
    fam["duplicates"] = one(dup[rng.permutation(len(dup))], 8, 0.5)
    c = rng.permutation(np.stack(np.meshgrid(*[np.arange(-2, 3)] * 3, indexing="ij"), -1).reshape(-1, 3))[:20]
    c = c.astype(f32)
    offs = np.array([[3, 4, 0], [4, 0, 3], [0, 3, 4], [5, 0, 0]], f32) / f32(16)
    o = offs[rng.integers(0, 4, len(c))]
    on = (c + o).astype(f32)
    c2 = (c + f32(10)).astype(f32)                                # a second copy, moved one ulp inside
    inside = (c2 + o).astype(f32)
    inside[:, 0] = np.where(o[:, 0] != 0, np.nextafter(inside[:, 0], c2[:, 0]), inside[:, 0])
    inside[:, 1] = np.where(o[:, 0] == 0, np.nextafter(inside[:, 1], c2[:, 1]), inside[:, 1])
    fam["r2_boundary"] = one(np.concatenate([c, on, c2, inside]), 4, 0.3125)
    g = np.stack(np.meshgrid(*[np.arange(6)] * 3, indexing="ij"), -1).reshape(-1, 3).astype(f32)
    fam["lattice_ties"] = one(g[rng.permutation(len(g))], 5, 1.5)
    nf = rng.uniform(-0.5, 0.5, (60, 3)).astype(f32)
    for k, v in enumerate((np.nan, np.inf, -np.inf, np.nan, np.inf, -np.inf)):
        nf[7 * k + 3, k % 3] = v
    fam["nonfinite"] = one(nf, 6, 0.4)
    line = knn_long_line(n_pairs=24, seed=1)[0]
    fam["long_line"] = one(line, 2, 0.2)
    lens = np.array([50, 0, 7], np.int64)
    rag = np.zeros((3, 50, 3), f32)
    for n, L in enumerate(lens):
        rag[n, :L] = rng.uniform(-0.3, 0.3, (L, 3))
    fam["ragged"] = (rag, lens, 7, 0.3)
    return fam


if __name__ == "__main__":
    main()
