"""Time ops.poisson_reconstruction (csrc/poisson.cu) at depth 8 and 9 from 100k and 1M samples of a torus.

    python scripts/poisson_time.py [--warmup 1] [--iters 3]

Per case: the whole call (median of CUDA-event times after warm-up), then from one more call the per-level device times
dss_poisson_solve reports (set-up: occupied cells, splat, right-hand side, diagonal, start residual; CG) and CG
iterations, the extraction (dss_marching_tetrahedra, both of its calls) and the mesh size.  Prints one JSON line per
case, the card name and its power limit first."""
import argparse
import ctypes as C
import json

import torch

from timing import card, median_ms
from meshes import torus
from dss_b200 import _lib
from dss_b200.ops import marching_tetrahedra, poisson_reconstruction
from dss_b200.utils.create_mvr_data import sample_points_from_mesh


def levels(p, n, depth):
    """per-level {setup_ms, cg_ms, iterations} of one dss_poisson_solve call, and the grid it wrote"""
    R = 1 << depth
    chi = torch.empty((R + 1,) * 3, dtype=torch.float32, device=p.device)
    c, L, its, res = (C.c_float * 3)(), C.c_float(), C.c_int(), C.c_double()
    li, ms = (C.c_int * (depth + 1))(), (C.c_float * (2 * (depth + 1)))()
    _lib.check(_lib.load().dss_poisson_solve(_lib.ctx(p.device), _lib.ptr(p), _lib.ptr(n), p.shape[0], depth,
                                             _lib.ptr(chi), c, C.byref(L), C.byref(its), C.byref(res), li, ms,
                                             _lib.stream_ptr(p.device)), "dss_poisson_solve")
    out = {l: {"setup_ms": round(ms[2 * l], 3), "cg_ms": round(ms[2 * l + 1], 3), "iterations": li[l]}
           for l in range(depth + 1) if li[l] or ms[2 * l + 1]}
    return out, chi, torch.tensor(list(c)), L.value, res.value


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--iters", type=int, default=3)
    opt = ap.parse_args()
    dev = torch.device("cuda:0")
    gpu = card()
    print(json.dumps({"card": gpu["name"], "power_limit": gpu["power_limit"]}), flush=True)
    v, f = torus()
    v, f = v.to(dev), f[:, [0, 2, 1]].to(dev)     # outward winding
    g = torch.Generator(device=dev).manual_seed(0)
    pts, nrm = sample_points_from_mesh(v, f, 1_000_000, generator=g)
    for P in (100_000, 1_000_000):
        p, n = pts[:P].contiguous(), nrm[:P].contiguous()
        for depth in (8, 9):
            res = {"P": P, "depth": depth}
            res["total_ms"] = median_ms(lambda: poisson_reconstruction(p, n, depth=depth), opt.warmup, opt.iters)
            lv, chi, c, L, residual = levels(p, n, depth)
            res["levels"] = lv
            res["residual"] = residual
            res["extract_ms"] = median_ms(lambda: marching_tetrahedra(chi, c, L), 1, opt.iters)
            verts, faces = marching_tetrahedra(chi, c, L)
            res["verts"], res["faces"] = int(verts.shape[0]), int(faces.shape[0])
            res["scratch_gb"] = round(_lib.scratch_bytes(dev) / 1e9, 2)
            print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
