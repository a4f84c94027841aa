"""CPU oracle for the DSS splatting hot path -- TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
import this package.  dss_b200/ never does: the product path fails loudly without its CUDA
library instead of falling back to anything here.

Thin numpy/ctypes front for oracle/dss_oracle.c (each C function cites the reference file:line it
restates).  Parity status: pinned against the reference's own CPU code compiled from
/root/reference (oracle/_ref, oracle/build_ref.py) and the fixtures under tests/golden/.
"""
import ctypes as C
import os

import numpy as np

from .build import build_oracle, LIB

_lib = None


def lib():
    global _lib
    if _lib is None:
        build_oracle()
        _lib = C.CDLL(LIB)
        _lib.oracle_rasterize_coarse.restype = C.c_long
        _lib.oracle_num_threads.restype = C.c_int
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _i64(a):
    return np.ascontiguousarray(a, dtype=np.int64)


def _i32(a):
    return np.ascontiguousarray(a, dtype=np.int32)


def num_threads():
    return int(lib().oracle_num_threads())


def set_num_threads(n):
    lib().oracle_set_num_threads(C.c_int(int(n)))


def splat_points_naive(points, ellipse, cutoff, radii, first_idx, num_pts, depth_merge, S, K,
                       fma_mode=0, bbox_and=False):
    """-> idx (N,S,S,K) i32, zbuf, qvalue f32, occ (N,S,S) f32.  rasterize_points.cu:131-212."""
    points, ellipse, cutoff, radii = _f32(points), _f32(ellipse), _f32(cutoff), _f32(radii)
    first_idx, num_pts = _i64(first_idx), _i64(num_pts)
    N = len(num_pts)
    idx = np.empty((N, S, S, K), np.int32)
    zbuf = np.empty((N, S, S, K), np.float32)
    q = np.empty((N, S, S, K), np.float32)
    occ = np.empty((N, S, S), np.float32)
    lib().oracle_splat_points_naive(_p(points), _p(ellipse), _p(cutoff), _p(radii), _p(first_idx),
                                    _p(num_pts), C.c_int(N), C.c_float(depth_merge), C.c_int(S),
                                    C.c_int(K), C.c_int(fma_mode), C.c_int(int(bbox_and)),
                                    _p(idx), _p(zbuf), _p(q), _p(occ))
    return idx, zbuf, q, occ


def splat_points_binned(points, ellipse, cutoff, radii, first_idx, num_pts, depth_merge, S, K,
                        bin_size, fma_mode=0):
    """Same outputs via coarse bins + per-pixel scan.  rasterize_points.cu:293-432, 506-597."""
    points, ellipse, cutoff, radii = _f32(points), _f32(ellipse), _f32(cutoff), _f32(radii)
    first_idx, num_pts = _i64(first_idx), _i64(num_pts)
    N = len(num_pts)
    idx = np.empty((N, S, S, K), np.int32)
    zbuf = np.empty((N, S, S, K), np.float32)
    q = np.empty((N, S, S, K), np.float32)
    occ = np.empty((N, S, S), np.float32)
    lib().oracle_splat_points_binned(_p(points), _p(ellipse), _p(cutoff), _p(radii), _p(first_idx),
                                     _p(num_pts), C.c_int(N), C.c_float(depth_merge), C.c_int(S),
                                     C.c_int(K), C.c_int(bin_size), C.c_int(fma_mode),
                                     _p(idx), _p(zbuf), _p(q), _p(occ))
    return idx, zbuf, q, occ


def rasterize_coarse(points, radii, first_idx, num_pts, S, bin_size):
    """-> (bin_offsets (N*B*B+1,) i64, bin_ids i32 ascending per bin).  rasterize_points.cu:293-432."""
    points, radii = _f32(points), _f32(radii)
    first_idx, num_pts = _i64(first_idx), _i64(num_pts)
    N = len(num_pts)
    B = 1 + (S - 1) // bin_size
    off = np.zeros(N * B * B + 1, np.int64)
    total = lib().oracle_rasterize_coarse(_p(points), _p(radii), _p(first_idx), _p(num_pts), C.c_int(N),
                                          C.c_int(S), C.c_int(bin_size), _p(off), None)
    ids = np.empty(max(int(total), 1), np.int32)
    lib().oracle_rasterize_coarse(_p(points), _p(radii), _p(first_idx), _p(num_pts), C.c_int(N),
                                  C.c_int(S), C.c_int(bin_size), _p(off), _p(ids))
    return off, ids[: int(total)]


def blend_forward(idx, qvalue, occ, scaler, colours):
    """-> (N,S,S,C+1).  renderer.py:53-78 + norm_weighted_sum [ext]."""
    idx, qvalue, occ, scaler, colours = _i32(idx), _f32(qvalue), _f32(occ), _f32(scaler), _f32(colours)
    K = idx.shape[-1]
    Cc = colours.shape[1]
    npix = idx.size // K
    out = np.empty(idx.shape[:-1] + (Cc + 1,), np.float32)
    lib().oracle_blend_forward(_p(idx), _p(qvalue), _p(occ), _p(scaler), _p(colours), C.c_long(npix),
                               C.c_int(K), C.c_int(Cc), _p(out))
    return out


def blend_backward_colours(idx, qvalue, scaler, grad_image, P):
    idx, qvalue, scaler, grad_image = _i32(idx), _f32(qvalue), _f32(scaler), _f32(grad_image)
    K = idx.shape[-1]
    Cc = grad_image.shape[-1] - 1
    npix = idx.size // K
    out = np.zeros((P, Cc), np.float32)
    lib().oracle_blend_backward_colours(_p(idx), _p(qvalue), _p(scaler), _p(grad_image), C.c_long(npix),
                                        C.c_int(K), C.c_int(Cc), C.c_long(P), _p(out))
    return out


def visibility(idx, P):
    idx = _i32(idx)
    K = idx.shape[-1]
    vis = np.zeros(P, np.uint8)
    lib().oracle_visibility(_p(idx), C.c_long(idx.size // K), C.c_int(K), C.c_long(P), _p(vis))
    return vis


def search_radius(radii, vis, first_idx, num_pts, radii_s):
    radii, first_idx, num_pts = _f32(radii), _i64(first_idx), _i64(num_pts)
    vis = np.ascontiguousarray(vis, np.uint8)
    rs = np.zeros(len(num_pts), np.float32)
    lib().oracle_search_radius(_p(radii), _p(vis), _p(first_idx), _p(num_pts), C.c_int(len(num_pts)),
                               C.c_float(radii_s), _p(rs))
    return rs


def occ_backward_fast(points, radii, vis, rs, grad_occ, first_idx, num_pts, bruteforce=False, fma_mode=0,
                      stats=False):
    """-> (grad_f32 (P,2), grad_f64 (P,2)).  rasterize_points_backward.cu:85-178.

    fma_mode: the rounding of d2 = dx*dx + dy*dy in the disc test -- 0: two products and a sum (the reference's x86
    build), 1: fmaf(dx, dx, dy*dy) (the reference's CUDA build and our kernels).  stats=True appends a dict with
    "abs" (P,2), the per-point float64 sums of |dx/den*g| and |dy/den*g| over the contributing pairs, and "pairs"
    (P,) int32, their number.  bruteforce=True visits every pixel for every point; grad_f32 is then None."""
    points, radii, rs, grad_occ = _f32(points), _f32(radii), _f32(rs), _f32(grad_occ)
    first_idx, num_pts = _i64(first_idx), _i64(num_pts)
    vis = np.ascontiguousarray(vis, np.uint8)
    N, S = grad_occ.shape[0], grad_occ.shape[1]
    P = points.shape[0]
    g64 = np.zeros((P, 2), np.float64)
    a64 = np.zeros((P, 2), np.float64) if stats else None
    npairs = np.zeros(P, np.int32) if stats else None
    g32 = None
    if bruteforce:
        lib().oracle_occ_backward_fast_bruteforce(_p(points), _p(radii), _p(vis), _p(rs), _p(grad_occ),
                                                  _p(first_idx), _p(num_pts), C.c_int(N), C.c_int(S),
                                                  C.c_int(int(fma_mode)), _p(g64), _p(a64), _p(npairs))
    else:
        g32 = np.zeros((P, 2), np.float32)
        lib().oracle_occ_backward_fast(_p(points), _p(radii), _p(vis), _p(rs), _p(grad_occ), _p(first_idx),
                                       _p(num_pts), C.c_int(N), C.c_int(S), C.c_int(int(fma_mode)), _p(g32), _p(g64),
                                       _p(a64), _p(npairs))
    if stats:
        return g32, g64, dict(abs=a64, pairs=npairs)
    return g32, g64


def occ_backward_slow(points, radii, grad_occ, first_idx, num_pts, radii_s, cpu_twin=False):
    """rasterize_points.cu:673-760 (cpu_twin: rasterize_points_cpu.cpp:380-477)."""
    points, radii, grad_occ = _f32(points), _f32(radii), _f32(grad_occ)
    first_idx, num_pts = _i64(first_idx), _i64(num_pts)
    N, S = grad_occ.shape[0], grad_occ.shape[1]
    g = np.zeros((points.shape[0], 2), np.float32)
    lib().oracle_occ_backward_slow(_p(points), _p(radii), _p(grad_occ), _p(first_idx), _p(num_pts),
                                   C.c_int(N), C.c_int(S), C.c_float(radii_s), C.c_int(int(cpu_twin)), _p(g))
    return g


def zbuf_backward(idx, grad_zbuf, P):
    idx, grad_zbuf = _i32(idx), _f32(grad_zbuf)
    K = idx.shape[-1]
    z = np.zeros(P, np.float32)
    lib().oracle_zbuf_backward(_p(idx), _p(grad_zbuf), C.c_long(idx.size // K), C.c_int(K), _p(z))
    return z


def exclusive_scan_i32(a):
    a = _i32(a)
    out = np.empty_like(a)
    lib().oracle_exclusive_scan_i32(_p(a), C.c_int(a.size), _p(out))
    return out


def insert_points_2d(points, lengths, params, G):
    points, lengths, params = _f32(points), _i64(lengths), _f32(params)
    N, P = points.shape[0], points.shape[1]
    cnt = np.zeros((N, G), np.int32)
    cell = np.full((N, P), -1, np.int32)
    slot = np.full((N, P), -1, np.int32)
    lib().oracle_insert_points_2d(_p(points), _p(lengths), _p(params), C.c_int(N), C.c_int(P), C.c_int(G),
                                  _p(cnt), _p(cell), _p(slot))
    return cnt, cell, slot


def counting_sort_2d(points, lengths, cell, slot, off):
    points, lengths = _f32(points), _i64(lengths)
    cell, slot, off = _i32(cell), _i32(slot), _i32(off)
    N, P = points.shape[0], points.shape[1]
    G = off.shape[1]
    sp = np.zeros((N, P, 2), np.float32)
    si = np.full((N, P), -1, np.int32)
    lib().oracle_counting_sort_2d(_p(points), _p(lengths), _p(cell), _p(slot), _p(off), C.c_int(N), C.c_int(P),
                                  C.c_int(G), _p(sp), _p(si))
    return sp, si


def preprocess_f64(M, V, pts, nrm, h, cutoff, sigma, S):
    """Double-precision per-(point,view) info.  rasterizer.py:443-565.
    -> dict(ndc (N*P0,3), ellipse (.,3), radii (.,2), scaler (.,), jac (.,3,2))"""
    M, V, pts, nrm, h = _f32(M), _f32(V), _f32(pts), _f32(nrm), _f32(h)
    N, P0 = M.shape[0], pts.shape[0]
    per_splat = int(h.size == N * P0 and h.size != N)
    P = N * P0
    ndc = np.empty((P, 3)); ell = np.empty((P, 3)); rad = np.empty((P, 2)); sc = np.empty(P)
    jac = np.empty((P, 3, 2))
    lib().oracle_preprocess_f64(_p(M), _p(V), _p(pts), _p(nrm), _p(h), C.c_int(per_splat), C.c_int(N),
                                C.c_long(P0), C.c_float(cutoff), C.c_float(sigma), C.c_int(S), _p(ndc),
                                _p(ell), _p(rad), _p(sc), _p(jac))
    return dict(ndc=ndc, ellipse=ell, radii=rad, scaler=sc, jac=jac)


def knn_brute(queries, qfirst, qnum, points, first, num, K, r):
    """-> (dists (Pq,K) f32 ascending, idxs (Pq,K) i32 local to the cloud), -1 padded.
    external/FRNN/frnn/csrc/bruteforce/bruteforce_cpu.cpp:8-64."""
    queries, points = _f32(queries), _f32(points)
    qfirst, qnum, first, num = _i64(qfirst), _i64(qnum), _i64(first), _i64(num)
    assert K <= 64
    d = np.full((queries.shape[0], K), -1, np.float32)
    i = np.full((queries.shape[0], K), -1, np.int32)
    lib().oracle_knn_brute(_p(queries), _p(qfirst), _p(qnum), _p(points), _p(first), _p(num), C.c_int(len(num)),
                           C.c_int(K), C.c_float(r), _p(d), _p(i))
    return d, i
