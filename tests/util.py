"""Seeded synthetic scenes shared by tests, smoke() and bench.py (SURVEY.md section 8d), the helpers that store
and read what the reference's own kernels computed on them (tests/golden/), and the float64 reference of the fused
backward (render_backward_f64)."""
import ctypes as C
import os

import numpy as np
import torch

from dss_b200 import _lib, ops
from dss_b200.core.camera import FoVPerspectiveCameras, look_at_view_transform, camera_matrices

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
# outputs of the reference's CUDA kernels (oracle/_ref/dss_ref_cuda on an H100), minted by tests/golden/make_golden_ref_cuda.py
REF_CUDA_GOLDEN = os.path.join(GOLDEN_DIR, "ref_cuda_witness.npz")


def golden_case(path, case):
    """The arrays stored for `case` in a golden file (keys "<case>__<name>")."""
    d = np.load(path)
    out = {k[len(case) + 2:]: d[k] for k in d.files if k.startswith(case + "__")}
    assert out, "no golden data for %s in %s" % (case, path)
    return out


def sample_rows(n, k, seed):
    """A fixed, sorted sample of min(k, n) of the indices 0..n-1."""
    return np.sort(np.random.default_rng(seed).choice(n, min(k, n), replace=False))


def row_hash(a):
    """(M, ...) -> (M,) uint64: an exact hash of the bit patterns of each row (32-bit elements)."""
    b = np.ascontiguousarray(a).reshape(a.shape[0], -1).view(np.uint32).astype(np.uint64)
    h = np.full(b.shape[0], 14695981039346656037, np.uint64)
    for k in range(b.shape[1]):
        h = (h ^ b[:, k]) * np.uint64(1099511628211)
    return h


def digest(a):
    """One exact, position-sensitive uint64 digest of the bit patterns of a whole 32-bit array."""
    b = np.ascontiguousarray(a).reshape(-1).view(np.uint32).astype(np.uint64)
    w = np.arange(b.size, dtype=np.uint64) * np.uint64(2654435761) + np.uint64(97)
    return np.uint64((b * w + b).sum(dtype=np.uint64))


def sphere_cloud(P0, seed=0, radius=0.5):
    """P0 points uniform on a sphere of radius 0.5 (the training init, config.py:177-182),
    outward normals, random colours."""
    g = torch.Generator().manual_seed(1234 + seed)
    p = torch.nn.functional.normalize(torch.randn(P0, 3, generator=g), dim=1)
    colours = torch.rand(P0, 3, generator=g)
    return (radius * p).contiguous(), p.clone().contiguous(), colours.contiguous()


def random_cameras(N, seed=0, dist=(1.2, 2.2), znear=0.1, zfar=100.0):
    """Look-at cameras as DSS/core/camera.py:42-51 samples them (fov 60, znear 0.1, zfar 100)."""
    g = torch.Generator().manual_seed(4321 + seed)
    d = torch.rand(N, generator=g) * (dist[1] - dist[0]) + dist[0]
    azim = torch.rand(N, generator=g) * 360 - 180
    elev = torch.rand(N, generator=g) * 180 - 90
    at = torch.rand(N, 3, generator=g) * 0.1 - 0.05
    R, T = look_at_view_transform(d, elev, azim, at=at)
    return FoVPerspectiveCameras(znear=znear, zfar=zfar, R=R, T=T)


def scene(P0, N, seed=0):
    pts, nrm, col = sphere_cloud(P0, seed)
    cams = random_cameras(N, seed)
    proj, view = camera_matrices(cams)
    return pts, nrm, col, proj, view, cams


def packed_offsets(N, P0):
    first = torch.arange(N, dtype=torch.int64) * P0
    num = torch.full((N,), P0, dtype=torch.int64)
    return first, num


def random_screen_splats(P, N, S, seed=0, rad_px=(0.8, 4.0), z=(0.5, 3.0), behind_frac=0.05, ragged=True):
    """Random packed screen-space splats for the _C-level operators: points (P,3), ellipse (P,3),
    cutoff (P,), radii (P,2), first_idx, num_points.  Radii are the exact bbox of the conic at cutoff."""
    rng = np.random.default_rng(100 + seed)
    pts = np.concatenate([rng.uniform(-1.05, 1.05, (P, 2)), rng.uniform(z[0], z[1], (P, 1))], 1).astype(np.float32)
    behind = rng.random(P) < behind_frac
    pts[behind, 2] = -pts[behind, 2]
    pix = 2.0 / S
    # random SPD 2x2 variance -> conic = inverse
    s1 = rng.uniform(rad_px[0] * pix, rad_px[1] * pix, P)
    s2 = rng.uniform(rad_px[0] * pix, rad_px[1] * pix, P)
    th = rng.uniform(0, np.pi, P)
    c, s = np.cos(th), np.sin(th)
    G00 = (c * s1) ** 2 + (s * s2) ** 2
    G11 = (s * s1) ** 2 + (c * s2) ** 2
    G01 = c * s * (s1 ** 2 - s2 ** 2)
    det = G00 * G11 - G01 ** 2
    cutoff = rng.uniform(0.5, 2.0, P).astype(np.float32)
    ell = np.stack([G11 / det, -2 * G01 / det, G00 / det], 1).astype(np.float32)
    rad = np.stack([np.sqrt(cutoff * G00), np.sqrt(cutoff * G11)], 1).astype(np.float32)
    if ragged and N > 1:
        cuts = np.sort(rng.choice(np.arange(1, P), N - 1, replace=False))
        bounds = np.concatenate([[0], cuts, [P]])
    else:
        bounds = np.linspace(0, P, N + 1).astype(np.int64)
    first = bounds[:-1].astype(np.int64)
    num = (bounds[1:] - bounds[:-1]).astype(np.int64)
    return pts, ell, cutoff, rad, first, num


def backward_via_lib(out, pts, proj, view, first, num, shared, prm, grad_image, grad_zbuf, repeat_camera=1):
    """dss_render_backward with grad_ndc set, then `repeat_camera` calls of dss_camera_backward (as ops.py does) ->
    (grad_ndc (P,3), grad_points (P0,3) / (P,3), [(grad_proj, grad_view)] of every repetition).  No forward cell counts
    are passed, so the backward runs its own count pass."""
    dev = pts.device
    N = proj.shape[0]
    P0 = pts.shape[0]
    P = N * P0 if shared else P0
    a = _lib.RenderArgs()
    ops._fill_common(a, pts, None, None, proj, view, None, first, num, shared, N, P0, P, prm)
    a.records, a.idx, a.weights, a.visible = (_lib.ptr(t) for t in (out.records, out.idx, out.weights, out.visible))
    a.grad_image, a.grad_zbuf = _lib.ptr(grad_image), _lib.ptr(grad_zbuf)
    # rows that no view range covers are never written (ops.py zero-fills them the same way)
    grad_points = torch.zeros_like(pts)
    grad_ndc = torch.zeros((P, 3), dtype=torch.float32, device=dev)
    a.grad_points_world, a.grad_ndc = _lib.ptr(grad_points), _lib.ptr(grad_ndc)
    lib, ctx, st = _lib.load(), _lib.ctx(dev), _lib.stream_ptr(dev)
    _lib.check(lib.dss_render_backward(ctx, C.byref(a), st), "dss_render_backward")
    res = []
    for _ in range(repeat_camera):
        gP, gV = (torch.full((N, 4, 4), float("nan"), device=dev) for _ in range(2))
        _lib.check(lib.dss_camera_backward(ctx, C.byref(a), _lib.ptr(gP), _lib.ptr(gV), None, st), "dss_camera_backward")
        res.append((gP, gV))
    torch.cuda.synchronize(dev)
    return grad_ndc, grad_points, res


def _npy(t):
    return t.detach().cpu().numpy() if torch.is_tensor(t) else np.asarray(t)


def view_ranges(N, P0, first, num):
    """(first, num) as int64 numpy arrays; a shared cloud (first = None) of P0 points is N ranges of P0 slots"""
    if first is None:
        return np.arange(N, dtype=np.int64) * P0, np.full(N, P0, np.int64)
    return _npy(first).astype(np.int64), _npy(num).astype(np.int64)


def preprocess_f64_slots(pts, nrm, proj, view, h, prm, first=None, num=None):
    """oracle.preprocess_f64 for every slot of a shared (first = None) or packed cloud: one call per view on that view's
    slice of the points, the normals and h (per view (N,), or per splat (P,) -- the slice then sets its per_splat mode)
    -> dict of (P, .) float64 arrays ndc, radii, scaler, jac; rows outside every view range are NaN."""
    import oracle
    pts, nrm, projn, viewn, h = _npy(pts), _npy(nrm), _npy(proj), _npy(view), _npy(h).reshape(-1)
    N, shared = projn.shape[0], first is None
    first, num = view_ranges(N, pts.shape[0], first, num)
    P = N * pts.shape[0] if shared else pts.shape[0]
    per_splat = h.size == P and h.size != N
    out = dict(ndc=np.full((P, 3), np.nan), radii=np.full((P, 2), np.nan), scaler=np.full(P, np.nan),
               jac=np.full((P, 3, 2), np.nan))
    for n in range(N):
        f, m = int(first[n]), int(num[n])
        if m == 0:
            continue
        src = slice(0, m) if shared else slice(f, f + m)
        pre = oracle.preprocess_f64(projn[n:n + 1], viewn[n:n + 1], pts[src], nrm[src],
                                    h[f:f + m] if per_splat else h[n:n + 1], prm.cutoff_threshold,
                                    prm.antialiasing_sigma, prm.image_size)
        for k in out:
            out[k][f:f + m] = pre[k]
    return out


def render_backward_f64(ndc, radii, idx, qvalue, scaler, pts, proj, view, prm, grad_image, grad_zbuf=None,
                        first=None, num=None):
    """Float64 reference of the whole fused backward (dss_render_backward) on a forward's own fragments.

    ndc (P,3), radii (P,2)     : the per-slot screen records the forward rasterized (records[:, :3], records[:, 3:5])
    idx, qvalue (N,S,S,K)       : its fragments;  scaler (P,): its per-slot scaler
    pts (P0,3) / (P,3)          : world points of a shared cloud (first = num = None) or of the packed slots
    proj, view (N,4,4)          : the cameras; prm: the SplatParams of the call
    grad_image (N,S,S,4), grad_zbuf (N,S,S,K) or None

    Composes the oracle: visibility -> exact lower median per (ragged) view -> occupancy gather (its float64 sums) ->
    z-buffer scatter (float64) -> clip of the 3-vector (rasterizer.py:667-673) in float64 -> chain through the float64
    Jacobian of oracle.preprocess_f64 and V[:3, 2] (the view depth) -> world gradient; and the colour gradient.
    Returns a dict of float64 arrays:
      ndc (P,3)       clipped NDC gradient per slot;   ndc_raw (P,3): the same before the clip
      ndc_err32 (P,)  per slot, |fp32 oracle - float64| of the pre-clip vector (fp32 sums in pixel order)
      world           (P0,3) summed over the views (shared) or (P,3) per packed row (rows no range covers: 0)
      colours (P,3)   colour gradient per slot
      vis (P,) uint8, rs (N,): the visibility and search radius it used
    """
    import oracle
    ndc = np.ascontiguousarray(_npy(ndc), np.float32)
    radii = np.ascontiguousarray(_npy(radii), np.float32)
    idx = np.ascontiguousarray(_npy(idx), np.int32)
    qvalue, scaler = _npy(qvalue), _npy(scaler)
    pts, viewn = _npy(pts), _npy(view)
    gi = np.ascontiguousarray(_npy(grad_image), np.float32)
    N, P = viewn.shape[0], ndc.shape[0]
    shared = first is None
    first, num = view_ranges(N, pts.shape[0], first, num)
    vis = oracle.visibility(idx, P)
    rs = oracle.search_radius(radii, vis, first, num, prm.radii_backward_scaler)
    g32, g64 = oracle.occ_backward_fast(ndc, radii, vis, rs, np.ascontiguousarray(gi[..., 3]), first, num)
    raw = np.concatenate([g64, np.zeros((P, 1))], 1)
    raw32 = np.concatenate([g32.astype(np.float64), np.zeros((P, 1))], 1)
    if grad_zbuf is not None:
        gz = np.ascontiguousarray(_npy(grad_zbuf), np.float32)
        # rasterize_points.cu:823-846: every fragment up to the first empty one
        live = np.cumprod(idx >= 0, axis=-1).astype(bool)
        np.add.at(raw[:, 2], idx[live], gz[live].astype(np.float64))
        raw32[:, 2] = oracle.zbuf_backward(idx, gz, P)
    err32 = np.linalg.norm(raw32 - raw, axis=1)
    g = raw.copy()
    if prm.clip_pts_grad > 0:
        nrm = np.linalg.norm(g, axis=1, keepdims=True)
        g = g / np.maximum(nrm, 1e-12) * np.minimum(nrm, prm.clip_pts_grad)
    # chain: d ndc_xy / d world = J (float64, from the world points; the normals and h do not enter it),
    # d z_view / d world = V[:3, 2]
    jac = preprocess_f64_slots(pts, np.zeros_like(pts), proj, view, np.ones(N, np.float32), prm,
                               None if shared else first, None if shared else num)["jac"]
    world = np.zeros((pts.shape[0], 3))
    for n in range(N):
        f, m = int(first[n]), int(num[n])
        gs = g[f:f + m]
        w = np.einsum("pkj,pj->pk", jac[f:f + m], gs[:, :2]) + gs[:, 2:3] * viewn[n, :3, 2].astype(np.float64)[None]
        if shared:
            world[:m] += w
        else:
            world[f:f + m] += w
    colours = oracle.blend_backward_colours(idx, qvalue, scaler, gi, P).astype(np.float64)
    return dict(ndc=g, ndc_raw=raw, ndc_err32=err32, world=world, colours=colours, vis=vis, rs=rs)


def render_backward_f64_of(out, pts, proj, view, prm, grad_image, grad_zbuf=None, first=None, num=None):
    """render_backward_f64 on the fragments of render_points(..., return_fragments=True)"""
    return render_backward_f64(out.records[:, :3], out.records[:, 3:5], out.idx, out.qvalue, out.scaler, pts, proj,
                               view, prm, grad_image, grad_zbuf, first, num)
