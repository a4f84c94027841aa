"""Fused surface-splatting render operator (autograd.Function) over the C ABI.

forward  = dss_render_forward : per-(point,view) EWA preprocess -> tile binning (on-device prefix sum) ->
           per-tile top-K rasterization + normalised blend              (rasterizer.py:584-664, renderer.py:36-82)
backward = dss_render_backward: visibility / median radius -> occupancy gather -> colour scatter ->
           z scatter -> per-point clip -> chain to world space           (rasterizer.py:788-977, 667-673)
           [+ dss_camera_backward when proj, view or the shading's camera centres require grad]
           [+ dss_light_backward when the shading's lights or ambient colour require grad]

Gradients follow the reference exactly: positions receive the occupancy surrogate gradient (and the
z-buffer gradient when one is supplied), colours receive the compositor gradient, the cameras (proj, view,
shading camera centres) and the shading's lights receive what the reference's differentiable transform and shading
give them, the shininess and the per-point ellipse parameters are constants (computed under no_grad and detached:
rasterizer.py:606-608, 562-565).
"""
import ctypes as C
from typing import NamedTuple, Optional

import torch

from . import _lib

__all__ = ["SplatParams", "Shading", "make_shading", "RenderOutput", "render_points", "preprocess_points",
           "point_filters", "point_filters_no_views", "set_point_filters", "local_frames", "MeshRender", "render_mesh", "chamfer_distance",
           "PointMeshDistance", "point_mesh_distance"]


class SplatParams(NamedTuple):
    image_size: int = 256
    points_per_pixel: int = 5
    cutoff_threshold: float = 1.0
    depth_merging_threshold: float = 0.05
    antialiasing_sigma: float = 1.0
    radii_backward_scaler: float = 5.0
    clip_pts_grad: float = -1.0
    backface_culling: bool = False
    znear: float = 1.0
    zfar: float = 100.0


class Shading(NamedTuple):
    """Fused per-point shading (SURVEY.md 8(f)3): pass as ``shading=`` with the per-point albedo as ``colours`` (per
    world point of a shared cloud, or per packed row).  Build it from the light objects with :func:`make_shading`."""
    lights: torch.Tensor         # (L,9) {direction | location, diffuse rgb, specular rgb}, or (N,L,9): a set per view
    ambient: torch.Tensor        # (3,), or (N,3) with per-view lights
    cam_centres: torch.Tensor    # (N,3) camera centres in world space
    light_type: int = 0          # 0 directional, 1 point
    shininess: float = 64.0


class RenderOutput(NamedTuple):
    image: torch.Tensor      # (N,S,S,4) rgb + occupancy
    idx: torch.Tensor        # (N,S,S,K) int32
    zbuf: Optional[torch.Tensor]
    qvalue: Optional[torch.Tensor]
    weights: torch.Tensor    # (N,S,S,K) normalised blend weights
    visible: torch.Tensor    # (P,) uint8
    records: torch.Tensor    # (P,8) {x,y,z,rx, ry,a,b,c}
    scaler: torch.Tensor     # (P,)


def _fill_shading(a, sh, albedo):
    a.shade = 1
    a.n_lights = int(sh.lights.shape[-2])
    a.lights_per_view = int(sh.lights.dim() == 3)
    a.light_type = int(sh.light_type)
    a.shininess = float(sh.shininess)
    a.albedo, a.lights, a.ambient, a.cam_centres = _lib.ptr(albedo), _lib.ptr(sh.lights), _lib.ptr(sh.ambient), \
        _lib.ptr(sh.cam_centres)


def _check_shading(sh, N, dev):
    per_view = sh.lights.dim() == 3
    if (sh.lights.dim() not in (2, 3) or sh.lights.shape[-1] != 9 or not (1 <= sh.lights.shape[-2] <= _lib.MAX_LIGHTS)
            or (per_view and sh.lights.shape[0] != N)):
        raise RuntimeError("shading.lights must be (L,9) or, per view, (%d,L,9) with 1 <= L <= %d, got %s"
                           % (N, _lib.MAX_LIGHTS, tuple(sh.lights.shape)))
    if tuple(sh.ambient.shape) != ((N, 3) if per_view else (3,)) or tuple(sh.cam_centres.shape) != (N, 3):
        raise RuntimeError("shading.ambient must be (3,), or (N,3) with per-view lights, and shading.cam_centres (N,3)")
    _lib.require_cuda(sh.lights, sh.ambient, sh.cam_centres)
    return Shading(_lib.as_f32(sh.lights.detach(), "lights"), _lib.as_f32(sh.ambient.detach(), "ambient"),
                   _lib.as_f32(sh.cam_centres.detach(), "cam_centres"), int(sh.light_type), float(sh.shininess))


def _fill_common(a, points, normals, colours, proj, view, h, first_idx, num_points, shared, N, P0, P, prm):
    a.points_world = _lib.ptr(points)
    a.normals_world = _lib.ptr(normals)
    a.colours = _lib.ptr(colours)
    a.proj = _lib.ptr(proj)
    a.view = _lib.ptr(view)
    a.h = _lib.ptr(h)
    a.first_idx = _lib.ptr(first_idx)
    a.num_points = _lib.ptr(num_points)
    a.n_views = N
    a.shared_cloud = int(shared)
    a.P0 = P0
    a.P = P
    a.h_per_splat = int(h is not None and h.numel() == P and h.numel() != N)
    a.image_size = int(prm.image_size)
    a.points_per_pixel = int(prm.points_per_pixel)
    a.backface_culling = int(bool(prm.backface_culling))
    a.cutoff_threshold = float(prm.cutoff_threshold)
    a.depth_merging_threshold = float(prm.depth_merging_threshold)
    a.antialiasing_sigma = float(prm.antialiasing_sigma)
    a.znear = float(prm.znear)
    a.zfar = float(prm.zfar)
    a.radii_backward_scaler = float(prm.radii_backward_scaler)
    a.clip_pts_grad = float(prm.clip_pts_grad)


def _layout(points, proj, first_idx, num_points, shared):
    N = proj.shape[0]
    if shared:
        if N > _lib.MAX_SHARED_VIEWS:   # the backward's chain kernel holds the view matrices in shared memory
            raise RuntimeError("a shared cloud takes at most %d views per call, got %d" % (_lib.MAX_SHARED_VIEWS, N))
        P0 = points.shape[0]
        return N, P0, N * P0
    if first_idx is None or num_points is None:
        raise RuntimeError("packed clouds need cloud_to_packed_first_idx and num_points_per_cloud")
    P = points.shape[0]
    # the kernels read both arrays as int64[N] and index the packed arrays with them: check before any launch
    # (their VALUES stay on the device -- reading them back would put a host sync into every forward; rows that no
    #  range covers get zero gradients, see backward)
    for name, t in (("cloud_to_packed_first_idx", first_idx), ("num_points_per_cloud", num_points)):
        if t.dtype != torch.int64 or tuple(t.shape) != (N,):
            raise RuntimeError("%s must be an int64 tensor of shape (%d,), got %s %s"
                               % (name, N, t.dtype, tuple(t.shape)))
    return N, P, P   # P0 is only an upper bound on the points of one view in packed mode


def _splat_shape(h, frames, rows, N, P):
    """(h_c, frames_c) for the kernel: exactly one of the isotropic / invariant scale h ((N,) or (P,)) and the
    anisotropic frames ((rows, 8) records of :func:`local_frames`, rows = P0 for a shared cloud, P packed)"""
    if (h is None) == (frames is None):
        raise RuntimeError("pass exactly one of h (isotropic / invariant splats) and frames (anisotropic splats)")
    if frames is None:
        h_c = _lib.as_f32(h.detach().reshape(-1), "h")
        if h_c.numel() not in (N, P):
            raise RuntimeError("h must have N or P elements")
        return h_c, None
    f = _lib.as_f32(frames.detach(), "frames")
    if tuple(f.shape) != (rows, 8):
        raise RuntimeError("frames must have shape (%d, 8), got %s" % (rows, tuple(f.shape)))
    if f.data_ptr() % 16:
        f = f.clone()
    return None, f


class _RenderFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, points, normals, colours, proj, view, h, first_idx, num_points, shared, prm, want_frags,
                grad_sync=None, shading=None, cam_centres=None, lights=None, ambient=None, frames=None,
                deterministic=False):
        # cam_centres, lights and ambient are the shading's tensors, passed on their own so that autograd tracks them
        dev = _lib.require_cuda(points, normals, colours, proj, view, h, first_idx, num_points, frames)
        points_c = _lib.as_f32(points.detach(), "points")
        normals_c = _lib.as_f32(normals.detach(), "normals")
        colours_c = _lib.as_f32(colours.detach(), "colours")
        proj_c = _lib.as_f32(proj.detach(), "proj")
        view_c = _lib.as_f32(view.detach(), "view")
        N, P0, P = _layout(points_c, proj_c, first_idx, num_points, shared)
        h_c, frames_c = _splat_shape(h, frames, P0 if shared else P, N, P)
        if shading is not None:
            if tuple(colours_c.shape) != (P0, 3):
                raise RuntimeError("fused shading takes the per-point albedo as colours: (%d, 3) for a %s, got %s"
                                   % (P0, "shared cloud" if shared else "packed cloud, one row per packed point",
                                      tuple(colours_c.shape)))
            if not shared and grad_sync is not None:
                raise RuntimeError("grad_sync does not take packed clouds with fused shading")
            shading = _check_shading(shading, N, dev)
        shared_col = bool(shared) and (N > 1 or shading is not None) and tuple(colours_c.shape) == (P0, 3)
        if tuple(colours_c.shape) != (P, 3) and not shared_col:
            raise RuntimeError("colours must have shape (%d, 3)%s, got %s"
                               % (P, " or (%d, 3)" % P0 if shared else "", tuple(colours_c.shape)))
        if tuple(proj_c.shape) != (N, 4, 4) or tuple(view_c.shape) != (N, 4, 4):
            raise RuntimeError("proj and view must have shape (N,4,4)")
        S, K = int(prm.image_size), int(prm.points_per_pixel)
        if K > _lib.MAX_POINTS_PER_PIXEL:
            raise RuntimeError("Must have points_per_pixel <= %d" % _lib.MAX_POINTS_PER_PIXEL)
        f32 = dict(dtype=torch.float32, device=dev)
        records = torch.empty((P, 8), **f32)
        scaler = torch.empty((P,), **f32)
        image = torch.empty((N, S, S, 4), **f32)
        idx = torch.empty((N, S, S, K), dtype=torch.int32, device=dev)
        weights = torch.empty((N, S, S, K), **f32)
        # (capacity rounded up to 4 bytes: the blend epilogue sets the bytes with word atomics when it also counts the
        #  visible splats per backward-binning cell, see dss_render_args.cell_counts)
        visible = torch.empty(((P + 3) // 4 * 4,), dtype=torch.uint8, device=dev)[:P]
        # one counter per backward-binning cell: the size dss_render_args.cell_counts states (include/dss_b200.h)
        OB = (S + 31) // 32
        cell_counts = torch.empty((N * OB * OB * 1024,), dtype=torch.int32, device=dev)
        zbuf = torch.empty((N, S, S, K), **f32) if want_frags else None
        qvalue = torch.empty((N, S, S, K), **f32) if want_frags else None
        fi = first_idx.contiguous() if first_idx is not None else None
        npts = num_points.contiguous() if num_points is not None else None
        a = _lib.RenderArgs()
        _fill_common(a, points_c, normals_c, colours_c, proj_c, view_c, h_c, fi, npts, shared, N, P0, P, prm)
        a.frames = _lib.ptr(frames_c)
        a.shared_colours = int(shared_col)
        shaded = None
        if shading is not None:
            shaded = torch.empty((P, 3), **f32)
            _fill_shading(a, shading, colours_c)
            a.shaded = _lib.ptr(shaded)
        a.records, a.scaler, a.image, a.idx = _lib.ptr(records), _lib.ptr(scaler), _lib.ptr(image), _lib.ptr(idx)
        a.weights, a.visible, a.zbuf, a.qvalue = _lib.ptr(weights), _lib.ptr(visible), _lib.ptr(zbuf), _lib.ptr(qvalue)
        a.cell_counts = _lib.ptr(cell_counts)
        with torch.cuda.device(dev):
            rc = _lib.load().dss_render_forward(_lib.ctx(dev), C.byref(a), _lib.stream_ptr(dev))
        _lib.check(rc, "dss_render_forward")
        # no zero-filled gradients for the outputs nobody differentiates (idx, weights, records ... would cost five
        # fill kernels over ~400 MB per backward); backward() handles None
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(points_c, proj_c, view_c, records, idx, weights, visible, fi, npts)
        ctx.shading = (shading, normals_c, colours_c) if shading is not None else None
        ctx.deterministic = bool(deterministic)
        ctx.cell_counts = cell_counts
        ctx.meta = (shared, prm, N, P0, P, want_frags, shared_col, grad_sync)
        outs = (image, idx, weights, visible, records, scaler)
        if want_frags:
            ctx.mark_non_differentiable(idx, weights, visible, records, scaler, qvalue)
            return outs + (zbuf, qvalue)
        ctx.mark_non_differentiable(idx, weights, visible, records, scaler)
        return outs

    @staticmethod
    def backward(ctx, grad_image, *rest):
        points_c, proj_c, view_c, records, idx, weights, visible, fi, npts = ctx.saved_tensors
        shared, prm, N, P0, P, want_frags, shared_col, grad_sync = ctx.meta
        dev = points_c.device
        grad_zbuf = rest[5] if (want_frags and len(rest) > 5) else None
        if grad_image is None:
            grad_image = torch.zeros((N, prm.image_size, prm.image_size, 4), dtype=torch.float32, device=dev)
        grad_image = _lib.as_f32(grad_image, "grad_image")
        if grad_zbuf is not None:
            grad_zbuf = _lib.as_f32(grad_zbuf, "grad_zbuf")
        shade = ctx.shading
        # with fused shading the colour scatter fills a (P,3) scratch (d L / d shaded colour) that the shading backward
        # turns into d albedo / d normal / d position
        grad_colours = torch.empty((P if (shade is not None or not shared_col) else P0, 3), dtype=torch.float32, device=dev)
        grad_normals = None
        # packed clouds: rows no view range covers are never written by the kernels
        grad_points = torch.empty_like(points_c) if shared else torch.zeros_like(points_c)
        a = _lib.RenderArgs()
        _fill_common(a, points_c, None, None, proj_c, view_c, None, fi, npts, shared, N, P0, P, prm)
        a.records, a.idx, a.weights, a.visible = _lib.ptr(records), _lib.ptr(idx), _lib.ptr(weights), _lib.ptr(visible)
        a.cell_counts = _lib.ptr(ctx.cell_counts)
        a.shared_colours = int(shared_col)
        a.grad_image, a.grad_zbuf = _lib.ptr(grad_image), _lib.ptr(grad_zbuf)
        a.grad_colours, a.grad_points_world = _lib.ptr(grad_colours), _lib.ptr(grad_points)
        grad_albedo = grad_pshade = None
        if shade is not None:
            sh, normals_c, albedo_c = shade
            # per world point (shared cloud) or per packed row, whose uncovered rows the kernels never write
            alloc = torch.empty if shared else torch.zeros
            grad_albedo, grad_normals, grad_pshade = (alloc((P0, 3), dtype=torch.float32, device=dev) for _ in range(3))
            _fill_shading(a, sh, albedo_c)
            a.deterministic_colours = int(ctx.deterministic)
            a.normals_world = _lib.ptr(normals_c)
            a.grad_albedo, a.grad_normals_world = _lib.ptr(grad_albedo), _lib.ptr(grad_normals)
            a.grad_points_shading = _lib.ptr(grad_pshade)
        # camera gradients: only when asked for (the (P,3) NDC gradient is 96 MB at 1M points x 8 views)
        want_cam = ctx.needs_input_grad[3] or ctx.needs_input_grad[4] or ctx.needs_input_grad[13]
        grad_proj = grad_view = grad_cam = None
        if want_cam:
            grad_ndc = torch.empty((P, 3), dtype=torch.float32, device=dev)
            a.grad_ndc = _lib.ptr(grad_ndc)
            grad_proj, grad_view = (torch.empty((N, 4, 4), dtype=torch.float32, device=dev) for _ in range(2))
            if shade is not None and ctx.needs_input_grad[13]:
                grad_cam = torch.empty((N, 3), dtype=torch.float32, device=dev)
        # light gradients: only when asked for, in the shape of the shading's tensors
        grad_lights = grad_amb = None
        if shade is not None:
            sh = shade[0]
            grad_lights = torch.empty_like(sh.lights) if ctx.needs_input_grad[14] else None
            grad_amb = torch.empty_like(sh.ambient) if ctx.needs_input_grad[15] else None
        want_light = grad_lights is not None or grad_amb is not None
        lib = _lib.load()

        def light_backward():
            # reads the d L / d shaded scratch in grad_colours
            a.grad_colours = _lib.ptr(grad_colours)
            rc = lib.dss_light_backward(_lib.ctx(dev), C.byref(a), _lib.ptr(grad_lights), _lib.ptr(grad_amb),
                                        _lib.stream_ptr(dev))
            _lib.check(rc, "dss_light_backward")

        def camera_backward():
            # reads grad_ndc and (shading) the d L / d shaded scratch in grad_colours
            a.grad_colours = _lib.ptr(grad_colours)
            rc = lib.dss_camera_backward(_lib.ctx(dev), C.byref(a), _lib.ptr(grad_proj), _lib.ptr(grad_view),
                                         _lib.ptr(grad_cam), _lib.stream_ptr(dev))
            _lib.check(rc, "dss_camera_backward")

        with torch.cuda.device(dev):
            if grad_sync is None:
                rc = lib.dss_render_backward(_lib.ctx(dev), C.byref(a), _lib.stream_ptr(dev))
                _lib.check(rc, "dss_render_backward")
                if want_cam:
                    camera_backward()
                if want_light:
                    light_backward()
            else:
                # data-parallel step (dss_b200/parallel.py): the colour gradients are final after the colour scatter --
                # reduce them over the ranks on a side stream while the occupancy path runs here
                main, side = torch.cuda.current_stream(dev), grad_sync.side_stream(dev)
                side.wait_stream(main)
                with torch.cuda.stream(side):
                    rc = lib.dss_colour_backward(_lib.ctx(dev), C.byref(a), _lib.stream_ptr(dev))
                    _lib.check(rc, "dss_colour_backward")
                    if shade is not None:
                        shade_done = torch.cuda.Event()
                        shade_done.record(side)
                        grad_sync.reduce_early(grad_albedo, grad_normals)
                    else:
                        grad_sync.reduce_early(grad_colours)
                a.grad_colours = _lib.ptr(None)
                rc = lib.dss_render_backward(_lib.ctx(dev), C.byref(a), _lib.stream_ptr(dev))
                _lib.check(rc, "dss_render_backward")
                if shade is not None:
                    main.wait_event(shade_done)
                    grad_points += grad_pshade           # position gradient through the shading
                if want_cam:
                    # the rank's own views: no collective (shared camera parameters are the caller's to reduce)
                    camera_backward()
                if want_light:
                    # after the shading work of the side stream (waited for above); no collective either
                    light_backward()
                grad_sync.reduce_late(grad_points)
                grad_sync.join(dev)
        cams = (grad_proj, grad_view) + (None,) * 8 + (grad_cam, grad_lights, grad_amb, None, None)
        if shade is not None:
            return (grad_points, grad_normals, grad_albedo) + cams
        return (grad_points, None, grad_colours) + cams


def render_points(points, normals, colours, proj, view, h, params: SplatParams, first_idx=None, num_points=None,
                  shared_cloud=True, return_fragments=False, grad_sync=None, shading=None, frames=None,
                  deterministic=False) -> RenderOutput:
    """Render ``N`` views of an oriented point cloud to RGBA.

    points, normals : (P0,3) when ``shared_cloud`` (one cloud seen from N cameras) else packed (P,3)
    colours         : (N*P0,3) / (P,3) per-(view,point) features (e.g. shaded rgb), or (P0,3) per-point
                      features used by every view of a shared cloud (gradient then summed over the views)
    proj, view      : (N,4,4) full-projection and world-to-view matrices, row-vector convention; when they require
                      grad they receive the gradient of the screen positions (proj: x, y; view: the depth)
    h               : (N,) per-view or (P,) per-splat variance scale (rasterizer.py:293-402), or None with ``frames``
    frames          : anisotropic splats (``Vrk_invariant`` and ``Vrk_isotropic`` off, rasterizer.py:256-291): the
                      (P0,8) (shared cloud) or (P,8) (packed) records of :func:`local_frames`, in place of ``h``; the
                      splat's world variance is l1 f1 f1^T + l2 f2 f2^T.  Constants, as in the reference: the normals
                      then receive only the shading's gradient
    shading         : optional Shading -- `colours` is then the per-point albedo, (P0,3) for a shared cloud or (P,3),
                      one row per packed point, for packed clouds, and the colour of every (view, point) is computed in
                      the preprocess kernel: albedo * (ambient + diffuse) + specular (DSS/core/texture.py:74-127), with
                      view n's lights and camera centre for the rows of view n; gradients flow to the albedo, the
                      NORMALS, the positions and, when they require grad, shading.cam_centres, shading.lights and
                      shading.ambient (hence to the light objects' tensors through make_shading); the shininess stays
                      a constant.  Packed rows that no view range covers get zero gradients.
    grad_sync       : optional dss_b200.parallel.GradSync -- the backward then returns gradients already summed over the
                      ranks of a view-sharded step, the collectives overlapped with the backward kernels (not with
                      fused shading of packed clouds)
    deterministic   : with ``shading``, the backward sums d L / d shaded in 64-bit fixed point, so that its gradients are
                      the same bits on every run (the training step asks for it: the loop's resume relies on it); off,
                      float atomics add those terms in arrival order, which is faster at large P
    """
    outs = _RenderFunction.apply(points, normals, colours, proj, view, h, first_idx, num_points,
                                 bool(shared_cloud), params, bool(return_fragments), grad_sync, shading,
                                 *((shading.cam_centres, shading.lights, shading.ambient) if shading is not None
                                   else (None, None, None)), frames, bool(deterministic))
    image, idx, weights, visible, records, scaler = outs[:6]
    zbuf, qvalue = (outs[6], outs[7]) if return_fragments else (None, None)
    return RenderOutput(image, idx, zbuf, qvalue, weights, visible, records, scaler)


def point_filters(out: RenderOutput, mask_img, group=None):
    """The visibility and inmask point filters of the reference's ``Model.forward`` (point_modeling.py:172-173,
    188-212) for the SHARED cloud that ``render_points`` drew in ``out``: ``visibility`` = visible in any view,
    ``inmask`` = visibility and, in any view, torch's ``grid_sample(mask, clamp(-xy, -1, 1))`` (bilinear, reflection
    padding, align_corners=False) != 0 at the NDC position the render projected the point to (csrc/point_filter.cu).
    A non-finite projected position is outside the mask.

    ``mask_img``: the N ground-truth masks, (N,H,W) or (N,1,H,W), float32, uint8 or bool, any strides (read in place),
    of any size H x W.  Returns ``(visibility, inmask)``, (P0,) bool.  One launch, no host synchronisation.

    ``group``: a torch.distributed process group whose ranks each rendered some of the views of one shared cloud: the
    filters are then those of all the views, the same on every rank (exact: ORs of bytes).  Two launches and two
    all-reduces (MAX) of P0 bytes: this rank's visibility, ORed over the ranks, gates ``dss_point_filters_gated``,
    whose inmask is ORed over the ranks in turn.  A rank without views calls :func:`point_filters_no_views`."""
    N = out.image.shape[0]
    P = out.records.shape[0]
    if out.image.dim() != 4 or tuple(out.records.shape[1:]) != (8,) or P % N or tuple(out.visible.shape) != (P,):
        raise RuntimeError("out must be the RenderOutput of a shared cloud: records (N*P0, 8) and visible (N*P0,)")
    if mask_img.dim() == 4 and mask_img.shape[1] == 1:
        mask_img = mask_img[:, 0]
    if mask_img.dim() != 3 or mask_img.shape[0] != N or mask_img.shape[1] < 1 or mask_img.shape[2] < 1:
        raise RuntimeError("mask_img must have shape (%d, H, W) or (%d, 1, H, W), got %s" % (N, N, tuple(mask_img.shape)))
    if mask_img.dtype not in (torch.float32, torch.uint8, torch.bool):
        raise TypeError("mask_img must be float32, uint8 or bool, got %s" % mask_img.dtype)
    dev = _lib.require_cuda(out.records, out.visible, mask_img)
    P0 = P // N
    strides = (C.c_int64 * 3)(*mask_img.stride())
    head = (out.records, out.visible, 1, N, P0, mask_img, int(mask_img.dtype != torch.float32), strides,
            int(mask_img.shape[1]), int(mask_img.shape[2]))

    def launch(name, *tail):
        args = [_lib.ptr(a) if isinstance(a, torch.Tensor) or a is None else a for a in head + tail]
        with torch.cuda.device(dev):
            rc = getattr(_lib.load(), name)(_lib.ctx(dev), *args, _lib.stream_ptr(dev))
        _lib.check(rc, name)

    if group is None:
        visibility = torch.empty((P0,), dtype=torch.bool, device=dev)
        inmask = torch.empty((P0,), dtype=torch.bool, device=dev)
        launch("dss_point_filters", visibility, inmask)
        return visibility, inmask
    import torch.distributed as dist
    visibility, inmask = (torch.empty((P0,), dtype=torch.uint8, device=dev) for _ in range(2))
    launch("dss_point_filters", visibility, inmask)
    dist.all_reduce(visibility, op=dist.ReduceOp.MAX, group=group)
    launch("dss_point_filters_gated", visibility, visibility, inmask)
    dist.all_reduce(inmask, op=dist.ReduceOp.MAX, group=group)
    return visibility.view(torch.bool), inmask.view(torch.bool)


def point_filters_no_views(P0, device, group):
    """:func:`point_filters` with ``group`` on a rank that holds no views of the batch: the same two all-reduces, with
    zero contributions, so that the ranks with views do not wait for it.  Returns the (P0,) filters of all views."""
    import torch.distributed as dist
    visibility, inmask = (torch.zeros((int(P0),), dtype=torch.uint8, device=device) for _ in range(2))
    dist.all_reduce(visibility, op=dist.ReduceOp.MAX, group=group)
    dist.all_reduce(inmask, op=dist.ReduceOp.MAX, group=group)
    return visibility.view(torch.bool), inmask.view(torch.bool)


def set_point_filters(points_filter, out: RenderOutput, mask_img):
    """Set ``points_filter`` (a ``PointCloudsFilters``) to the (1, P0) ``visibility`` and ``inmask`` of
    :func:`point_filters`, the filters ``ProjectionLoss`` / ``RepulsionLoss`` read: one call in place of
    point_modeling.py:188-212.  Returns ``points_filter``."""
    visibility, inmask = point_filters(out, mask_img)
    points_filter.set_filter(visibility=visibility[None], inmask=inmask[None])
    return points_filter


def make_shading(lights, view_matrices, shininess=64.0) -> Shading:
    """Shading record for the fused route from a DirectionalLights / PointLights object (dss_b200.core.lighting) and the
    (N,4,4) world-to-view matrices of the step's cameras.  Lights of batch 1 are shared by the views, lights of batch N
    give every view its own set (see pack_lights).  The camera centres and the light rows stay differentiable functions
    of `view_matrices` and of the light tensors, so learnable cameras and lights receive the shading's gradient too."""
    from .core.lighting import pack_lights
    from .core.texture import camera_centres
    rows, ambient, kind = pack_lights(lights)
    N = view_matrices.shape[0]
    if rows.dim() == 3 and rows.shape[0] != N:
        raise ValueError("the lights have batch %d: the fused shading takes lights of batch 1 or N = %d"
                         % (rows.shape[0], N))
    dev = view_matrices.device
    return Shading(rows.to(dev), ambient.to(dev), camera_centres(view_matrices).contiguous().float(), kind, float(shininess))


def preprocess_points(points, normals, proj, view, h, params: SplatParams, first_idx=None, num_points=None,
                      shared_cloud=True, frames=None):
    """Per-(point,view) screen-space info only (rasterizer.py:525-565 + the transform of :614).  Pass exactly one of
    ``h`` and ``frames``, as for :func:`render_points`.

    Returns dict(ndc (P,3), ellipse_params (P,3), radii (P,2), scaler (P,), cutoff_threshold (P,))."""
    dev = _lib.require_cuda(points, normals, proj, view, h, first_idx, num_points, frames)
    points_c, normals_c = _lib.as_f32(points.detach(), "points"), _lib.as_f32(normals.detach(), "normals")
    proj_c, view_c = _lib.as_f32(proj.detach(), "proj"), _lib.as_f32(view.detach(), "view")
    N, P0, P = _layout(points_c, proj_c, first_idx, num_points, shared_cloud)
    h_c, frames_c = _splat_shape(h, frames, P0 if shared_cloud else P, N, P)
    f32 = dict(dtype=torch.float32, device=dev)
    ndc, ell = torch.empty((P, 3), **f32), torch.empty((P, 3), **f32)
    radii, scaler = torch.empty((P, 2), **f32), torch.empty((P,), **f32)
    fi = first_idx.contiguous() if first_idx is not None else None
    npts = num_points.contiguous() if num_points is not None else None
    a = _lib.RenderArgs()
    _fill_common(a, points_c, normals_c, None, proj_c, view_c, h_c, fi, npts, shared_cloud, N, P0, P, params)
    a.frames = _lib.ptr(frames_c)
    a.ndc, a.ellipse, a.radii, a.scaler = _lib.ptr(ndc), _lib.ptr(ell), _lib.ptr(radii), _lib.ptr(scaler)
    with torch.cuda.device(dev):
        rc = _lib.load().dss_preprocess(_lib.ctx(dev), C.byref(a), _lib.stream_ptr(dev))
    _lib.check(rc, "dss_preprocess")
    return {"ndc": ndc, "ellipse_params": ell, "radii": radii, "scaler": scaler,
            "cutoff_threshold": torch.full((P,), float(params.cutoff_threshold), **f32)}


LOCAL_FRAME_K = 8   # neighbourhood of the anisotropic kernel (rasterizer.py:272-273)


def local_frames(points, first_idx=None, num_points=None):
    """Per-point principal frames of the anisotropic reconstruction kernel (``Vrk_invariant`` and ``Vrk_isotropic``
    off: DSS/core/rasterizer.py:256-291 over DSS/utils/mathHelper.py:34-91).  ``points`` (P0,3), one cloud, or packed
    (P,3) with ``first_idx`` / ``num_points`` (N,) int64 as for ``knn_points_packed``.

    Returns (P0|P, 8) float32 records {f1.xyz, l1, f2.xyz, l2}: l0 <= l1 <= l2 the eigenvalues of the population
    covariance of each point's 8 nearest neighbours (itself included) and f1, f2 the eigenvectors of the two largest,
    solved in float64 (csrc/local_frames.cu).  Rows with fewer than 8 finite neighbours (a non-finite point, a packed
    cloud of fewer than 8 points) are NaN.  Two launches (the K-NN and the frames kernel), no host synchronisation; a
    single cloud of at most 8 points raises ValueError as the reference does (mathHelper.py:57-61), packed clouds are
    not checked on the host.  No gradients (the reference computes the frames under no_grad)."""
    from .frnn_grid import knn_points_packed
    dev = _lib.require_cuda(points, first_idx, num_points)
    if points.dim() != 2 or points.shape[1] != 3:
        raise RuntimeError("points must have shape (P, 3)")
    if (first_idx is None) != (num_points is None):
        raise RuntimeError("pass both first_idx and num_points, or neither")
    pts = _lib.as_f32(points.detach(), "points")
    P = pts.shape[0]
    single = first_idx is None
    if single:
        if P <= LOCAL_FRAME_K:
            raise ValueError("the anisotropic kernel needs clouds of more than %d points (the neighbourhood size), "
                             "got %d" % (LOCAL_FRAME_K, P))
        first_idx = torch.zeros((1,), dtype=torch.int64, device=dev)
        num_points = torch.full((1,), P, dtype=torch.int64, device=dev)
    fi, npts = first_idx.contiguous(), num_points.contiguous()
    _, idx = knn_points_packed(pts, fi, npts, LOCAL_FRAME_K, -1.0)
    frames = torch.empty((P, 8), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        rc = _lib.load().dss_local_frames(_lib.ctx(dev), _lib.ptr(pts), _lib.ptr(None if single else fi),
                                          _lib.ptr(None if single else npts), int(npts.shape[0]), P, _lib.ptr(idx),
                                          _lib.ptr(frames), _lib.stream_ptr(dev))
    _lib.check(rc, "dss_local_frames")
    return frames


class MeshRender(NamedTuple):
    image: Optional[torch.Tensor]   # (N,S,S,4) flat-shaded rgb + coverage, or None without shading
    pix_to_face: torch.Tensor       # (N,S,S) int32 face index in the mesh, -1 where no face covers the pixel
    zbuf: torch.Tensor              # (N,S,S) float32 view-space depth of that face, -1 where none


def render_mesh(verts, faces, proj, view, image_size, shading: Optional[Shading] = None) -> MeshRender:
    """Rasterize one opaque triangle mesh into N views: the closest face per pixel and, with ``shading``, its flat
    shading -- pytorch3d's ``MeshRasterizer`` (blur_radius 0, faces_per_pixel 1, no perspective correction, no back-face
    culling) + ``HardFlatShader`` as the reference's scripts/create_mvr_data_from_mesh.py uses them (csrc/mesh_raster.cu;
    the rules are in include/dss_b200.h).

    verts (V,3) f32, faces (F,3) integer (every index in [0, V), checked here), proj / view (N,4,4) as for
    :func:`render_points`.  ``shading``: a :class:`Shading` (:func:`make_shading`), lights shared or per view,
    directional or point; the vertex colours and materials are ones.  Forward only (no gradients).  Background pixels
    are (1, 1, 1, 0); alpha is the coverage mask."""
    dev = _lib.require_cuda(verts, faces, proj, view)
    v = _lib.as_f32(verts.detach(), "verts")
    if v.dim() != 2 or v.shape[1] != 3:
        raise RuntimeError("verts must have shape (V, 3), got %s" % (tuple(v.shape),))
    if faces.dim() != 2 or faces.shape[1] != 3 or faces.dtype.is_floating_point or faces.dtype == torch.bool:
        raise RuntimeError("faces must be an integer tensor of shape (F, 3), got %s %s" % (faces.dtype, tuple(faces.shape)))
    V, F = v.shape[0], faces.shape[0]
    if F and (int(faces.min()) < 0 or int(faces.max()) >= V):
        raise ValueError("face indices must lie in [0, %d)" % V)
    if V >= 2 ** 31 or F >= 2 ** 31:
        raise ValueError("at most 2^31 - 1 vertices and faces")
    f = faces.detach().to(torch.int32).contiguous()
    proj_c, view_c = _lib.as_f32(proj.detach(), "proj"), _lib.as_f32(view.detach(), "view")
    N = proj_c.shape[0]
    if tuple(proj_c.shape) != (N, 4, 4) or tuple(view_c.shape) != (N, 4, 4) or N < 1:
        raise RuntimeError("proj and view must have shape (N,4,4), N >= 1")
    S = int(image_size)
    if S < 1:
        raise RuntimeError("image_size must be positive")
    pix_to_face = torch.empty((N, S, S), dtype=torch.int32, device=dev)
    zbuf = torch.empty((N, S, S), dtype=torch.float32, device=dev)
    image = None
    sh_args = (0, 0, 0, 0.0, None, None, None)
    if shading is not None:
        sh = _check_shading(shading, N, dev)
        image = torch.empty((N, S, S, 4), dtype=torch.float32, device=dev)
        sh_args = (int(sh.lights.shape[-2]), sh.light_type, int(sh.lights.dim() == 3), sh.shininess, sh.lights,
                   sh.ambient, sh.cam_centres)
    with torch.cuda.device(dev):
        rc = _lib.load().dss_rasterize_mesh(
            _lib.ctx(dev), _lib.ptr(v), V, _lib.ptr(f), F, _lib.ptr(proj_c), _lib.ptr(view_c), N, S,
            *sh_args[:4], *(_lib.ptr(t) for t in sh_args[4:]), _lib.ptr(pix_to_face), _lib.ptr(zbuf), _lib.ptr(image),
            _lib.stream_ptr(dev))
    _lib.check(rc, "dss_rasterize_mesh")
    return MeshRender(image, pix_to_face, zbuf)


def _chamfer_input(points, lengths, normals, name):
    """pytorch3d's _handle_pointcloud_input in the dss_knn_points layout: a cloud object gives its packed rows and its
    own normals; a padded (N,P,3) tensor is passed as packed with gaps (cloud n owns rows [n P, n P + lengths[n]))."""
    if hasattr(points, "points_packed"):
        pts, nrm = points.points_packed(), points.normals_packed()
        first, num = points.cloud_to_packed_first_idx(), points.num_points_per_cloud()
        N = len(points)
    else:
        if not torch.is_tensor(points) or points.dim() != 3 or points.shape[2] != 3:
            raise ValueError("%s must be a PointClouds3D or a padded (N, P, 3) tensor" % name)
        if normals is not None and tuple(normals.shape) != tuple(points.shape):
            raise ValueError("%s_normals must have the shape of %s, got %s" % (name, name, tuple(normals.shape)))
        N, P = points.shape[0], points.shape[1]
        pts, nrm = points.reshape(N * P, 3), None if normals is None else normals.reshape(N * P, 3)
        if lengths is not None and (not torch.is_tensor(lengths) or lengths.dim() != 1 or lengths.shape[0] != N):
            raise ValueError("Expected %s_lengths to be of shape (N,) = (%d,), got %s"
                             % (name, N, tuple(lengths.shape) if torch.is_tensor(lengths) else type(lengths).__name__))
        first = torch.arange(N, dtype=torch.int64, device=points.device) * P
        # a length outside [0, P] would read another cloud's or no storage: clamped on the device, no host sync
        num = (torch.full((N,), P, dtype=torch.int64, device=points.device) if lengths is None
               else lengths.to(device=points.device, dtype=torch.int64).clamp(0, P))
    for t in (pts, nrm):
        if t is not None and t.requires_grad:
            raise RuntimeError("chamfer_distance is an evaluation metric without a backward: pass tensors that do not "
                               "require grad (detach them, or call it under torch.no_grad())")
    return pts, nrm, first.contiguous(), num.contiguous(), N


def chamfer_distance(x, y, x_lengths=None, y_lengths=None, x_normals=None, y_normals=None, batch_reduction="mean",
                     point_reduction="mean"):
    """pytorch3d's ``chamfer_distance`` [ext, pytorch3d 0.4.0] as the reference's ``Trainer.evaluate_3d`` calls it
    (DSS/training/trainer.py:158-160), forward only (csrc/chamfer.cu, the rules in include/dss_b200.h).

    ``x`` / ``y``: ``PointClouds3D`` (their own lengths and normals are used) or padded (N,P,3) float32 CUDA tensors with
    optional ``*_lengths`` (N,) and ``*_normals`` (N,P,3).  Per cloud n: the sum over x's rows of the squared distance
    to the nearest row of y (smallest (distance, index)), the same from y to x, and with both normals the sums of
    1 - |cosine_similarity(eps=1e-6)| against the nearest row's normal.  ``point_reduction`` "mean" divides each sum by
    its cloud's length, "sum" keeps it; ``batch_reduction`` "mean" or "sum" reduces over n, ``None`` keeps (N,).
    Returns ``(cham_x + cham_y, cham_norm_x + cham_norm_y or None)`` as float32 device tensors.  A row without a
    neighbour (a NaN or infinite coordinate, an empty other cloud) makes its cloud's terms NaN; padding rows are never
    read.  No gradients: inputs that require grad raise RuntimeError.  No host synchronisation."""
    if batch_reduction not in ("mean", "sum", None):
        raise ValueError('batch_reduction must be one of ["mean", "sum"] or None')
    if point_reduction not in ("mean", "sum"):
        raise ValueError('point_reduction must be one of ["mean", "sum"]')
    sums, xc, yc, with_normals = _chamfer_sums(x, y, x_lengths, y_lengths, x_normals, y_normals)
    terms = sums
    if point_reduction == "mean":
        terms = sums / torch.stack([xc, yc, xc, yc], 1).to(torch.float64)
    if batch_reduction is not None:
        terms = terms.sum(0)
        if batch_reduction == "mean":
            terms = terms / sums.shape[0]
    dist = (terms[..., 0] + terms[..., 1]).float()
    return dist, (terms[..., 2] + terms[..., 3]).float() if with_normals else None


def _chamfer_sums(x, y, x_lengths=None, y_lengths=None, x_normals=None, y_normals=None):
    """dss_chamfer on chamfer_distance's inputs -> (sums (N,4) float64 {sum_x d, sum_y d, sum_x c, sum_y c}, x lengths,
    y lengths, whether both normals were given)"""
    xp, xn, xf, xc, N = _chamfer_input(x, x_lengths, x_normals, "x")
    yp, yn, yf, yc, Ny = _chamfer_input(y, y_lengths, y_normals, "y")
    dev = _lib.require_cuda(xp, xn, xf, xc, yp, yn, yf, yc)
    if Ny != N:
        raise ValueError("y does not have the correct shape: %d clouds against %d" % (Ny, N))
    with_normals = xn is not None and yn is not None
    xp, yp = _lib.as_f32(xp, "x"), _lib.as_f32(yp, "y")
    xn, yn = (_lib.as_f32(xn, "x_normals"), _lib.as_f32(yn, "y_normals")) if with_normals else (None, None)
    sums = torch.zeros((N, 4), dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        rc = _lib.load().dss_chamfer(_lib.ctx(dev), _lib.ptr(xp), _lib.ptr(xn), _lib.ptr(xf), _lib.ptr(xc),
                                     xp.shape[0], _lib.ptr(yp), _lib.ptr(yn), _lib.ptr(yf), _lib.ptr(yc), yp.shape[0],
                                     N, _lib.ptr(sums), _lib.stream_ptr(dev))
    _lib.check(rc, "dss_chamfer")
    return sums, xc, yc, with_normals


class PointMeshDistance(NamedTuple):
    sq_dists: torch.Tensor            # (P,) float32 squared distance to the nearest face, NaN for a non-finite query
    face_idx: torch.Tensor            # (P,) int64 that face, -1 where there is none
    closest: Optional[torch.Tensor]   # (P,3) float32 the closest point on it, or None when not asked for


def point_mesh_distance(points, verts, faces, return_closest=False, _face_tests=None) -> PointMeshDistance:
    """Exact distance from every point to one triangle mesh (csrc/mesh_distance.cu; the rules are in
    include/dss_b200.h): each face is the closed triangle of its vertices, distances are formed in float64 and rounded
    once, a tie goes to the smaller face index, and the result equals a brute force over all faces.

    points (P,3) and verts (V,3) float32 CUDA tensors, faces (F,3) integer with every index in [0, V) (checked here).
    A point with a NaN or infinite coordinate gets NaN / -1; faces on a non-finite vertex are never nearest; without a
    usable face every point gets NaN / -1.  Forward only: inputs that require grad raise RuntimeError.  The call
    synchronises the host once, to size the search structure."""
    dev = _lib.require_cuda(points, verts, faces)
    for name, t in (("points", points), ("verts", verts)):
        if t.requires_grad:
            raise RuntimeError("point_mesh_distance has no backward: pass %s that does not require grad (detach it, "
                               "or call it under torch.no_grad())" % name)
    p, v = _lib.as_f32(points, "points"), _lib.as_f32(verts, "verts")
    if p.dim() != 2 or p.shape[1] != 3:
        raise RuntimeError("points must have shape (P, 3), got %s" % (tuple(p.shape),))
    if v.dim() != 2 or v.shape[1] != 3:
        raise RuntimeError("verts must have shape (V, 3), got %s" % (tuple(v.shape),))
    if faces.dim() != 2 or faces.shape[1] != 3 or faces.dtype.is_floating_point or faces.dtype == torch.bool:
        raise RuntimeError("faces must be an integer tensor of shape (F, 3), got %s %s" % (faces.dtype, tuple(faces.shape)))
    P, V, F = p.shape[0], v.shape[0], faces.shape[0]
    if P >= 2 ** 31 or V >= 2 ** 31 or F >= 2 ** 31:
        raise ValueError("at most 2^31 - 1 points, vertices and faces")
    if F and (int(faces.min()) < 0 or int(faces.max()) >= V):
        raise ValueError("face indices must lie in [0, %d)" % V)
    f = faces.to(torch.int32).contiguous()
    sq = torch.empty(P, dtype=torch.float32, device=dev)
    idx = torch.empty(P, dtype=torch.int32, device=dev)
    closest = torch.empty((P, 3), dtype=torch.float32, device=dev) if return_closest else None
    with torch.cuda.device(dev):
        rc = _lib.load().dss_point_mesh_distance(_lib.ctx(dev), _lib.ptr(p), P, _lib.ptr(v), V, _lib.ptr(f), F,
                                                 _lib.ptr(sq), _lib.ptr(idx), _lib.ptr(closest), _lib.ptr(_face_tests),
                                                 _lib.stream_ptr(dev))
    _lib.check(rc, "dss_point_mesh_distance")
    return PointMeshDistance(sq, idx.long(), closest)
