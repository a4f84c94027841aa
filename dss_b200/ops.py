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
import math
from typing import NamedTuple, Optional

import torch

from . import _lib

__all__ = ["SplatParams", "Shading", "make_shading", "RenderOutput", "render_points", "preprocess_points",
           "point_filters", "point_filters_no_views", "set_point_filters", "local_frames", "PointNormals",
           "estimate_normals", "Outliers", "outlier_ratio", "Upsampled", "upsample_schedule", "upsample_points",
           "denoise_normals", "Projected", "project_to_surface", "l0_smooth", "MeshRender", "render_mesh", "chamfer_distance",
           "PointMeshDistance", "point_mesh_distance", "PoissonMesh", "poisson_reconstruction", "marching_tetrahedra",
           "ImageMetrics", "image_metrics", "gather_views", "shared_cloud_splats", "render_data_views", "evaluate_2d",
           "Coverage", "accumulate_coverage", "point_coverage", "check_rigid_cameras", "pose_cameras"]


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
    depth: Optional[torch.Tensor] = None   # (N,S,S) sum_k w_k z_k, with depth=True


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
    """(N, P0, P, first_idx, num_points) of a render call; a shared cloud reads no offsets (None)"""
    N = proj.shape[0]
    if shared:
        if N > _lib.MAX_SHARED_VIEWS:   # the backward's chain kernel holds the view matrices in shared memory
            raise RuntimeError("a shared cloud takes at most %d views per call, got %d" % (_lib.MAX_SHARED_VIEWS, N))
        P0 = points.shape[0]
        return N, P0, N * P0, None, None
    # packed rows that no view's range covers get zero gradients, see backward
    P = points.shape[0]
    return (N, P, P) + _lib.cloud_offsets(first_idx, num_points, N)   # P0 only bounds one view's points when packed


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
                deterministic=False, want_depth=False):
        # cam_centres, lights and ambient are the shading's tensors, passed on their own so that autograd tracks them
        dev = _lib.require_cuda(points, normals, colours, proj, view, h, first_idx, num_points, frames)
        points_c = _lib.as_f32(points.detach(), "points")
        normals_c = _lib.as_f32(normals.detach(), "normals")
        colours_c = _lib.as_f32(colours.detach(), "colours")
        proj_c = _lib.as_f32(proj.detach(), "proj")
        view_c = _lib.as_f32(view.detach(), "view")
        N, P0, P, fi, npts = _layout(points_c, proj_c, first_idx, num_points, shared)
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
        depth = torch.empty((N, S, S), **f32) if want_depth else None
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
        a.depth = _lib.ptr(depth)
        _lib.call("dss_render_forward", dev, C.byref(a))
        # no zero-filled gradients for the outputs nobody differentiates (idx, weights, records ... would cost five
        # fill kernels over ~400 MB per backward); backward() handles None
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(points_c, proj_c, view_c, records, idx, weights, visible, fi, npts)
        ctx.shading = (shading, normals_c, colours_c) if shading is not None else None
        ctx.deterministic = bool(deterministic)
        ctx.cell_counts = cell_counts
        ctx.meta = (shared, prm, N, P0, P, want_frags, shared_col, grad_sync)
        ctx.want_depth = bool(want_depth)
        outs = (image, idx, weights, visible, records, scaler)
        tail = (depth,) if want_depth else ()
        if want_frags:
            ctx.mark_non_differentiable(idx, weights, visible, records, scaler, qvalue)
            return outs + (zbuf, qvalue) + tail
        ctx.mark_non_differentiable(idx, weights, visible, records, scaler)
        return outs + tail

    @staticmethod
    def backward(ctx, grad_image, *rest):
        points_c, proj_c, view_c, records, idx, weights, visible, fi, npts = ctx.saved_tensors
        shared, prm, N, P0, P, want_frags, shared_col, grad_sync = ctx.meta
        dev = points_c.device
        grad_zbuf = rest[5] if want_frags else None
        grad_depth = rest[-1] if ctx.want_depth else None
        if grad_image is None:
            grad_image = torch.zeros((N, prm.image_size, prm.image_size, 4), dtype=torch.float32, device=dev)
        grad_image = _lib.as_f32(grad_image, "grad_image")
        if grad_zbuf is not None:
            grad_zbuf = _lib.as_f32(grad_zbuf, "grad_zbuf")
        if grad_depth is not None:
            grad_depth = _lib.as_f32(grad_depth, "grad_depth")
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
        a.grad_depth = _lib.ptr(grad_depth)
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

        def light_backward():
            # reads the d L / d shaded scratch in grad_colours
            a.grad_colours = _lib.ptr(grad_colours)
            _lib.call("dss_light_backward", dev, C.byref(a), grad_lights, grad_amb)

        def camera_backward():
            # reads grad_ndc and (shading) the d L / d shaded scratch in grad_colours
            a.grad_colours = _lib.ptr(grad_colours)
            _lib.call("dss_camera_backward", dev, C.byref(a), grad_proj, grad_view, grad_cam)

        if grad_sync is None:
            _lib.call("dss_render_backward", dev, C.byref(a))
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
                _lib.call("dss_colour_backward", dev, C.byref(a))
                if shade is not None:
                    shade_done = torch.cuda.Event()
                    shade_done.record(side)
                    grad_sync.reduce_early(grad_albedo, grad_normals)
                else:
                    grad_sync.reduce_early(grad_colours)
            a.grad_colours = _lib.ptr(None)
            _lib.call("dss_render_backward", dev, C.byref(a))
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
        cams = (grad_proj, grad_view) + (None,) * 8 + (grad_cam, grad_lights, grad_amb, None, None, None)
        if shade is not None:
            return (grad_points, grad_normals, grad_albedo) + cams
        return (grad_points, None, grad_colours) + cams


def render_points(points, normals, colours, proj, view, h, params: SplatParams, first_idx=None, num_points=None,
                  shared_cloud=True, return_fragments=False, grad_sync=None, shading=None, frames=None,
                  deterministic=False, depth=False) -> RenderOutput:
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
    depth           : also return ``RenderOutput.depth``, the (N,S,S) depth of the blend D = sum_k w_k z_k over the
                      pixel's K-list (``weights`` and the records' view depth z; 0 where the list is empty), one launch
                      more.  Differentiable: its gradient reaches each listed record's view depth as sum g_D w_k -- the
                      weights held constant, as the reference holds the blend weights -- summed in 64-bit fixed point
                      (the same bits on every run), and from there the positions and, when they require grad, ``proj``
                      and ``view``
    """
    outs = _RenderFunction.apply(points, normals, colours, proj, view, h, first_idx, num_points,
                                 bool(shared_cloud), params, bool(return_fragments), grad_sync, shading,
                                 *((shading.cam_centres, shading.lights, shading.ambient) if shading is not None
                                   else (None, None, None)), frames, bool(deterministic), bool(depth))
    image, idx, weights, visible, records, scaler = outs[:6]
    zbuf, qvalue = (outs[6], outs[7]) if return_fragments else (None, None)
    return RenderOutput(image, idx, zbuf, qvalue, weights, visible, records, scaler, outs[-1] if depth else None)


def _shared_render_masks(out: RenderOutput, mask_img):
    """``(device, P0, head)`` of a shared-cloud render and its N masks, checked: ``head`` the leading C-ABI arguments
    (records, visible, shared_cloud, N, P0, mask, mask_kind, mask_strides, H, W) of dss_point_filters and
    dss_point_coverage"""
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
    return dev, P0, (out.records, out.visible, 1, N, P0, mask_img, int(mask_img.dtype != torch.float32), strides,
                     int(mask_img.shape[1]), int(mask_img.shape[2]))


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
    dev, P0, head = _shared_render_masks(out, mask_img)
    if group is None:
        visibility = torch.empty((P0,), dtype=torch.bool, device=dev)
        inmask = torch.empty((P0,), dtype=torch.bool, device=dev)
        _lib.call("dss_point_filters", dev, *head, visibility, inmask)
        return visibility, inmask
    import torch.distributed as dist
    visibility, inmask = (torch.empty((P0,), dtype=torch.uint8, device=dev) for _ in range(2))
    _lib.call("dss_point_filters", dev, *head, visibility, inmask)
    dist.all_reduce(visibility, op=dist.ReduceOp.MAX, group=group)
    _lib.call("dss_point_filters_gated", dev, *head, visibility, visibility, inmask)
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


class Coverage(NamedTuple):
    seen: torch.Tensor       # (P0,) int32: the views in which the point is in some pixel's K-list
    outside: torch.Tensor    # (P0,) int32: the views in which it is kept, in the frame and over background


def accumulate_coverage(out: RenderOutput, mask_img, seen, outside):
    """Add the view coverage of the SHARED cloud that ``render_points`` drew in ``out`` to the (P0,) int32 counters
    ``seen`` and ``outside`` (csrc/prune.cu; the rule is in include/dss_b200.h): ``seen[i]`` += the number of views in
    which point i is in some pixel's K-list (``out.visible``), ``outside[i]`` += the number of views in which the
    preprocess kept it (record z > 0), it projects inside the frame (finite x, y with ``|x|, |y| <= 1``) and the
    ``mask_img`` sample there, the one :func:`point_filters` takes, is zero.  Not gated on visibility: a visual-hull
    test.  ``mask_img`` as :func:`point_filters` takes it.  One launch, no host synchronisation, deterministic:
    capturable.  Returns ``Coverage(seen, outside)``."""
    dev, P0, head = _shared_render_masks(out, mask_img)
    for name, t in (("seen", seen), ("outside", outside)):
        if not isinstance(t, torch.Tensor) or t.dtype != torch.int32 or tuple(t.shape) != (P0,) \
                or not t.is_contiguous() or t.device != dev:
            raise RuntimeError("%s must be a contiguous int32 tensor of shape (%d,) on %s, got %s" % (
                name, P0, dev, "%s %s on %s" % (t.dtype, tuple(t.shape), t.device) if isinstance(t, torch.Tensor)
                else type(t).__name__))
    _lib.call("dss_point_coverage", dev, *head, seen, outside)
    return Coverage(seen, outside)


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
    N, P0, P, fi, npts = _layout(points_c, proj_c, first_idx, num_points, shared_cloud)
    h_c, frames_c = _splat_shape(h, frames, P0 if shared_cloud else P, N, P)
    f32 = dict(dtype=torch.float32, device=dev)
    ndc, ell = torch.empty((P, 3), **f32), torch.empty((P, 3), **f32)
    radii, scaler = torch.empty((P, 2), **f32), torch.empty((P,), **f32)
    a = _lib.RenderArgs()
    _fill_common(a, points_c, normals_c, None, proj_c, view_c, h_c, fi, npts, shared_cloud, N, P0, P, params)
    a.frames = _lib.ptr(frames_c)
    a.ndc, a.ellipse, a.radii, a.scaler = _lib.ptr(ndc), _lib.ptr(ell), _lib.ptr(radii), _lib.ptr(scaler)
    _lib.call("dss_preprocess", dev, C.byref(a))
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
    single = first_idx is None and num_points is None
    pts, fi, npts = _lib.packed_cloud(points, first_idx, num_points)
    P = pts.shape[0]
    if single and P <= LOCAL_FRAME_K:
        raise ValueError("the anisotropic kernel needs clouds of more than %d points (the neighbourhood size), "
                         "got %d" % (LOCAL_FRAME_K, P))
    _, idx = knn_points_packed(pts, fi, npts, LOCAL_FRAME_K, -1.0)
    frames = torch.empty((P, 8), dtype=torch.float32, device=pts.device)
    _lib.call("dss_local_frames", pts.device, pts, None if single else fi, None if single else npts,
              int(npts.shape[0]), P, idx, frames)
    return frames


class PointNormals(NamedTuple):
    normals: torch.Tensor             # (P,3) float32, unit; NaN on an invalid row
    root: torch.Tensor                # (P,) int32 local index of the row's component root, -1 when not oriented
    parent: torch.Tensor              # (P,) int32 local index of the row's tree parent, -1 at a root / when not oriented


def estimate_normals(points, k=20, orient=True, first_idx=None, num_points=None) -> PointNormals:
    """Normals of clouds that carry none (csrc/normals.cu; the rules are in include/dss_b200.h and DESIGN.md): PCA over
    each point's ``k`` nearest neighbours of its cloud (itself included), solved in float64, and with ``orient`` the
    signs propagated along the minimum spanning forest of the k-NN graph under the weight 1 - |n_i . n_j| from the
    point of largest z of each component, whose normal is made to point up (Hoppe et al. 1992, meshlab's "Compute
    normals for point sets").  On a closed surface the normals then point outwards.  Without ``orient`` each normal's
    component of largest magnitude is positive.  Orientation is consistent within a connected component only:
    ``root`` tells the components apart.

    ``points`` (P,3) float32 CUDA tensor, one cloud, or packed with ``first_idx`` / ``num_points`` (N,) int64 as for
    ``knn_points_packed``; each cloud is handled on its own, and packed rows outside every cloud are not written.
    ``k`` in [3, 32] (meshlab's default 20).  A row with a non-finite point or fewer than ``k`` finite neighbours gets a
    NaN normal and root = parent = -1.  Two library calls (the K-NN and the estimate), no host synchronisation, the same
    bits on every call.  No gradients."""
    from .frnn_grid import knn_points_packed
    pts, fi, npts = _lib.packed_cloud(points, first_idx, num_points)
    k = _lib.check_k(k, 3, 32)
    dev, P = pts.device, pts.shape[0]
    if P >= 2 ** 30:
        raise ValueError("at most 2^30 - 1 points")
    normals = torch.empty((P, 3), dtype=torch.float32, device=dev)
    root = torch.full((P,), -1, dtype=torch.int32, device=dev)
    parent = torch.full((P,), -1, dtype=torch.int32, device=dev)
    if P == 0:
        return PointNormals(normals, root, parent)
    _, idx = knn_points_packed(pts, fi, npts, k, -1.0)
    _lib.call("dss_estimate_normals", dev, pts, fi, npts, int(npts.shape[0]), P, idx, k, int(bool(orient)), normals,
              root, parent)
    return PointNormals(normals, root, parent)


class Outliers(NamedTuple):
    keep: torch.Tensor                # (P,) bool: ratio < tolerance (False on an invalid row and outside every cloud)
    ratio: torch.Tensor               # (P,) float64 l0 / (l0 + l1 + l2); NaN on an invalid row and outside every cloud


def outlier_ratio(points, k=16, tolerance=0.05, first_idx=None, num_points=None) -> Outliers:
    """The planarity test of the reference's ``remove_outliers`` (DSS/core/cloud.py:363-378; csrc/normals.cu, the
    rules are in include/dss_b200.h): ``ratio = l0 / (l0 + l1 + l2)``, the smallest eigenvalue of the population
    covariance of each point's ``k`` nearest neighbours of its cloud (itself included) over the three, from the same
    float64 PCA as :func:`estimate_normals`, and ``keep = ratio < tolerance`` in float64.

    ``points`` (P,3) float32 CUDA tensor, one cloud, or packed with ``first_idx`` / ``num_points`` (N,) int64 as for
    ``knn_points_packed``.  ``k`` in [3, 32].  A row with a non-finite point or fewer than ``k`` finite neighbours, and
    a row whose neighbours all coincide (0 / 0), get ratio NaN and are not kept.  Two library calls (the K-NN and the
    ratio), no host synchronisation, so the call can be captured in a CUDA graph; the same bits on every call."""
    from .frnn_grid import knn_points_packed
    pts, fi, npts = _lib.packed_cloud(points, first_idx, num_points)
    k = _lib.check_k(k, 3, 32)
    dev, P = pts.device, pts.shape[0]
    if P >= 2 ** 30:
        raise ValueError("at most 2^30 - 1 points")
    keep = torch.zeros((P,), dtype=torch.bool, device=dev)
    ratio = torch.full((P,), float("nan"), dtype=torch.float64, device=dev)
    if P == 0:
        return Outliers(keep, ratio)
    _, idx = knn_points_packed(pts, fi, npts, k, -1.0)
    _lib.call("dss_outlier_ratio", dev, pts, fi, npts, int(npts.shape[0]), P, idx, k, float(tolerance), ratio, keep)
    return Outliers(keep, ratio)


class Upsampled(NamedTuple):
    points: torch.Tensor              # (M,3) float32, packed: cloud n owns rows [first_idx[n], first_idx[n] + num_points[n])
    normals: Optional[torch.Tensor]   # (M,3) float32 or None
    features: Optional[torch.Tensor]  # (M,D) float32 or None
    first_idx: torch.Tensor           # (N,) int64
    num_points: torch.Tensor          # (N,) int64, the targets
    parents: torch.Tensor             # (M,2) int32 (i, j*) local to the cloud; (-1, -1) on an input row


def upsample_schedule(num_points, targets, k=16):
    """The sizes of every cloud before each round and after the last: a list of R + 1 lists of N ints.  Each round adds
    ``min(n - c, c // 10)`` points to a cloud of ``c`` points and target ``n``, until every cloud has reached its
    target.  Raises ValueError for a target below the cloud's size, and for a cloud that has to grow but has at most
    ``k`` or fewer than 10 points (the rounds would then need missing neighbours or never end)."""
    c, n = [int(x) for x in num_points], [int(x) for x in targets]
    if len(c) != len(n):
        raise ValueError("%d targets for %d clouds" % (len(n), len(c)))
    for i, (ci, ni) in enumerate(zip(c, n)):
        if ni < ci:
            raise ValueError("cloud %d: the target %d is below its %d points" % (i, ni, ci))
        if ni > ci and (ci <= k or ci < 10):
            raise ValueError("cloud %d: %d points cannot grow with k = %d: it needs more than k and at least 10 points"
                             % (i, ci, k))
    rounds = [c]
    while any(ci < ni for ci, ni in zip(c, n)):
        c = [ci + min(ni - ci, ci // 10) for ci, ni in zip(c, n)]
        rounds.append(c)
    return rounds


def _read_clouds(fi, npts, P, *per_cloud):
    """The one host synchronisation of upsample_points and _rimls_setup: every cloud's first row and size (int64) and
    the per-cloud values ``per_cloud``, (N,) or (N,c) each, as the columns of one (N, c...) float64 array, in one copy.
    ValueError when a cloud's range leaves the P rows."""
    import numpy as np
    N = fi.shape[0]
    # clamped to [-1, P + 1], which float64 holds exactly and where a range past the rows stays past them
    offsets = (fi.clamp(-1, P + 1), npts.clamp(-1, P + 1))
    info = torch.cat([t.double().reshape(N, -1) for t in offsets + per_cloud], 1).cpu().numpy()
    first, num = info[:, 0].astype(np.int64), info[:, 1].astype(np.int64)
    if (first < 0).any() or (num < 0).any() or (first > P - num).any():
        raise ValueError("first_idx / num_points leave the points")
    return first, num, info[:, 2:]


def upsample_points(points, n, k=16, normals=None, features=None, first_idx=None, num_points=None) -> Upsampled:
    """Densify point clouds as the reference's ``upsample`` does (DSS/core/cloud.py:555-632; csrc/upsample.cu, the rules
    are in include/dss_b200.h and DESIGN.md): in every round each cloud of ``c`` points gains ``min(n - c, c // 10)``
    points, one next to each of its sparsest neighbourhoods.  For a point p and its ``k`` nearest other points q_j the
    candidates are (q_j + 2 p) / 3; a point's sparsity is the largest over j of the distance from candidate j to its
    nearest q; the points of largest sparsity (ties: the smaller index) each add their sparsest candidate.  With
    ``normals`` a child's normal is normalize(2 n_p + n_q) of the unit normals, with ``features`` (colours or any D) its
    feature is (f_q + 2 f_p) / 3.

    ``points`` (P,3) float32 CUDA tensor, one cloud, or packed with ``first_idx`` / ``num_points`` (N,) int64 as for
    ``knn_points_packed`` (gaps allowed); ``normals`` (P,3) / ``features`` (P,D) float32 in the same rows.  ``n`` an int
    or N ints: the size of every cloud afterwards.  ``k`` in [3, 31].  The result is packed without gaps; each cloud
    keeps its input rows first, in their order, and each round's points follow in the order of their parents' indices,
    so an index never changes and ``parents`` stays valid.  Raises ValueError for a non-finite coordinate, a target
    below a cloud's size, and a cloud that has to grow with at most ``k`` or fewer than 10 points.

    Synchronises once, to read the sizes; then one library call (per round the K-NN and five kernels), the same bits on
    every call.  No gradients."""
    import numpy as np
    dev = _lib.require_cuda(points, normals, features)
    pts, fi, npts = _lib.packed_cloud(points, first_idx, num_points)
    k = _lib.check_k(k, 3, 31)
    P = pts.shape[0]
    nrm = None if normals is None else _lib.as_f32(normals.detach(), "normals")
    if nrm is not None and tuple(nrm.shape) != (P, 3):
        raise RuntimeError("normals must have shape (P, 3)")
    ftr = None if features is None else _lib.as_f32(features.detach(), "features")
    if ftr is not None and (ftr.dim() != 2 or ftr.shape[0] != P or ftr.shape[1] < 1):
        raise RuntimeError("features must have shape (P, D)")
    N = int(npts.shape[0])
    if N < 1:
        raise ValueError("no clouds")
    # the one synchronisation: every cloud's first row, size and count of non-finite rows
    bad = torch.zeros((P + 1,), dtype=torch.int64, device=dev)
    bad[1:] = torch.cumsum((~torch.isfinite(pts).all(1)).to(torch.int64), 0)
    first_h, num_h, info = _read_clouds(fi, npts, P, bad[(fi + npts).clamp(0, P)] - bad[fi.clamp(0, P)])
    if info[:, 0].any():
        raise ValueError("non-finite coordinates in cloud(s) %s" % np.flatnonzero(info[:, 0]).tolist())
    if torch.is_tensor(n):
        n = n.tolist()
    targets = [int(n)] * N if np.ndim(n) == 0 else [int(x) for x in n]
    sched = upsample_schedule(num_h, targets, k)
    rounds = len(sched) - 1
    sizes = np.asarray(sched, dtype=np.int64)
    out_num = sizes[-1]
    out_first = np.concatenate([[0], np.cumsum(out_num)[:-1]]).astype(np.int64)
    M = int(out_num.sum())
    if M >= 2 ** 31 - 1:
        raise ValueError("at most 2^31 - 2 points in all")
    knn_num = np.where(sizes[1:] > sizes[:-1], sizes[:-1], 0)
    src = np.concatenate([np.arange(f, f + c) for f, c in zip(first_h, num_h)] + [np.zeros(0, np.int64)])
    dst = np.concatenate([np.arange(f, f + c) for f, c in zip(out_first, num_h)] + [np.zeros(0, np.int64)])
    table = torch.from_numpy(np.concatenate([out_first, sizes.ravel(), knn_num.ravel(), src, dst])).to(dev)
    o = torch.split(table, [N, sizes.size, knn_num.size, src.size, dst.size])
    first_d, sizes_d, knn_d, src_d, dst_d = (t.contiguous() for t in o)
    out_pts = torch.empty((M, 3), dtype=torch.float32, device=dev)
    out_pts[dst_d] = pts[src_d]
    out_nrm = out_ftr = None
    if nrm is not None:
        out_nrm = torch.empty((M, 3), dtype=torch.float32, device=dev)
        out_nrm[dst_d] = nrm[src_d]
    if ftr is not None:
        out_ftr = torch.empty((M, ftr.shape[1]), dtype=torch.float32, device=dev)
        out_ftr[dst_d] = ftr[src_d]
    parents = torch.full((M, 2), -1, dtype=torch.int32, device=dev)
    if rounds > 0:
        _lib.call("dss_upsample_points", dev, out_pts, out_nrm, out_ftr, 0 if ftr is None else int(ftr.shape[1]),
                  first_d, sizes_d, knn_d, N, M, rounds, k, parents)
    return Upsampled(out_pts, out_nrm, out_ftr, first_d, sizes_d[rounds * N:], parents)


def _rimls_radius(diag, count, k, scale):
    """The neighbourhood radius of one cloud of the RIMLS calls, in float64: ``min(scale * avg * k, 0.2)`` with
    ``avg = sqrt(diag / count)`` (0 for an empty cloud)"""
    if count <= 0:
        return 0.0
    return min(scale * math.sqrt(diag / count) * k, 0.2)


def _rimls_setup(points, normals, k, first_idx, num_points, scale):
    """Checks and the one host synchronisation of denoise_normals / project_to_surface: (pts, nrm, first_idx,
    num_points, knn_idx (P, k + 1), radius (N,) float64) on the device"""
    import numpy as np
    from .frnn_grid import knn_points_packed
    dev = _lib.require_cuda(points, normals)
    pts, fi, npts = _lib.packed_cloud(points, first_idx, num_points)
    k = _lib.check_k(k, 3, 31)
    nrm = _lib.as_f32(normals.detach(), "normals")
    P = pts.shape[0]
    if tuple(nrm.shape) != (P, 3):
        raise RuntimeError("normals must have shape (P, 3)")
    if P >= 2 ** 31 - 1:
        raise ValueError("at most 2^31 - 2 points")
    N = int(npts.shape[0])
    if N < 1:
        raise ValueError("no clouds")
    # the cloud of every row (id + 1, 0 in the gaps), then in one read-back: every cloud's first row, size, count of
    # rows with a non-finite point or normal, and bounding box
    ids = torch.arange(1, N + 1, dtype=torch.int64, device=dev)
    mark = torch.zeros((P + 1,), dtype=torch.int64, device=dev)
    mark.index_add_(0, fi.clamp(0, P), ids)
    mark.index_add_(0, (fi + npts).clamp(0, P), -ids)
    cloud = torch.cumsum(mark[:P], 0).clamp(0, N)
    bad = ~(torch.isfinite(pts).all(1) & torch.isfinite(nrm).all(1))
    nbad = torch.zeros((N + 1,), dtype=torch.float64, device=dev).index_add_(0, cloud, bad.double())
    idx3 = cloud[:, None].expand(P, 3)
    lo = torch.full((N + 1, 3), float("inf"), device=dev).scatter_reduce(0, idx3, pts, "amin")
    hi = torch.full((N + 1, 3), -float("inf"), device=dev).scatter_reduce(0, idx3, pts, "amax")
    first_h, num_h, info = _read_clouds(fi, npts, P, nbad[1:], lo[1:], hi[1:])
    order = np.lexsort((num_h, first_h))
    if (first_h[order][1:] < (first_h + num_h)[order][:-1]).any():
        raise ValueError("the clouds' ranges overlap")
    if info[:, 0].any():
        raise ValueError("non-finite points or normals in cloud(s) %s" % np.flatnonzero(info[:, 0]).tolist())
    radius = []
    for n in range(N):
        d = info[n, 4:7] - info[n, 1:4]
        diag = math.sqrt((float(d[0]) * float(d[0]) + float(d[1]) * float(d[1])) + float(d[2]) * float(d[2])) \
            if num_h[n] > 0 else 0.0
        radius.append(_rimls_radius(diag, int(num_h[n]), k, scale))
    radius = torch.tensor(radius, dtype=torch.float64, device=dev)
    idx = knn_points_packed(pts, fi, npts, k + 1, -1.0)[1] if P > 0 else None
    return pts, nrm, fi, npts, idx, radius


def denoise_normals(points, normals, k=16, sharpness_sigma=30.0, first_idx=None, num_points=None):
    """Smooth the normals of point clouds as the reference's ``denoise_normals`` does (DSS/core/cloud.py:515-553;
    csrc/rimls.cu, the rules are in include/dss_b200.h and DESIGN.md): each row's unit normal becomes
    ``normalize(sum_j w_j n_j / sum_j w_j)`` over its ``k`` nearest other points of its cloud within ``r = min(4 avg k,
    0.2)``, ``avg = sqrt(diag / c)`` of the cloud's bounding-box diagonal and size, with ``w_j = exp(-d_j^2 c / 2)
    exp(-((1 - n_i.n_j) / sharpness_sigma)^2)``, zero beyond ``d_j^2 > 32 / c``.  A row whose weights are all zero keeps
    its own unit normal.

    ``points``, ``normals`` (P,3) float32 CUDA tensors, one cloud, or packed with ``first_idx`` / ``num_points`` (N,)
    int64 as for ``knn_points_packed`` (gaps allowed).  ``k`` in [3, 31].  Float64 throughout, rounded once to float32.
    Raises ValueError for non-finite points or normals.  Synchronises once, to read the clouds' bounding boxes; then
    the K-NN and one launch.  Returns the (P,3) float32 normals; rows outside every cloud are copied from ``normals``."""
    pts, nrm, fi, npts, idx, radius = _rimls_setup(points, normals, k, first_idx, num_points, 4.0)
    out = nrm.clone()
    if pts.shape[0] > 0:
        _lib.call("dss_denoise_normals", pts.device, pts, nrm, fi, npts, int(npts.shape[0]), pts.shape[0], idx, int(k),
                  radius, float(sharpness_sigma), out)
    return out


class Projected(NamedTuple):
    points: torch.Tensor              # (P,3) float32, the projected positions
    iterations: torch.Tensor          # (P,) int32, the outer iterations that moved each row


def project_to_surface(points, normals, k=31, max_proj_iters=10, max_est_iters=5, first_idx=None,
                       num_points=None) -> Projected:
    """Move every point onto the RIMLS surface (robust implicit moving least squares) of its cloud's samples, as the
    reference's ``project_to_latent_surface`` does (DSS/core/cloud.py:442-513; csrc/rimls.cu, the rules are in
    include/dss_b200.h and DESIGN.md), with the samples -- the input points and their unit normals -- fixed for the
    whole call.  Each row fits the surface to its ``k`` nearest other points within ``r = min(16 avg k, 0.2)``, in at
    most ``max_est_iters`` robust reweighting steps, moves along ``-f grad f``, and repeats up to ``max_proj_iters``
    times while it moved farther than 5e-4.  A row without a neighbour at a positive distance within ``r`` stays.

    ``points``, ``normals`` (P,3) float32 CUDA tensors, one cloud, or packed with ``first_idx`` / ``num_points`` (N,)
    int64 as for ``knn_points_packed`` (gaps allowed).  ``k`` in [3, 31].  Float64 throughout, rounded once to float32;
    the inputs are not modified and the normals are not updated.  Raises ValueError for non-finite points or normals.
    Synchronises once, to read the clouds' bounding boxes; then the K-NN and one launch, the same bits on every call.
    Rows outside every cloud are copied from ``points``.  No gradients."""
    for name, v in (("max_proj_iters", max_proj_iters), ("max_est_iters", max_est_iters)):
        if isinstance(v, bool) or int(v) != v or v < 0:
            raise ValueError("%s must be a non-negative integer, got %r" % (name, v))
    pts, nrm, fi, npts, idx, radius = _rimls_setup(points, normals, k, first_idx, num_points, 16.0)
    out = pts.clone()
    iterations = torch.zeros((pts.shape[0],), dtype=torch.int32, device=pts.device)
    if pts.shape[0] > 0:
        _lib.call("dss_project_to_surface", pts.device, pts, nrm, fi, npts, int(npts.shape[0]), pts.shape[0], idx,
                  int(k), radius, int(max_proj_iters), int(max_est_iters), out, iterations)
    return Projected(out, iterations)


L0_MAX_SIZE = 2048   # DSS_L0_MAX_SIZE


def _five_smooth(n):
    for p in (2, 3, 5):
        while n % p == 0:
            n //= p
    return n == 1


def l0_size_error(n):
    """None when ``n`` is an image side ``l0_smooth`` accepts (2 .. 2048, no prime factor above 5), otherwise the
    message of its ValueError, which names the nearest accepted side (the smaller one on a tie)"""
    if 2 <= n <= L0_MAX_SIZE and _five_smooth(n):
        return None
    near = min((m for m in range(2, L0_MAX_SIZE + 1) if _five_smooth(m)), key=lambda m: (abs(m - n), m))
    return ("l0_smooth takes image sides in [2, %d] with no prime factor above 5; %d is not one (nearest: %d)"
            % (L0_MAX_SIZE, n, near))


def l0_smooth(images, lmd=0.05):
    """L0 gradient-minimisation smoothing (Xu et al. 2011), as the reference's ``L0Smooth(images, lmd)`` computes it
    per image (DSS/misc/imageFilters.py:133-180; csrc/l0_smooth.cu, the rules are in include/dss_b200.h and DESIGN.md):
    20 rounds, beta = 0.1 doubling to 52428.8; each round zeroes the periodic forward differences (hp, vp) of the
    estimate where sum_c(hp^2 + vp^2) < lmd / beta and solves S = ifft2(fft2(I + beta div) / (1 + beta D)) on periodic
    boundaries.  Edges whose contrast survives the threshold stay sharp; everything between them flattens.

    ``images`` (N, H, W, C) float32 or float64 CUDA tensor, any strides, C in {1, 3}; H and W in [2, 2048] with no prime
    factor above 5 (ValueError otherwise, naming the nearest accepted size).  ``lmd`` >= 0; 0 returns the input.
    Float64 throughout on the device; returns a new contiguous tensor of the input's dtype.  One library call, no host
    synchronisation, the same bits on every call: capturable.  No gradients."""
    if not torch.is_tensor(images):
        raise TypeError("images must be a tensor")
    if images.dim() != 4:
        raise ValueError("images must have shape (N, H, W, C), got %d dimensions" % images.dim())
    N, H, W, Cn = (int(v) for v in images.shape)
    if Cn not in (1, 3):
        raise ValueError("images must have C = 1 or 3 channels, got %d" % Cn)
    if images.dtype not in (torch.float32, torch.float64):
        raise TypeError("images must be float32 or float64, got %s" % images.dtype)
    dev = _lib.require_cuda(images)
    for n in (H, W):
        msg = l0_size_error(n)
        if msg is not None:
            raise ValueError(msg)
    lmd = float(lmd)
    if not (math.isfinite(lmd) and lmd >= 0.0):
        raise ValueError("lmd must be finite and >= 0, got %r" % lmd)
    img = images.detach()
    out = torch.empty((N, H, W, Cn), dtype=img.dtype, device=dev)
    if N > 0:
        strides = (C.c_int64 * 4)(*img.stride())
        _lib.call("dss_l0_smooth", dev, img, int(img.dtype == torch.float64), strides, N, H, W, Cn, lmd, out)
    return out


class MeshRender(NamedTuple):
    image: Optional[torch.Tensor]   # (N,S,S,4) flat-shaded rgb + coverage, or None without shading
    pix_to_face: torch.Tensor       # (N,S,S) int32 face index in the mesh, -1 where no face covers the pixel
    zbuf: torch.Tensor              # (N,S,S) float32 view-space depth of that face, -1 where none


def _mesh_input(verts, faces):
    """(verts (V,3) float32, faces (F,3) int32, V, F) of a triangle mesh: faces integer, every index in [0, V), at most
    2^31 - 1 vertices and faces"""
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
    return v, faces.detach().to(torch.int32).contiguous(), V, F


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
    v, f, V, F = _mesh_input(verts, faces)
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
    _lib.call("dss_rasterize_mesh", dev, v, V, f, F, proj_c, view_c, N, S, *sh_args, pix_to_face, zbuf, image)
    return MeshRender(image, pix_to_face, zbuf)


def _chamfer_input(points, lengths, normals, name):
    """pytorch3d's _handle_pointcloud_input in the dss_knn_points layout: a cloud object gives its packed rows and its
    own normals; a padded (N,P,3) tensor is passed as packed with gaps (cloud n owns rows [n P, n P + lengths[n]))."""
    if hasattr(points, "points_packed"):
        pts, nrm = points.points_packed(), points.normals_packed()
        N = len(points)
        first, num = _lib.cloud_offsets(points.cloud_to_packed_first_idx(), points.num_points_per_cloud(), N)
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
    _lib.call("dss_chamfer", dev, xp, xn, xf, xc, xp.shape[0], yp, yn, yf, yc, yp.shape[0], N, sums)
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
    p = _lib.as_f32(points, "points")
    if p.dim() != 2 or p.shape[1] != 3:
        raise RuntimeError("points must have shape (P, 3), got %s" % (tuple(p.shape),))
    v, f, V, F = _mesh_input(verts, faces)
    P = p.shape[0]
    if P >= 2 ** 31:
        raise ValueError("at most 2^31 - 1 points, vertices and faces")
    sq = torch.empty(P, dtype=torch.float32, device=dev)
    idx = torch.empty(P, dtype=torch.int32, device=dev)
    closest = torch.empty((P, 3), dtype=torch.float32, device=dev) if return_closest else None
    _lib.call("dss_point_mesh_distance", dev, p, P, v, V, f, F, sq, idx, closest, _face_tests)
    return PointMeshDistance(sq, idx.long(), closest)


class PoissonMesh(NamedTuple):
    verts: torch.Tensor               # (V,3) float32 on the device of the input
    faces: torch.Tensor               # (F,3) int64, each face's normal pointing outwards
    grid: Optional[torch.Tensor]      # (R+1, R+1, R+1) float32 chi (negative inside), or None when not asked for
    origin: torch.Tensor              # (3,) float32 (CPU): the centre c the grid is placed around
    side: float                       # L, the grid's edge length: node (i, j, k) lies at c + (h (i, j, k) - 0.5) L
    iterations: int                   # CG iterations of the finest level
    residual: float                   # its final relative residual |r| / |b|


def marching_tetrahedra(grid, origin, side):
    """The chi = 0 surface of a node grid (csrc/poisson.cu; the rules are in include/dss_b200.h): every cube split into
    6 Kuhn tetrahedra, one vertex per crossing edge, faces oriented from chi < 0 (inside) to chi >= 0 (outside).

    grid (R+1, R+1, R+1) float32 CUDA tensor, x-major; origin the centre c (3 numbers or a tensor), side the edge L:
    node (i, j, k) lies at c + (h (i, j, k) - 0.5) L with h = 1 / R.  Returns (verts (V,3) float32, faces (F,3) int64),
    vertices ordered by (node, edge direction), faces by (cube, tetrahedron, triangle).  Synchronises the host twice:
    once to size the outputs, once in the call that fills them."""
    dev = _lib.require_cuda(grid)
    g = _lib.as_f32(grid, "grid")
    if g.dim() != 3 or g.shape[0] != g.shape[1] or g.shape[0] != g.shape[2] or g.shape[0] < 2:
        raise RuntimeError("grid must have shape (R+1, R+1, R+1) with R >= 1, got %s" % (tuple(g.shape),))
    if g.requires_grad:
        raise RuntimeError("marching_tetrahedra has no backward: pass a grid that does not require grad")
    R = g.shape[0] - 1
    c = (C.c_float * 3)(*[float(v) for v in (origin.tolist() if torch.is_tensor(origin) else origin)])
    nv, nf = C.c_int64(0), C.c_int64(0)
    verts = torch.empty((0, 3), dtype=torch.float32, device=dev)
    faces = torch.empty((0, 3), dtype=torch.int32, device=dev)
    if _lib.call("dss_marching_tetrahedra", dev, g, R, c, float(side), None, 0, None, 0, C.byref(nv), C.byref(nf),
                 capacity=True) == _lib.DSS_E_CAPACITY:
        # counts beyond int32 are not allocated: the library refuses them in the second call
        if nv.value < 2 ** 31 and nf.value < 2 ** 31:
            verts = torch.empty((nv.value, 3), dtype=torch.float32, device=dev)
            faces = torch.empty((nf.value, 3), dtype=torch.int32, device=dev)
        _lib.call("dss_marching_tetrahedra", dev, g, R, c, float(side), verts, verts.shape[0], faces, faces.shape[0],
                  C.byref(nv), C.byref(nf))
    return verts, faces.long()


def poisson_reconstruction(points, normals, depth=8, return_grid=False) -> PoissonMesh:
    """Screened Poisson surface reconstruction of an oriented cloud (csrc/poisson.cu; the discretisation is in
    include/dss_b200.h): the indicator chi on the 2^depth grid around the usable samples, then its chi = 0 surface by
    :func:`marching_tetrahedra`.  What the reference's ``Generator.generate_mesh`` gets from pymeshlab's
    ``surface_reconstruction_screened_poisson(depth=8)``, with trilinear elements instead of Kazhdan's B-splines.

    points, normals (P,3) float32 CUDA tensors; a row with a non-finite value or a zero normal is ignored, normals need
    not be unit.  depth in [2, 9].  Without a usable sample, or when they all coincide, the mesh is empty.  The result
    is the same bits for any order of the rows.  Forward only: inputs that require grad raise RuntimeError.  The host
    synchronises once every few dozen CG iterations (DESIGN.md)."""
    dev = _lib.require_cuda(points, normals)
    for name, t in (("points", points), ("normals", normals)):
        if t.requires_grad:
            raise RuntimeError("poisson_reconstruction has no backward: pass %s that does not require grad (detach it, "
                               "or call it under torch.no_grad())" % name)
    p, n = _lib.as_f32(points, "points"), _lib.as_f32(normals, "normals")
    if p.dim() != 2 or p.shape[1] != 3 or n.shape != p.shape:
        raise RuntimeError("points and normals must both have shape (P, 3), got %s and %s"
                           % (tuple(p.shape), tuple(n.shape)))
    if not 2 <= int(depth) <= 9:
        raise ValueError("depth must lie in [2, 9], got %r" % (depth,))
    depth = int(depth)
    P, R = p.shape[0], 1 << depth
    if P >= 2 ** 31:
        raise ValueError("at most 2^31 - 1 samples")
    chi = torch.empty((R + 1, R + 1, R + 1), dtype=torch.float32, device=dev)
    c, L = (C.c_float * 3)(), C.c_float(0.0)
    its, res = C.c_int(0), C.c_double(0.0)
    _lib.call("dss_poisson_solve", dev, p, n, P, depth, chi, c, C.byref(L), C.byref(its), C.byref(res), None, None)
    origin = torch.tensor(list(c), dtype=torch.float32)
    verts, faces = marching_tetrahedra(chi, origin, L.value)
    return PoissonMesh(verts, faces, chi if return_grid else None, origin, L.value, its.value, res.value)


class PoissonDiskSamples(NamedTuple):
    points: torch.Tensor              # (n,3) float32 on the device of the input, in pool order
    normals: torch.Tensor             # (n,3) float32 unit normal of each sample's face
    radius: float                     # the disk radius the count was reached at


def sample_points_poisson_disk(verts, faces, num_samples, geodesic=False, seed=0) -> PoissonDiskSamples:
    """Poisson-disk samples of a triangle mesh (csrc/mesh_sample.cu; the rule is in include/dss_b200.h): a dart throw
    over a pool of 20 x ``num_samples`` area-weighted samples drawn from ``seed``, at the radius whose count lies within
    0.5 % of ``num_samples`` (meshlab's ``generate_sampling_poisson_disk`` with ``exactnumflag``, the reference's
    evaluation ground truth).  ``geodesic`` measures meshlab's approximate geodesic distance instead of the Euclidean
    one.  The same inputs give the same bits.

    verts (V,3) float32 CUDA tensor, faces (F,3) integer with every index in [0, V) (checked here).  Faces with a
    non-finite vertex or zero area are never sampled; without a usable face the result is empty with radius 0.
    Forward only.  The host synchronises once per few selection rounds (DESIGN.md)."""
    dev = _lib.require_cuda(verts, faces)
    if verts.requires_grad:
        raise RuntimeError("sample_points_poisson_disk has no backward: pass verts that do not require grad")
    v, f, V, F = _mesh_input(verts, faces)
    N = int(num_samples)
    if N < 1 or _lib.PD_MONTECARLO_RATE * N >= 2 ** 31:
        raise ValueError("num_samples must lie in [1, %d], got %r" % ((2 ** 31 - 1) // _lib.PD_MONTECARLO_RATE,
                                                                     num_samples))
    n, r = C.c_int64(0), C.c_double(0.0)
    # room for a count within the tolerance, which is what the search nearly always returns; a call that finds more
    # (its probes all missed the tolerance) is repeated with room for exactly that many
    cap = N + N // 200
    for first in (True, False):
        points = torch.empty((cap, 3), dtype=torch.float32, device=dev)
        normals = torch.empty((cap, 3), dtype=torch.float32, device=dev)
        if _lib.call("dss_sample_mesh_poisson_disk", dev, v, V, f, F, N, int(bool(geodesic)), int(seed) & (2 ** 64 - 1),
                     points, normals, cap, C.byref(n), C.byref(r), capacity=first) != _lib.DSS_E_CAPACITY:
            break
        cap = n.value
    return PoissonDiskSamples(points[:n.value], normals[:n.value], r.value)


def poisson_disk_stats(device=None):
    """{"probes", "radii", "counts", "rounds", "stage_ms"} of the last :func:`sample_points_poisson_disk` call on the
    device: per probe its radius, sample count and selection rounds; stage_ms the pool build, the radius search, the
    final selection (0 when the returned probe was the last) and the output, in milliseconds."""
    probes = C.c_int(0)
    radii = (C.c_double * _lib.PD_MAX_PROBES)()
    counts = (C.c_int64 * _lib.PD_MAX_PROBES)()
    rounds = (C.c_int * _lib.PD_MAX_PROBES)()
    ms = (C.c_float * 4)()
    _lib.check(_lib.load().dss_poisson_disk_stats(_lib.ctx(device), C.byref(probes), radii, counts, rounds, ms),
               "dss_poisson_disk_stats")
    k = probes.value
    return {"probes": k, "radii": list(radii[:k]), "counts": list(counts[:k]), "rounds": list(rounds[:k]),
            "stage_ms": list(ms)}


class ImageMetrics(NamedTuple):
    iou: torch.Tensor                 # () float64: mean over the views of 1 - I / eps_denom(U)
    psnr: torch.Tensor                # () float64: mean over the views of the summed-channel squared error per pixel
    per_view: torch.Tensor            # (V,5) float64 rows (I, U, E, iou, psnr)


def image_metrics(pred_rgba, gt_rgb, gt_mask) -> ImageMetrics:
    """The reference's image-space validation metrics (``Trainer.eval_step``, DSS/training/trainer.py:173-212) of
    renders against their ground truth (csrc/image_metrics.cu; the rules are in include/dss_b200.h).

    ``pred_rgba`` (V,s,s,4) float32: the renders, used as they are (no clamping).  ``gt_rgb`` (V,H,W,3) float32, any
    strides (``img.permute(0, 2, 3, 1)`` of an (V,3,H,W) batch reads in place), and ``gt_mask`` (V,H,W) or (V,1,H,W)
    float32, uint8 or bool, its value used: the ground truth at the data's resolution, resized to s x s inside the
    kernel as ``F.interpolate(mode='bilinear', align_corners=False)`` does it (s == H reads it unchanged).  Per view
    ``iou`` = ``IouLoss`` = 1 - I / eps_denom(U) with I = sum m alpha, U = sum (m + alpha - m alpha) (an empty view
    scores 1), and ``psnr`` = ``L2Loss(channel_dim=1)`` = the mean over the pixels of the squared RGB error summed over
    the channels (an error, not a ratio in dB, despite the reference's name); both means are over the views, as
    ``BaseTrainer.evaluate`` takes them.  Device tensors; two launches, no host synchronisation, the same bits on every
    call.  No gradients."""
    dev = _lib.require_cuda(pred_rgba, gt_rgb, gt_mask)
    pred = _lib.as_f32(pred_rgba.detach(), "pred_rgba")
    if pred.dim() != 4 or pred.shape[3] != 4 or pred.shape[1] != pred.shape[2] or pred.shape[0] < 1:
        raise RuntimeError("pred_rgba must have shape (V, s, s, 4), V >= 1, got %s" % (tuple(pred.shape),))
    V, s = pred.shape[0], pred.shape[1]
    if gt_rgb.dtype != torch.float32:
        raise TypeError("gt_rgb must be float32, got %s" % gt_rgb.dtype)
    if gt_rgb.dim() != 4 or gt_rgb.shape[0] != V or gt_rgb.shape[3] != 3:
        raise RuntimeError("gt_rgb must have shape (%d, H, W, 3), got %s" % (V, tuple(gt_rgb.shape)))
    H, W = gt_rgb.shape[1], gt_rgb.shape[2]
    mask = gt_mask.detach()
    if mask.dim() == 4 and mask.shape[1] == 1:
        mask = mask[:, 0]
    if tuple(mask.shape) != (V, H, W):
        raise RuntimeError("gt_mask must have shape (%d, %d, %d) or (%d, 1, %d, %d), got %s"
                           % (V, H, W, V, H, W, tuple(gt_mask.shape)))
    if mask.dtype not in (torch.float32, torch.uint8, torch.bool):
        raise TypeError("gt_mask must be float32, uint8 or bool, got %s" % mask.dtype)
    mask = mask.contiguous()
    if pred.data_ptr() % 16:
        pred = pred.clone()
    per_view = torch.empty((V, 5), dtype=torch.float64, device=dev)
    means = torch.empty((2,), dtype=torch.float64, device=dev)
    gt = gt_rgb.detach()
    _lib.call("dss_image_metrics", dev, pred, s, gt, (C.c_int64 * 4)(*gt.stride()), mask,
              int(mask.dtype != torch.float32), V, H, W, per_view, means)
    return ImageMetrics(means[0], means[1], per_view)


def gather_views(store, idx, img, mask):
    """Views ``idx`` of a device-resident view store into the training step's ground truth (csrc/views.cu; the rules
    are in include/dss_b200.h).  ``store`` (V,H,W,4) contiguous, r, g, b, mask per pixel: uint8 (rgb u / 255 as
    correctly rounded float32 division, mask u != 0) or float32 (copied bit for bit).  ``idx`` (B,) int64 on the
    store's device, every value in [0, V): NOT checked here (that would read the indices back); the caller checks them
    on the host before it uploads them.  ``img`` (B,H,W,3) and ``mask`` (B,H,W) float32 contiguous outputs, written in
    place and returned.  One launch on the current stream, no allocation, no host synchronisation: capturable."""
    dev = _lib.require_cuda(store, idx, img, mask)
    if store.dtype not in (torch.uint8, torch.float32) or store.dim() != 4 or store.shape[3] != 4 \
            or not store.is_contiguous():
        raise RuntimeError("store must be a contiguous (V, H, W, 4) uint8 or float32 tensor, got %s %s"
                           % (store.dtype, tuple(store.shape)))
    V, H, W = store.shape[:3]
    if idx.dtype != torch.int64 or idx.dim() != 1:
        raise RuntimeError("idx must be an int64 tensor of shape (B,), got %s %s" % (idx.dtype, tuple(idx.shape)))
    B = idx.shape[0]
    for name, t, shape in (("img", img, (B, H, W, 3)), ("mask", mask, (B, H, W))):
        if t.dtype != torch.float32 or tuple(t.shape) != shape or not t.is_contiguous():
            raise RuntimeError("%s must be a contiguous float32 tensor of shape %s, got %s %s"
                               % (name, shape, t.dtype, tuple(t.shape)))
    if B > 65535:
        raise ValueError("gather_views takes at most 65535 views at a time, got %d" % B)
    _lib.call("dss_gather_views", dev, store, int(store.dtype == torch.float32), V, H, W, idx, B, img, mask)
    return img, mask


RIGID_TOLERANCE = 1e-4     # max |R R^T - I| and |last column - (0, 0, 0, 1)| of a camera the pose map takes


def check_rigid_cameras(view0, tol=RIGID_TOLERANCE):
    """Refuse with ValueError world-to-view matrices ``view0`` (V,4,4), row-vector convention, that the pose map cannot
    invert as rigid motions: a 3x3 block R with ``max |R R^T - I| > tol`` or ``det R <= 0``, or a last column further
    than ``tol`` from (0, 0, 0, 1).  Reads the matrices to the host: a set-up check, once per set of cameras."""
    m = torch.as_tensor(view0).detach().to("cpu", torch.float64)
    if m.dim() != 3 or tuple(m.shape[1:]) != (4, 4):
        raise ValueError("camera matrices must be (V, 4, 4), got %s" % (tuple(m.shape),))
    R = m[:, :3, :3]
    ortho = (R @ R.transpose(1, 2) - torch.eye(3, dtype=torch.float64)).abs().amax((1, 2))
    col = (m[:, :, 3] - torch.tensor([0.0, 0.0, 0.0, 1.0], dtype=torch.float64)).abs().amax(1)
    bad = (ortho > tol) | (col > tol) | (torch.linalg.det(R) <= 0) | ~torch.isfinite(m).all(2).all(1)
    if bool(bad.any()):
        v = int(bad.nonzero()[0, 0])
        raise ValueError("camera %d is not a rigid world-to-view transform within %g (max |R R^T - I| = %.3g, det R = "
                         "%.6g, last column %s): the pose refinement takes rotations and translations only"
                         % (v, tol, float(ortho[v]), float(torch.linalg.det(R[v])), m[v, :, 3].tolist()))


class _PoseCameras(torch.autograd.Function):
    @staticmethod
    def forward(ctx, poses, idx, view0, proj0):
        dev = poses.device
        V, B = poses.shape[0], idx.shape[0]
        view = torch.empty((B, 4, 4), dtype=torch.float32, device=dev)
        proj = torch.empty((B, 4, 4), dtype=torch.float32, device=dev)
        p = poses.detach()
        _lib.call("dss_pose_forward", dev, p, idx, V, B, view0, proj0, view, proj)
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(p, idx, view0, proj0)
        return view, proj

    @staticmethod
    def backward(ctx, grad_view, grad_proj):
        p, idx, view0, proj0 = ctx.saved_tensors
        g = lambda t, name: None if t is None else _lib.as_f32(t, name)
        grad = torch.empty_like(p)
        _lib.call("dss_pose_backward", p.device, p, idx, p.shape[0], idx.shape[0], view0, proj0,
                  g(grad_view, "grad_view"), g(grad_proj, "grad_proj"), grad)
        return grad, None, None, None


def pose_cameras(poses, idx, view0, proj0):
    """The refined cameras of a batch of views (csrc/poses.cu; the map is in include/dss_b200.h): ``poses`` (V,6)
    float32, one correction (rotation vector, translation) per view applied in the camera frame; ``idx`` (B,) int64 the
    batch's views (repeats allowed), every value in [0, V): NOT checked here (that would read them back; out of range
    gives NaN cameras); ``view0`` / ``proj0`` (V,4,4) float32 the views' world-to-view and full projection matrices,
    whose 3x3 view blocks must be rotations (:func:`check_rigid_cameras`, which the callers run once at set-up).
    Returns ``(view, proj)`` (B,4,4): ``view0[idx] E`` and ``view0[idx] E view0[idx]^-1 proj0[idx]``, ``view0`` /
    ``proj0`` bit for bit where a pose is zero.  Differentiable in ``poses`` only; the backward writes every row of the
    (V,6) gradient, summing repeated views in batch order, the same bits on every run.  One launch each way, no scratch,
    no host synchronisation: capturable."""
    _lib.require_cuda(poses, idx, view0, proj0)
    if poses.dtype != torch.float32 or poses.dim() != 2 or poses.shape[1] != 6 or poses.shape[0] < 1:
        raise RuntimeError("poses must be a float32 (V, 6) tensor with V >= 1, got %s %s"
                           % (poses.dtype, tuple(poses.shape)))
    V = poses.shape[0]
    if idx.dtype != torch.int64 or idx.dim() != 1:
        raise RuntimeError("idx must be an int64 tensor of shape (B,), got %s %s" % (idx.dtype, tuple(idx.shape)))
    for name, t in (("view0", view0), ("proj0", proj0)):
        if t.dtype != torch.float32 or tuple(t.shape) != (V, 4, 4):
            raise RuntimeError("%s must be a float32 tensor of shape (%d, 4, 4), got %s %s"
                               % (name, V, t.dtype, tuple(t.shape)))
    return _PoseCameras.apply(poses.contiguous(), idx.contiguous(), view0.detach().contiguous(),
                              proj0.detach().contiguous())


def shared_cloud_splats(points, n_views, Vrk_invariant=True, Vrk_isotropic=True, frnn_radius=0.2):
    """``(h, frames)`` for :func:`render_points` of ``n_views`` views of ONE shared cloud, as the training step sizes its
    splats: the spacing rule of ``SurfaceSplatting._compute_h`` (one h per view with ``Vrk_invariant``, one per point
    with ``Vrk_isotropic``) or, with both off, the cloud's anisotropic :func:`local_frames`.  Computed without grad."""
    from .core.rasterizer import point_sq_spacing, splat_variance_scale
    with torch.no_grad():
        if Vrk_invariant or Vrk_isotropic:
            h = splat_variance_scale([point_sq_spacing(points, frnn_radius)], Vrk_invariant).repeat(n_views)
            return h, None
        return None, local_frames(points)


def _data_view_renderer(points, normals, colours, data, Vrk_invariant, Vrk_isotropic, frnn_radius, shininess):
    """render(params, views, depth=False) -> the ``RenderOutput`` whose image :func:`render_data_views` returns (with
    ``depth``, its depth map too), with what does not depend on the views (the cloud's splat sizes, all the views' cameras and lights on the device) computed once"""
    from .core.camera import camera_matrices
    from .core.lighting import pack_lights
    from .core.texture import camera_centres
    from .utils.dataset import DeviceViews
    dev = _lib.require_cuda(points, normals, colours)
    # the training loop's matrices and light rows, bit for bit: all the views' projections, then the batch's
    if isinstance(data, DeviceViews):
        lights_of = None if data.light_cls is None else data.lights
        proj_all, view_all = data.proj, data.camera_mat
    else:
        lp = data.light_props(dev)
        lights_of = None if lp is None else \
            (lambda idx: lp[0](**{k: v.index_select(0, idx) for k, v in lp[1].items()}, device=dev))
        proj_all = camera_matrices(data.get_cameras())[0].to(dev)
        view_all = torch.from_numpy(data.camera_mat[:len(data)]).to(dev)
    if lights_of is None:
        raise ValueError("the data has no lights_%d entries: the views are shaded with the data's lights")
    p, c = points.detach(), colours.detach()
    n = torch.nn.functional.normalize(normals.detach(), dim=-1)
    h1, frames = shared_cloud_splats(p, 1, Vrk_invariant, Vrk_isotropic, frnn_radius)

    def render(params, views, depth=False):
        idx = torch.as_tensor(list(views), dtype=torch.int64, device=dev)
        rows, ambient, kind = pack_lights(lights_of(idx))
        view = view_all.index_select(0, idx)
        with torch.no_grad():
            shading = Shading(rows, ambient, camera_centres(view).contiguous(), kind, float(shininess))
            return render_points(p, n, c, proj_all.index_select(0, idx), view,
                                 None if h1 is None else h1.repeat(idx.shape[0]), params, shading=shading,
                                 deterministic=True, frames=frames, depth=depth)
    return render


def render_data_views(points, normals, colours, data, params: SplatParams, views, Vrk_invariant=True,
                      Vrk_isotropic=True, frnn_radius=0.2, shininess=64.0, depth=False):
    """(len(views), S, S, 4) renders, S = ``params.image_size``, of one shared cloud from the cameras of ``data``'s
    views ``views`` (an ``MVRData``: its ``get_cameras()`` projections and ``camera_mat`` view matrices, or the same
    held by a ``DeviceViews``) with fused shading by each view's own lights (``data.light_props``), as the training
    step renders a batch: unit normals, the splats of :func:`shared_cloud_splats`, ``colours`` the albedo.  Forward
    only.  With ``depth``: ``(images, depth maps (len(views), S, S))``, the depth of ``render_points(..., depth=True)``."""
    out = _data_view_renderer(points, normals, colours, data, Vrk_invariant, Vrk_isotropic, frnn_radius,
                              shininess)(params, views, depth=depth)
    return (out.image, out.depth) if depth else out.image


def evaluate_2d(points, normals, colours, data, params: SplatParams, image_size, batch=1, Vrk_invariant=True,
                Vrk_isotropic=True, frnn_radius=0.2, shininess=64.0):
    """The reference's ``Trainer.evaluate_2d`` for a point cloud: every view of ``data`` rendered at ``image_size`` x
    ``image_size`` with the splat renderer, ``batch`` views at a time (:func:`render_data_views` with ``params`` at
    that size), scored by :func:`image_metrics` against the view's ground truth.  ``data``: a ``DeviceViews`` (the
    training loop passes its own, so a validation uploads nothing) or an ``MVRData`` with images and masks, whose
    ``device_views`` this builds first.  The ground truth of each batch is gathered from the views' store
    (:func:`gather_views`).  Returns ``{"iou", "psnr"}`` (float64 device scalars, the means over all the views) and
    ``"per_view"`` (V,5) float64 rows (I, U, E, iou, psnr).  Uses no random numbers and none of a training step's
    buffers."""
    from .utils.dataset import DeviceViews
    dev = _lib.require_cuda(points, normals, colours)
    if not isinstance(data, DeviceViews):
        if data.images is None or data.masks is None:
            raise ValueError("evaluate_2d needs the data's images and masks")
        data = data.device_views(dev)
    prm = params._replace(image_size=int(image_size))
    V, B = len(data), max(1, int(batch))
    render = _data_view_renderer(points, normals, colours, data, Vrk_invariant, Vrk_isotropic, frnn_radius, shininess)
    rows = []
    for i in range(0, V, B):
        views = list(range(i, min(i + B, V)))
        image = render(prm, views).image
        rgb, mask = data.gather(data.upload(views))
        rows.append(image_metrics(image, rgb, mask).per_view)
    per_view = torch.cat(rows)
    means = per_view[:, 3:].mean(0)
    return {"iou": means[0], "psnr": means[1], "per_view": per_view}


def point_coverage(points, normals, data, params: SplatParams, batch=1, views=None, Vrk_invariant=True,
                   Vrk_isotropic=True, frnn_radius=0.2) -> Coverage:
    """The view coverage of one shared cloud over views of ``data``: :func:`accumulate_coverage` of the renders of
    ``views`` (default all of ``data``'s views), ``batch`` at a time, each against its ground-truth masks, gathered from
    the views' store (:func:`gather_views`).  The renders are :func:`render_data_views`' at ``params`` (unit normals,
    the splats of :func:`shared_cloud_splats`); a point's K-list membership in a view depends on that view alone, so the
    counts do not depend on ``batch``.  ``data``: a ``DeviceViews`` or an ``MVRData`` with images and masks, whose
    ``device_views`` this builds first.  Returns ``Coverage(seen, outside)``, (P0,) int32 counts of views."""
    from .utils.dataset import DeviceViews
    dev = _lib.require_cuda(points, normals)
    if not isinstance(data, DeviceViews):
        if data.images is None or data.masks is None:
            raise ValueError("point_coverage needs the data's images and masks")
        data = data.device_views(dev)
    views = list(range(len(data))) if views is None else list(views)
    B = max(1, int(batch))
    P0 = points.shape[0]
    cov = Coverage(torch.zeros((P0,), dtype=torch.int32, device=dev), torch.zeros((P0,), dtype=torch.int32, device=dev))
    if not views:
        return cov
    # the albedo and the shininess change the shading alone, not which points a view keeps or draws
    render = _data_view_renderer(points, normals, torch.ones_like(points), data, Vrk_invariant, Vrk_isotropic,
                                 frnn_radius, 64.0)
    for i in range(0, len(views), B):
        part = views[i:i + B]
        out = render(params, part)
        _, mask = data.gather(data.upload(part))
        accumulate_coverage(out, mask, *cov)
    return cov
