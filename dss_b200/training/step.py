"""The reference's training step on the fused path: ``Trainer.compute_loss`` + ``loss.backward()``
(DSS/training/trainer.py:275-331, DSS/models/point_modeling.py:135-214) for one shared cloud of P0 points and a batch of
N views, with the settings ``configs/dss.yml`` trains with:

1. ``F.normalize(normals)`` (point_modeling.py:84-86);
2. the splat size from a K-NN of the current points (rasterizer.py:293-342, ``Vrk_invariant`` / ``Vrk_isotropic``), or,
   with both off (``configs/default.yaml``), the anisotropic splats' local frames (rasterizer.py:256-291);
3. ``render_points`` with fused shading: the batch's lights, and camera centres derived from the batch's view matrices;
4. ``image_loss`` (trainer.py:332-376);
5. ``point_filters``: the visibility and inmask filters (point_modeling.py:172-173, 188-212);
6. the fused ``ProjectionLoss`` and ``RepulsionLoss`` over a rebuilt K-NN (trainer.py:305-319), each skipped when its
   lambda is 0;
7. ``loss.backward()``.

Gradients land on the step's OWN leaves (``step.points``, ``step.normals``, ``step.colours``: fresh copies of what was
passed in, the ones named in ``learn`` requiring grad); the optimizer stays with the caller, who updates those leaves in
place.  ``step.loss`` holds the trainer's loss dict as device scalars, ``step.image`` the render, ``step.visibility`` and
``step.inmask`` the (P0,) filters.

:class:`TrainStep` runs the step eagerly, on one GPU or, with a ``GradSync`` of world size G > 1, view-sharded over G
ranks: each rank holds the whole cloud and passes its own views, and every rank finishes with the loss, filters and
gradients of one step over all the views.  :class:`GraphedTrainStep` runs on one GPU.  :class:`GraphedTrainStep` captures it once in a CUDA graph: every piece is
free of host synchronisation, so one replay computes the whole step.  Between replays ``load()`` copies the next batch
into the step's static inputs.  Host-side settings are frozen into a capture; when one of them changes (``params``, e.g.
its ``radii_backward_scaler``, which the trainer's scheduler lowers, or a lambda), or when another library call has
reallocated the scratch buffers the graph uses, the next ``replay()`` captures again.
"""
import torch
import torch.distributed as dist
import torch.nn.functional as F

from .. import _lib
from ..core.cloud import PointClouds3D, PointCloudsFilters
from ..core.lighting import pack_lights
from ..core.texture import camera_centres
from ..graph import GraphedStep
from ..ops import (LOCAL_FRAME_K, Shading, SplatParams, point_filters, point_filters_no_views, pose_cameras,
                   render_points, shared_cloud_splats)
from .losses import ProjectionLoss, RepulsionLoss, depth_loss, fused_image_loss_targets, image_loss

__all__ = ["TrainStep", "GraphedTrainStep"]

_LEARNABLE = ("points", "normals", "colours")


class TrainStep:
    """One training step, eager.  ``points``, ``normals``, ``colours`` (P0,3) float32 CUDA: the world cloud and its
    albedo.  ``params``: the rasterizer settings (``SplatParams``).  The remaining settings default to the trainer's and
    ``configs/dss.yml``'s.  ``step(img, mask_img, proj, view, lights)`` runs the step on a batch and returns the loss dict:
    ``img`` (N,H,W,3) float32 ground truth (any strides), ``mask_img`` (N,H,W) or (N,1,H,W) float32, uint8 or bool,
    ``proj`` / ``view`` (N,4,4) as ``render_points`` takes them, ``lights`` a ``DirectionalLights`` / ``PointLights``
    of batch 1 or N (dss_b200.core.lighting).

    ``grad_sync``: a ``dss_b200.parallel.GradSync`` of world size G > 1 shards the step by views.  Every rank builds its
    TrainStep from the same cloud and settings and calls ``step`` with its own views (``assign_views`` deals them; a
    rank may hold none: pass tensors of batch 0, its lights are not read), in the same order as the other ranks.
    The loss is the one over all the views (image-loss sums, one all-reduce of 5 doubles), the point filters those of
    all the views (two all-reduces of P0 bytes), the render gradients arrive summed over the ranks through
    ``GradSync``, and the regularisers run replicated on every rank: each rank ends with the same ``step.loss``,
    ``step.visibility``, ``step.inmask`` and gradients on its leaves, so identical optimizer steps keep the replicas
    identical.  The ranks must agree on P0, the kind of lights, the lambdas and ``params``; that is not checked (it would
    take a host synchronisation).  With G = 1 or no ``grad_sync`` the step runs as on one GPU.

    ``Vrk_invariant`` / ``Vrk_isotropic`` select the splat shape as in the rasterizer settings: one h per view, one h
    per point, or, with both False (``configs/default.yaml``), anisotropic splats from the local frames of every point's
    8 nearest neighbours (``local_frames``, computed every step from the current points; a view-sharded step computes
    them on every rank from the same cloud, no collective).  The anisotropic kernel needs P0 > 8.

    ``poses`` (V,6) float32 with ``views`` (the ``DeviceViews`` of the data, whose cameras must be rigid): the step also
    learns one camera correction per view (``ops.pose_cameras``) on its own leaf ``step.poses``, a copy of ``poses``.
    ``step(..., idx=idx)`` then renders with the refined cameras of the batch's views ``idx`` ((B,) int64 on the
    device, the views ``proj`` / ``view`` are the unrefined cameras of), which receive the render's and the shading
    camera centres' gradients, and ``step.poses.grad`` holds the (V,6) gradient after the step.  View-sharded, every
    rank's gradient rows of its own views are summed over the ranks with one all-reduce of 6 V floats (a rank without
    views adds zeros), so every rank holds the same gradient.  At zero poses the step computes the loss, image,
    filters and cloud gradients of the step without ``poses``.

    ``lambda_dr_depth`` > 0 adds the dense depth term ``loss_dr_depth`` (``losses.depth_loss``) to the loss and to the
    loss dict: the render's depth map (``render_points(..., depth=True)``) against the batch's ``depth`` (N,S,S) float32
    view-space depth, passed as ``step(..., depth=depth)``, over the pixels inside the ground-truth mask and the render's
    alpha whose depth is finite and inside (znear, zfar) of ``params``.  Its gradient reaches the points (and the poses)
    through the render's view-depth gradient.  View-sharded, its two sums are all-reduced (2 doubles).  At 0 (the
    default) the step reads no depth and computes what it computes without the term."""

    def __init__(self, points, normals, colours, params: SplatParams, *, learn=("points", "normals"),
                 Vrk_invariant=True, Vrk_isotropic=True, frnn_radius=0.2, shininess=64.0, lambda_dr_rgb=1.0,
                 lambda_dr_silhouette=1.0, lambda_dr_proj=0.01, lambda_dr_repel=0.0, knn_k=12, filter_scale=2.0,
                 sharpness_sigma=0.75, grad_sync=None, poses=None, views=None, lambda_dr_depth=0.0):
        dev = _lib.require_cuda(points, normals, colours, poses)
        for name, t in (("points", points), ("normals", normals), ("colours", colours)):
            if t.dtype != torch.float32 or t.dim() != 2 or tuple(t.shape) != (points.shape[0], 3):
                raise RuntimeError("%s must be a float32 (P0, 3) tensor, got %s %s" % (name, t.dtype, tuple(t.shape)))
        if any(name not in _LEARNABLE for name in learn):
            raise ValueError("learn takes names out of %s, got %s" % (_LEARNABLE, tuple(learn)))
        if not (Vrk_invariant or Vrk_isotropic) and points.shape[0] <= LOCAL_FRAME_K:
            raise ValueError("the anisotropic kernel (Vrk_invariant and Vrk_isotropic off) needs more than %d points, "
                             "got %d" % (LOCAL_FRAME_K, points.shape[0]))
        self._sync = grad_sync if grad_sync is not None and grad_sync.world_size > 1 else None
        # image_loss and point_filters take None as "not sharded": GradSync's default group is named explicitly
        self._group = None if self._sync is None else (grad_sync.group if grad_sync.group is not None
                                                       else dist.group.WORLD)
        self.device = dev
        leaf = lambda t, name: t.detach().clone().requires_grad_(name in learn)
        self.points, self.normals, self.colours = leaf(points, "points"), leaf(normals, "normals"), \
            leaf(colours, "colours")
        self.params = params
        self.Vrk_invariant, self.frnn_radius, self.shininess = bool(Vrk_invariant), float(frnn_radius), float(shininess)
        self.Vrk_isotropic = bool(Vrk_isotropic)
        self.lambda_dr_rgb, self.lambda_dr_silhouette = float(lambda_dr_rgb), float(lambda_dr_silhouette)
        self.lambda_dr_proj, self.lambda_dr_repel = float(lambda_dr_proj), float(lambda_dr_repel)
        self.knn_k, self.filter_scale, self.sharpness_sigma = int(knn_k), float(filter_scale), float(sharpness_sigma)
        self.lambda_dr_depth = float(lambda_dr_depth)
        if not 0.0 <= self.lambda_dr_depth < float("inf"):
            raise ValueError("lambda_dr_depth must be a finite number >= 0, got %r" % (lambda_dr_depth,))
        # the cloud's point count as a device tensor made once: PointClouds3D would build it from a host list, a copy
        # that a capture cannot take
        self._num = torch.full((1,), points.shape[0], dtype=torch.int64, device=dev)
        self.loss = self.image = self.visibility = self.inmask = None
        self.poses = self._cameras = None
        if poses is not None:
            if views is None:
                raise ValueError("learning camera poses needs the views' cameras: pass views=DeviceViews")
            V = len(views)
            if poses.dtype != torch.float32 or tuple(poses.shape) != (V, 6):
                raise RuntimeError("poses must be a float32 (%d, 6) tensor, one row per view, got %s %s"
                                   % (V, poses.dtype, tuple(poses.shape)))
            views.check_rigid()
            self.poses = poses.detach().clone().requires_grad_(True)
            self._cameras = (views.camera_mat, views.proj)

    def settings(self):
        """every host-side value the step bakes into its launches"""
        return (tuple(self.params), self.Vrk_invariant, self.Vrk_isotropic, self.frnn_radius, self.shininess,
                self.lambda_dr_rgb, self.lambda_dr_silhouette, self.lambda_dr_proj, self.lambda_dr_repel, self.knn_k,
                self.filter_scale, self.sharpness_sigma, self.poses is not None, self.lambda_dr_depth)

    def _check_batch(self, img, mask_img, proj, view, depth=None):
        _lib.require_cuda(self.points, img, mask_img, proj, view, depth)
        if not fused_image_loss_targets(img, mask_img):
            raise TypeError("img must be float32 and mask_img float32, uint8 or bool, neither requiring grad; got %s "
                            "and %s" % (img.dtype, mask_img.dtype))
        N = proj.shape[0]
        if tuple(proj.shape) != (N, 4, 4) or tuple(view.shape) != (N, 4, 4):
            raise RuntimeError("proj and view must have shape (N, 4, 4)")
        S = int(self.params.image_size)
        if tuple(img.shape) != (N, S, S, 3):
            raise RuntimeError("img must have shape (N, S, S, 3) = %s, got %s" % ((N, S, S, 3), tuple(img.shape)))
        if self.lambda_dr_depth > 0 and (depth is None or depth.dtype != torch.float32 or tuple(depth.shape) != (N, S, S)
                                         or depth.requires_grad):
            raise RuntimeError("a step with lambda_dr_depth > 0 takes the batch's depth maps: depth, a float32 tensor "
                               "of shape %s not requiring grad, got %s" % ((N, S, S), None if depth is None else
                                                                           "%s %s" % (depth.dtype, tuple(depth.shape))))

    def __call__(self, img, mask_img, proj, view, lights, idx=None, depth=None):
        self._check_batch(img, mask_img, proj, view, depth)
        if self.poses is not None:
            if idx is None or idx.dtype != torch.int64 or tuple(idx.shape) != (proj.shape[0],) \
                    or idx.device != self.device:
                raise RuntimeError("a step that learns poses takes the batch's views: idx, an int64 tensor of shape "
                                   "(%d,) on %s" % (proj.shape[0], self.device))
        if self._sync is not None and proj.shape[0] == 0:
            return self._run(img, mask_img, proj, view, None, None, None, idx, depth)
        rows, ambient, kind = pack_lights(lights)
        return self._run(img, mask_img, proj, view, rows.detach(), ambient.detach(), kind, idx, depth)

    def _run(self, img, mask_img, proj, view, rows, ambient, light_type, idx=None, depth_gt=None):
        for t in (self.points, self.normals, self.colours, self.poses):
            if t is not None:
                t.grad = None
        N, dev = proj.shape[0], self.device
        if self.poses is not None and N > 0:
            view, proj = pose_cameras(self.poses, idx, *self._cameras)
        normals = F.normalize(self.normals, dim=-1)
        want_depth = self.lambda_dr_depth > 0
        if N == 0:
            # a rank of a view-sharded step without views: the collectives of the others, with zero contributions
            S = int(self.params.image_size)
            image = torch.zeros((0, S, S, 4), dtype=torch.float32, device=dev)
            # (in the order of the branch below: collectives pair up by their order on the group)
            loss = image_loss(image, img, mask_img, self.lambda_dr_rgb, self.lambda_dr_silhouette, group=self._group)
            if want_depth:
                loss_depth = depth_loss(image[..., 0], image, depth_gt, mask_img, self.lambda_dr_depth,
                                        self.params.znear, self.params.zfar, group=self._group)
            visibility, inmask = point_filters_no_views(self.points.shape[0], dev, self._group)
            rendered = _NoViews.apply(self.points, normals, self.colours, self._sync)
        else:
            h, frames = shared_cloud_splats(self.points, N, self.Vrk_invariant, self.Vrk_isotropic, self.frnn_radius)
            shading = Shading(rows, ambient, camera_centres(view).contiguous(), light_type, self.shininess)
            out = render_points(self.points, normals, self.colours, proj, view, h, self.params, shading=shading,
                                deterministic=True,
                                grad_sync=self._sync, frames=frames, depth=want_depth)
            loss = image_loss(out.image, img, mask_img, self.lambda_dr_rgb, self.lambda_dr_silhouette,
                              group=self._group)
            if want_depth:
                loss_depth = depth_loss(out.depth, out.image, depth_gt, mask_img, self.lambda_dr_depth,
                                        self.params.znear, self.params.zfar, group=self._group)
            visibility, inmask = point_filters(out, mask_img, group=self._group)
            image, rendered = out.image, None
        cloud = PointClouds3D([self.points], [normals])
        cloud._cache["num"] = self._num
        points_filter = PointCloudsFilters(dev, visibility=visibility[None], inmask=inmask[None])
        zero = torch.zeros((), dtype=torch.float32, device=dev)
        reg = {}
        for key, lam, cls in (("loss_dr_proj", self.lambda_dr_proj, ProjectionLoss),
                              ("loss_dr_repel", self.lambda_dr_repel, RepulsionLoss)):
            reg[key] = zero
            if lam > 0:
                fn = cls(reduction="mean", knn_k=self.knn_k, filter_scale=self.filter_scale,
                         sharpness_sigma=self.sharpness_sigma)
                reg[key] = fn(cloud, rebuild_knn=True, points_filter=points_filter) * lam
        # trainer.py:313: loss = proj + repel + the image loss
        total = reg["loss_dr_proj"] + reg["loss_dr_repel"] + loss["loss"]
        if want_depth:
            total = total + loss_depth
        if rendered is not None:
            total = total + rendered
        total.backward()
        if self.poses is not None:
            if self.poses.grad is None:       # a rank without views
                self.poses.grad = torch.zeros_like(self.poses)
            if self._sync is not None:
                dist.all_reduce(self.poses.grad, op=dist.ReduceOp.SUM, group=self._group)
        self.loss = {"loss": total.detach(), "loss_dr_rgb": loss["loss_dr_rgb"].detach(),
                     "loss_dr_silhouette": loss["loss_dr_silhouette"].detach(),
                     "loss_dr_proj": reg["loss_dr_proj"].detach(), "loss_dr_repel": reg["loss_dr_repel"].detach()}
        if want_depth:
            self.loss["loss_dr_depth"] = loss_depth.detach()
        self.image, self.visibility, self.inmask = image.detach(), visibility, inmask
        return self.loss


class _NoViews(torch.autograd.Function):
    """The render of a view-sharded step's rank that holds no views: 0 forward; backward, the all-reduces that
    render_points' backward makes through GradSync (d albedo and d normal on its side stream, then d position), with
    zero contributions, so that this rank receives the other ranks' render gradients."""

    @staticmethod
    def forward(ctx, points, normals, albedo, sync):
        ctx.sync, ctx.P0 = sync, points.shape[0]
        return points.new_zeros(())

    @staticmethod
    def backward(ctx, grad):
        sync, dev = ctx.sync, grad.device
        g_points, g_normals, g_albedo = (torch.zeros((ctx.P0, 3), dtype=torch.float32, device=dev) for _ in range(3))
        main, side = torch.cuda.current_stream(dev), sync.side_stream(dev)
        side.wait_stream(main)
        with torch.cuda.stream(side):
            sync.reduce_early(g_albedo, g_normals)
        sync.reduce_late(g_points)
        sync.join(dev)
        return g_points, g_normals, g_albedo, None


class GraphedTrainStep(TrainStep, GraphedStep):
    """:class:`TrainStep` captured in a CUDA graph.  The step owns static copies of the first batch
    (``step.img``, ``step.mask_img``, ``step.proj``, ``step.view`` and the packed light rows); ``load(img, mask_img,
    proj, view, lights)`` copies the next batch into them in place (same shapes, same kind of lights) and ``replay()``
    runs the step on them::

        step = GraphedTrainStep(points, normals, colours, params, img, mask_img, proj, view, lights)
        for batch in loader:
            step.load(*batch)
            step.replay()            # step.loss, step.image, step.visibility, step.inmask; gradients on the leaves
            optimizer.step()         # over step.points, step.normals: updated in place

    ``replay()`` captures again, first, when :meth:`settings` differ from those of the capture (``step.params =
    step.params._replace(radii_backward_scaler=...)``, ``step.lambda_dr_proj = ...``).  As for ``GraphedRenderStep``,
    the forward's tile-list capacity is frozen into the capture: replays stay correct when the lists outgrow it, and
    :meth:`stale` tells when a new capture (:meth:`capture`) would be faster.  The capture holds the library's scratch
    buffers; when a library call outside the step has reallocated them (the library's scratch total changed), the next
    ``replay()`` captures again too.

    :meth:`from_views` builds the step on views resident on the device instead: the capture gathers each batch itself,
    and ``load_views(idx)`` takes the place of ``load``.  Only such a step learns camera poses (``poses=``): the capture
    runs the pose map on the gathered index, and ``step.poses`` is one more leaf."""
    _OUTPUTS = ("loss", "image", "visibility", "inmask")

    def __init__(self, points, normals, colours, params: SplatParams, img, mask_img, proj, view, lights, warmup=3,
                 _views=None, depth=None, **settings):
        sync = settings.get("grad_sync")
        if sync is not None and sync.world_size > 1:
            raise NotImplementedError("GraphedTrainStep runs on one GPU; a view-sharded step runs eagerly: "
                                      "TrainStep(..., grad_sync=...)")
        if settings.get("poses") is not None and _views is None:
            raise ValueError("a graphed step learns camera poses on device views: GraphedTrainStep.from_views(..., "
                             "poses=...)")
        super().__init__(points, normals, colours, params, views=None if _views is None else _views[0], **settings)
        self._check_batch(img, mask_img, proj, view, depth)
        rows, ambient, self._light_type = pack_lights(lights)
        # static inputs (clone keeps a permuted view's strides)
        self.img, self.mask_img = img.detach().clone(), mask_img.detach().clone()
        self.proj, self.view = proj.detach().float().contiguous().clone(), view.detach().float().contiguous().clone()
        self.lights, self.ambient = rows.detach().clone(), ambient.detach().clone()
        self.depth = depth.detach().clone() if self.lambda_dr_depth > 0 else None
        # from_views: the device views and the static (B,) index the capture gathers the batch with
        self._views, self._index = _views if _views is not None else (None, None)
        self._warmup = max(1, int(warmup))
        self._leaves = (self.points, self.normals, self.colours) + ((self.poses,) if self.poses is not None else ())
        self.capture()

    @classmethod
    def from_views(cls, points, normals, colours, params: SplatParams, views, idx, warmup=3, **settings):
        """The step on views resident on the device (``views``: a ``DeviceViews``), first on views ``idx`` (a host
        list).  The capture begins with the batch: the gather of the images and masks into ``step.img`` /
        ``step.mask_img`` and the selection of ``step.proj``, ``step.view`` and the light rows, all from one static
        (B,) device index; ``load_views(idx)`` sets that index and ``replay()`` runs the whole iteration::

            step = GraphedTrainStep.from_views(points, normals, colours, params, views, order[:B])
            for idx in batches:
                step.load_views(idx)
                step.replay()
                optimizer.step()

        The batch is the one ``load(*views.batch(idx))`` would copy in, bit for bit.  ``load()`` refuses such a step:
        the capture's gather would overwrite what it copied."""
        if views.light_cls is None:
            raise ValueError("the training step shades every view with its lights, and the views have none")
        index = views.upload(idx)
        depth = None
        if float(settings.get("lambda_dr_depth", 0.0)) > 0:
            if views.depth is None:
                raise ValueError("lambda_dr_depth > 0 needs the views' depth maps (MVRData(..., load_dense_depth=True))")
            depth = views.depth_at(index)
        return cls(points, normals, colours, params, *views.batch_at(index), warmup=warmup, _views=(views, index),
                   depth=depth, **settings)

    def _gather(self):
        """the batch of the static index into the static inputs: the start of a from_views capture"""
        views, index = self._views, self._index
        views.gather(index, self.img, self.mask_img)
        torch.index_select(views.proj, 0, index, out=self.proj)
        torch.index_select(views.camera_mat, 0, index, out=self.view)
        if self.depth is not None:
            torch.index_select(views.depth, 0, index, out=self.depth)
        # pack_lights on the batch's light properties, as the step packs the lights it is handed: the ambient colour is
        # summed over the lights per batch, in the order torch's reduction takes for the batch's shape
        rows, ambient, _ = pack_lights(views.lights(index))
        self.lights.copy_(rows)
        self.ambient.copy_(ambient)

    def _eager(self):
        if self._views is not None:
            self._gather()
        return self._run(self.img, self.mask_img, self.proj, self.view, self.lights, self.ambient, self._light_type,
                         self._index, self.depth)

    def load_views(self, idx):
        """the next batch of a :meth:`from_views` step: the host list ``idx`` (as many views as the capture's, checked
        by ``DeviceViews.check`` before anything is copied) into the static index, without blocking, from a fresh
        pinned tensor"""
        if self._views is None:
            raise RuntimeError("load_views() needs a step made by GraphedTrainStep.from_views; use load()")
        idx = self._views.check(idx)
        if len(idx) != self._index.shape[0]:
            raise ValueError("load_views() takes the capture's %d views, got %d" % (self._index.shape[0], len(idx)))
        self._index.copy_(torch.tensor(idx, dtype=torch.int64).pin_memory(), non_blocking=True)

    def load(self, img, mask_img, proj, view, lights, depth=None):
        """copy the next batch into the static inputs (no synchronisation); ``depth`` with ``lambda_dr_depth`` > 0"""
        if self._views is not None:
            raise RuntimeError("this step gathers its batch from device views inside the capture, which would "
                               "overwrite a loaded batch: use load_views(idx)")
        self._check_batch(img, mask_img, proj, view, depth)
        rows, ambient, kind = pack_lights(lights)
        if kind != self._light_type or rows.shape != self.lights.shape or ambient.shape != self.ambient.shape:
            raise ValueError("the lights must keep the kind and shape of the capture: %s %s, got %s %s"
                             % (self._light_type, tuple(self.lights.shape), kind, tuple(rows.shape)))
        pairs = ((self.img, img), (self.mask_img, mask_img), (self.proj, proj), (self.view, view),
                 (self.lights, rows), (self.ambient, ambient)) + (((self.depth, depth),) if self.depth is not None else ())
        for dst, src in pairs:
            if dst.shape != src.shape or dst.dtype != src.dtype:
                raise ValueError("load() takes a batch of the capture's shapes and dtypes: %s %s, got %s %s"
                                 % (tuple(dst.shape), dst.dtype, tuple(src.shape), src.dtype))
            dst.copy_(src.detach())
