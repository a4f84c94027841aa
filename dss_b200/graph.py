"""CUDA-graph replay of a whole render step (forward + backward) for loops with fixed shapes.

A step is ~30 kernel launches and two ctypes calls; at the headline size the launches hide behind the GPU work, at the
smaller BASELINE clouds (100k points) they need not.  The C library never synchronises or
allocates in steady state (DESIGN.md "Host side"), so the whole step can be captured once and replayed:

    step = GraphedRenderStep(points, normals, colours, proj, view, h, params, grad_image)
    step.replay()                    # image in step.image, gradients in step.grad_points / step.grad_colours
    step.points.data.add_(...)       # update the step's OWN static leaves in place (optimizer step), replay again

With ``targets=(img, mask_img, lambda_rgb, lambda_silhouette)`` instead of ``grad_image`` the captured step is render
forward -> ``image_loss`` (dss_b200.training.losses, its fused route) -> backward of ``loss``: the step owns static copies
``step.img`` / ``step.mask_img`` that the caller updates in place between replays (the next batch), and ``step.loss``
holds the loss dict's device scalars of the last replay.

The step owns its differentiated inputs (`step.points`, `step.colours`, `step.normals`: fresh leaf copies of what was passed
in): a leaf that has already been through an eager backward on the default stream carries an AccumulateGrad node bound
to that stream, and synchronising with the legacy default stream is not capturable.

:class:`GraphedStep` is the capture and replay that this step and ``dss_b200.training.step.GraphedTrainStep`` share.
The graph holds the library's scratch buffers, which a library call outside the step reallocates when it needs more (a
larger image or cloud, say): the next ``replay()`` then captures again, so that the graph never reads freed memory.

Sizes decided on the host at capture time are frozen into the graph: the forward's tile-list capacity and the staged
window of the occupancy gather.  Both have on-device fallbacks (tiles whose list outgrew the buffer are rasterized from
the records; views whose window does not fit take the direct gather), so a replay is always CORRECT; `stale()` tells when
re-capturing would make it faster again.
"""
import contextlib
import ctypes as C

import torch

from . import _lib
from .ops import render_points
from .training.losses import fused_image_loss_targets, image_loss

__all__ = ["GraphedStep", "GraphedRenderStep"]


class GraphedStep:
    """A step captured in one CUDA graph.  A subclass defines ``_eager()``, which runs the step from leaves without
    gradients and sets the attributes named in ``_OUTPUTS``, and sets ``device``, ``_warmup`` (eager runs before a
    capture) and ``_leaves`` (the tensors whose gradients the step computes) before it calls :meth:`capture`.
    :meth:`replay` returns the first of the outputs."""
    _OUTPUTS = ()

    def settings(self):
        """every host-side value the step bakes into its launches: when it changes, the next replay captures again"""
        return ()

    def _capturing(self):
        """context around the capture, for what must not run inside one"""
        return contextlib.nullcontext()

    def capture(self):
        """warm up on a side stream (sizes the library's scratch and the caching allocator), then capture the step"""
        dev = self.device
        self.graph = None
        s = torch.cuda.Stream(device=dev)
        s.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(s):
            for _ in range(self._warmup):
                self._eager()
        torch.cuda.current_stream(dev).wait_stream(s)
        torch.cuda.synchronize(dev)
        self._capacity_at_capture = _lib.tile_total(dev)
        for t in self._leaves:
            t.grad = None
        graph = torch.cuda.CUDAGraph(keep_graph=True)    # (kept for kernel_nodes)
        with self._capturing(), torch.cuda.graph(graph):
            self._eager()
        graph.instantiate()
        # the library's scratch only grows, by reallocation: a different total means that a buffer the graph uses moved
        self.graph, self._captured, self._scratch = graph, self.settings(), _lib.scratch_bytes(dev)
        # what every replay rewrites: re-attached after each replay, so that an optimizer's zero_grad(set_to_none=True)
        # or an eager call in between does not detach them
        self._outputs = tuple(getattr(self, name) for name in self._OUTPUTS)
        self._grads = tuple(t.grad for t in self._leaves)

    def replay(self):
        if self.settings() != self._captured or _lib.scratch_bytes(self.device) != self._scratch:
            self.capture()
        self.graph.replay()
        for name, value in zip(self._OUTPUTS, self._outputs):
            setattr(self, name, value)
        for t, g in zip(self._leaves, self._grads):
            t.grad = g
        return self._outputs[0]

    def stale(self, slack=1.2) -> bool:
        """True when the tile lists have outgrown what they were at capture time by more than `slack` (the replay is
        still correct -- overflowing tiles are rasterized from the records -- but a fresh capture will be faster)."""
        now = _lib.tile_total(self.device)
        return self._capacity_at_capture > 0 and now > slack * 1.25 * self._capacity_at_capture

    def kernel_nodes(self) -> int:
        """the number of kernel launches one replay makes (kernel nodes of the captured graph)"""
        rt = C.CDLL("libcudart.so.12")
        g = C.c_void_p(self.graph.raw_cuda_graph())
        count = C.c_size_t(0)
        if rt.cudaGraphGetNodes(g, None, C.byref(count)):
            raise RuntimeError("cudaGraphGetNodes failed")
        nodes = (C.c_void_p * count.value)()
        if rt.cudaGraphGetNodes(g, nodes, C.byref(count)):
            raise RuntimeError("cudaGraphGetNodes failed")
        kinds = C.c_int(0)
        n = 0
        for node in nodes:
            if rt.cudaGraphNodeGetType(C.c_void_p(node), C.byref(kinds)):
                raise RuntimeError("cudaGraphNodeGetType failed")
            n += kinds.value == 0     # cudaGraphNodeTypeKernel
        return n


class GraphedRenderStep(GraphedStep):
    _OUTPUTS = ("image", "visible", "loss", "grad_points", "grad_colours", "grad_normals")

    def __init__(self, points, normals, colours, proj, view, h, params, grad_image=None, shading=None, warmup=3,
                 grad_sync=None, targets=None):
        if (grad_image is None) == (targets is None):
            raise ValueError("pass exactly one of grad_image and targets=(img, mask_img, lambda_rgb, lambda_silhouette)")
        if targets is not None:
            img, mask_img, lambda_rgb, lambda_sil = targets
            _lib.require_cuda(points, img, mask_img)
            # the step differentiates its own detached copies; the torch body would wait for the device, which a
            # capture cannot do
            if not fused_image_loss_targets(img.detach(), mask_img.detach()):
                raise TypeError("targets must be a float32 img and a float32, uint8 or bool mask_img (the fused image "
                                "loss); got %s and %s" % (img.dtype, mask_img.dtype))
            # static copies the caller refills in place between replays (clone keeps a permuted view's strides)
            self.img, self.mask_img = img.detach().clone(), mask_img.detach().clone()
            self._lambdas = (float(lambda_rgb), float(lambda_sil))
        self.loss = None
        dev = _lib.require_cuda(points, normals, colours, proj, view, h, grad_image)
        self.device = dev
        leaf = lambda t: t.detach().clone().requires_grad_(True)
        self.points, self.colours = leaf(points), leaf(colours)
        self.normals = leaf(normals) if shading is not None else normals.detach().clone()
        self._leaves = (self.points, self.colours, self.normals)
        # the cameras and the lights (shared or per view) are constants of the captured step (no gradients to them)
        self._args = (self.points, self.normals, self.colours, proj.detach(), view.detach(), h, params)
        self._shading = shading._replace(cam_centres=shading.cam_centres.detach(), lights=shading.lights.detach(),
                                         ambient=shading.ambient.detach()) if shading is not None else None
        if grad_sync is not None and grad_sync.world_size > 1:
            # capturing the two overlapped NCCL all-reduces (issued from two streams inside the
            # backward) deadlocks at replay -- a view-sharded step is launched eagerly
            raise NotImplementedError("GraphedRenderStep does not capture the multi-GPU gradient exchange; "
                                      "call render_points(..., grad_sync=...) eagerly")
        self._sync = grad_sync
        self.grad_image = grad_image
        self._warmup = max(1, warmup)
        self.capture()

    @contextlib.contextmanager
    def _capturing(self):
        timing = getattr(self._sync, "timing", False)
        if self._sync is not None:
            self._sync.timing = False    # no timing events inside a capture
        try:
            yield
        finally:
            if self._sync is not None:
                self._sync.timing = timing

    def _eager(self):
        for t in self._leaves:
            t.grad = None
        points, normals, colours, proj, view, h, params = self._args
        out = render_points(points, normals, colours, proj, view, h, params, shading=self._shading, grad_sync=self._sync)
        if self.grad_image is not None:
            out.image.backward(self.grad_image)
        else:
            self.loss = image_loss(out.image, self.img, self.mask_img, *self._lambdas)
            self.loss["loss"].backward()
        self.image, self.visible = out.image, out.visible
        self.grad_points, self.grad_colours, self.grad_normals = (t.grad for t in self._leaves)
