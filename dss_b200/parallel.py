"""View-sharded data parallelism for the splatting path (SURVEY.md section 8e).

Views are independent units: the views of a step are dealt to the G ranks (one process per GPU), every rank holds the
full cloud, renders and back-propagates its own views, and the per-point gradients (d position | d normal | d colour)
are summed over the ranks so that identical optimizer steps need no parameter broadcast.  No other collective is on
the path, and none is needed inside the kernels.

The exchange is OVERLAPPED with the backward pass instead of trailing it (one all-reduce of a
``torch.cat`` copy behind the last kernel would add its whole time to the step).  The colour-side gradients are final as
soon as the colour scatter has run, long before the occupancy path finishes, so :class:`GradSync` reduces them on a
side stream while the occupancy gather (the longest kernel of the backward) is still running; only the position
gradients, final after the last kernel, are reduced behind it.  No staging copy: both collectives run in place on
the tensors the backward returns.

Works with any torch.distributed backend ("nccl" over NVLink between GPUs, "gloo" in the CPU tests).
"""
from typing import List, Optional, Sequence, Tuple

import torch
import torch.distributed as dist

__all__ = ["shard_views", "assign_views", "view_costs_from_cameras", "GradSync", "pack_point_grads",
           "unpack_point_grads", "allreduce_point_grads", "allreduce_visibility", "replicas_differ", "check_replicas",
           "agree_any"]


def shard_views(n_views: int, world_size: int, rank: int) -> Tuple[int, int]:
    """Contiguous [start, stop) slice of the view batch owned by ``rank`` (sizes differ by at most one)."""
    if world_size <= 0 or not (0 <= rank < world_size):
        raise ValueError("bad world_size/rank")
    base, extra = divmod(n_views, world_size)
    start = rank * base + min(rank, extra)
    return start, start + base + (1 if rank < extra else 0)


def assign_views(costs: Sequence[float], world_size: int) -> List[List[int]]:
    """Deal views to ranks so that every rank gets the same NUMBER of views (+-1) and about the same COST.

    Views differ up to 3x in cost (a close camera covers more pixels and has a wider backward window) and the slowest
    rank sets the step time.  Views are sorted by decreasing cost and dealt in snake order (0..G-1, G-1..0, ...): equal
    counts by construction, and the cost sums differ by at most one view's cost.  ``costs`` can be any estimate -- the
    previous step's per-view visible-point count times its search radius squared, or :func:`view_costs_from_cameras`.
    Returns ``world_size`` lists of view indices (each sorted ascending)."""
    if world_size <= 0:
        raise ValueError("bad world_size")
    order = sorted(range(len(costs)), key=lambda i: (-float(costs[i]), i))
    out: List[List[int]] = [[] for _ in range(world_size)]
    for k, v in enumerate(order):
        r = k % world_size
        if (k // world_size) % 2 == 1:
            r = world_size - 1 - r
        out[r].append(v)
    return [sorted(x) for x in out]


def view_costs_from_cameras(view_matrices: torch.Tensor) -> torch.Tensor:
    """Cheap cost estimate from the world-to-view matrices (N,4,4; row-vector convention): the projected area of the
    object, hence the number of covered tiles and the area of the backward window, falls with the squared camera
    distance."""
    t = view_matrices[:, 3, :3].double()
    return 1.0 / (t * t).sum(-1).clamp_min(1e-12)


class GradSync:
    """Sums the per-point gradients over the ranks, overlapped with the backward pass.

    Pass an instance as ``grad_sync=`` to :func:`dss_b200.ops.render_points`.  The backward then
      1. runs the colour scatter on this object's side stream and calls :meth:`reduce_early` on the colour-side
         gradients there (the collective starts while the occupancy path runs on the main stream),
      2. runs the occupancy path and the chain kernel on the main stream and calls :meth:`reduce_late` on the position
         gradients,
      3. makes the main stream wait for the side stream (:meth:`join`).
    With world size 1 (or torch.distributed not initialised) every method is a no-op apart from the stream handling, so
    the same training step runs on one GPU.  ``timing=True`` records CUDA events around both collectives; read them
    with :meth:`timings_ms` (synchronises)."""

    def __init__(self, group=None, timing: bool = False):
        self.group = group
        self.timing = timing
        self._side = {}
        self._events = []
        self.bytes_reduced = 0
        self.calls = 0

    # -- plumbing --------------------------------------------------------------------------------
    @property
    def world_size(self) -> int:
        if not (dist.is_available() and dist.is_initialized()):
            return 1
        return dist.get_world_size(self.group)

    def side_stream(self, device) -> "torch.cuda.Stream":
        key = torch.device(device).index
        if key not in self._side:
            self._side[key] = torch.cuda.Stream(device=device)
        return self._side[key]

    def _reduce(self, tensors: Sequence[Optional[torch.Tensor]]):
        tensors = [t for t in tensors if t is not None]
        if not tensors or self.world_size == 1:
            return
        ev = None
        if self.timing and tensors[0].is_cuda:
            ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
            ev[0].record()
        for t in tensors:
            dist.all_reduce(t, op=dist.ReduceOp.SUM, group=self.group)
            self.bytes_reduced += t.numel() * t.element_size()
        if ev is not None:
            ev[1].record()
            self._events.append(ev)

    # -- called by the backward ------------------------------------------------------------------
    def reduce_early(self, *tensors):
        """colour-side gradients (d colour, d normal): issued on the CURRENT stream, which is the side stream."""
        self._reduce(tensors)

    def reduce_late(self, *tensors):
        """position gradients: issued on the current (main) stream behind the chain kernel."""
        self._reduce(tensors)
        self.calls += 1

    def join(self, device):
        torch.cuda.current_stream(device).wait_stream(self.side_stream(device))

    # -- reporting -------------------------------------------------------------------------------
    def timings_ms(self) -> float:
        """Total device time of the recorded collectives (both streams; they overlap with compute)."""
        total = 0.0
        for a, b in self._events:
            b.synchronize()
            total += a.elapsed_time(b)
        self._events = []
        return total

    def reset_counters(self):
        self._events = []
        self.bytes_reduced = 0
        self.calls = 0


def pack_point_grads(grad_points: Optional[torch.Tensor], grad_normals: Optional[torch.Tensor],
                     grad_colours: Optional[torch.Tensor], P0: int, device=None) -> torch.Tensor:
    """(P0, 9) fp32 buffer [d pos | d normal | d colour]; missing parts are zero.  (For callers that want ONE collective
    behind the backward; :class:`GradSync` needs no packing.)"""
    ref = next(t for t in (grad_points, grad_normals, grad_colours) if t is not None)
    buf = torch.zeros((P0, 9), dtype=torch.float32, device=device if device is not None else ref.device)
    for i, t in enumerate((grad_points, grad_normals, grad_colours)):
        if t is not None:
            buf[:, 3 * i: 3 * i + 3] = t
    return buf


def unpack_point_grads(buf: torch.Tensor):
    return buf[:, 0:3], buf[:, 3:6], buf[:, 6:9]


def allreduce_point_grads(buf: torch.Tensor, group=None, async_op: bool = False):
    """Sum the packed gradient buffer over all ranks, in place.  Returns the work handle when async."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return None
    return dist.all_reduce(buf, op=dist.ReduceOp.SUM, group=group, async_op=async_op)


def allreduce_visibility(visible: torch.Tensor, group=None):
    """any-over-views visibility (point_modeling.py:172-173) across ranks: one tiny all-reduce(max)."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return visible
    v = visible.to(torch.uint8)
    dist.all_reduce(v, op=dist.ReduceOp.MAX, group=group)
    return v.to(visible.dtype)


def replicas_differ(tensors: Sequence[torch.Tensor], group=None) -> bool:
    """True when the ranks' ``tensors`` (float32, any shapes, the same on every rank) are not the same bits on every
    rank; every rank gets the same answer.  The float32 bit patterns, viewed as int32, and their complements go through
    ONE all-reduce(MAX): max(~x) = ~min(x), so an element differs somewhere exactly when its max and min differ.  Bits,
    not values: a 1-ulp difference, +0.0 against -0.0 and NaNs of other payloads all count.  Ends in a host
    synchronisation (the answer is a Python bool); False without a group of more than one rank."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return False
    bits = torch.cat([t.detach().reshape(-1).view(torch.int32) for t in tensors])
    both = torch.cat([bits, ~bits])
    dist.all_reduce(both, op=dist.ReduceOp.MAX, group=group)
    n = bits.numel()
    return bool((both[:n] != ~both[n:]).any())


def check_replicas(named: Sequence[Tuple[str, torch.Tensor]], group=None):
    """Raise RuntimeError on every rank when :func:`replicas_differ` finds the ``(name, tensor)`` pairs differ between
    the ranks: replicas of a data-parallel model that drifted apart would otherwise train on silently."""
    if replicas_differ([t for _, t in named], group):
        raise RuntimeError("the ranks' replicas differ: %s are not the same bits on every rank"
                           % ", ".join(name for name, _ in named))


def agree_any(flag: bool, group=None) -> bool:
    """True on every rank when ``flag`` is true on any rank: one all-reduce(MAX) of a host int32 over ``group``, which
    must take CPU tensors (gloo).  It waits for the other ranks but adds no device synchronisation."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return bool(flag)
    t = torch.tensor([1 if flag else 0], dtype=torch.int32)
    dist.all_reduce(t, op=dist.ReduceOp.MAX, group=group)
    return bool(t.item())
