"""Data-parallel plumbing for the hot path: one process per GPU, one flat gradient bucket, one NCCL all-reduce per
optimizer step over NVLink/NVSwitch.

The reference has no distributed code at all (SURVEY.md §2.1: a single ``gpu`` argument in
holocron/trainer/core.py:52, 90-104). The path shards by batch: every rank runs the same fused kernels on its shard,
BatchNorm statistics stay per-GPU (the reference uses plain ``nn.BatchNorm2d``), and the only exchange is the mean of the
parameter gradients. A model converted with ``nn.SyncBatchNorm.convert_sync_batchnorm`` also all-reduces the statistics of
each BatchNorm step (``nn/_fused.py``, DESIGN.md §6). ``torch.distributed`` (backend ``nccl`` on GPUs, ``gloo`` in the CPU tests) is the plumbing.

Design: all ``.grad`` tensors are views into ONE contiguous fp32 bucket (allocated once, laid out in reverse
registration order = roughly the order backward produces them), so
  * backward accumulates straight into the bucket (no per-step flatten copy),
  * the all-reduce is a single collective on the bucket (size ~100 MB for RepVGG: latency-, not bandwidth-bound),
  * the fused optimizer kernels read the reduced gradients in place through the same pointers.
"""
from typing import Iterable, List, Optional

import torch
import torch.distributed as dist
from torch import Tensor, nn


class GradBucket:
    """Flat fp32 gradient storage whose slices are installed as the parameters' ``.grad``."""

    def __init__(self, params: Iterable[nn.Parameter], direct: bool = True) -> None:
        """``direct``: allow the backward kernels of this package (weight-gradient reduction, BatchNorm parameter
        gradients) to ADD their results straight into the bucket views and hand ``None`` to autograd for those
        parameters, instead of materialising a gradient tensor that AccumulateGrad adds with one more element-wise kernel
        per parameter and step (207 launches per RepVGG-A0 step). Tensor hooks registered on such parameters do not fire."""
        self.params: List[nn.Parameter] = [p for p in params if p.requires_grad]
        if not self.params:
            raise ValueError("no trainable parameters")
        dev = self.params[0].device
        # 64-element alignment keeps every view 256-byte aligned for the vectorised optimizer kernels
        offsets, total = [], 0
        for p in reversed(self.params):
            offsets.append(total)
            total += (p.numel() + 63) // 64 * 64
        self.flat = torch.zeros(total, device=dev, dtype=torch.float32)
        self.views: List[Tensor] = []
        for p, off in zip(reversed(self.params), offsets):
            chunk = self.flat[off:off + p.numel()]
            if p.ndim == 4 and p.is_contiguous(memory_format=torch.channels_last) and not p.is_contiguous():
                n, c, h, w = p.shape
                view = chunk.view(n, h, w, c).permute(0, 3, 1, 2)
            else:
                view = chunk.view(p.shape) if p.is_contiguous() else chunk.view(-1)[:p.numel()].view(p.shape)
            self.views.append(view)
            p.grad = view
            p._hb_direct_grad = bool(direct)

    def zero_(self) -> None:
        """Replaces ``optimizer.zero_grad()``: one memset, gradients stay bound to the bucket."""
        self.flat.zero_()
        for p, v in zip(reversed(self.params), self.views):
            if p.grad is not v:
                p.grad = v

    def all_reduce_mean(self, group: Optional[dist.ProcessGroup] = None, async_op: bool = False):
        """Averages the bucket across ranks (sum all-reduce on the pre-scaled bucket)."""
        if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
            return None
        self.flat.mul_(1.0 / dist.get_world_size(group))
        return dist.all_reduce(self.flat, op=dist.ReduceOp.SUM, group=group, async_op=async_op)


class OverlappedReducer:
    """Gradient all-reduce split into a few chunks that are launched on a SIDE stream while backward is still running.

    The bucket is laid out in reverse registration order, so the gradients of the layers behind a given module form a
    PREFIX of the flat buffer. A tensor hook on the output of each boundary module fires when autograd has the gradient of
    that activation, i.e. after every backward node behind it has been launched; with the bucket in ``direct`` mode their
    kernels have then already added the parameter gradients into the bucket (stream order), so the prefix up to that
    boundary is final and its all-reduce (pre-scaled by 1 / world) can start: an event links the side stream behind the
    work issued so far. :meth:`finish` reduces the remaining tail and joins the streams before the optimizer. Everything is
    stream-ordered (no host synchronisation), so the whole thing is captured into the step's CUDA graph like any other
    launch. RepVGG-A0: 80 MB of the 104 MB bucket belong to the last stage and leave while the other 24 blocks are still in
    backward; the un-overlapped tail shrinks to the first stages' ~2 MB.
    """

    def __init__(self, bucket: GradBucket, boundaries: List[nn.Module], group: Optional[dist.ProcessGroup] = None) -> None:
        self.bucket, self.group = bucket, group
        self.world = dist.get_world_size(group) if (dist.is_available() and dist.is_initialized()) else 1
        self.side = torch.cuda.Stream() if bucket.flat.is_cuda else None
        # prefix end (in elements) of the bucket once everything AFTER boundary module b has been produced
        offset_of = {}
        total = 0
        for p in reversed(bucket.params):
            offset_of[id(p)] = total
            total += (p.numel() + 63) // 64 * 64
        self.total = total
        self.ends: List[int] = []
        for mod in boundaries:
            own = [id(p) for p in mod.parameters()]
            own = [i for i in own if i in offset_of]
            if not own:
                raise ValueError("boundary module without trainable parameters")
            # parameters registered after the module's own ones sit before its LAST parameter's offset
            self.ends.append(min(offset_of[i] for i in own))
        if sorted(self.ends, reverse=True) != self.ends or len(set(self.ends)) != len(self.ends):
            raise ValueError("boundary modules must be given in forward order")
        self._done = 0                 # elements already handed to the side stream in this step
        self.enabled = True            # set False to run a backward pass without any collective (rank-local profiling)
        self._handles = []
        for k, mod in enumerate(boundaries):
            mod.register_forward_hook(self._make_forward_hook(len(boundaries) - 1 - k))
        # hook k (k = 0 for the LAST boundary) covers the prefix [ .. ends_sorted[k])
        self._ends_by_fire = list(reversed(self.ends))

    def _make_forward_hook(self, fire_index: int):
        def fwd_hook(_m, _inp, out):
            if self.world > 1 and torch.is_grad_enabled() and isinstance(out, torch.Tensor) and out.requires_grad:
                out.register_hook(lambda g, k=fire_index: self._reduce_upto(self._ends_by_fire[k]))
            return None
        return fwd_hook

    def _reduce_upto(self, end: int) -> None:
        if self.world == 1 or not self.enabled or end <= self._done:
            return None
        chunk = self.bucket.flat[self._done:end]
        if self.side is None:          # CPU tensors (gloo tests): same chunking, no streams
            chunk.mul_(1.0 / self.world)
            dist.all_reduce(chunk, op=dist.ReduceOp.SUM, group=self.group)
        else:
            ev = torch.cuda.Event()
            ev.record(torch.cuda.current_stream())
            self.side.wait_event(ev)
            with torch.cuda.stream(self.side):
                chunk.mul_(1.0 / self.world)
                dist.all_reduce(chunk, op=dist.ReduceOp.SUM, group=self.group)
        self._done = end
        return None

    def finish(self) -> None:
        """Reduces what is left (the first layers' gradients) and makes the current stream wait for every chunk."""
        if self.world == 1:
            return
        self._reduce_upto(self.total)
        if self.side is not None:
            torch.cuda.current_stream().wait_stream(self.side)
        self._done = 0

    @staticmethod
    def stage_boundaries(model: nn.Module, max_chunks: int = 4) -> List[nn.Module]:
        """Default boundaries: the top-level stages of ``model.features`` that own parameters (all but the first)."""
        feats = getattr(model, "features", None)
        if not isinstance(feats, nn.Sequential):
            return []
        stages = [m for m in feats.children() if any(p.requires_grad for p in m.parameters())]
        return stages[1:-1][-(max_chunks - 1):] if len(stages) > 2 else []


def broadcast_parameters(module: nn.Module, src: int = 0, group: Optional[dist.ProcessGroup] = None) -> None:
    """Makes every rank start from rank ``src``'s parameters and buffers (replicas are kept identical afterwards by the
    gradient all-reduce alone)."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return
    with torch.no_grad():
        for t in list(module.parameters()) + list(module.buffers()):
            dist.broadcast(t.data, src=src, group=group)


def shard_batch(global_batch: int, rank: int, world_size: int) -> range:
    """Contiguous batch shard of rank ``rank`` (remainder spread over the first ranks)."""
    base, rem = divmod(global_batch, world_size)
    start = rank * base + min(rank, rem)
    return range(start, start + base + (1 if rank < rem else 0))
