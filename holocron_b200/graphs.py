"""CUDA-graph capture of a whole training step (forward + loss + backward + gradient all-reduce + optimizer).

The reference has no counterpart (it is eager PyTorch); this is the device-side answer to the ~650 kernel launches and
the Python / autograd bookkeeping of one RepVGG step: the step is captured ONCE into a ``torch.cuda.CUDAGraph`` and
replayed, so the host cost per step is one graph launch. Requirements (all met by this package's ops):

* no host synchronisation inside the step (no ``.item()``, no data-dependent Python control flow);
* static shapes and static input buffers (``static_inputs`` are refilled with ``copy_`` before each replay);
* gradients live in persistent storage (:class:`holocron_b200.distributed.GradBucket` views) and the optimizer is
  constructed with ``capturable=True`` so that its step counter lives on the device.

Filters are re-packed to bf16 inside the captured step (the packing kernels are part of the graph), so in-place
parameter updates are always seen.
"""
from typing import Callable, Sequence

import torch
from torch import Tensor

from ._lib import lib

__all__ = ["GraphedTrainStep"]


class GraphedTrainStep:
    """``step_fn(*static_inputs) -> loss`` captured into a CUDA graph.

    Args:
        step_fn: runs one full training step on the given tensors and returns the (device) loss tensor
        example_inputs: tensors with the shapes / dtypes / device of every later call
        warmup: eager executions on a side stream before the capture (allocator, lazy initialisation, autotuning).
            At least TWO are always run: the first builds the lazily-created device tables (multi-tensor filter packing,
            optimizer tensor tables - pageable host-to-device copies, illegal during capture), the second exercises the
            steady-state path that is then captured. NOTE: warm-up executions are REAL training steps - they update the
            parameters, the optimizer state and the BatchNorm running statistics.
    """

    def __init__(self, step_fn: Callable[..., Tensor], example_inputs: Sequence[Tensor], warmup: int = 3) -> None:
        self.static_inputs = [t.clone() for t in example_inputs]
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(max(2, warmup)):
                step_fn(*self.static_inputs)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        before = lib().hb_launch_count()
        # capture on the stream of the warm-up: autograd's AccumulateGrad nodes were created there
        with torch.cuda.graph(self.graph, stream=side):
            self.static_loss = step_fn(*self.static_inputs)
        #: kernels of this library recorded in the graph (= launched by every replay)
        self.launches_per_replay = int(lib().hb_launch_count() - before)

    def __call__(self, *inputs: Tensor) -> Tensor:
        for dst, src in zip(self.static_inputs, inputs):
            if dst is not src:
                dst.copy_(src, non_blocking=True)
        self.graph.replay()
        return self.static_loss
