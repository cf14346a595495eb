"""LARS on the fused multi-tensor kernels — API mirror of holocron/optim/lars.py."""
import ctypes
from typing import Callable, Dict, Iterable, Optional, Tuple

import torch
from torch.optim import Optimizer

from .._lib import check, lib, ptr, stream_ptr
from ._multi_tensor import TensorTable, as_layout, bump_versions

__all__ = ["LARS"]

_cf = ctypes.c_float


class LARS(Optimizer):
    """LARS (https://arxiv.org/abs/1708.03888) with the reference's update (lars.py:91-135): SGD (momentum, dampening,
    Nesterov) whose step is scaled per tensor by ``||p|| / (||g|| + wd * ||p||)`` (1 when either norm is zero).

    Reference behaviour kept: ``scale_clip`` is stored (default ``(0.0, 10.0)``) but never applied; with weight decay the
    gradient tensor itself becomes ``g + wd * p`` (the reference adds in place); the first momentum buffer is a copy of that
    gradient; ``lr`` must be a python float. The reference compares both norms on the host (two synchronisations per
    tensor); here a group is two launches (norms, then the update) and nothing syncs."""

    def __init__(self, params: Iterable, lr: float = 1e-3, momentum: float = 0.0, dampening: float = 0.0,
                 weight_decay: float = 0.0, nesterov: bool = False, scale_clip: Optional[Tuple[float, float]] = None) -> None:
        if not isinstance(lr, float) or lr < 0.0:
            raise ValueError(f"Invalid learning rate: {lr}")
        if momentum < 0.0:
            raise ValueError(f"Invalid momentum value: {momentum}")
        if weight_decay < 0.0:
            raise ValueError(f"Invalid weight_decay value: {weight_decay}")
        defaults = {"lr": lr, "momentum": momentum, "dampening": dampening, "weight_decay": weight_decay, "nesterov": nesterov}
        if nesterov and (momentum <= 0 or dampening != 0):
            raise ValueError("Nesterov momentum requires a momentum and zero dampening")
        super().__init__(params, defaults)
        self.scale_clip = scale_clip if scale_clip is not None else (0.0, 10.0)
        self._tables = {}

    def __setstate__(self, state: Dict[str, torch.Tensor]) -> None:
        super().__setstate__(state)
        for group in self.param_groups:
            group.setdefault("nesterov", False)
        self._tables = {}

    @torch.no_grad()
    def step(self, closure: Optional[Callable[[], float]] = None) -> Optional[float]:  # type: ignore[override]
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for gi, group in enumerate(self.param_groups):
            momentum = group["momentum"]
            fresh, seasoned = [], []      # tensors whose momentum buffer is created by this step / already exists
            for p in group["params"]:
                if p.grad is None:
                    continue
                if p.grad.is_sparse:
                    raise RuntimeError(f"{self.__class__.__name__} does not support sparse gradients")
                # the kernel updates the gradient in place (weight decay): give it the parameter's layout for good
                p.grad = as_layout(p.grad, p)
                if momentum != 0 and "momentum_buffer" not in self.state[p]:
                    self.state[p]["momentum_buffer"] = torch.empty_like(p, memory_format=torch.preserve_format)
                    fresh.append(p)
                else:
                    seasoned.append(p)
            for first, plist in ((1, fresh), (0, seasoned)):
                if not plist:
                    continue
                table = self._tables.setdefault((gi, first), TensorTable())
                table.update([p.data for p in plist], [p.grad for p in plist],
                             ms=[self.state[p]["momentum_buffer"] for p in plist] if momentum != 0 else None)
                check(lib().hb_lars_step(ptr(table.metas), ptr(table.chunks), table.num_chunks, table.num_tensors,
                                         _cf(group["lr"]), _cf(momentum), _cf(group["dampening"]), _cf(group["weight_decay"]),
                                         int(bool(group["nesterov"])), first, ptr(table.scratch), stream_ptr()), "hb_lars_step")
                bump_versions(plist)
        return loss
