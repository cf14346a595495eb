"""LAMB on the fused multi-tensor kernels — API mirror of holocron/optim/lamb.py."""
import ctypes
from typing import Callable, Iterable, Optional, Tuple

import torch
from torch.optim import Optimizer

from .._lib import check, lib, ptr, stream_ptr
from ._multi_tensor import TensorTable, as_layout, bump_versions, collect_step, device_local_lr

__all__ = ["LAMB"]

_cf = ctypes.c_float


class LAMB(Optimizer):
    """LAMB (https://arxiv.org/abs/1904.00962) with the reference's update (lamb.py:79-137): Adam moments WITHOUT
    bias correction, ``update = m / (sqrt(v) + eps) + wd * p`` and a LARS trust ratio
    ``clamp(||p||, *scale_clip) / ||update||`` (1 when either norm is zero).

    The reference computes both norms with ``.sum().sqrt()`` and compares them on the host (two device
    synchronisations per tensor and step); here the norms of all tensors are reduced on the device by the first
    kernel and consumed by the second, and ``state['local_lr']`` is a 0-dim device tensor (never a python ``1``).
    """

    def __init__(self, params: Iterable, lr: float = 1e-3, betas: Tuple[float, float] = (0.9, 0.999), eps: float = 1e-8,
                 weight_decay: float = 0.0, scale_clip: Optional[Tuple[float, float]] = None) -> None:
        if lr < 0.0:
            raise ValueError(f"Invalid learning rate: {lr}")
        if eps < 0.0:
            raise ValueError(f"Invalid epsilon value: {eps}")
        if not 0.0 <= betas[0] < 1.0:
            raise ValueError(f"Invalid beta parameter at index 0: {betas[0]}")
        if not 0.0 <= betas[1] < 1.0:
            raise ValueError(f"Invalid beta parameter at index 1: {betas[1]}")
        defaults = {"lr": lr, "betas": betas, "eps": eps, "weight_decay": weight_decay}
        super().__init__(params, defaults)
        self.scale_clip = scale_clip if scale_clip is not None else (0.0, 10.0)
        self._tables = {}

    @torch.no_grad()
    def step(self, closure: Optional[Callable[[], float]] = None) -> Optional[float]:  # type: ignore[override]
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for gi, group in enumerate(self.param_groups):
            plist = collect_step(self, group)
            if not plist:
                continue
            states = [self.state[p] for p in plist]
            device_local_lr(states)
            table = self._tables.setdefault(gi, TensorTable())
            table.update([p.data for p in plist], [as_layout(p.grad, p) for p in plist], ms=[s["exp_avg"] for s in states],
                         vs=[s["exp_avg_sq"] for s in states], auxs=[s["local_lr"] for s in states])
            beta1, beta2 = group["betas"]
            check(lib().hb_lamb_step(ptr(table.metas), ptr(table.chunks), table.num_chunks, table.num_tensors,
                                     _cf(group["lr"]), _cf(beta1), _cf(beta2), _cf(group["eps"]),
                                     _cf(group["weight_decay"]), _cf(self.scale_clip[0]), _cf(self.scale_clip[1]),
                                     ptr(table.scratch), stream_ptr()), "hb_lamb_step")
            bump_versions(plist)
        return loss

    def _init_state(self, p: torch.Tensor, state: dict, group: dict) -> None:
        state["exp_avg"] = torch.zeros_like(p.data, memory_format=torch.preserve_format)
        state["exp_avg_sq"] = torch.zeros_like(p.data, memory_format=torch.preserve_format)
