"""RaLars on the fused multi-tensor kernels — API mirror of holocron/optim/ralars.py."""
import ctypes
import math
from typing import Callable, Iterable, Optional, Tuple

import torch
from torch.optim import Optimizer

from .._lib import check, lib, ptr, stream_ptr
from ._multi_tensor import TensorTable, bump_versions, table_key
from .adabelief import _as_layout

__all__ = ["RaLars"]

_cf = ctypes.c_float


class RaLars(Optimizer):
    """RAdam + LARS (reference ralars.py:56-140): Adam moments; while the length of the approximated SMA exceeds 4 the
    update is the variance-rectified Adam ratio ``r_t * (m / bc1) / (sqrt(v / bc2) + eps)``, otherwise the bias-corrected
    momentum (or the unrectified ratio with ``force_adaptive_momentum``); ``+ wd * p``; then the LARS trust ratio
    ``clamp(||p||, *scale_clip) / ||update||`` (1 when either is zero) scales the step. ``state['local_lr']`` is a 0-dim
    device tensor.

    The rectification branch depends on the step count only, so it is chosen on the host; the two norms never leave the
    device (the reference compares them on the host: two synchronisations per tensor). Two launches per group."""

    def __init__(self, params: Iterable, lr: float = 1e-3, betas: Tuple[float, float] = (0.9, 0.999), eps: float = 1e-8,
                 weight_decay: float = 0.0, force_adaptive_momentum: bool = False,
                 scale_clip: Optional[Tuple[float, float]] = None) -> None:
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
        self.force_adaptive_momentum = force_adaptive_momentum
        self.scale_clip = scale_clip if scale_clip is not None else (0, 10)
        self._tables = {}

    def __setstate__(self, state) -> None:
        super().__setstate__(state)
        self._tables = {}

    @torch.no_grad()
    def step(self, closure: Optional[Callable[[], float]] = None) -> Optional[float]:  # type: ignore[override]
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for gi, group in enumerate(self.param_groups):
            beta1, beta2 = group["betas"]
            if not isinstance(group.get("sma_inf"), float):
                group["sma_inf"] = 2 / (1 - beta2) - 1
            sma_inf = group["sma_inf"]
            by_step = {}
            for p in group["params"]:
                if p.grad is None:
                    continue
                if p.grad.is_sparse:
                    raise RuntimeError(f"{self.__class__.__name__} does not support sparse gradients")
                state = self.state[p]
                if len(state) == 0:
                    state["step"] = 0
                    state["exp_avg"] = torch.zeros_like(p.data)
                    state["exp_avg_sq"] = torch.zeros_like(p.data)
                if not isinstance(state.get("local_lr"), torch.Tensor):
                    state["local_lr"] = torch.ones((), device=p.device, dtype=torch.float32)
                state["step"] += 1
                by_step.setdefault(state["step"], []).append(p)
            for step, plist in by_step.items():
                bias_correction2 = 1 - beta2 ** step
                sma_t = sma_inf - 2 * step * (1 - bias_correction2) / bias_correction2
                if sma_t > 4:
                    mode = 0
                    r_t = math.sqrt((sma_t - 4) * (sma_t - 2) * sma_inf / ((sma_inf - 4) * (sma_inf - 2) * sma_t))
                else:
                    mode, r_t = (1 if self.force_adaptive_momentum else 2), 1.0
                table = self._tables.setdefault(table_key(gi, step, by_step), TensorTable())
                st = [self.state[p] for p in plist]
                table.update([p.data for p in plist], [_as_layout(p.grad, p) for p in plist], [s["exp_avg"] for s in st],
                             [s["exp_avg_sq"] for s in st], None, [s["local_lr"] for s in st])
                check(lib().hb_ralars_step(ptr(table.metas), ptr(table.chunks), table.num_chunks, table.num_tensors,
                                           _cf(group["lr"]), _cf(beta1), _cf(beta2), _cf(group["eps"]),
                                           _cf(group["weight_decay"]), _cf(self.scale_clip[0]), _cf(self.scale_clip[1]), mode,
                                           _cf(r_t), int(step), ptr(table.scratch), stream_ptr()), "hb_ralars_step")
                bump_versions(plist)
        return loss
