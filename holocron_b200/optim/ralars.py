"""RaLars on the fused multi-tensor kernels — API mirror of holocron/optim/ralars.py."""
import ctypes
import math
from typing import Iterable, List, Optional, Tuple

import torch
from torch import Tensor
from torch.optim import Optimizer

from .._lib import check, lib, ptr, stream_ptr
from ._multi_tensor import StepByCount, TensorTable, device_local_lr

__all__ = ["RaLars"]

_cf = ctypes.c_float


class RaLars(StepByCount, Optimizer):
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

    def _init_state(self, p: Tensor, state: dict, group: dict) -> None:
        state["exp_avg"] = torch.zeros_like(p.data)
        state["exp_avg_sq"] = torch.zeros_like(p.data)

    def _columns(self, group: dict, states: List[dict]) -> dict:
        device_local_lr(states)
        return {"ms": "exp_avg", "vs": "exp_avg_sq", "auxs": "local_lr"}

    def _launch(self, table: TensorTable, group: dict, step: int, step_dev: Optional[Tensor],
                ctl: Optional[Tensor]) -> None:
        beta1, beta2 = group["betas"]
        if not isinstance(group.get("sma_inf"), float):
            group["sma_inf"] = 2 / (1 - beta2) - 1
        sma_inf = group["sma_inf"]
        bias_correction2 = 1 - beta2 ** step
        sma_t = sma_inf - 2 * step * (1 - bias_correction2) / bias_correction2
        if sma_t > 4:
            mode = 0
            r_t = math.sqrt((sma_t - 4) * (sma_t - 2) * sma_inf / ((sma_inf - 4) * (sma_inf - 2) * sma_t))
        else:
            mode, r_t = (1 if self.force_adaptive_momentum else 2), 1.0
        check(lib().hb_ralars_step(ptr(table.metas), ptr(table.chunks), table.num_chunks, table.num_tensors,
                                   _cf(group["lr"]), _cf(beta1), _cf(beta2), _cf(group["eps"]), _cf(group["weight_decay"]),
                                   _cf(self.scale_clip[0]), _cf(self.scale_clip[1]), mode, _cf(r_t), int(step),
                                   ptr(table.scratch), stream_ptr()), "hb_ralars_step")
