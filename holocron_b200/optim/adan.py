"""Adan on the fused multi-tensor kernel — API mirror of holocron/optim/adan.py."""
import ctypes
from typing import Iterable, List, Optional, Tuple

import torch
from torch import Tensor
from torch.optim import Adam

from .._lib import check, lib, ptr, stream_ptr
from ._multi_tensor import StepByCount, TensorTable, functional_step

__all__ = ["Adan", "adan"]

_cf = ctypes.c_float


def _launch(table: TensorTable, step: int, amsgrad: bool, beta1: float, beta2: float, beta3: float, lr: float,
            weight_decay: float, eps: float, step_dev: Optional[Tensor] = None, ctl: Optional[Tensor] = None) -> None:
    check(lib().hb_adan_step(ptr(table.metas), ptr(table.chunks), table.num_chunks, _cf(lr), _cf(beta1), _cf(beta2),
                             _cf(beta3), _cf(eps), _cf(weight_decay), int(amsgrad), int(step), ptr(step_dev), ptr(ctl),
                             stream_ptr()), "hb_adan_step")


class Adan(StepByCount, Adam):
    """Adan (https://arxiv.org/abs/2208.06677) with the reference's exact update (adan.py:145-199): ``exp_avg`` (EMA of the
    gradient), ``exp_avg_sq`` (EMA of the gradient DIFFERENCE), ``exp_avg_delta`` (EMA of ``(g + beta2 * diff)^2``), all
    bias-corrected; ``p -= lr * (m / bc1 + beta2 * v / bc2) / (sqrt(n) / sqrt(bc3) + eps)`` and, with weight decay, the L2
    term folded into the gradient plus ``p /= 1 + wd * lr``.

    Quirk kept: the reference allocates ``state['prev_grad']`` but never writes it, so the "difference" is taken against
    zeros unless a loaded state says otherwise; the kernel reads the tensor and leaves it untouched as well. Same
    constructor (three betas) and ``state_dict`` layout as the reference. One launch per group: 40 B / parameter instead
    of ~16 ATen kernels per tensor."""

    _step_on_device = True
    _full_aux = True

    def __init__(self, params: Iterable, lr: float = 1e-3, betas: Tuple[float, float, float] = (0.98, 0.92, 0.99),
                 eps: float = 1e-8, weight_decay: float = 0.0, amsgrad: bool = False, capturable: bool = False) -> None:
        super().__init__(params, lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=amsgrad,  # type: ignore[arg-type]
                         capturable=bool(capturable))
        self._tables = {}
        self._step_dev = {}

    def __setstate__(self, state) -> None:
        super().__setstate__(state)
        self._tables = {}
        self._step_dev = {}

    def _init_state(self, p: Tensor, state: dict, group: dict) -> None:
        for key in ("exp_avg", "exp_avg_sq", "exp_avg_delta"):
            state[key] = torch.zeros_like(p, memory_format=torch.preserve_format)
        if group["amsgrad"]:
            state["max_exp_avg_delta"] = torch.zeros_like(p, memory_format=torch.preserve_format)
        state["prev_grad"] = torch.zeros_like(p, memory_format=torch.preserve_format)

    def _columns(self, group: dict, states: List[dict]) -> dict:
        return {"ms": "exp_avg", "vs": "exp_avg_sq", "vmaxs": "max_exp_avg_delta" if group["amsgrad"] else None,
                "auxs": "prev_grad", "exts": "exp_avg_delta"}

    def _launch(self, table: TensorTable, group: dict, step: int, step_dev: Optional[Tensor],
                ctl: Optional[Tensor]) -> None:
        _launch(table, step, group["amsgrad"], *group["betas"], group["lr"], group["weight_decay"], group["eps"], step_dev,
                ctl)


def adan(params: List[Tensor], grads: List[Tensor], prev_grads: List[Tensor], exp_avgs: List[Tensor],
         exp_avg_sqs: List[Tensor], exp_avg_deltas: List[Tensor], max_exp_avg_deltas: List[Tensor], state_steps: List[int],
         amsgrad: bool, beta1: float, beta2: float, beta3: float, lr: float, weight_decay: float, eps: float) -> None:
    """Functional API (reference adan.py:145-199): one fused launch per distinct step value."""
    functional_step(params, grads, state_steps,
                    lambda table, step: _launch(table, step, amsgrad, beta1, beta2, beta3, lr, weight_decay, eps),
                    full_aux=True, ms=exp_avgs, vs=exp_avg_sqs, vmaxs=max_exp_avg_deltas if amsgrad else None,
                    auxs=prev_grads, exts=exp_avg_deltas)
