"""AdEMAMix on the fused multi-tensor kernel — API mirror of holocron/optim/ademamix.py."""
import ctypes
from typing import Iterable, List, Optional, Tuple

import torch
from torch import Tensor
from torch.optim import Optimizer

from .._lib import check, lib, ptr, stream_ptr
from ._multi_tensor import StepByCount, TensorTable, functional_step

__all__ = ["AdEMAMix", "ademamix"]

_cf = ctypes.c_float


def _launch(table: TensorTable, step: int, beta1: float, beta2: float, beta3: float, alpha: float, lr: float,
            weight_decay: float, eps: float, step_dev: Optional[Tensor] = None, ctl: Optional[Tensor] = None) -> None:
    check(lib().hb_ademamix_step(ptr(table.metas), ptr(table.chunks), table.num_chunks, _cf(lr), _cf(beta1), _cf(beta2),
                                 _cf(beta3), _cf(alpha), _cf(eps), _cf(weight_decay), int(step), ptr(step_dev), ptr(ctl),
                                 stream_ptr()), "hb_ademamix_step")


class AdEMAMix(StepByCount, Optimizer):
    """AdEMAMix (https://arxiv.org/abs/2409.03137) with the reference's update (ademamix.py:138-176): a fast,
    bias-corrected gradient EMA ``exp_avg`` (beta1), a slow uncorrected one ``exp_avg_slow`` (beta3), Adam's second moment
    ``exp_avg_sq`` (beta2): ``p -= lr * (m1 / bc1 + alpha * m2) / (sqrt(nu) / sqrt(bc2) + eps)``; L2 weight decay is folded
    into the gradient. Same constructor, validation and ``state_dict`` layout as the reference; one launch per group
    (36 B / parameter)."""

    def __init__(self, params: Iterable, lr: float = 1e-3, betas: Tuple[float, float, float] = (0.9, 0.999, 0.9999),
                 alpha: float = 5.0, eps: float = 1e-8, weight_decay: float = 0.0) -> None:
        if lr < 0.0:
            raise ValueError(f"Invalid learning rate: {lr}")
        if eps < 0.0:
            raise ValueError(f"Invalid epsilon value: {eps}")
        for idx, beta in enumerate(betas):
            if not 0.0 <= beta < 1.0:
                raise ValueError(f"Invalid beta parameter at index {idx}: {beta}")
        defaults = {"lr": lr, "betas": betas, "alpha": alpha, "eps": eps, "weight_decay": weight_decay}
        super().__init__(params, defaults)
        self._tables = {}

    def __setstate__(self, state) -> None:
        super().__setstate__(state)
        self._tables = {}

    def _init_state(self, p: Tensor, state: dict, group: dict) -> None:
        for key in ("exp_avg", "exp_avg_slow", "exp_avg_sq"):
            state[key] = torch.zeros_like(p, memory_format=torch.preserve_format)

    def _columns(self, group: dict, states: List[dict]) -> dict:
        return {"ms": "exp_avg", "vs": "exp_avg_sq", "exts": "exp_avg_slow"}

    def _launch(self, table: TensorTable, group: dict, step: int, step_dev: Optional[Tensor],
                ctl: Optional[Tensor]) -> None:
        _launch(table, step, *group["betas"], group["alpha"], group["lr"], group["weight_decay"], group["eps"], None, ctl)


def ademamix(params: List[Tensor], grads: List[Tensor], exp_avgs: List[Tensor], exp_avgs_slow: List[Tensor],
             exp_avg_sqs: List[Tensor], state_steps: List[int], beta1: float, beta2: float, beta3: float, alpha: float,
             lr: float, weight_decay: float, eps: float) -> None:
    """Functional API (reference ademamix.py:138-176): one fused launch per distinct step value."""
    functional_step(params, grads, state_steps,
                    lambda table, step: _launch(table, step, beta1, beta2, beta3, alpha, lr, weight_decay, eps),
                    ms=exp_avgs, vs=exp_avg_sqs, exts=exp_avgs_slow)
