"""TAdam on the fused multi-tensor kernels — API mirror of holocron/optim/tadam.py."""
import ctypes
from typing import Iterable, List, Optional, Tuple

import torch
from torch import Tensor
from torch.optim import Optimizer

from .._lib import check, lib, ptr, stream_ptr
from ._multi_tensor import StepByCount, TensorTable, functional_step

__all__ = ["TAdam", "tadam"]

_cf = ctypes.c_float


def _launch(table: TensorTable, step: int, amsgrad: bool, beta1: float, beta2: float, lr: float, weight_decay: float,
            eps: float, dof: Optional[float]) -> None:
    check(lib().hb_tadam_step(ptr(table.metas), ptr(table.chunks), table.num_chunks, table.num_tensors, _cf(lr),
                              _cf(beta1), _cf(beta2), _cf(eps), _cf(weight_decay), int(amsgrad),
                              _cf(-1.0 if dof is None else dof), int(step), None, ptr(table.scratch), stream_ptr()),
          "hb_tadam_step")


class TAdam(StepByCount, Optimizer):
    """TAdam (https://arxiv.org/abs/2003.00179), the reference's update (tadam.py:160-212): Student-t weighted first
    moment ``w_t = (dof + d) / (dof + sum((g - m)^2 / (v + eps)))``, ``W_t <- W_t (2 beta1 - 1) / beta1 + w_t``.
    State: ``step`` (python int), ``exp_avg``, ``exp_avg_sq``, ``W_t`` (1-element tensor), ``max_exp_avg_sq``.
    Three launches per parameter group (reduce, update, W_t) instead of ~14 per tensor."""

    def __init__(self, params: Iterable, lr: float = 1e-3, betas: Tuple[float, float] = (0.9, 0.999), eps: float = 1e-8,
                 weight_decay: float = 0.0, amsgrad: bool = False, dof: Optional[float] = None) -> None:
        if lr < 0.0:
            raise ValueError(f"Invalid learning rate: {lr}")
        if eps < 0.0:
            raise ValueError(f"Invalid epsilon value: {eps}")
        if not 0.0 <= betas[0] < 1.0:
            raise ValueError(f"Invalid beta parameter at index 0: {betas[0]}")
        if not 0.0 <= betas[1] < 1.0:
            raise ValueError(f"Invalid beta parameter at index 1: {betas[1]}")
        if weight_decay < 0.0:
            raise ValueError(f"Invalid weight_decay value: {weight_decay}")
        defaults = {"lr": lr, "betas": betas, "eps": eps, "weight_decay": weight_decay, "amsgrad": amsgrad, "dof": dof}
        super().__init__(params, defaults)
        self._tables = {}

    def __setstate__(self, state) -> None:
        super().__setstate__(state)
        for group in self.param_groups:
            group.setdefault("amsgrad", False)
        self._tables = {}

    def _init_state(self, p: Tensor, state: dict, group: dict) -> None:
        state["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
        state["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
        if group["amsgrad"]:
            state["max_exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
        beta1 = group["betas"][0]
        state["W_t"] = beta1 / (1 - beta1) * torch.ones(1, dtype=p.data.dtype, device=p.data.device)

    def _columns(self, group: dict, states: List[dict]) -> dict:
        return {"ms": "exp_avg", "vs": "exp_avg_sq", "vmaxs": "max_exp_avg_sq" if group["amsgrad"] else None,
                "auxs": "W_t"}

    def _launch(self, table: TensorTable, group: dict, step: int, step_dev: Optional[Tensor],
                ctl: Optional[Tensor]) -> None:
        _launch(table, step, group["amsgrad"], *group["betas"], group["lr"], group["weight_decay"], group["eps"],
                group["dof"])


def tadam(params: List[Tensor], grads: List[Tensor], exp_avgs: List[Tensor], exp_avg_sqs: List[Tensor],
          max_exp_avg_sqs: List[Tensor], W_ts: List[Tensor], state_steps: List[int], amsgrad: bool, beta1: float,  # noqa: N803
          beta2: float, lr: float, weight_decay: float, eps: float, dof: float) -> None:
    """Functional API (reference tadam.py:160-212)."""
    functional_step(params, grads, state_steps,
                    lambda table, step: _launch(table, step, amsgrad, beta1, beta2, lr, weight_decay, eps, dof),
                    ms=exp_avgs, vs=exp_avg_sqs, vmaxs=max_exp_avg_sqs if amsgrad else None, auxs=W_ts)
