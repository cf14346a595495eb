"""TAdam on the fused multi-tensor kernels — API mirror of holocron/optim/tadam.py."""
import ctypes
from typing import Callable, Iterable, List, Optional, Tuple

import torch
from torch import Tensor
from torch.optim import Optimizer

from .._lib import check, lib, ptr, stream_ptr
from ._multi_tensor import TensorTable, bump_versions, table_key
from .adabelief import _as_layout

__all__ = ["TAdam", "tadam"]

_cf = ctypes.c_float


def _launch(table: TensorTable, step: int, amsgrad: bool, beta1: float, beta2: float, lr: float, weight_decay: float,
            eps: float, dof: Optional[float]) -> None:
    check(lib().hb_tadam_step(ptr(table.metas), ptr(table.chunks), table.num_chunks, table.num_tensors, _cf(lr),
                              _cf(beta1), _cf(beta2), _cf(eps), _cf(weight_decay), int(amsgrad),
                              _cf(-1.0 if dof is None else dof), int(step), None, ptr(table.scratch), stream_ptr()),
          "hb_tadam_step")


class TAdam(Optimizer):
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

    @torch.no_grad()
    def step(self, closure: Optional[Callable[[], float]] = None) -> Optional[float]:  # type: ignore[override]
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for gi, group in enumerate(self.param_groups):
            beta1, beta2 = group["betas"]
            by_step = {}
            for p in group["params"]:
                if p.grad is None:
                    continue
                if p.grad.is_sparse:
                    raise RuntimeError(f"{self.__class__.__name__} does not support sparse gradients")
                state = self.state[p]
                if len(state) == 0:
                    state["step"] = 0
                    state["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    state["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    if group["amsgrad"]:
                        state["max_exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    state["W_t"] = beta1 / (1 - beta1) * torch.ones(1, dtype=p.data.dtype, device=p.data.device)
                state["step"] += 1
                by_step.setdefault(state["step"], []).append(p)
            for step, plist in by_step.items():
                table = self._tables.setdefault(table_key(gi, step, by_step), TensorTable())
                table.update([p.data for p in plist], [_as_layout(p.grad, p) for p in plist],
                             [self.state[p]["exp_avg"] for p in plist], [self.state[p]["exp_avg_sq"] for p in plist],
                             [self.state[p]["max_exp_avg_sq"] for p in plist] if group["amsgrad"] else None,
                             [self.state[p]["W_t"] for p in plist])
                _launch(table, step, group["amsgrad"], beta1, beta2, group["lr"], group["weight_decay"], group["eps"],
                        group["dof"])
                bump_versions(plist)
        return loss


def tadam(params: List[Tensor], grads: List[Tensor], exp_avgs: List[Tensor], exp_avg_sqs: List[Tensor],
          max_exp_avg_sqs: List[Tensor], W_ts: List[Tensor], state_steps: List[int], amsgrad: bool, beta1: float,  # noqa: N803
          beta2: float, lr: float, weight_decay: float, eps: float, dof: float) -> None:
    """Functional API (reference tadam.py:160-212)."""
    by_step = {}
    for i, s in enumerate(state_steps):
        by_step.setdefault(int(s), []).append(i)
    for step, idx in by_step.items():
        table = TensorTable()
        table.update([params[i].detach() for i in idx], [_as_layout(grads[i], params[i]) for i in idx],
                     [exp_avgs[i] for i in idx], [exp_avg_sqs[i] for i in idx],
                     [max_exp_avg_sqs[i] for i in idx] if amsgrad else None, [W_ts[i] for i in idx])
        _launch(table, step, amsgrad, beta1, beta2, lr, weight_decay, eps, dof)
        bump_versions([params[i] for i in idx])
