"""Adan on the fused multi-tensor kernel — API mirror of holocron/optim/adan.py."""
import ctypes
from typing import Callable, Iterable, List, Optional, Tuple

import torch
from torch import Tensor
from torch.optim import Adam

from .._lib import check, lib, ptr, stream_ptr
from ._multi_tensor import TensorTable, bump_versions, table_key
from .adabelief import _as_layout

__all__ = ["Adan", "adan"]

_cf = ctypes.c_float


def _launch(table: TensorTable, step: int, amsgrad: bool, beta1: float, beta2: float, beta3: float, lr: float,
            weight_decay: float, eps: float, step_dev: Optional[Tensor] = None, ctl: Optional[Tensor] = None) -> None:
    check(lib().hb_adan_step(ptr(table.metas), ptr(table.chunks), table.num_chunks, _cf(lr), _cf(beta1), _cf(beta2),
                             _cf(beta3), _cf(eps), _cf(weight_decay), int(amsgrad), int(step), ptr(step_dev), ptr(ctl),
                             stream_ptr()), "hb_adan_step")


class Adan(Adam):
    """Adan (https://arxiv.org/abs/2208.06677) with the reference's exact update (adan.py:145-199): ``exp_avg`` (EMA of the
    gradient), ``exp_avg_sq`` (EMA of the gradient DIFFERENCE), ``exp_avg_delta`` (EMA of ``(g + beta2 * diff)^2``), all
    bias-corrected; ``p -= lr * (m / bc1 + beta2 * v / bc2) / (sqrt(n) / sqrt(bc3) + eps)`` and, with weight decay, the L2
    term folded into the gradient plus ``p /= 1 + wd * lr``.

    Quirk kept: the reference allocates ``state['prev_grad']`` but never writes it, so the "difference" is taken against
    zeros unless a loaded state says otherwise; the kernel reads the tensor and leaves it untouched as well. Same
    constructor (three betas) and ``state_dict`` layout as the reference. One launch per group: 40 B / parameter instead
    of ~16 ATen kernels per tensor."""

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

    @torch.no_grad()
    def step(self, closure: Optional[Callable[[], float]] = None) -> Optional[float]:  # type: ignore[override]
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        ctl = getattr(self, "_hb_ctl", None)
        for gi, group in enumerate(self.param_groups):
            by_step = {}
            for p in group["params"]:
                if p.grad is None:
                    continue
                if p.grad.is_sparse:
                    raise RuntimeError(f"{self.__class__.__name__} does not support sparse gradients")
                state = self.state[p]
                if len(state) == 0:
                    state["step"] = 0
                    for key in ("exp_avg", "exp_avg_sq", "exp_avg_delta"):
                        state[key] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    if group["amsgrad"]:
                        state["max_exp_avg_delta"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    state["prev_grad"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                state["step"] += 1
                by_step.setdefault(state["step"], []).append(p)
            beta1, beta2, beta3 = group["betas"]
            for step, plist in by_step.items():
                key = table_key(gi, step, by_step)
                table = self._tables.setdefault(key, TensorTable())
                st = [self.state[p] for p in plist]
                table.update([p.data for p in plist], [_as_layout(p.grad, p) for p in plist], [s["exp_avg"] for s in st],
                             [s["exp_avg_sq"] for s in st],
                             [s["max_exp_avg_delta"] for s in st] if group["amsgrad"] else None,
                             [s["prev_grad"] for s in st], [s["exp_avg_delta"] for s in st], full_aux=True)
                step_dev = None
                if group.get("capturable"):
                    step_dev = self._step_dev.get(key)
                    if step_dev is None:
                        step_dev = torch.full((1,), step - 1, device=plist[0].device, dtype=torch.int32)
                        self._step_dev[key] = step_dev
                    check(lib().hb_step_increment(ptr(step_dev), ptr(ctl), stream_ptr()), "hb_step_increment")
                _launch(table, step, group["amsgrad"], beta1, beta2, beta3, group["lr"], group["weight_decay"], group["eps"],
                        step_dev, ctl)
                bump_versions(plist)
        return loss


def adan(params: List[Tensor], grads: List[Tensor], prev_grads: List[Tensor], exp_avgs: List[Tensor],
         exp_avg_sqs: List[Tensor], exp_avg_deltas: List[Tensor], max_exp_avg_deltas: List[Tensor], state_steps: List[int],
         amsgrad: bool, beta1: float, beta2: float, beta3: float, lr: float, weight_decay: float, eps: float) -> None:
    """Functional API (reference adan.py:145-199): one fused launch per distinct step value."""
    by_step = {}
    for i, s in enumerate(state_steps):
        by_step.setdefault(int(s), []).append(i)
    for step, idx in by_step.items():
        table = TensorTable()
        table.update([params[i].detach() for i in idx], [_as_layout(grads[i], params[i]) for i in idx],
                     [exp_avgs[i] for i in idx], [exp_avg_sqs[i] for i in idx],
                     [max_exp_avg_deltas[i] for i in idx] if amsgrad else None, [prev_grads[i] for i in idx],
                     [exp_avg_deltas[i] for i in idx], full_aux=True)
        _launch(table, step, amsgrad, beta1, beta2, beta3, lr, weight_decay, eps)
        bump_versions([params[i] for i in idx])
