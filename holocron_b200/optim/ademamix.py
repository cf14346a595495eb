"""AdEMAMix on the fused multi-tensor kernel — API mirror of holocron/optim/ademamix.py."""
import ctypes
from typing import Callable, Iterable, List, Optional, Tuple

import torch
from torch import Tensor
from torch.optim import Optimizer

from .._lib import check, lib, ptr, stream_ptr
from ._multi_tensor import TensorTable, bump_versions, table_key
from .adabelief import _as_layout

__all__ = ["AdEMAMix", "ademamix"]

_cf = ctypes.c_float


def _launch(table: TensorTable, step: int, beta1: float, beta2: float, beta3: float, alpha: float, lr: float,
            weight_decay: float, eps: float, step_dev: Optional[Tensor] = None, ctl: Optional[Tensor] = None) -> None:
    check(lib().hb_ademamix_step(ptr(table.metas), ptr(table.chunks), table.num_chunks, _cf(lr), _cf(beta1), _cf(beta2),
                                 _cf(beta3), _cf(alpha), _cf(eps), _cf(weight_decay), int(step), ptr(step_dev), ptr(ctl),
                                 stream_ptr()), "hb_ademamix_step")


class AdEMAMix(Optimizer):
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
                    for key in ("exp_avg", "exp_avg_slow", "exp_avg_sq"):
                        state[key] = torch.zeros_like(p, memory_format=torch.preserve_format)
                state["step"] += 1
                by_step.setdefault(state["step"], []).append(p)
            beta1, beta2, beta3 = group["betas"]
            for step, plist in by_step.items():
                table = self._tables.setdefault(table_key(gi, step, by_step), TensorTable())
                st = [self.state[p] for p in plist]
                table.update([p.data for p in plist], [_as_layout(p.grad, p) for p in plist], [s["exp_avg"] for s in st],
                             [s["exp_avg_sq"] for s in st], None, None, [s["exp_avg_slow"] for s in st])
                _launch(table, step, beta1, beta2, beta3, group["alpha"], group["lr"], group["weight_decay"], group["eps"],
                        None, ctl)
                bump_versions(plist)
        return loss


def ademamix(params: List[Tensor], grads: List[Tensor], exp_avgs: List[Tensor], exp_avgs_slow: List[Tensor],
             exp_avg_sqs: List[Tensor], state_steps: List[int], beta1: float, beta2: float, beta3: float, alpha: float,
             lr: float, weight_decay: float, eps: float) -> None:
    """Functional API (reference ademamix.py:138-176): one fused launch per distinct step value."""
    by_step = {}
    for i, s in enumerate(state_steps):
        by_step.setdefault(int(s), []).append(i)
    for step, idx in by_step.items():
        table = TensorTable()
        table.update([params[i].detach() for i in idx], [_as_layout(grads[i], params[i]) for i in idx],
                     [exp_avgs[i] for i in idx], [exp_avg_sqs[i] for i in idx], None, None, [exp_avgs_slow[i] for i in idx])
        _launch(table, step, beta1, beta2, beta3, alpha, lr, weight_decay, eps)
        bump_versions([params[i] for i in idx])
