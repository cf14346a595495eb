"""AdamP on the fused multi-tensor kernels — API mirror of holocron/optim/adamp.py (the reference training scripts' default
optimizer, references/classification/train.py:340)."""
import ctypes
from typing import Callable, Iterable, List, Optional, Tuple

import torch
from torch import Tensor
from torch.optim import Adam

from .._lib import check, lib, ptr, stream_ptr
from ._multi_tensor import TensorTable, bump_versions, table_key
from .adabelief import _as_layout

__all__ = ["AdamP", "adamp"]

_cf = ctypes.c_float


def _launch(table: TensorTable, step: int, amsgrad: bool, beta1: float, beta2: float, lr: float, weight_decay: float,
            eps: float, delta: float, step_dev: Optional[Tensor] = None, ctl: Optional[Tensor] = None) -> None:
    if table.scratch is None or table.scratch.numel() < 4 * table.num_tensors:
        table.scratch = torch.zeros(4 * max(1, table.num_tensors), device=table.metas.device, dtype=torch.float64)
    check(lib().hb_adamp_step(ptr(table.metas), ptr(table.chunks), table.num_chunks, table.num_tensors, _cf(lr), _cf(beta1),
                              _cf(beta2), _cf(eps), _cf(weight_decay), int(amsgrad), _cf(delta), int(step), ptr(step_dev),
                              ptr(ctl), ptr(table.scratch), stream_ptr()), "hb_adamp_step")


class AdamP(Adam):
    """AdamP (https://arxiv.org/abs/2006.08217) with the reference's exact update (adamp.py:144-191): Adam moments with
    bias correction and L2 weight decay folded into the gradient; when the gradient is almost orthogonal to the weight
    tensor, ``cosine_similarity(p, g) < delta / sqrt(numel)``, the component of the update along the weights is removed:
    ``pt -= <p_hat, pt> p_hat`` with ``p_hat = p / (||p|| + eps)``.

    Same constructor (``delta=0.1`` after Adam's arguments) and ``state_dict`` layout (``step`` python int, ``exp_avg``,
    ``exp_avg_sq``, ``max_exp_avg_sq``) as the reference, which inherits ``torch.optim.Adam``. The reference issues ~15 ATen
    kernels and one host synchronisation (the python ``if`` on the cosine) per parameter tensor; here a parameter group is
    two launches (moments + the four per-tensor reductions, then the apply pass: 40 B / parameter) and nothing syncs.
    ``capturable=True`` keeps the step count on the device (CUDA-graph replay), like :class:`AdaBelief`."""

    def __init__(self, params: Iterable, lr: float = 1e-3, betas: Tuple[float, float] = (0.9, 0.999), eps: float = 1e-8,
                 weight_decay: float = 0.0, amsgrad: bool = False, delta: float = 0.1, capturable: bool = False) -> None:
        super().__init__(params, lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=amsgrad,
                         capturable=bool(capturable))
        self.delta = delta
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
                    state["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    state["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    if group["amsgrad"]:
                        state["max_exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                state["step"] += 1
                by_step.setdefault(state["step"], []).append(p)
            beta1, beta2 = group["betas"]
            for step, plist in by_step.items():
                key = table_key(gi, step, by_step)
                table = self._tables.setdefault(key, TensorTable())
                table.update([p.data for p in plist], [_as_layout(p.grad, p) for p in plist],
                             [self.state[p]["exp_avg"] for p in plist], [self.state[p]["exp_avg_sq"] for p in plist],
                             [self.state[p]["max_exp_avg_sq"] for p in plist] if group["amsgrad"] else None, None)
                step_dev = None
                if group.get("capturable"):
                    step_dev = self._step_dev.get(key)
                    if step_dev is None:
                        step_dev = torch.full((1,), step - 1, device=plist[0].device, dtype=torch.int32)
                        self._step_dev[key] = step_dev
                    check(lib().hb_step_increment(ptr(step_dev), ptr(ctl), stream_ptr()), "hb_step_increment")
                _launch(table, step, group["amsgrad"], beta1, beta2, group["lr"], group["weight_decay"], group["eps"],
                        self.delta, step_dev, ctl)
                bump_versions(plist)
        return loss


def adamp(params: List[Tensor], grads: List[Tensor], exp_avgs: List[Tensor], exp_avg_sqs: List[Tensor],
          max_exp_avg_sqs: List[Tensor], state_steps: List[int], amsgrad: bool, beta1: float, beta2: float, lr: float,
          weight_decay: float, eps: float, delta: float) -> None:
    """Functional API (reference adamp.py:144-191): one pair of fused launches per distinct step value."""
    by_step = {}
    for i, s in enumerate(state_steps):
        by_step.setdefault(int(s), []).append(i)
    for step, idx in by_step.items():
        table = TensorTable()
        table.update([params[i].detach() for i in idx], [_as_layout(grads[i], params[i]) for i in idx],
                     [exp_avgs[i] for i in idx], [exp_avg_sqs[i] for i in idx],
                     [max_exp_avg_sqs[i] for i in idx] if amsgrad else None, None)
        _launch(table, step, amsgrad, beta1, beta2, lr, weight_decay, eps, delta)
        bump_versions([params[i] for i in idx])
