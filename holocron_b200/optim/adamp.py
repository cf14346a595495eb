"""AdamP on the fused multi-tensor kernels — API mirror of holocron/optim/adamp.py (the reference training scripts' default
optimizer, references/classification/train.py:340)."""
import ctypes
from typing import Iterable, List, Optional, Tuple

import torch
from torch import Tensor
from torch.optim import Adam

from .._lib import check, lib, ptr, stream_ptr
from ._multi_tensor import StepByCount, TensorTable, functional_step

__all__ = ["AdamP", "adamp"]

_cf = ctypes.c_float


def _launch(table: TensorTable, step: int, amsgrad: bool, beta1: float, beta2: float, lr: float, weight_decay: float,
            eps: float, delta: float, step_dev: Optional[Tensor] = None, ctl: Optional[Tensor] = None) -> None:
    check(lib().hb_adamp_step(ptr(table.metas), ptr(table.chunks), table.num_chunks, table.num_tensors, _cf(lr), _cf(beta1),
                              _cf(beta2), _cf(eps), _cf(weight_decay), int(amsgrad), _cf(delta), int(step), ptr(step_dev),
                              ptr(ctl), ptr(table.scratch), stream_ptr()), "hb_adamp_step")


class AdamP(StepByCount, Adam):
    """AdamP (https://arxiv.org/abs/2006.08217) with the reference's exact update (adamp.py:144-191): Adam moments with
    bias correction and L2 weight decay folded into the gradient; when the gradient is almost orthogonal to the weight
    tensor, ``cosine_similarity(p, g) < delta / sqrt(numel)``, the component of the update along the weights is removed:
    ``pt -= <p_hat, pt> p_hat`` with ``p_hat = p / (||p|| + eps)``.

    Same constructor (``delta=0.1`` after Adam's arguments) and ``state_dict`` layout (``step`` python int, ``exp_avg``,
    ``exp_avg_sq``, ``max_exp_avg_sq``) as the reference, which inherits ``torch.optim.Adam``. The reference issues ~15 ATen
    kernels and one host synchronisation (the python ``if`` on the cosine) per parameter tensor; here a parameter group is
    two launches (moments + the four per-tensor reductions, then the apply pass: 40 B / parameter) and nothing syncs.
    ``capturable=True`` keeps the step count on the device (CUDA-graph replay), like :class:`AdaBelief`."""

    _step_on_device = True

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

    def _init_state(self, p: Tensor, state: dict, group: dict) -> None:
        state["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
        state["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
        if group["amsgrad"]:
            state["max_exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)

    def _columns(self, group: dict, states: List[dict]) -> dict:
        return {"ms": "exp_avg", "vs": "exp_avg_sq", "vmaxs": "max_exp_avg_sq" if group["amsgrad"] else None}

    def _launch(self, table: TensorTable, group: dict, step: int, step_dev: Optional[Tensor],
                ctl: Optional[Tensor]) -> None:
        _launch(table, step, group["amsgrad"], *group["betas"], group["lr"], group["weight_decay"], group["eps"], self.delta,
                step_dev, ctl)


def adamp(params: List[Tensor], grads: List[Tensor], exp_avgs: List[Tensor], exp_avg_sqs: List[Tensor],
          max_exp_avg_sqs: List[Tensor], state_steps: List[int], amsgrad: bool, beta1: float, beta2: float, lr: float,
          weight_decay: float, eps: float, delta: float) -> None:
    """Functional API (reference adamp.py:144-191): one pair of fused launches per distinct step value."""
    functional_step(params, grads, state_steps,
                    lambda table, step: _launch(table, step, amsgrad, beta1, beta2, lr, weight_decay, eps, delta),
                    ms=exp_avgs, vs=exp_avg_sqs, vmaxs=max_exp_avg_sqs if amsgrad else None)
