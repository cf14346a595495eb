"""AdaBelief on the fused multi-tensor kernel — API mirror of holocron/optim/adabelief.py."""
import ctypes
from typing import Iterable, List, Optional, Tuple

import torch
from torch import Tensor
from torch.optim import Adam

from .._lib import check, lib, ptr, stream_ptr
from ._multi_tensor import StepByCount, TensorTable, functional_step

__all__ = ["AdaBelief", "adabelief"]

_cf = ctypes.c_float


def _launch(table: TensorTable, step: int, amsgrad: bool, beta1: float, beta2: float, lr: float, weight_decay: float,
            eps: float, step_dev: Optional[Tensor] = None, ctl: Optional[Tensor] = None) -> None:
    check(lib().hb_adabelief_step(ptr(table.metas), ptr(table.chunks), table.num_chunks, _cf(lr), _cf(beta1), _cf(beta2),
                                  _cf(eps), _cf(weight_decay), int(amsgrad), int(step), ptr(step_dev), ptr(ctl),
                                  stream_ptr()), "hb_adabelief_step")


class AdaBelief(StepByCount, Adam):
    """AdaBelief (https://arxiv.org/abs/2010.07468) with the reference's exact update (adabelief.py:121-167):
    L2 weight decay folded into the gradient, no ``+eps`` inside the belief EMA, bias-corrected step.

    Same constructor arguments and ``state_dict`` layout (``step`` python int, ``exp_avg``, ``exp_avg_sq``,
    ``max_exp_avg_sq``) as the reference, which inherits ``torch.optim.Adam.__init__``; Adam's implementation
    switches (``foreach``, ``fused``, ...) are accepted and ignored. One kernel launch per parameter group and
    step value instead of ~9 per tensor.

    ``capturable=True`` (Adam's flag) keeps the step count of each group in a device counter that the kernels read for
    the bias corrections, so that a captured CUDA graph of ``step()`` stays correct when replayed
    (:class:`holocron_b200.utils.GraphedTrainStep`); ``state['step']`` then only advances when Python runs ``step()``.
    """

    _step_on_device = True

    def __init__(self, params: Iterable, lr: float = 1e-3, betas: Tuple[float, float] = (0.9, 0.999), eps: float = 1e-8,
                 weight_decay: float = 0, amsgrad: bool = False, **kwargs) -> None:
        # the reference inherits torch.optim.Adam.__init__ (adabelief.py:16): same validation, same defaults keys.
        # Adam's implementation switches are accepted; `foreach` / `fused` select torch code paths that do not exist
        # here (always ONE fused multi-tensor launch per group) and are only recorded, while flags that would change
        # the arithmetic of the kernel are refused instead of being silently ignored.
        if kwargs.get("maximize"):
            raise NotImplementedError("AdaBelief(maximize=True): the fused kernel implements gradient descent only")
        if kwargs.get("differentiable"):
            raise NotImplementedError("AdaBelief(differentiable=True) is not supported by the fused kernel")
        unknown = set(kwargs) - {"foreach", "maximize", "capturable", "differentiable", "fused", "decoupled_weight_decay"}
        if unknown:
            raise TypeError(f"unexpected keyword arguments {sorted(unknown)}")
        if kwargs.get("decoupled_weight_decay"):
            raise NotImplementedError("AdaBelief folds weight decay into the gradient (reference adabelief.py:149-150)")
        switches = {k: kwargs[k] for k in ("foreach", "fused") if k in kwargs}
        super().__init__(params, lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=amsgrad,
                         capturable=bool(kwargs.get("capturable", False)))
        for group in self.param_groups:
            group.update(switches)
        self.defaults.update(switches)
        self._tables = {}
        self._step_dev = {}

    def __setstate__(self, state) -> None:
        super().__setstate__(state)
        for group in self.param_groups:
            group.setdefault("amsgrad", False)
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
        _launch(table, step, group["amsgrad"], *group["betas"], group["lr"], group["weight_decay"], group["eps"], step_dev,
                ctl)


def adabelief(params: List[Tensor], grads: List[Tensor], exp_avgs: List[Tensor], exp_avg_sqs: List[Tensor],
              max_exp_avg_sqs: List[Tensor], state_steps: List[int], amsgrad: bool, beta1: float, beta2: float, lr: float,
              weight_decay: float, eps: float) -> None:
    """Functional API (reference adabelief.py:121-167): one fused launch per distinct step value."""
    functional_step(params, grads, state_steps,
                    lambda table, step: _launch(table, step, amsgrad, beta1, beta2, lr, weight_decay, eps),
                    ms=exp_avgs, vs=exp_avg_sqs, vmaxs=max_exp_avg_sqs if amsgrad else None)
