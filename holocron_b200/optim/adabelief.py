"""AdaBelief on the fused multi-tensor kernel — API mirror of holocron/optim/adabelief.py."""
import ctypes
from typing import Callable, Iterable, List, Optional, Tuple

import torch
from torch import Tensor
from torch.optim import Adam

from .._lib import check, lib, ptr, stream_ptr
from ._multi_tensor import TensorTable, bump_versions, table_key, effective_strides

__all__ = ["AdaBelief", "adabelief"]

_cf = ctypes.c_float


def _launch(table: TensorTable, step: int, amsgrad: bool, beta1: float, beta2: float, lr: float, weight_decay: float,
            eps: float, step_dev: Optional[Tensor] = None, ctl: Optional[Tensor] = None) -> None:
    check(lib().hb_adabelief_step(ptr(table.metas), ptr(table.chunks), table.num_chunks, _cf(lr), _cf(beta1), _cf(beta2),
                                  _cf(eps), _cf(weight_decay), int(amsgrad), int(step), ptr(step_dev), ptr(ctl),
                                  stream_ptr()), "hb_adabelief_step")


class AdaBelief(Adam):
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

    @torch.no_grad()
    def step(self, closure: Optional[Callable[[], float]] = None) -> Optional[float]:  # type: ignore[override]
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        # device control block of holocron_b200.trainer.TrainStep (lr / beta1 schedule, NaN-skip flag), if any
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
                table = self._tables.setdefault(table_key(gi, step, by_step), TensorTable())
                grads = [_as_layout(p.grad, p) for p in plist]
                table.update([p.data for p in plist], grads, [self.state[p]["exp_avg"] for p in plist],
                             [self.state[p]["exp_avg_sq"] for p in plist],
                             [self.state[p]["max_exp_avg_sq"] for p in plist] if group["amsgrad"] else None, None)
                step_dev = None
                if group.get("capturable"):
                    key = table_key(gi, step, by_step)
                    step_dev = self._step_dev.get(key)
                    if step_dev is None:
                        step_dev = torch.full((1,), step - 1, device=plist[0].device, dtype=torch.int32)
                        self._step_dev[key] = step_dev
                    check(lib().hb_step_increment(ptr(step_dev), ptr(ctl), stream_ptr()), "hb_step_increment")
                _launch(table, step, group["amsgrad"], beta1, beta2, group["lr"], group["weight_decay"], group["eps"],
                        step_dev, ctl)
                bump_versions(plist)
        return loss


def _as_layout(g: Tensor, p: Tensor) -> Tensor:
    """Gradient with the parameter's strides (copy only when autograd produced a different layout)."""
    if g.dtype != torch.float32:
        g = g.float()
    if g.shape == p.shape and effective_strides(g) == effective_strides(p):
        return g
    out = torch.empty_like(p)
    out.copy_(g)
    return out


def adabelief(params: List[Tensor], grads: List[Tensor], exp_avgs: List[Tensor], exp_avg_sqs: List[Tensor],
              max_exp_avg_sqs: List[Tensor], state_steps: List[int], amsgrad: bool, beta1: float, beta2: float, lr: float,
              weight_decay: float, eps: float) -> None:
    """Functional API (reference adabelief.py:121-167): one fused launch per distinct step value."""
    by_step = {}
    for i, s in enumerate(state_steps):
        by_step.setdefault(int(s), []).append(i)
    for step, idx in by_step.items():
        table = TensorTable()
        table.update([params[i].detach() for i in idx], [_as_layout(grads[i], params[i]) for i in idx],
                     [exp_avgs[i] for i in idx], [exp_avg_sqs[i] for i in idx],
                     [max_exp_avg_sqs[i] for i in idx] if amsgrad else None, None)
        _launch(table, step, amsgrad, beta1, beta2, lr, weight_decay, eps)
        bump_versions([params[i] for i in idx])
