"""Lookahead on the fused weight-synchronisation kernel — API mirror of holocron/optim/wrapper.py (Lookahead)."""
import ctypes
from collections import OrderedDict, defaultdict
from typing import Any, Callable, Dict, Optional

import torch
from torch.optim.optimizer import Optimizer

from .._lib import check, lib, ptr, stream_ptr
from ._multi_tensor import TensorTable, bump_versions

__all__ = ["Lookahead"]


class Lookahead(Optimizer):
    """Lookahead wrapper (https://arxiv.org/abs/1907.08610), reference wrapper.py:10-135: the base optimizer updates the
    fast weights; every ``sync_period`` steps ``slow += sync_rate * (fast - slow); fast = slow``.

    Same attributes as the reference (``base_optimizer``, ``fast_steps``, ``defaults``, ``param_groups`` holding the SLOW
    copies, ``state_dict()['base_state_dict']``, ``repr``). The reference synchronises tensor by tensor with three ATen
    kernels and a temporary each; here one launch covers a parameter group (16 B / parameter). Like the reference the
    constructor does not run ``Optimizer.__init__``; the hook registries newer torch versions expect are created so that
    ``state_dict`` / ``load_state_dict`` work (they raise ``AttributeError`` on the reference with torch >= 2.0)."""

    def __init__(self, base_optimizer: torch.optim.Optimizer, sync_rate: float = 0.5, sync_period: int = 6) -> None:
        if sync_rate < 0 or sync_rate > 1:
            raise ValueError(f"expected positive float lower than 1 as sync_rate, received: {sync_rate}")
        if not isinstance(sync_period, int) or sync_period < 1:
            raise ValueError(f"expected positive integer as sync_period, received: {sync_period}")
        self.defaults = {"sync_rate": sync_rate, "sync_period": sync_period}
        self.state = defaultdict(dict)
        self.base_optimizer = base_optimizer
        self.fast_steps = 0
        self.param_groups = []
        for name in ("_optimizer_step_pre_hooks", "_optimizer_step_post_hooks", "_optimizer_state_dict_pre_hooks",
                     "_optimizer_state_dict_post_hooks", "_optimizer_load_state_dict_pre_hooks",
                     "_optimizer_load_state_dict_post_hooks"):
            setattr(self, name, OrderedDict())
        self._tables = {}
        for group in self.base_optimizer.param_groups:
            self._add_param_group(group)

    def __getstate__(self) -> Dict[str, Any]:
        return {
            "defaults": self.defaults,
            "state": self.state,
            "base_state": self.base_optimizer.__getstate__(),
            "fast_steps": self.fast_steps,
            "param_groups": self.param_groups,
        }

    def state_dict(self) -> Dict[str, Any]:
        return dict(**super().state_dict(), base_state_dict=self.base_optimizer.state_dict())

    def load_state_dict(self, state_dict: Dict[str, Any]) -> None:
        self.base_optimizer.load_state_dict(state_dict["base_state_dict"])
        super().load_state_dict({k: v for k, v in state_dict.items() if k != "base_state_dict"})
        self._tables = {}

    def zero_grad(self, set_to_none: bool = True) -> None:
        self.base_optimizer.zero_grad(set_to_none)

    def step(self, closure: Optional[Callable[[], float]] = None) -> Optional[float]:  # type: ignore[override]
        loss = self.base_optimizer.step(closure)
        self.fast_steps += 1
        if self.fast_steps % self.defaults["sync_period"] == 0:
            self.sync_params(self.defaults["sync_rate"])
        return loss

    def __repr__(self) -> str:
        format_string = self.__class__.__name__ + " ("
        optimizer_repr = self.base_optimizer.__repr__().replace("\n", "\n\t")
        format_string += f"\nbase_optimizer={optimizer_repr},"
        for arg, val in self.defaults.items():
            format_string += f"\n{arg}={val},"
        format_string += "\n)"
        return format_string

    def _add_param_group(self, param_group: Dict[str, Any]) -> None:
        """Adds the slow copy of a parameter group of the base optimizer."""
        group = {"params": [p.clone().detach() for p in param_group["params"]], "lr": param_group["lr"]}
        self.param_groups.append(group)

    def add_param_group(self, param_group: Dict[str, Any]) -> None:
        """Adds a parameter group to the base optimizer (fast weights) and its slow copy."""
        self.base_optimizer.add_param_group(param_group)
        self._add_param_group(self.base_optimizer.param_groups[-1])

    @torch.no_grad()
    def sync_params(self, sync_rate: float = 0.0) -> None:
        """slow_param <- slow_param + sync_rate * (fast_param - slow_param); fast_param <- slow_param."""
        for gi, (fast_group, slow_group) in enumerate(zip(self.base_optimizer.param_groups, self.param_groups)):
            fast = [p.data for p in fast_group["params"]]
            if not fast:
                continue
            table = self._tables.setdefault(gi, TensorTable())
            table.update(fast, None, ms=[p.data for p in slow_group["params"]])
            check(lib().hb_lookahead_sync(ptr(table.metas), ptr(table.chunks), table.num_chunks, ctypes.c_float(sync_rate),
                                          stream_ptr()), "hb_lookahead_sync")
            bump_versions(fast_group["params"])
