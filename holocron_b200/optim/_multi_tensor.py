"""Device-resident tensor tables for the multi-tensor optimizer kernels (holocron_b200/csrc/optim.cu), and the host steps
the fused optimizers share around their launches."""
from typing import Callable, Dict, List, Optional, Sequence

import numpy as np
import torch
from torch import Tensor

from .._lib import check, lib, ptr, require_cuda, stream_ptr


def effective_strides(t: Tensor):
    """Strides of the dims that matter (size-1 dims can carry any stride, e.g. 1x1 filters in channels_last)."""
    return tuple(s for s, n in zip(t.stride(), t.shape) if n != 1)


def _dense(t: Tensor) -> bool:
    """Non-overlapping and dense: some permutation of the dims is contiguous, so the storage is one flat run of numel
    elements and an element-wise kernel may walk it in memory order."""
    expect = 1
    for stride, n in sorted((s, n) for s, n in zip(t.stride(), t.shape) if n != 1):
        if stride != expect:
            return False
        expect *= n
    return True


def _same_dense_layout(ts: Sequence[Optional[Tensor]]) -> bool:
    ref = next(t for t in ts if t is not None)
    for t in ts:
        if t is None:
            continue
        if t.shape != ref.shape or effective_strides(t) != effective_strides(ref):
            return False
    return _dense(ref)


class TensorTable:
    """Packs (param, grad, exp_avg, exp_avg_sq, [max_exp_avg_sq], [aux]) pointers of a parameter group into the
    device table + chunk list the kernels index. Rebuilt only when a pointer changes (e.g. after
    ``Trainer._reset_opt`` rewrites the optimizer state, reference trainer/core.py:238-252)."""

    def __init__(self) -> None:
        self.key = None
        self.metas: Optional[Tensor] = None
        self.chunks: Optional[Tensor] = None
        self.num_chunks = 0
        self.num_tensors = 0
        self.scratch: Optional[Tensor] = None
        self.held = None

    def update(self, params: List[Tensor], grads: Optional[List[Tensor]], ms: Optional[List[Tensor]] = None,
               vs: Optional[List[Tensor]] = None, vmaxs: Optional[List[Tensor]] = None, auxs: Optional[List[Tensor]] = None,
               exts: Optional[List[Tensor]] = None, full_aux: bool = False) -> None:
        """Columns: parameter, gradient, two state tensors, amsgrad maximum, ``aux`` (a 1-element per-tensor scalar such as
        TAdam's ``W_t`` / the LARS trust ratio, or - ``full_aux`` - a full-size tensor such as Adan's ``prev_grad``) and
        ``ext`` (a third full-size state tensor: Adan's ``exp_avg_delta``, AdEMAMix's ``exp_avg_slow``)."""
        none = [None] * len(params)
        cols = [params, grads or none, ms or none, vs or none, vmaxs or none, auxs or none, exts or none]
        # the kernels read these through raw pointers: a gradient copied into the parameter's layout for this call only
        # must stay allocated until the next call, or the caller's next allocation (AdamP's scratch, a device step counter)
        # lands in its memory before the launch has read it
        self.held = cols
        key = tuple(0 if t is None else t.data_ptr() for col in cols for t in col)
        if key == self.key:
            return
        dev = params[0].device
        chunk = lib().hb_optim_chunk_elems()
        rows, chunk_rows = [], []
        for i, p in enumerate(params):
            group = [col[i] for col in cols]
            require_cuda(*[t for t in group if t is not None])
            full = group[:5] + [group[6]] + ([group[5]] if full_aux else [])
            for t in full:
                if t is not None and t.dtype != torch.float32:
                    raise TypeError("the fused optimizers keep parameters, gradients and state in float32")
            if not _same_dense_layout(full):
                raise RuntimeError("parameter, gradient and optimizer state must share one dense memory layout")
            rows.append([0 if t is None else t.data_ptr() for t in group] + [p.numel()])
            n_chunks = (p.numel() + chunk - 1) // chunk
            chunk_rows.append(np.stack([np.full(n_chunks, i, dtype=np.int32), np.arange(n_chunks, dtype=np.int32)], 1))
        metas = np.asarray(rows, dtype=np.int64)
        chunks = np.concatenate(chunk_rows, 0) if chunk_rows else np.zeros((0, 2), np.int32)
        self.metas = torch.from_numpy(metas).to(dev)
        self.chunks = torch.from_numpy(np.ascontiguousarray(chunks)).to(dev)
        self.num_chunks = int(chunks.shape[0])
        self.num_tensors = len(params)
        # per-tensor sums of the reducing kernels: 4 doubles per tensor for AdamP, at most 2 for the others
        self.scratch = torch.zeros(4 * max(1, len(params)), device=dev, dtype=torch.float64)
        self.key = key


def table_key(gi: int, step: int, by_step) -> tuple:
    """Key of the table (and device step counter) of the parameters of group ``gi`` that sit at ``step``. Parameters of one
    group at different step counts (a parameter whose gradient appeared later) are keyed by their distance from the group's
    lowest count, which stays the same from call to call; keyed by the count itself the caches would grow by one entry
    per call."""
    return (gi, step - min(by_step) if len(by_step) > 1 else -1)


def bump_versions(params: Sequence[Tensor]) -> None:
    """The kernels write parameters through raw pointers; tell autograd / the filter-packing cache they changed."""
    torch.autograd.graph.increment_version(list(params))


def as_layout(g: Tensor, p: Tensor) -> Tensor:
    """Gradient with the parameter's dtype and strides (a copy only when autograd or the caller produced another)."""
    if g.dtype == p.dtype and g.shape == p.shape and effective_strides(g) == effective_strides(p):
        return g
    out = torch.empty_like(p)
    out.copy_(g)
    return out


def collect_step(opt, group: dict) -> List[Tensor]:
    """The parameters of ``group`` that have a gradient, each counted one step further: a sparse gradient is refused and
    the state of a parameter seen for the first time is created (``step`` 0, then the optimizer's
    ``_init_state(p, state, group)``) before ``state["step"]`` advances."""
    plist = []
    for p in group["params"]:
        if p.grad is None:
            continue
        if p.grad.is_sparse:
            raise RuntimeError(f"{opt.__class__.__name__} does not support sparse gradients")
        state = opt.state[p]
        if len(state) == 0:
            state["step"] = 0
            opt._init_state(p, state, group)
        state["step"] += 1
        plist.append(p)
    return plist


def device_local_lr(states: List[dict]) -> None:
    """LAMB and RaLars write each tensor's trust ratio into ``state["local_lr"]``, a 0-dim device tensor; a state loaded
    from the reference holds a python number there (or nothing)."""
    for state in states:
        if not isinstance(state.get("local_lr"), torch.Tensor):
            state["local_lr"] = torch.ones((), device=state["exp_avg"].device, dtype=torch.float32)


class StepByCount:
    """``step()`` of the optimizers whose update depends on each parameter's own step count (bias corrections): the
    parameters of a group that sit at one count share a table (``_tables[table_key(...)]``) and a launch.

    A subclass gives ``_init_state(p, state, group)``, ``_columns(group, states)`` (the state key of each column of
    :meth:`TensorTable.update` it fills, or None) and ``_launch(table, group, step, step_dev, ctl)``, its ABI call.
    ``ctl`` is the device control block of :class:`holocron_b200.trainer.TrainStep`, if one is attached. With
    ``_step_on_device`` and a group built with ``capturable=True``, each count also lives in a device counter
    (``_step_dev``, same key) that the kernels read for the bias corrections and that advances on the device unless the
    control block skips the update, so that a captured CUDA graph of ``step()`` stays correct when replayed."""

    _step_on_device = False
    _full_aux = False       # the aux column is a full-size tensor (Adan's prev_grad)

    @torch.no_grad()
    def step(self, closure: Optional[Callable[[], float]] = None) -> Optional[float]:
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        ctl = getattr(self, "_hb_ctl", None)
        for gi, group in enumerate(self.param_groups):
            by_step = {}
            for p in collect_step(self, group):
                by_step.setdefault(self.state[p]["step"], []).append(p)
            for step, plist in by_step.items():
                key = table_key(gi, step, by_step)
                table = self._tables.setdefault(key, TensorTable())
                states = [self.state[p] for p in plist]
                cols = self._columns(group, states)
                table.update([p.data for p in plist], [as_layout(p.grad, p) for p in plist],
                             **{col: None if k is None else [s[k] for s in states] for col, k in cols.items()},
                             full_aux=self._full_aux)
                step_dev = None
                if self._step_on_device and group.get("capturable"):
                    step_dev = self._step_dev.get(key)
                    if step_dev is None:
                        step_dev = torch.full((1,), step - 1, device=plist[0].device, dtype=torch.int32)
                        self._step_dev[key] = step_dev
                    check(lib().hb_step_increment(ptr(step_dev), ptr(ctl), stream_ptr()), "hb_step_increment")
                self._launch(table, group, step, step_dev, ctl)
                bump_versions(plist)
        return loss


def functional_step(params: List[Tensor], grads: List[Tensor], state_steps: List[int],
                    launch: Callable[[TensorTable, int], None], full_aux: bool = False,
                    **columns: Optional[List[Tensor]]) -> None:
    """The functional forms: one table and one ``launch(table, step)`` per distinct step count. ``columns`` are the state
    columns of :meth:`TensorTable.update` over all parameters (None: no such column)."""
    by_step: Dict[int, List[int]] = {}
    for i, s in enumerate(state_steps):
        by_step.setdefault(int(s), []).append(i)
    for step, idx in by_step.items():
        table = TensorTable()
        table.update([params[i].detach() for i in idx], [as_layout(grads[i], params[i]) for i in idx],
                     **{k: None if col is None else [col[i] for i in idx] for k, col in columns.items()}, full_aux=full_aux)
        launch(table, step)
        bump_versions([params[i] for i in idx])
