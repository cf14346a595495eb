"""Device-resident tensor tables for the multi-tensor optimizer kernels (holocron_b200/csrc/optim.cu)."""
from typing import List, Optional, Sequence

import numpy as np
import torch
from torch import Tensor

from .._lib import lib, require_cuda


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

    def update(self, params: List[Tensor], grads: Optional[List[Tensor]], ms: Optional[List[Tensor]],
               vs: Optional[List[Tensor]], vmaxs: Optional[List[Tensor]], auxs: Optional[List[Tensor]],
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
        self.scratch = torch.zeros(2 * max(1, len(params)), device=dev, dtype=torch.float64)
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
