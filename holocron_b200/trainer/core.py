"""The reference's training-loop semantics as a data-parallel, CUDA-graph-capturable step.

Reference: ``Trainer._fit_epoch`` / ``_backprop_step`` / ``_reset_opt`` / ``_reset_scheduler``
(holocron/trainer/core.py:135-165, 184-208, 238-269). Per iteration the reference does, on one GPU and with two host
synchronisations (``torch.isfinite(batch_loss)`` and ``batch_loss.item()``):

    loss = criterion(model(x), target)
    if not skip_nan_loss or isfinite(loss):  loss.backward();  every `gradient_acc` iterations:
        [clip_grad_norm_(params, grad_clip)] ; optimizer.step() ; optimizer.zero_grad()
    else: nan_cnt += 1 (ValueError beyond nan_tolerance)
    scheduler.step()                       # OneCycleLR (cycles lr AND beta1) | CosineAnnealingLR, once per iteration

:class:`TrainStep` keeps exactly these semantics but makes every decision on the device, so the whole iteration is one
CUDA-graph replay and one process per GPU can be driven without the host in the loop:

* gradients accumulate in the flat :class:`~holocron_b200.distributed.GradBucket` (the backward kernels add into it);
* one NCCL all-reduce (mean) of the bucket per optimizer update when a process group is active;
* ``clip_grad_norm_`` = two launches on the flat bucket (``hb_grad_clip_norm``: fixed-order norm, in-place scaling; a
  NaN norm makes every gradient NaN, as ``clip_grad_norm_`` does);
* the schedule is a device table ``[total_iterations][lr, beta1]`` produced by running the reference's own torch scheduler
  classes on the host once; a device control block (``train_ctl.cu``) selects the row of the current iteration and the
  optimizer kernels read lr / beta1 from it;
* a non-finite loss sets a device flag: that window's optimizer update is skipped (parameters, moments and step count
  untouched, bucket zeroed) and a device counter of consecutive bad windows backs ``nan_tolerance``
  (checked by :meth:`TrainStep.check`, one synchronisation when the caller wants it - e.g. once per epoch).

Deviation (documented): with ``gradient_acc > 1`` the reference skips only the offending micro-batch and still applies the
other micro-batches of the window; here the whole window's update is skipped (a NaN gradient cannot be un-added from the
accumulation buffer without a synchronisation or a second buffer). With ``gradient_acc == 1`` the two coincide.
"""
import ctypes
from typing import Any, Callable, Dict, Optional, Sequence

import torch
from torch import Tensor, nn
from torch.optim.lr_scheduler import CosineAnnealingLR, OneCycleLR

from .._lib import check, lib, ptr, stream_ptr
from ..distributed import GradBucket

__all__ = ["TrainStep", "lr_schedule_table"]


def lr_schedule_table(optimizer: torch.optim.Optimizer, lr: float, total_iterations: int, sched_type: str = "onecycle",
                      **kwargs: Any) -> Tensor:
    """``[total_iterations, 2]`` fp32 table of (lr, beta1) that the reference's scheduler would set on the FIRST parameter
    group at iterations 0, 1, ... (reference core.py:262-269: ``OneCycleLR(optimizer, lr, total)`` - which also cycles
    ``betas[0]`` - or ``CosineAnnealingLR(optimizer, total)``). Produced by running torch's scheduler on a shadow optimizer
    with the same group hyper-parameters; beta1 = -1 where the scheduler does not touch it."""
    group = optimizer.param_groups[0]
    betas = group.get("betas")
    p = nn.Parameter(torch.zeros(1))
    kw = {"lr": lr} if sched_type == "cosine" else {"lr": group["lr"]}
    shadow = torch.optim.Adam([p], betas=tuple(betas), **kw) if betas is not None else torch.optim.SGD([p], momentum=0.9, **kw)
    if sched_type == "onecycle":
        sched = OneCycleLR(shadow, lr, total_iterations, **kwargs)
    elif sched_type == "cosine":
        sched = CosineAnnealingLR(shadow, total_iterations, **kwargs)
    else:
        raise ValueError(f"The following scheduler type is not supported: {sched_type}")
    rows = []
    for i in range(total_iterations):
        g = shadow.param_groups[0]
        rows.append([g["lr"], g["betas"][0] if (betas is not None and sched_type == "onecycle") else -1.0])
        shadow.step()
        if i + 1 < total_iterations:
            sched.step()
    return torch.tensor(rows, dtype=torch.float32)


class TrainStep:
    """One training iteration with the reference Trainer's semantics (see the module docstring).

    Args:
        model, criterion, optimizer: as given to the reference ``Trainer``; ``optimizer`` must be one of this package's fused
            optimizers that understand the device control block (``AdaBelief``, ``AdamP``) built with ``capturable=True``.
        gradient_acc: optimizer update every ``gradient_acc`` iterations (reference ``Trainer(gradient_acc=...)``)
        grad_clip: max global L2 norm (``clip_grad_norm_``) or None
        skip_nan_loss, nan_tolerance: reference ``Trainer(skip_nan_loss=..., nan_tolerance=...)``
        schedule: ``[iterations, 2]`` (lr, beta1) table from :func:`lr_schedule_table`, or None (fixed hyper-parameters)
        graph: capture the iteration(s) into CUDA graphs (static shapes, device-resident criterion)
    """

    def __init__(self, model: nn.Module, criterion: Callable[..., Tensor], optimizer: torch.optim.Optimizer,
                 gradient_acc: int = 1, grad_clip: Optional[float] = None, skip_nan_loss: bool = False, nan_tolerance: int = 5,
                 schedule: Optional[Tensor] = None, graph: bool = True, process_group=None,
                 forward_loss: Optional[Callable[..., Tensor]] = None) -> None:
        self.model, self.criterion, self.optimizer = model, criterion, optimizer
        # `forward_loss(*batch) -> loss` replaces `criterion(model(x), *targets)` (detectors compute their own losses)
        self.forward_loss = forward_loss
        self.gradient_acc = int(gradient_acc)
        self.grad_clip = None if grad_clip is None else float(grad_clip)
        self.skip_nan_loss, self.nan_tolerance = bool(skip_nan_loss), int(nan_tolerance)
        self.process_group = process_group
        params = [p for p in model.parameters() if p.requires_grad]
        if not params:
            raise AssertionError("All parameters are frozen")
        dev = params[0].device
        self.bucket = GradBucket(params)
        L = lib()
        self.ctl = torch.zeros(L.hb_train_ctl_bytes() // 4, device=dev, dtype=torch.float32)
        group = optimizer.param_groups[0]
        self.ctl[0] = float(group["lr"])
        self.ctl[1] = -1.0
        self.schedule = None if schedule is None else schedule.to(device=dev, dtype=torch.float32).contiguous()
        self._clip_scratch = torch.empty(L.hb_grad_clip_partials_max(), device=dev, dtype=torch.float64)
        optimizer._hb_ctl = self.ctl           # the fused optimizers read lr / beta1 / skip from the control block
        self._count = 0                        # iterations inside the current accumulation window (host bookkeeping)
        self.iterations = 0                    # the reference Trainer's `step`
        self.epoch, self.start_epoch, self.min_loss = 0, 0, float("inf")
        self._graphs: Dict[bool, Any] = {}
        self._use_graph = bool(graph)

    # ---- the two kinds of iteration: accumulate only / accumulate + update --------------------------------------
    def _iteration(self, update: bool, *batch: Tensor) -> Tensor:
        L = lib()
        if self.forward_loss is not None:
            loss = self.forward_loss(*batch)
        else:
            x, target = batch[0], batch[1:]
            loss = self.criterion(self.model(x), *target)
        loss32 = loss.detach().float().reshape(1)
        check(L.hb_train_ctl_observe(ptr(self.ctl), ptr(loss32), int(self.skip_nan_loss), stream_ptr()), "hb_train_ctl_observe")
        loss.backward()
        if update:
            check(L.hb_train_ctl_step(ptr(self.ctl), ptr(self.schedule), 0 if self.schedule is None else self.schedule.shape[0],
                                      0, stream_ptr()), "hb_train_ctl_step")
            self.bucket.all_reduce_mean(self.process_group)
            if self.grad_clip is not None:
                check(L.hb_grad_clip_norm(ptr(self.bucket.flat), self.bucket.flat.numel(), ctypes.c_float(self.grad_clip),
                                          ptr(self._clip_scratch), ptr(self.ctl), stream_ptr()), "hb_grad_clip_norm")
            self.optimizer.step()
            self.bucket.zero_()
            check(L.hb_train_ctl_step(ptr(self.ctl), None, 0, 1, stream_ptr()), "hb_train_ctl_step")
        check(L.hb_train_ctl_tick(ptr(self.ctl), stream_ptr()), "hb_train_ctl_tick")
        return loss

    def __call__(self, *batch: Tensor) -> Tensor:
        """Runs one iteration on ``(x, *targets)``; returns the (device) loss. No host synchronisation."""
        self._count += 1
        update = self._count == self.gradient_acc
        if update:
            self._count = 0
        self.iterations += 1
        if not self._use_graph:
            return self._iteration(update, *batch)
        g = self._graphs.get(update)
        if g is None:
            from ..graphs import GraphedTrainStep
            # warm-up iterations would advance the device state: snapshot and restore everything they touch
            snap = self._snapshot()
            g = GraphedTrainStep(lambda *b: self._iteration(update, *b), batch, warmup=2)
            self._restore(snap)
            self._graphs[update] = g
        return g(*batch)

    def _snapshot(self):
        st = {"ctl": self.ctl.clone(), "flat": self.bucket.flat.clone(),
              "params": [p.detach().clone() for p in self.model.parameters()],
              "buffers": [b.detach().clone() for b in self.model.buffers()],
              "opt": [{k: (v.clone() if isinstance(v, Tensor) else v) for k, v in s.items()} for s in self.optimizer.state.values()],
              "steps": {k: v.clone() for k, v in getattr(self.optimizer, "_step_dev", {}).items()}}
        return st

    def _restore(self, st) -> None:
        with torch.no_grad():
            self.ctl.copy_(st["ctl"])
            self.bucket.flat.copy_(st["flat"])
            for p, q in zip(self.model.parameters(), st["params"]):
                p.copy_(q)
            for b, q in zip(self.model.buffers(), st["buffers"]):
                b.copy_(q)
            for i, s in enumerate(self.optimizer.state.values()):
                if i < len(st["opt"]):
                    for k, v in st["opt"][i].items():
                        if isinstance(v, Tensor):
                            s[k].copy_(v)
                        else:
                            s[k] = v
                else:                          # state created lazily by the warm-up updates: back to its initial value
                    for k, v in s.items():
                        if isinstance(v, Tensor):
                            v.zero_()
                        elif k == "step":
                            s[k] = 0
            for k, v in st["steps"].items():
                self.optimizer._step_dev[k].copy_(v)
            for k, v in getattr(self.optimizer, "_step_dev", {}).items():
                if k not in st["steps"]:
                    v.zero_()
        torch.autograd.graph.increment_version(list(self.model.parameters()))

    # ---- checkpoints: the reference's on-disk layout (holocron/trainer/core.py:106-133) --------------------------
    def save(self, output_file: str) -> None:
        """``{"epoch", "step", "min_loss", "model": state_dict}`` written with the legacy (non-zipfile) serialisation,
        exactly what the reference ``Trainer.save`` writes (optimizer / scheduler state is not part of it there either), so
        that ``references/clean_checkpoint.py`` and the reference ``Trainer.load`` read it unchanged."""
        torch.save({"epoch": self.epoch, "step": self.iterations, "min_loss": self.min_loss,
                    "model": self.model.state_dict()}, output_file, _use_new_zipfile_serialization=False)

    def load(self, state: Dict[str, Any]) -> None:
        """Resumes from a checkpoint dict of the reference layout (reference ``Trainer.load``, core.py:123-133)."""
        self.start_epoch = state["epoch"]
        self.epoch = self.start_epoch
        self.iterations = state["step"]
        self.min_loss = state["min_loss"]
        self.model.load_state_dict(state["model"])
        torch.autograd.graph.increment_version(list(self.model.parameters()))   # packed bf16 filters are stale now

    # ---- host-visible state (each property synchronises) --------------------------------------------------------
    def state(self) -> Dict[str, float]:
        c = self.ctl.cpu()
        ints = c.view(torch.int32)
        return {"lr": float(c[0]), "beta1": float(c[1]), "skip": int(ints[2]), "iter": int(ints[4]), "nan_run": int(ints[5]),
                "opt_steps": int(ints[6]), "grad_norm": float(c[7])}

    def check(self) -> None:
        """Raises like the reference (core.py:157-159) once the loss has been NaN/inf for more than ``nan_tolerance``
        consecutive updates. One device synchronisation - call it as often as the reference's progress bar would matter."""
        if self.state()["nan_run"] > self.nan_tolerance:
            raise ValueError(f"loss value has been NaN or inf for more than {self.nan_tolerance} steps.")
