"""The reference's trainer classes on top of :class:`~holocron_b200.trainer.core.TrainStep` — API mirror of
holocron/trainer/core.py (Trainer :26-451), classification.py (ClassificationTrainer :21-159, BinaryClassificationTrainer
:162-232), segmentation.py (SegmentationTrainer :15-83) and detection.py (assign_iou :17-32, DetectionTrainer :35-126).

Same constructor arguments, same public methods (``fit_n_epochs``, ``find_lr``, ``check_setup``, ``evaluate``, ``save`` /
``load``, ``to_cuda``), same checkpoint layout, same printed lines. What differs is where the decisions of an iteration are
taken:

* with one of this package's fused optimizers that read the device control block (``AdaBelief``, ``AdamP``, ``Adan``,
  ``AdEMAMix`` built with ``capturable=True``) an iteration is one :class:`TrainStep` call: gradient accumulation, global-norm
  clipping, the OneCycle / cosine schedule (lr and beta1 from a device table), the NaN-skip decision and the NaN counter all
  live on the device; the host reads the loss back only every ``log_every`` iterations (the reference synchronises twice per
  iteration: ``torch.isfinite(loss)`` and ``loss.item()``), and ``Trainer(graph=True)`` replays the iteration as a CUDA graph
  (static batch shapes: use ``drop_last=True``);
* with any other ``torch.optim.Optimizer`` the iteration is the reference's own sequence (``_backprop_step``: backward,
  clip, step, zero_grad, scheduler.step, host-side NaN test) - this is also what runs for CPU models.

``amp`` is accepted for compatibility: the CUDA kernels of this package compute in bf16 with fp32 accumulation whatever the
flag says (no loss scaling needed), stock torch modules are wrapped in bf16 autocast when it is set.
Evaluation accumulates its sums on the device and synchronises once per call instead of two to four times per batch
(under ``torch.no_grad()``; the reference uses ``inference_mode``).
Progress bars (fastprogress) and plots (matplotlib) are optional: losses and learning rates are always recorded in
``loss_recorder`` / ``lr_recorder``; the plotting methods raise ImportError when matplotlib is missing."""
import contextlib
import math
from collections import defaultdict
from typing import Any, Callable, Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
import torch
from torch import Tensor, nn
from torch.optim.lr_scheduler import CosineAnnealingLR, MultiplicativeLR, OneCycleLR

from .._lib import check, lib, ptr, require_cuda, stream_ptr
from ..transforms._table import upload
from .core import TrainStep, lr_schedule_table
from .utils import freeze_bn, freeze_model, split_normalization_params

__all__ = ["BinaryClassificationTrainer", "ClassificationTrainer", "DetectionTrainer", "SegmentationTrainer", "Trainer",
           "assign_iou", "assign_iou_batch"]

ParamSeq = Sequence[torch.nn.Parameter]


def _reads_control_block(optimizer: torch.optim.Optimizer) -> bool:
    from .. import optim
    return isinstance(optimizer, (optim.AdaBelief, optim.AdamP, optim.Adan, optim.AdEMAMix)) and \
        all(g.get("capturable", False) for g in optimizer.param_groups or [optimizer.defaults])


class Trainer:
    """Baseline trainer (reference trainer/core.py:26-451). Extra keyword arguments: ``graph`` (CUDA-graph replay of the
    iteration on the device path), ``log_every`` (loss read-back period of the device path), ``process_group`` (data-parallel
    gradient mean over NCCL inside the step)."""

    def __init__(self, model: nn.Module, train_loader, val_loader, criterion: nn.Module, optimizer: torch.optim.Optimizer,
                 gpu: Optional[int] = None, output_file: str = "./checkpoint.pth", amp: bool = False,
                 skip_nan_loss: bool = False, nan_tolerance: int = 5, gradient_acc: int = 1,
                 gradient_clip: Optional[float] = None, on_epoch_end: Optional[Callable[[Dict[str, float]], Any]] = None,
                 graph: bool = False, log_every: int = 50, process_group=None) -> None:
        self.model = model
        self.train_loader = train_loader
        self.val_loader = val_loader
        self.criterion = criterion
        self.optimizer = optimizer
        self.amp = amp
        self.on_epoch_end = on_epoch_end
        self.skip_nan_loss = skip_nan_loss
        self.nan_tolerance = nan_tolerance
        self.gradient_acc = gradient_acc
        self.grad_clip = gradient_clip
        self.output_file = output_file
        self.graph, self.log_every, self.process_group = graph, max(1, int(log_every)), process_group
        self.step = 0
        self.start_epoch = 0
        self.epoch = 0
        self._grad_count = 0
        self.min_loss = math.inf
        self.gpu = gpu
        self._params: Tuple[ParamSeq, ParamSeq] = ([], [])
        self.lr_recorder: List[float] = []
        self.loss_recorder: List[float] = []
        self._train_step: Optional[TrainStep] = None
        self.set_device(gpu)
        self._reset_opt(self.optimizer.defaults["lr"])

    # ------------------------------------------------------------------------------------------------ devices / files
    def set_device(self, gpu: Optional[int] = None) -> None:
        if isinstance(gpu, int):
            if not torch.cuda.is_available():
                raise AssertionError("PyTorch cannot access your GPU. Please investigate!")
            if gpu >= torch.cuda.device_count():
                raise ValueError("Invalid device index")
            torch.cuda.set_device(gpu)
            self.model = self.model.cuda()
            if isinstance(self.criterion, torch.nn.Module):
                self.criterion = self.criterion.cuda()

    def save(self, output_file: str) -> None:
        """``{"epoch", "step", "min_loss", "model"}`` in the legacy serialisation (reference core.py:106-121)."""
        torch.save({"epoch": self.epoch, "step": self.step, "min_loss": self.min_loss, "model": self.model.state_dict()},
                   output_file, _use_new_zipfile_serialization=False)

    def load(self, state: Dict[str, Any]) -> None:
        self.start_epoch = state["epoch"]
        self.epoch = self.start_epoch
        self.step = state["step"]
        self.min_loss = state["min_loss"]
        self.model.load_state_dict(state["model"])
        torch.autograd.graph.increment_version(list(self.model.parameters()))   # packed bf16 filters are stale now

    def to_cuda(self, x, target):
        if isinstance(self.gpu, int):
            if self.gpu >= torch.cuda.device_count():
                raise ValueError("Invalid device index")
            return self._to_cuda(x, target)
        return x, target

    @staticmethod
    def _to_cuda(x: Tensor, target: Tensor) -> Tuple[Tensor, Tensor]:
        return x.cuda(non_blocking=True), target.cuda(non_blocking=True)

    # ------------------------------------------------------------------------------------------------ one iteration
    def _autocast(self):
        on_cuda = next(self.model.parameters()).is_cuda
        return torch.autocast("cuda", dtype=torch.bfloat16) if (self.amp and on_cuda) else contextlib.nullcontext()

    def _get_loss(self, x: Tensor, target: Tensor, return_logits: bool = False) -> Union[Tensor, Tuple[Tensor, Tensor]]:
        with self._autocast():
            out = self.model(x)
            loss = self.criterion(out.float() if out.is_floating_point() else out, target)
        return (loss, out) if return_logits else loss

    def _backprop_step(self, loss: Tensor) -> None:
        """Host-driven update of the generic path (reference core.py:184-208; bf16 needs no GradScaler)."""
        self._grad_count += 1
        loss.backward()
        if self._grad_count == self.gradient_acc:
            if isinstance(self.grad_clip, float):
                nn.utils.clip_grad_norm_(self.model.parameters(), self.grad_clip)
            self.optimizer.step()
            self.optimizer.zero_grad()
            self._grad_count = 0

    def _device_path(self) -> bool:
        return next(self.model.parameters()).is_cuda and _reads_control_block(self.optimizer)

    def _make_step(self, schedule: Optional[Tensor], skip_nan_loss: Optional[bool] = None) -> TrainStep:
        self._train_step = TrainStep(
            self.model, self.criterion, self.optimizer, gradient_acc=self.gradient_acc,
            grad_clip=self.grad_clip if isinstance(self.grad_clip, float) else None,
            skip_nan_loss=self.skip_nan_loss if skip_nan_loss is None else skip_nan_loss, nan_tolerance=self.nan_tolerance,
            schedule=schedule, graph=self.graph, process_group=self.process_group,
            forward_loss=lambda x, target: self._get_loss(x, target))
        return self._train_step

    def _fit_epoch(self, mb: Any = None) -> None:
        """One pass over ``train_loader`` (reference core.py:135-165)."""
        freeze_bn(self.model.train())
        if self._train_step is not None:
            last = None
            for idx, (x, target) in enumerate(self.train_loader):
                x, target = self.to_cuda(x, target)
                last = self._train_step(x, target)
                self.step += 1
                if (idx + 1) % self.log_every == 0:
                    self._train_step.check()                      # raises past `nan_tolerance` consecutive NaN updates
                    self.loss_recorder.append(float(last.detach()))
            if last is not None:
                self._train_step.check()
            self.epoch += 1
            return
        nan_cnt = 0
        for x, target in self.train_loader:
            x, target = self.to_cuda(x, target)
            batch_loss = self._get_loss(x, target)
            if not self.skip_nan_loss or torch.isfinite(batch_loss):
                nan_cnt = 0
                self._backprop_step(batch_loss)
            else:
                nan_cnt += 1
                if nan_cnt > self.nan_tolerance:
                    raise ValueError(f"loss value has been NaN or inf for more than {self.nan_tolerance} steps.")
            self.scheduler.step()
            self.step += 1
        self.epoch += 1

    # ------------------------------------------------------------------------------------------------ optimizer set-up
    def _set_params(self, norm_weight_decay: Optional[float] = None) -> None:
        if not any(p.requires_grad for p in self.model.parameters()):
            raise AssertionError("All parameters are frozen")
        if norm_weight_decay is None:
            self._params = [p for p in self.model.parameters() if p.requires_grad], []
        else:
            self._params = split_normalization_params(self.model)

    def _reset_opt(self, lr: float, norm_weight_decay: Optional[float] = None) -> None:
        """Fresh optimizer state and parameter groups (reference core.py:238-252)."""
        self.optimizer.defaults["lr"] = lr
        self.optimizer.state = defaultdict(dict)
        self.optimizer.param_groups = []
        self._set_params(norm_weight_decay)
        if norm_weight_decay is None:
            self.optimizer.add_param_group({"params": self._params[0]})
        else:
            wd_groups = [norm_weight_decay, self.optimizer.defaults.get("weight_decay", 0)]
            for _params, _wd in zip(self._params, wd_groups):
                if len(_params) > 0:
                    self.optimizer.add_param_group({"params": _params, "weight_decay": _wd})
        self.optimizer.zero_grad()
        # the fused optimizers keep per-group device tables and device step counters next to `state`: start them afresh too
        for attr in ("_tables", "_step_dev"):
            if isinstance(getattr(self.optimizer, attr, None), dict):
                getattr(self.optimizer, attr).clear()
        self._train_step = None
        self._grad_count = 0

    def _reset_scheduler(self, lr: float, num_epochs: int, sched_type: str = "onecycle", **kwargs: Any) -> None:
        """OneCycleLR (lr and beta1) / CosineAnnealingLR over ``num_epochs * len(train_loader)`` iterations (reference
        core.py:254-269); on the device path the same torch classes fill the schedule table of the step."""
        total = num_epochs * len(self.train_loader)
        if sched_type not in ("onecycle", "cosine"):
            raise ValueError(f"The following scheduler type is not supported: {sched_type}")
        if self._device_path():
            self._make_step(lr_schedule_table(self.optimizer, lr, total, sched_type, **kwargs))
            return
        if sched_type == "onecycle":
            self.scheduler = OneCycleLR(self.optimizer, lr, total, **kwargs)
        else:
            self.scheduler = CosineAnnealingLR(self.optimizer, total, **kwargs)

    @torch.no_grad()
    def evaluate(self):  # noqa: ANN201
        raise NotImplementedError

    @staticmethod
    def _eval_metrics_str(eval_metrics) -> str:  # noqa: ANN001
        raise NotImplementedError

    # ------------------------------------------------------------------------------------------------ public loops
    def fit_n_epochs(self, num_epochs: int, lr: float, freeze_until: Optional[str] = None, sched_type: str = "onecycle",
                     norm_weight_decay: Optional[float] = None, **kwargs: Any) -> None:
        """Trains for ``num_epochs`` epochs, evaluating and checkpointing after each (reference core.py:271-315)."""
        freeze_model(self.model.train(), freeze_until)
        self._reset_opt(lr, norm_weight_decay)
        self._reset_scheduler(lr, num_epochs, sched_type, **kwargs)
        for _ in range(num_epochs):
            self._fit_epoch()
            eval_metrics = self.evaluate()
            print(f"Epoch {self.epoch}/{self.start_epoch + num_epochs} - {self._eval_metrics_str(eval_metrics)}")  # noqa: T201
            if eval_metrics["val_loss"] < self.min_loss:
                print(f"Validation loss decreased {self.min_loss:.4} --> {eval_metrics['val_loss']:.4}: saving state...")  # noqa: T201
                self.min_loss = eval_metrics["val_loss"]
                self.save(self.output_file)
            if self.on_epoch_end is not None:
                self.on_epoch_end(eval_metrics)

    def find_lr(self, freeze_until: Optional[str] = None, start_lr: float = 1e-7, end_lr: float = 1,
                norm_weight_decay: Optional[float] = None, num_it: int = 100) -> None:
        """Learning-rate range test (reference core.py:317-370): ``num_it`` iterations at exponentially growing rates, losses
        in ``loss_recorder``, rates in ``lr_recorder``. Diagnostic: the loss is read back every iteration on both paths."""
        if num_it > len(self.train_loader):
            raise ValueError("the value of `num_it` needs to be lower than the number of available batches")
        freeze_model(self.model.train(), freeze_until)
        self._reset_opt(start_lr, norm_weight_decay)
        gamma = (end_lr / start_lr) ** (1 / (num_it - 1))
        self.lr_recorder = [start_lr * gamma**idx for idx in range(num_it)]
        self.loss_recorder = []
        step = scheduler = None
        if self._device_path():
            table = torch.tensor([[v, -1.0] for v in self.lr_recorder], dtype=torch.float32)
            step = self._make_step(table, skip_nan_loss=False)
        else:
            scheduler = MultiplicativeLR(self.optimizer, lambda step_: gamma)
        for batch_idx, (x, target) in enumerate(self.train_loader):
            x, target = self.to_cuda(x, target)
            if step is not None:
                batch_loss = step(x, target)
            else:
                batch_loss = self._get_loss(x, target)
                self._backprop_step(batch_loss)
                scheduler.step()
            if torch.isnan(batch_loss) or torch.isinf(batch_loss):
                if batch_idx == 0:
                    raise ValueError("loss value is NaN or inf.")
                break
            self.loss_recorder.append(batch_loss.item())
            if batch_idx + 1 == num_it:
                break
        self.lr_recorder = self.lr_recorder[: len(self.loss_recorder)]
        self._train_step = None

    def plot_recorder(self, beta: float = 0.95, **kwargs: Any) -> None:
        """Smoothed loss against learning rate after :meth:`find_lr` (reference core.py:372-404); needs matplotlib."""
        if len(self.lr_recorder) != len(self.loss_recorder) or len(self.lr_recorder) == 0:
            raise AssertionError("Please run the `lr_find` method first")
        import matplotlib.pyplot as plt
        import numpy as np
        smoothed_losses = []
        avg_loss = 0.0
        for idx, loss in enumerate(self.loss_recorder):
            avg_loss = beta * avg_loss + (1 - beta) * loss
            smoothed_losses.append(avg_loss / (1 - beta ** (idx + 1)))
        data_slice = slice(min(len(self.loss_recorder) // 10, 10),
                           -min(len(self.loss_recorder) // 20, 5) if len(self.loss_recorder) >= 20 else len(self.loss_recorder))
        vals = np.array(smoothed_losses[data_slice])
        min_idx = vals.argmin()
        max_val = vals[: min_idx + 1].max()
        delta = max_val - vals[min_idx]
        plt.plot(self.lr_recorder[data_slice], smoothed_losses[data_slice])
        plt.xscale("log")
        plt.xlabel("Learning Rate")
        plt.ylabel("Training loss")
        plt.ylim(vals[min_idx] - 0.1 * delta, max_val + 0.2 * delta)
        plt.grid(True, linestyle="--", axis="x")
        plt.show(**kwargs)

    def check_setup(self, freeze_until: Optional[str] = None, lr: float = 3e-4, norm_weight_decay: Optional[float] = None,
                    num_it: int = 100, **kwargs: Any) -> None:
        """Overfits one batch for ``num_it`` iterations (reference core.py:406-451): raises on a NaN / inf loss, records the
        losses in ``loss_recorder`` and plots them when matplotlib is available."""
        freeze_model(self.model.train(), freeze_until)
        self._reset_opt(lr, norm_weight_decay)
        x, target = next(iter(self.train_loader))
        x, target = self.to_cuda(x, target)
        step = self._make_step(None, skip_nan_loss=False) if self._device_path() else None
        losses = []
        for _ in range(num_it):
            if step is not None:
                batch_loss = step(x, target)
            else:
                batch_loss = self._get_loss(x, target)
                self._backprop_step(batch_loss)
            if torch.isnan(batch_loss) or torch.isinf(batch_loss):
                raise ValueError("loss value is NaN or inf.")
            losses.append(batch_loss.item())
        self.loss_recorder = losses
        self._train_step = None
        try:
            import matplotlib.pyplot as plt
        except ImportError:
            return
        plt.plot(range(len(losses)), losses)
        plt.xlabel("Optimization steps")
        plt.ylabel("Training loss")
        plt.grid(True, linestyle="--", axis="x")
        plt.show(**kwargs)


class ClassificationTrainer(Trainer):
    """Image classification (reference trainer/classification.py:21-159)."""

    is_binary: bool = False

    @torch.no_grad()
    def evaluate(self) -> Dict[str, float]:
        """Validation loss (NaN batches left out), top-1 and top-5 accuracy; sums stay on the device, one read-back."""
        self.model.eval()
        dev = next(self.model.parameters()).device
        acc = torch.zeros(4, device=dev, dtype=torch.float64)           # loss sum, valid batches, top-1 hits, top-5 hits
        num_samples = 0
        for x, target in self.val_loader:
            x, target = self.to_cuda(x, target)
            loss, out = self._get_loss(x, target, return_logits=True)
            ok = torch.isfinite(loss)
            pred = out.topk(5, dim=1)[1] if out.shape[1] >= 5 else out.argmax(dim=1, keepdim=True)
            correct = pred.eq(target.view(-1, 1).expand_as(pred))
            top5 = correct.any(dim=1).sum() if out.shape[1] >= 5 else correct.new_zeros(())
            acc += torch.stack([torch.where(ok, loss.double(), loss.new_zeros((), dtype=torch.float64)), ok.double(),
                                correct[:, 0].sum().double(), top5.double()])
            num_samples += x.shape[0]
        val_loss, valid, top1, top5 = acc.tolist()
        return {"val_loss": val_loss / valid if valid else float("nan"), "acc1": top1 / num_samples, "acc5": top5 / num_samples}

    @staticmethod
    def _eval_metrics_str(eval_metrics: Dict[str, float]) -> str:
        return (f"Validation loss: {eval_metrics['val_loss']:.4} "
                f"(Acc@1: {eval_metrics['acc1']:.2%}, Acc@5: {eval_metrics['acc5']:.2%})")


    @torch.no_grad()
    def plot_top_losses(self, mean: Tuple[float, float, float], std: Tuple[float, float, float],
                        classes: Optional[Sequence[str]] = None, num_samples: int = 12, **kwargs: Any) -> None:
        """The ``num_samples`` training samples with the highest loss (reference classification.py:77-159). The ranking -
        losses, predicted class and probability, targets, de-normalised images - is kept in ``self.top_losses`` (largest loss
        first); the grid of images is drawn when matplotlib is available (``kwargs`` go to ``plt.show``)."""
        if not self.is_binary and classes is None:
            raise AssertionError("arg 'classes' must be specified for multi-class classification")
        reduction = self.criterion.reduction
        self.criterion.reduction = "none"  # type: ignore[assignment]
        self.model.eval()
        kept: Optional[Dict[str, Tensor]] = None
        try:
            for x, target in self.train_loader:
                x, target = self.to_cuda(x, target)
                batch_loss, logits = self._get_loss(x, target, return_logits=True)
                logits = logits.float()
                if self.is_binary:
                    batch_loss = batch_loss.reshape(x.shape[0], -1).mean(1)
                    probs = torch.sigmoid(logits.reshape(x.shape[0], -1)[:, 0])
                    preds = (probs >= 0.5).long()
                else:
                    probs, preds = torch.softmax(logits, 1).max(dim=1)
                cur = {"losses": batch_loss.float(), "preds": preds, "probs": probs, "targets": target.reshape(x.shape[0], -1)[:, 0],
                       "images": x.float()}
                merged = cur if kept is None else {k: torch.cat((kept[k], v.to(kept[k].dtype))) for k, v in cur.items()}
                order = merged["losses"].argsort(descending=True)[:num_samples]
                kept = {k: v[order] for k, v in merged.items()}
        finally:
            self.criterion.reduction = reduction
        if kept is None:
            raise ValueError("the training loader is empty")
        dev = kept["images"].device
        images = kept["images"] * torch.tensor(std, device=dev).view(-1, 1, 1) + torch.tensor(mean, device=dev).view(-1, 1, 1)
        self.top_losses = {k: v.cpu() for k, v in kept.items() if k != "images"}
        self.top_losses["images"] = images.cpu()
        try:
            import matplotlib.pyplot as plt
            from torchvision.transforms.functional import to_pil_image
        except ImportError:
            return
        num_cols = 4
        num_rows = math.ceil(num_samples / num_cols)
        _, axes = plt.subplots(num_rows, num_cols, figsize=(20, 5), squeeze=False)
        for idx in range(images.shape[0]):
            ax = axes[idx // num_cols][idx % num_cols]
            ax.imshow(to_pil_image(self.top_losses["images"][idx].clamp(0, 1)))
            loss, prob = float(self.top_losses["losses"][idx]), float(self.top_losses["probs"][idx])
            tgt = self.top_losses["targets"][idx]
            if self.is_binary:
                ax.title.set_text(f"{loss:.3} / {prob:.2} / {float(tgt):.2}")
            else:
                ax.title.set_text(f"{loss:.3} / {classes[int(self.top_losses['preds'][idx])]} ({prob:.1%}) / {classes[int(tgt)]}")  # type: ignore[index]
            ax.axis("off")
        plt.show(**kwargs)


class BinaryClassificationTrainer(ClassificationTrainer):
    """Binary classification on one logit per sample (reference trainer/classification.py:162-232)."""

    is_binary: bool = True

    def _get_loss(self, x: Tensor, target: Tensor, return_logits: bool = False) -> Union[Tensor, Tuple[Tensor, Tensor]]:
        with self._autocast():
            out = self.model(x)
            out32 = out.float()
            loss = self.criterion(out32, target.to(dtype=out32.dtype).view_as(out32))   # targets may be stored as long
        return (loss, out) if return_logits else loss

    @torch.no_grad()
    def evaluate(self) -> Dict[str, float]:
        self.model.eval()
        dev = next(self.model.parameters()).device
        acc = torch.zeros(3, device=dev, dtype=torch.float64)           # loss sum, valid batches, per-sample accuracy sum
        num_samples = 0
        for x, target in self.val_loader:
            x, target = self.to_cuda(x, target)
            loss, out = self._get_loss(x, target, return_logits=True)
            ok = torch.isfinite(loss)
            hits = ((target.view_as(out) >= 0.5) == (torch.sigmoid(out.float()) >= 0.5)).sum().double() / out[0].numel()
            acc += torch.stack([torch.where(ok, loss.double(), loss.new_zeros((), dtype=torch.float64)), ok.double(), hits])
            num_samples += x.shape[0]
        val_loss, valid, top1 = acc.tolist()
        return {"val_loss": val_loss / valid if valid else float("nan"), "acc": top1 / num_samples}

    @staticmethod
    def _eval_metrics_str(eval_metrics: Dict[str, float]) -> str:
        return f"Validation loss: {eval_metrics['val_loss']:.4} (Acc: {eval_metrics['acc']:.2%})"


class SegmentationTrainer(Trainer):
    """Semantic segmentation (reference trainer/segmentation.py:15-83)."""

    def __init__(self, *args: Any, num_classes: int = 10, **kwargs: Any) -> None:
        super().__init__(*args, **kwargs)
        self.num_classes = num_classes

    @torch.no_grad()
    def evaluate(self, ignore_index: int = 255) -> Dict[str, float]:
        """Validation loss, global pixel accuracy and mean IoU from the confusion matrix (kept on the device)."""
        self.model.eval()
        dev = next(self.model.parameters()).device
        nc = self.num_classes
        conf_mat = torch.zeros((nc, nc), dtype=torch.int64, device=dev)
        acc = torch.zeros(2, device=dev, dtype=torch.float64)
        for x, target in self.val_loader:
            x, target = self.to_cuda(x, target)
            loss, out = self._get_loss(x, target, return_logits=True)
            ok = torch.isfinite(loss)
            acc += torch.stack([torch.where(ok, loss.double(), loss.new_zeros((), dtype=torch.float64)), ok.double()])
            pred = out.argmax(dim=1).flatten()
            target = target.flatten()
            k = (target >= 0) & (target < nc)
            # out-of-range targets (the ignore index) land in an extra bin that is dropped: no data-dependent gather
            inds = torch.where(k, nc * target.to(torch.int64) + pred, torch.full_like(pred, nc * nc))
            conf_mat += torch.bincount(inds, minlength=nc**2 + 1)[: nc**2].reshape(nc, nc)
        val_loss, valid = acc.tolist()
        diag = torch.diag(conf_mat)
        acc_global = (diag.sum() / conf_mat.sum()).item()
        mean_iou = (diag / (conf_mat.sum(1) + conf_mat.sum(0) - diag)).mean().item()
        return {"val_loss": val_loss / valid if valid else float("nan"), "acc_global": acc_global, "mean_iou": mean_iou}

    @staticmethod
    def _eval_metrics_str(eval_metrics: Dict[str, float]) -> str:
        return (f"Validation loss: {eval_metrics['val_loss']:.4} "
                f"(Acc: {eval_metrics['acc_global']:.2%} | Mean IoU: {eval_metrics['mean_iou']:.2%})")


def _pairwise_iou(gt_boxes: Tensor, pred_boxes: Tensor) -> Tensor:
    if gt_boxes.is_cuda:
        from ..ops.boxes import box_iou
    else:
        from torchvision.ops.boxes import box_iou
    return box_iou(gt_boxes, pred_boxes)


def assign_iou(gt_boxes: Tensor, pred_boxes: Tensor, iou_threshold: float = 0.5) -> Tuple[List[int], List[int]]:
    """Matches every ground-truth box to its best prediction (IoU >= threshold), one ground truth per prediction at most -
    reference trainer/detection.py:17-32 (pairwise IoU on the CUDA kernel for device tensors)."""
    iou = _pairwise_iou(gt_boxes, pred_boxes).max(dim=1)
    gt_kept = iou.values >= iou_threshold
    assign_unique = torch.unique(iou.indices[gt_kept])
    arange = torch.arange(gt_boxes.shape[0], device=gt_boxes.device)
    if iou.indices[gt_kept].shape[0] == assign_unique.shape[0]:
        return arange[gt_kept], iou.indices[gt_kept]  # type: ignore[return-value]
    gt_indices, pred_indices = [], []
    for pred_idx in assign_unique:
        selection = iou.values[gt_kept][iou.indices[gt_kept] == pred_idx].argmax()
        gt_indices.append(arange[gt_kept][iou.indices[gt_kept] == pred_idx][selection].item())
        pred_indices.append(pred_idx.item())
    return gt_indices, pred_indices


# the codes of hb_assign_iou_batch's descriptor rows (include/holocron_b200.h)
_BOX_CODES = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2, torch.float64: 4}
_LABEL_CODES = {torch.int64: 0, torch.int32: 1}
_MATCH_WORDS = 16
_INT32_MAX = 2 ** 31 - 1


def _match_table(gt_boxes: Sequence[Tensor], pred_boxes: Sequence[Tensor], gt_labels: Optional[Sequence[Tensor]],
                 pred_labels: Optional[Sequence[Tensor]]) -> Tuple[np.ndarray, List[int]]:
    """The descriptor rows of ``hb_assign_iou_batch`` (one per image: the boxes and labels are read in place through
    their strides) and each image's ground-truth count, refusing what the kernel does not read."""
    if len(gt_boxes) != len(pred_boxes):
        raise ValueError(f"{len(gt_boxes)} ground-truth sets but {len(pred_boxes)} prediction sets")
    labels = gt_labels is not None
    if labels and (pred_labels is None or len(gt_labels) != len(gt_boxes) or len(pred_labels) != len(gt_boxes)):
        raise ValueError("expected one ground-truth and one predicted label tensor per image")
    tensors = [*gt_boxes, *pred_boxes, *(gt_labels if labels else []), *(pred_labels if labels else [])]
    if len({t.device for t in tensors}) > 1:
        raise ValueError("all boxes and labels of a batch must be on one device")
    table = np.zeros((len(gt_boxes), _MATCH_WORDS), dtype=np.int64)
    ns, offset = [], 0
    for k, (g, p) in enumerate(zip(gt_boxes, pred_boxes)):
        for b in (g, p):
            if b.ndim != 2 or b.shape[1] != 4 or b.shape[0] > _INT32_MAX:
                raise ValueError(f"boxes are expected as (num_boxes, 4) tensors in xyxy format, got {tuple(b.shape)}")
            if b.dtype not in _BOX_CODES:
                raise TypeError(f"unsupported box dtype {b.dtype}: expected one of {', '.join(map(str, _BOX_CODES))}")
        n = int(g.shape[0])
        codes = _BOX_CODES[g.dtype] | _BOX_CODES[p.dtype] << 8
        row = [g.data_ptr(), p.data_ptr(), 0, 0, n, p.shape[0], *g.stride(), *p.stride(), 0, 0, 0, offset]
        if labels:
            gl, pl = gt_labels[k], pred_labels[k]
            for lab, m in ((gl, n), (pl, p.shape[0])):
                if lab.ndim != 1 or lab.shape[0] != m:
                    raise ValueError(f"{m} boxes but labels of shape {tuple(lab.shape)}")
                if lab.dtype not in _LABEL_CODES:
                    raise TypeError(f"unsupported label dtype {lab.dtype}: expected torch.int64 or torch.int32")
            codes |= _LABEL_CODES[gl.dtype] << 16 | _LABEL_CODES[pl.dtype] << 24
            row[2:4], row[10:12] = [gl.data_ptr(), pl.data_ptr()], [gl.stride(0), pl.stride(0)]
        row[12] = codes
        table[k, :14] = row
        ns.append(n)
        offset += n
    return table, ns


def _assign_batch(gt_boxes: Sequence[Tensor], pred_boxes: Sequence[Tensor], iou_threshold: float,
                  gt_labels: Optional[Sequence[Tensor]] = None, pred_labels: Optional[Sequence[Tensor]] = None,
                  counts: Optional[Tensor] = None) -> Tuple[Tensor, List[int]]:
    """One ``hb_assign_iou_batch`` launch over a non-empty batch: the flat int64 match vector and each image's
    ground-truth count. With labels, {assigned, correct} are added to ``counts`` (int64 [2] on the batch's device)."""
    require_cuda(*gt_boxes, *pred_boxes, *(gt_labels or ()), *(pred_labels or ()))
    table, ns = _match_table(gt_boxes, pred_boxes, gt_labels, pred_labels)
    device = gt_boxes[0].device
    with torch.cuda.device(device):
        match = torch.empty(sum(ns), dtype=torch.int64, device=device)
        scratch = torch.empty(2 * sum(ns), dtype=torch.int32, device=device)
        _dev, (descs,) = upload(device, table)
        check(lib().hb_assign_iou_batch(descs, len(ns), iou_threshold, ptr(scratch), ptr(match), ptr(counts),
                                        stream_ptr()), "hb_assign_iou_batch")
    return match, ns


def assign_iou_batch(gt_boxes: Sequence[Tensor], pred_boxes: Sequence[Tensor], iou_threshold: float = 0.5
                     ) -> List[Tensor]:
    """:func:`assign_iou` for every image of a batch in one CUDA launch, with no host synchronisation.

    ``gt_boxes[i]`` and ``pred_boxes[i]`` are image i's (n, 4) xyxy boxes (fp32, bf16, fp16 or fp64, any strides, all on
    one CUDA device; box arithmetic in fp32). Returns one int64 vector per image, views of one flat tensor: entry g is
    the prediction paired with ground-truth box g, or -1, so that {(g, m[g]) : m[g] >= 0} is the set of pairs
    ``assign_iou(gt_boxes[i], pred_boxes[i], iou_threshold)`` returns on CUDA tensors. The threshold is rounded to fp32,
    as torch rounds a scalar compared with an fp32 tensor."""
    if not gt_boxes and not pred_boxes:
        return []
    match, ns = _assign_batch(gt_boxes, pred_boxes, iou_threshold)
    return list(match.split(ns))


def _matchable(target: List[Dict[str, Tensor]], detections: List[Dict[str, Tensor]],
               counts: Optional[Tensor]) -> bool:
    """Whether hb_assign_iou_batch reads the batch: every box and label tensor on one CUDA device (counts' own, once
    it exists), in dtypes the kernel takes."""
    if not target or len(target) != len(detections):
        return False
    tensors = [d[k] for d in (*target, *detections) for k in ("boxes", "labels")]
    device = tensors[0].device if counts is None else counts.device
    return (device.type == "cuda" and all(t.device == device for t in tensors)
            and all(d["boxes"].dtype in _BOX_CODES and d["labels"].dtype in _LABEL_CODES
                    for d in (*target, *detections)))


class DetectionTrainer(Trainer):
    """Object detection: the model computes its own losses (reference trainer/detection.py:35-126)."""

    @staticmethod
    def _to_cuda(x: List[Tensor], target: List[Dict[str, Tensor]]):  # type: ignore[override]
        x = [_x.cuda(non_blocking=True) for _x in x]
        target = [{k: v.cuda(non_blocking=True) for k, v in t.items()} for t in target]
        return x, target

    def _get_loss(self, x: List[Tensor], target: List[Dict[str, Tensor]]) -> Tensor:  # type: ignore[override]
        with self._autocast():
            loss_dict = self.model(x, target)
        return sum(loss_dict.values())  # type: ignore[return-value]

    @staticmethod
    def _eval_metrics_str(eval_metrics: Dict[str, Optional[float]]) -> str:
        loc_str = f"{eval_metrics['loc_err']:.2%}" if isinstance(eval_metrics["loc_err"], float) else "N/A"
        clf_str = f"{eval_metrics['clf_err']:.2%}" if isinstance(eval_metrics["clf_err"], float) else "N/A"
        det_str = f"{eval_metrics['det_err']:.2%}" if isinstance(eval_metrics["det_err"], float) else "N/A"
        return f"Loc error: {loc_str} | Clf error: {clf_str} | Det error: {det_str}"

    @torch.no_grad()
    def evaluate(self, iou_threshold: float = 0.5) -> Dict[str, Optional[float]]:
        """Localisation / classification / end-to-end detection error rates (reference detection.py:77-126).

        Batches whose boxes and labels are all on one CUDA device are matched by one ``hb_assign_iou_batch`` launch
        each, their {assigned, correct} counts summed on the device and read back once per call; other batches take
        the reference's per-image loop."""
        self.model.eval()
        loc_assigns = 0
        correct, clf_error, loc_fn, loc_fp, num_samples = 0, 0, 0, 0, 0
        counts: Optional[Tensor] = None       # {assigned, correct} of the batches matched on the device
        dev_gt, dev_pred = 0, 0               # their ground-truth and predicted boxes
        for x, target in self.val_loader:
            x, target = self.to_cuda(x, target)
            with self._autocast():
                detections = self.model(x)
            num_samples += sum(t["boxes"].shape[0] for t in target)
            if _matchable(target, detections, counts):
                if counts is None:
                    counts = torch.zeros(2, dtype=torch.int64, device=target[0]["boxes"].device)
                _assign_batch([t["boxes"] for t in target], [d["boxes"] for d in detections], iou_threshold,
                              [t["labels"] for t in target], [d["labels"] for d in detections], counts)
                dev_gt += sum(t["boxes"].shape[0] for t in target)
                dev_pred += sum(d["boxes"].shape[0] for d in detections)
                continue
            for dets, t in zip(detections, target):
                if t["boxes"].shape[0] > 0 and dets["boxes"].shape[0] > 0:
                    gt_indices, pred_indices = assign_iou(t["boxes"], dets["boxes"], iou_threshold)
                    loc_assigns += len(gt_indices)
                    correct_ = (t["labels"][gt_indices] == dets["labels"][pred_indices]).sum().item()
                else:
                    gt_indices, pred_indices = [], []
                    correct_ = 0
                correct += correct_
                clf_error += len(gt_indices) - correct_
                loc_fn += t["boxes"].shape[0] - len(gt_indices)
                loc_fp += dets["boxes"].shape[0] - len(pred_indices)
        if counts is not None:
            assigned, correct_ = counts.tolist()
            loc_assigns += assigned
            correct += correct_
            clf_error += assigned - correct_
            loc_fn += dev_gt - assigned
            loc_fp += dev_pred - assigned
        nb_preds = num_samples - loc_fn + loc_fp
        loc_err = 1 - 2 * loc_assigns / (nb_preds + num_samples) if nb_preds + num_samples > 0 else None
        clf_err = 1 - correct / loc_assigns if loc_assigns > 0 else None
        det_err = 1 - 2 * correct / (nb_preds + num_samples) if nb_preds + num_samples > 0 else None
        return {"loc_err": loc_err, "clf_err": clf_err, "det_err": det_err, "val_loss": loc_err}
