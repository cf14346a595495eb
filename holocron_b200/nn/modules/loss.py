"""Loss modules on the hot path — mirrors holocron/nn/modules/loss.py (_Loss :25-47, FocalLoss :50-84,
MultiLabelCrossEntropy :87-103, ComplementCrossEntropy :106-125, ClassBalancedWrapper :128-160, MutualChannelLoss :163-192,
DiceLoss :195-219, PolyLoss :222-246)."""
from typing import Any, List, Optional, Union, cast

import torch
from torch import Tensor, nn

from .. import functional as F

__all__ = ["ClassBalancedWrapper", "ComplementCrossEntropy", "DiceLoss", "FocalLoss", "MultiLabelCrossEntropy",
           "MutualChannelLoss", "PolyLoss"]


class _Loss(nn.Module):
    """Base class: registers the class weights as a ``weight`` buffer (float w -> ``[w, 1 - w]``, list, or tensor)."""

    def __init__(self, weight: Optional[Union[float, List[float], Tensor]] = None, ignore_index: int = -100,
                 reduction: str = "mean") -> None:
        super().__init__()
        self.weight: Optional[Tensor]
        if isinstance(weight, (float, int)):
            self.register_buffer("weight", torch.Tensor([weight, 1 - weight]))
        elif isinstance(weight, list):
            self.register_buffer("weight", torch.Tensor(weight))
        elif isinstance(weight, Tensor):
            self.register_buffer("weight", weight)
        else:
            self.weight = None
        self.ignore_index = ignore_index
        if reduction not in ["none", "mean", "sum"]:
            raise NotImplementedError("argument reduction received an incorrect input")
        self.reduction = reduction


class FocalLoss(_Loss):
    """Focal loss (https://arxiv.org/abs/1708.02002): ``-(1 - p_t)^gamma * w_t log p_t`` on the fused kernel."""

    def __init__(self, gamma: float = 2.0, **kwargs: Any) -> None:
        super().__init__(**kwargs)
        self.gamma = gamma

    def forward(self, x: Tensor, target: Tensor) -> Tensor:
        return F.focal_loss(x, target, self.weight, self.ignore_index, self.reduction, self.gamma)

    def __repr__(self) -> str:
        return f"{self.__class__.__name__}(gamma={self.gamma}, reduction='{self.reduction}')"


class MultiLabelCrossEntropy(_Loss):
    """Cross entropy with multi-label (soft) targets ``(N, K, ...)``: ``-sum_k t_k w_k log p_k``."""

    def __init__(self, *args: Any, **kwargs: Any) -> None:
        super().__init__(*args, **kwargs)

    def forward(self, x: Tensor, target: Tensor) -> Tensor:
        return F.multilabel_cross_entropy(x, target, self.weight, self.ignore_index, self.reduction)

    def __repr__(self) -> str:
        return f"{self.__class__.__name__}(reduction='{self.reduction}')"


class ComplementCrossEntropy(_Loss):
    """Complement cross entropy (https://arxiv.org/abs/2009.02189): cross entropy plus ``gamma`` times the entropy of the
    normalised non-target probabilities."""

    def __init__(self, gamma: float = -1, **kwargs: Any) -> None:
        super().__init__(**kwargs)
        self.gamma = gamma

    def forward(self, x: Tensor, target: Tensor) -> Tensor:
        return F.complement_cross_entropy(x, target, self.weight, self.ignore_index, self.reduction, self.gamma)

    def __repr__(self) -> str:
        return f"{self.__class__.__name__}(gamma={self.gamma}, reduction='{self.reduction}')"


class ClassBalancedWrapper(nn.Module):
    """Class-balanced loss (https://arxiv.org/abs/1901.05555): sets the wrapped criterion's class weights to
    ``(1 - beta) / (1 - beta**num_samples)``, or multiplies its existing ``weight`` by them in place. Works around any
    criterion with a ``weight`` attribute (this package's losses, ``torch.nn.CrossEntropyLoss``, ...)."""

    def __init__(self, criterion: nn.Module, num_samples: Tensor, beta: float = 0.99) -> None:
        super().__init__()
        self.criterion = criterion
        self.beta = beta
        cb_weights = (1 - beta) / (1 - beta**num_samples)
        if self.criterion.weight is None:
            self.criterion.weight = cb_weights
        else:
            self.criterion.weight *= cb_weights.to(device=self.criterion.weight.device)

    def forward(self, x: Tensor, target: Tensor) -> Tensor:
        return cast(Tensor, self.criterion.forward(x, target))

    def __repr__(self) -> str:
        return f"{self.__class__.__name__}({self.criterion.__repr__()}, beta={self.beta})"


class MutualChannelLoss(_Loss):
    """Mutual channel loss (https://arxiv.org/abs/2002.04264) on ``(N, cnum * xi, ...)`` features. Draws a new channel mask
    on the host at every call, so it runs outside CUDA graph capture."""

    def __init__(self, weight: Optional[Union[float, List[float], Tensor]] = None, ignore_index: int = -100,
                 reduction: str = "mean", xi: int = 2, alpha: float = 1) -> None:
        super().__init__(weight, ignore_index, reduction)
        self.xi = xi
        self.alpha = alpha

    def forward(self, x: Tensor, target: Tensor) -> Tensor:
        return F.mutual_channel_loss(x, target, self.weight, self.ignore_index, self.reduction, self.xi, self.alpha)

    def __repr__(self) -> str:
        return f"{self.__class__.__name__}(reduction='{self.reduction}', xi={self.xi}, alpha={self.alpha})"


class DiceLoss(_Loss):
    """Dice loss (https://arxiv.org/abs/1606.04797) on probabilities. As in the reference only ``weight`` reaches the
    base class, so ``reduction`` always reads ``'mean'``."""

    def __init__(self, weight: Optional[Union[float, List[float], Tensor]] = None, gamma: float = 1.0,
                 eps: float = 1e-8) -> None:
        super().__init__(weight)
        self.gamma = gamma
        self.eps = eps

    def forward(self, x: Tensor, target: Tensor) -> Tensor:
        return F.dice_loss(x, target, self.weight, self.gamma, self.eps)

    def __repr__(self) -> str:
        return f"{self.__class__.__name__}(reduction='{self.reduction}', gamma={self.gamma}, eps={self.eps})"


class PolyLoss(_Loss):
    """Poly-1 loss (https://arxiv.org/abs/2204.12511): ``-log p_t + eps (1 - p_t)``, hard or soft targets."""

    def __init__(self, *args: Any, eps: float = 2.0, **kwargs: Any) -> None:
        super().__init__(*args, **kwargs)
        self.eps = eps

    def forward(self, x: Tensor, target: Tensor) -> Tensor:
        return F.poly_loss(x, target, self.eps, self.weight, self.ignore_index, self.reduction)

    def __repr__(self) -> str:
        return f"{self.__class__.__name__}(eps={self.eps}, reduction='{self.reduction}')"
