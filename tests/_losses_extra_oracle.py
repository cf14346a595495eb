"""fp32 CPU restatements of the reference's multilabel_cross_entropy, complement_cross_entropy and mutual_channel_loss
(holocron/nn/functional.py:150-319), differentiable with autograd. Test infrastructure only: the mutual channel loss takes
its channel mask as an argument instead of drawing it."""
from typing import Optional

import torch
import torch.nn.functional as F
from torch import Tensor


def _class_view(weight: Tensor, x: Tensor) -> Tensor:
    return weight.to(x.dtype).view(1, -1, *([1] * (x.ndim - 2)))


def _kept_classes(k: int, ignore_index: int):
    return [c for c in range(k) if not (0 <= ignore_index < k and c == ignore_index)]


def _reduce_positions(per_pos: Tensor, reduction: str) -> Tensor:
    if reduction == "sum":
        return per_pos.sum()
    if reduction == "mean":
        return per_pos.mean()
    return per_pos


def multilabel_cross_entropy(x: Tensor, target: Tensor, weight: Optional[Tensor] = None, ignore_index: int = -100,
                             reduction: str = "mean") -> Tensor:
    """-sum_k t_k w_k log_softmax(x)_k over the kept class columns; 'mean' over the N * spatial positions."""
    logp = F.log_softmax(x, dim=1)
    if weight is not None:
        logp = logp * _class_view(weight, x)
    per_class = -target * logp
    return _reduce_positions(per_class[:, _kept_classes(x.shape[1], ignore_index)].sum(1), reduction)


def complement_cross_entropy(x: Tensor, target: Tensor, weight: Optional[Tensor] = None, ignore_index: int = -100,
                             reduction: str = "mean", gamma: float = -1) -> Tensor:
    """torch's cross entropy + gamma * C, C = -1/(K-1) sum_{k != y, k kept} w_k q_k log q_k with q the softmax over the
    non-target classes."""
    ce = F.cross_entropy(x, target, weight, ignore_index=ignore_index, reduction=reduction)
    if gamma == 0:
        return ce
    k = x.shape[1]
    is_target = F.one_hot(target, k).movedim(-1, 1).bool()
    logq = F.log_softmax(x.masked_fill(is_target, float("-inf")), dim=1)
    logq = torch.where(is_target, torch.zeros_like(logq), logq)
    term = torch.where(is_target, torch.zeros_like(logq), logq.exp()) * logq
    if weight is not None:
        term = term * _class_view(weight, x)
    comp = -term[:, _kept_classes(k, ignore_index)].sum(1) / (k - 1)
    return ce + gamma * _reduce_positions(comp, reduction)


def mutual_channel_loss(x: Tensor, target: Tensor, mask: Tensor, weight: Optional[Tensor] = None,
                        ignore_index: int = -100, reduction: str = "mean", xi: int = 2, alpha: float = 1.0) -> Tensor:
    """discr - alpha * diversity for the given (cnum, xi) channel mask."""
    b, c = x.shape[:2]
    spatial = x.shape[2:]
    cnum = c // xi
    groups = x.reshape(b, cnum, xi, -1)
    # max(dim).values routes the gradient to the first maximal channel, as the reference's max does
    discr = (groups * mask.to(x.dtype).view(1, cnum, xi, 1)).max(dim=2).values.view(b, cnum, *spatial)
    w = weight.to(x.dtype) if weight is not None else None
    discr_loss = F.cross_entropy(discr, target, w, ignore_index=ignore_index, reduction=reduction)
    diversity = F.softmax(groups, dim=-1).max(dim=2).values.mean(dim=1)
    if reduction not in ("sum", "mean"):
        diversity = diversity.view(b, *spatial)
    return discr_loss - alpha * _reduce_positions(diversity, reduction)
