"""focal_loss / poly_loss / dice_loss / multilabel_cross_entropy / complement_cross_entropy / mutual_channel_loss on the
fused CUDA kernels (holocron_b200/csrc/losses.cu)."""
import ctypes
import math
from typing import Optional

import torch
from torch import Tensor

from .._lib import check, dtype_code, lib, ptr, require_cuda, stream_ptr

_cf = ctypes.c_float
_RED = {"none": 0, "mean": 1, "sum": 2}


def _nks(x: Tensor):
    n, k = x.shape[0], x.shape[1]
    s = 1
    for d in x.shape[2:]:
        s *= d
    return n, k, s


def _weight(weight, x: Tensor) -> Optional[Tensor]:
    if not isinstance(weight, Tensor):
        return None
    return weight.detach().to(device=x.device, dtype=torch.float32).contiguous()


def _index_targets(target: Tensor, n: int, s: int) -> Tensor:
    """Class-index targets as the flat int64 [N*S] vector the kernels read."""
    tc = target.contiguous().view(-1)
    if tc.dtype != torch.long:
        tc = tc.long()
    if tc.numel() != n * s:
        raise ValueError("target shape does not match the input's (N, ...) dims")
    return tc


def _position_buffers(x: Tensor, n: int, s: int, num_partials: int):
    """A forward's per-position loss, per-block partial sums (num_partials per block) and {sum, count, mean}."""
    loss_pos = torch.empty(n * s, device=x.device, dtype=torch.float32)
    partials = torch.empty(num_partials * lib().hb_loss_max_partials(), device=x.device, dtype=torch.float64)
    fwd_out = torch.empty(3, device=x.device, dtype=torch.float32)
    return loss_pos, partials, fwd_out


def _reduced(x: Tensor, loss_pos: Tensor, fwd_out: Tensor, reduction: int, flat: bool = False) -> Tensor:
    """mean, sum, or the per-position loss: flat [N*S], or shaped (N, ...) like x without its class axis."""
    if reduction == 1:
        return fwd_out[2].to(x.dtype)
    if reduction == 2:
        return fwd_out[0].to(x.dtype)
    out = loss_pos.to(x.dtype)
    return out if flat else out.view(x.shape[0], *x.shape[2:])


def _grad(gout: Tensor) -> Tensor:
    """The incoming gradient as the flat fp32 vector the backward kernels read."""
    return gout.detach().float().contiguous().view(-1)


class _HardLossFn(torch.autograd.Function):
    """kind 0: focal, 1: poly-1; hard (int64) targets."""

    @staticmethod
    def forward(ctx, x: Tensor, target: Tensor, weight: Optional[Tensor], ignore_index: int, reduction: int, kind: int,
                gamma: float, eps: float) -> Tensor:
        require_cuda(x, target)
        xc = x.contiguous()
        n, k, s = _nks(xc)
        tc = _index_targets(target, n, s)
        loss_pos, partials, fwd_out = _position_buffers(x, n, s, 2)
        check(lib().hb_cls_loss_hard_fwd(ptr(xc), ptr(tc), ptr(weight), ptr(loss_pos), ptr(partials), ptr(fwd_out), n,
                                         k, s, int(ignore_index), kind, _cf(gamma), _cf(eps), dtype_code(xc),
                                         stream_ptr()), "hb_cls_loss_hard_fwd")
        ctx.save_for_backward(xc, tc, weight, fwd_out)
        ctx.cfg = (n, k, s, int(ignore_index), reduction, kind, gamma, eps)
        return _reduced(x, loss_pos, fwd_out, reduction, flat=True)

    @staticmethod
    def backward(ctx, gout: Tensor):
        xc, tc, weight, fwd_out = ctx.saved_tensors
        n, k, s, ignore_index, reduction, kind, gamma, eps = ctx.cfg
        g = _grad(gout)
        dx = torch.empty_like(xc)
        check(lib().hb_cls_loss_hard_bwd(ptr(xc), ptr(tc), ptr(weight), ptr(g), ptr(fwd_out), ptr(dx), n, k, s,
                                         ignore_index, kind, _cf(gamma), _cf(eps), reduction, dtype_code(xc),
                                         stream_ptr()), "hb_cls_loss_hard_bwd")
        return dx, None, None, None, None, None, None, None


class _PolySoftFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x: Tensor, target: Tensor, weight: Optional[Tensor], ignore_index: int, reduction: int,
                eps: float) -> Tensor:
        require_cuda(x, target)
        xc = x.contiguous()
        tc = target.to(xc.dtype).contiguous()
        n, k, s = _nks(xc)
        loss_pos, partials, fwd_out = _position_buffers(x, n, s, 2)
        check(lib().hb_poly_soft_fwd(ptr(xc), ptr(tc), ptr(weight), ptr(loss_pos), ptr(partials), ptr(fwd_out), n, k,
                                     s, int(ignore_index), _cf(eps), dtype_code(xc), stream_ptr()), "hb_poly_soft_fwd")
        ctx.save_for_backward(xc, tc, weight)
        ctx.cfg = (n, k, s, int(ignore_index), reduction, eps)
        return _reduced(x, loss_pos, fwd_out, reduction)

    @staticmethod
    def backward(ctx, gout: Tensor):
        xc, tc, weight = ctx.saved_tensors
        n, k, s, ignore_index, reduction, eps = ctx.cfg
        g = _grad(gout)
        dx = torch.empty_like(xc)
        check(lib().hb_poly_soft_bwd(ptr(xc), ptr(tc), ptr(weight), ptr(g), ptr(dx), n, k, s, ignore_index, _cf(eps),
                                     reduction, dtype_code(xc), stream_ptr()), "hb_poly_soft_bwd")
        return dx, None, None, None, None, None


class _ComplementCEFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x: Tensor, target: Tensor, weight: Optional[Tensor], ignore_index: int, reduction: int,
                gamma: float) -> Tensor:
        require_cuda(x, target)
        xc = x.contiguous()
        n, k, s = _nks(xc)
        tc = _index_targets(target, n, s)
        loss_pos, partials, fwd_out = _position_buffers(x, n, s, 3)
        check(lib().hb_cce_fwd(ptr(xc), ptr(tc), ptr(weight), ptr(loss_pos), ptr(partials), ptr(fwd_out), n, k, s,
                               int(ignore_index), _cf(gamma), dtype_code(xc), stream_ptr()), "hb_cce_fwd")
        ctx.save_for_backward(xc, tc, weight, fwd_out)
        ctx.cfg = (n, k, s, int(ignore_index), reduction, gamma)
        return _reduced(x, loss_pos, fwd_out, reduction)

    @staticmethod
    def backward(ctx, gout: Tensor):
        xc, tc, weight, fwd_out = ctx.saved_tensors
        n, k, s, ignore_index, reduction, gamma = ctx.cfg
        g = _grad(gout)
        dx = torch.empty_like(xc)
        check(lib().hb_cce_bwd(ptr(xc), ptr(tc), ptr(weight), ptr(g), ptr(fwd_out), ptr(dx), n, k, s, ignore_index,
                               _cf(gamma), reduction, dtype_code(xc), stream_ptr()), "hb_cce_bwd")
        return dx, None, None, None, None, None


class _MutualChannelFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x: Tensor, target: Tensor, weight: Optional[Tensor], mask: Tensor, ignore_index: int,
                reduction: int, xi: int, alpha: float) -> Tensor:
        require_cuda(x, target)
        xc = x.contiguous()
        n, c, s = _nks(xc)
        cnum = c // xi
        tc = _index_targets(target, n, s)
        row_lse = torch.empty(n * c, device=x.device, dtype=torch.float32)
        lse_d = torch.empty(n * s, device=x.device, dtype=torch.float32)
        loss_pos, partials, fwd_out = _position_buffers(x, n, s, 3)
        check(lib().hb_mcl_fwd(ptr(xc), ptr(tc), ptr(weight), ptr(mask), ptr(row_lse), ptr(loss_pos), ptr(lse_d),
                               ptr(partials), ptr(fwd_out), n, cnum, xi, s, int(ignore_index), _cf(alpha),
                               dtype_code(xc), stream_ptr()), "hb_mcl_fwd")
        ctx.save_for_backward(xc, tc, weight, mask, row_lse, lse_d, fwd_out)
        ctx.cfg = (n, cnum, xi, s, int(ignore_index), reduction, alpha)
        return _reduced(x, loss_pos, fwd_out, reduction)

    @staticmethod
    def backward(ctx, gout: Tensor):
        xc, tc, weight, mask, row_lse, lse_d, fwd_out = ctx.saved_tensors
        n, cnum, xi, s, ignore_index, reduction, alpha = ctx.cfg
        g = _grad(gout)
        rdot = torch.empty_like(row_lse)
        dx = torch.empty_like(xc)
        check(lib().hb_mcl_bwd(ptr(xc), ptr(tc), ptr(weight), ptr(mask), ptr(row_lse), ptr(lse_d), ptr(g), ptr(fwd_out),
                               ptr(rdot), ptr(dx), n, cnum, xi, s, ignore_index, _cf(alpha), reduction, dtype_code(xc),
                               stream_ptr()), "hb_mcl_bwd")
        return dx, None, None, None, None, None, None, None


def _check_reduction(reduction: str) -> int:
    # the reference treats every value other than "sum" / "mean" as "none"
    return _RED.get(reduction, 0)


def focal_loss(x: Tensor, target: Tensor, weight: Optional[Tensor] = None, ignore_index: int = -100,
               reduction: str = "mean", gamma: float = 2.0) -> Tensor:
    """Focal loss — mirrors holocron/nn/functional.py:59-113, quirks included: the class weight scales
    ``log p_t`` only, ``ignore_index`` is honoured only inside ``[0, K)``, ``'mean'`` averages over the non-ignored
    positions and ``'none'`` is shaped like ``target``. Out-of-range targets give NaN (the reference raises from
    ``gather``; detecting it here would cost a device synchronisation)."""
    out = _HardLossFn.apply(x, target, _weight(weight, x), ignore_index, _check_reduction(reduction), 0, float(gamma), 0.0)
    if _check_reduction(reduction) == 0:
        return out.view(*target.shape)
    return out


def poly_loss(x: Tensor, target: Tensor, eps: float = 2.0, weight: Optional[Tensor] = None, ignore_index: int = -100,
              reduction: str = "mean") -> Tensor:
    """Poly-1 loss — mirrors holocron/nn/functional.py:540-613 for hard (``int64``, ``(N, ...)``) and soft
    (``(N, K, ...)``) targets. ``reduction='none'`` returns the flat ``(N*...,)`` vector for hard targets and
    ``(N, ...)`` for soft ones, as the reference does."""
    if target.ndim == x.ndim - 1:
        if target.dtype != torch.long:
            raise TypeError("target dtype is expected to be torch.int64")
        return _HardLossFn.apply(x, target, _weight(weight, x), ignore_index, _check_reduction(reduction), 1, 0.0,
                                 float(eps))
    if target.ndim != x.ndim or target.shape[0] != x.shape[0] or target.shape[1] != x.shape[1]:
        raise ValueError("invalid target shape")
    if isinstance(weight, Tensor) and x.ndim != 2:
        # the reference broadcasts weight.reshape(1, -1) against the LAST dim there, which is not a class weighting
        raise NotImplementedError("class weights with soft targets are only defined for (N, K) inputs")
    return _PolySoftFn.apply(x, target, _weight(weight, x), ignore_index, _check_reduction(reduction), float(eps))


class _DiceFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x: Tensor, target: Tensor, weight: Optional[Tensor], gamma: float, eps: float) -> Tensor:
        require_cuda(x, target)
        if x.ndim < 3:
            raise IndexError("Dimension out of range (dice_loss expects (N, K, ...) inputs with >= 3 dims)")
        xc = x.contiguous()
        tc = target.to(xc.dtype).contiguous()
        n, k, s = _nks(xc)
        sums = torch.empty(lib().hb_dice_scratch_doubles(k), device=x.device, dtype=torch.float64)
        out = torch.empty(1, device=x.device, dtype=torch.float32)
        coef = torch.empty(2 * k, device=x.device, dtype=torch.float32)
        check(lib().hb_dice_fwd(ptr(xc), ptr(tc), ptr(weight), ptr(sums), ptr(out), ptr(coef), n, k, s, _cf(gamma),
                                _cf(eps), dtype_code(xc), stream_ptr()), "hb_dice_fwd")
        ctx.save_for_backward(tc, coef)
        ctx.cfg = (n, k, s)
        return out[0].to(x.dtype)

    @staticmethod
    def backward(ctx, gout: Tensor):
        tc, coef = ctx.saved_tensors
        n, k, s = ctx.cfg
        g = _grad(gout)
        dx = torch.empty_like(tc)
        check(lib().hb_dice_bwd(ptr(tc), ptr(coef), ptr(g), ptr(dx), n, k, s, dtype_code(tc), stream_ptr()), "hb_dice_bwd")
        return dx, None, None, None, None


def dice_loss(x: Tensor, target: Tensor, weight: Optional[Tensor] = None, gamma: float = 1.0, eps: float = 1e-8) -> Tensor:
    """Dice loss on probabilities — mirrors holocron/nn/functional.py:503-537:
    ``1 - (1 + 1/gamma) * mean_k[(gamma*sum(x*t) + eps) / (sum(x + gamma*t) + eps)]`` with the sums taken jointly over
    batch and space. Two streaming reductions per class in one pass instead of 4 full-tensor temporaries."""
    return _DiceFn.apply(x, target, _weight(weight, x), float(gamma), float(eps))


def _torch_reduction(reduction: str) -> int:
    # the losses built on torch's cross_entropy reject what it rejects
    if reduction not in _RED:
        raise ValueError(f"{reduction} is not a valid value for reduction")
    return _RED[reduction]


def multilabel_cross_entropy(x: Tensor, target: Tensor, weight: Optional[Tensor] = None, ignore_index: int = -100,
                             reduction: str = "mean") -> Tensor:
    """Cross entropy with multi-label (soft) targets — mirrors holocron/nn/functional.py:150-191:
    ``-sum_k t_k w_k log_softmax(x)_k`` over the class axis. ``ignore_index`` drops that class column (only inside
    ``[0, K)``), ``weight`` scales the class axis for any rank, ``'mean'`` averages over the ``N * ...`` positions and
    ``'none'`` is shaped ``(N, ...)``. The soft-target poly-1 kernels with ``eps = 0``."""
    if target.shape != x.shape:
        raise ValueError("invalid target shape")
    return _PolySoftFn.apply(x, target, _weight(weight, x), ignore_index, _check_reduction(reduction), 0.0)


def complement_cross_entropy(x: Tensor, target: Tensor, weight: Optional[Tensor] = None, ignore_index: int = -100,
                             reduction: str = "mean", gamma: float = -1) -> Tensor:
    """Complement cross entropy (https://arxiv.org/abs/2009.02189) — mirrors holocron/nn/functional.py:194-255:
    ``cross_entropy(x, target, weight, ignore_index, reduction) + gamma * C`` with
    ``C = -1/(K-1) sum_{k != y} w_k q_k log q_k`` and ``q`` the softmax over the non-target classes. The cross-entropy
    part follows torch (any ``ignore_index`` drops the row, ``'mean'`` divides by the summed target weights); in ``C``
    ``ignore_index`` drops a class column (only inside ``[0, K)``) and ``'mean'`` averages over every position.
    ``gamma == 0`` is the cross entropy alone. Out-of-range targets give NaN (the reference raises)."""
    red = _torch_reduction(reduction)
    if target.ndim != x.ndim - 1:
        raise ValueError("complement_cross_entropy expects class-index targets of shape (N, ...)")
    if gamma != 0 and x.shape[1] == 1:
        raise ZeroDivisionError("complement_cross_entropy needs at least 2 classes (the term is scaled by 1 / (K - 1))")
    return _ComplementCEFn.apply(x, target.long(), _weight(weight, x), ignore_index, red, float(gamma))


def mutual_channel_mask(cnum: int, xi: int) -> Tensor:
    """The channel mask of the mutual channel loss, drawn as the reference draws it (holocron/nn/functional.py:290-294):
    ``ceil(xi / 2)`` ones per class, placed by one ``torch.randperm(xi)`` per class on the default CPU generator.
    Returns a float32 CPU tensor of shape ``(cnum, xi)``."""
    base = torch.zeros(xi)
    base[: math.ceil(xi / 2)] = 1
    mask = torch.zeros((cnum, xi))
    for idx in range(cnum):
        mask[idx] = base[torch.randperm(xi)]
    return mask


def mutual_channel_loss(x: Tensor, target: Tensor, weight: Optional[Tensor] = None, ignore_index: int = -100,
                        reduction: str = "mean", xi: int = 2, alpha: float = 1.0) -> Tensor:
    """Mutual channel loss (https://arxiv.org/abs/2002.04264) — mirrors holocron/nn/functional.py:258-319 on
    ``x`` of shape ``(N, cnum * xi, ...)``: ``discr - alpha * diversity``, where ``discr`` is torch's cross entropy of the
    per-class maxima of the randomly masked channels (masked channels enter as ``0 * x``) and ``diversity`` the mean over
    classes of the largest spatial softmax among a class' channels. Each call draws a new mask on the host, consuming the
    default CPU generator exactly as the reference does, so the loss cannot be captured into a CUDA graph."""
    b, c = x.shape[:2]
    cnum = c // xi
    if c % xi != 0:
        # what the reference's x.view(b, cnum, xi, -1) raises
        raise RuntimeError(f"shape '[{b}, {cnum}, {xi}, -1]' is invalid for input of size {x.numel()}")
    require_cuda(x, target)
    if torch.cuda.is_current_stream_capturing():
        raise RuntimeError("mutual_channel_loss draws a new channel mask on the host at every call and cannot run "
                           "inside CUDA graph capture; keep it out of the captured region (e.g. TrainStep(graph=False))")
    # pinned + non-blocking: a pageable copy would wait for the work already queued on the stream
    mask = mutual_channel_mask(cnum, xi).to(torch.uint8).view(-1).pin_memory().to(x.device, non_blocking=True)
    red = _torch_reduction(reduction)
    if target.ndim != x.ndim - 1:
        raise ValueError("mutual_channel_loss expects class-index targets of shape (N, ...)")
    return _MutualChannelFn.apply(x, target.long(), _weight(weight, x), mask, ignore_index, red, int(xi), float(alpha))
