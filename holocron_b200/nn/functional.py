"""Functional API mirroring ``holocron.nn.functional`` (reference holocron/nn/functional.py) for the hot-path ops.

Every function here launches the sm_90a kernels of ``libholocron_b200.so`` through the C ABI; inputs must be CUDA
tensors (there is no CPU fallback — the CPU restatement lives in ``oracle/`` and is test-only).
"""
from typing import Optional

import torch
from torch import Tensor

from .._lib import check, dtype_code, lib, ptr, require_cuda, stream_ptr
from ._losses import (complement_cross_entropy, dice_loss, focal_loss, multilabel_cross_entropy,  # noqa: F401
                      mutual_channel_loss, poly_loss)
from ._xcorr import add2d, norm_conv2d  # noqa: F401
from ._dropblock import dropblock2d  # noqa: F401
from ._pooling import z_pool  # noqa: F401

import ctypes

__all__ = ["add2d", "complement_cross_entropy", "concat_downsample2d", "dice_loss", "dropblock2d", "focal_loss", "hard_mish",
           "multilabel_cross_entropy", "mutual_channel_loss", "nl_relu", "norm_conv2d", "poly_loss", "z_pool"]

_cf = ctypes.c_float


def _dense(x: Tensor) -> bool:
    return x.is_contiguous() or (x.ndim == 4 and x.is_contiguous(memory_format=torch.channels_last))


class _HardMishFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x: Tensor, inplace: bool) -> Tensor:
        require_cuda(x)
        if not _dense(x):
            if inplace:
                raise RuntimeError("hard_mish(inplace=True) needs a dense (contiguous / channels_last) tensor")
            x = x.contiguous()
        if inplace:
            # autograd needs the pre-activation values: keep a copy (what PyTorch's own in-place mul_ does)
            if ctx.needs_input_grad[0]:
                ctx.save_for_backward(x.clone())
            out = x
            ctx.mark_dirty(x)
        else:
            ctx.save_for_backward(x)
            out = torch.empty_like(x)
        check(lib().hb_hard_mish_fwd(ptr(x), ptr(out), x.numel(), dtype_code(x), stream_ptr()), "hb_hard_mish_fwd")
        return out

    @staticmethod
    def backward(ctx, dy: Tensor):
        (x,) = ctx.saved_tensors
        dyc = dy.to(x.dtype)
        if dyc.stride() != x.stride():
            dyc = torch.empty_like(x).copy_(dyc)
        dx = torch.empty_like(x)
        check(lib().hb_hard_mish_bwd(ptr(x), ptr(dyc), ptr(dx), x.numel(), dtype_code(x), stream_ptr()),
              "hb_hard_mish_bwd")
        return dx, None


def hard_mish(x: Tensor, inplace: bool = False) -> Tensor:
    """HardMish activation ``x/2 * min(2, max(0, x + 2))`` — mirrors holocron/nn/functional.py:30-41.

    One 128-bit-vectorised HBM pass (the reference needs 3 ATen kernels and 2 temporaries). With
    ``inplace=True`` the returned tensor aliases ``x``.
    """
    return _HardMishFn.apply(x, inplace)


class _NLReluFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x: Tensor, beta: float, inplace: bool) -> Tensor:
        require_cuda(x)
        if not _dense(x):
            if inplace:
                raise RuntimeError("nl_relu(inplace=True) needs a dense (contiguous / channels_last) tensor")
            x = x.contiguous()
        out = x if inplace else torch.empty_like(x)
        check(lib().hb_nl_relu_fwd(ptr(x), ptr(out), x.numel(), _cf(beta), dtype_code(x), stream_ptr()),
              "hb_nl_relu_fwd")
        ctx.beta = beta
        ctx.from_out = inplace
        if inplace:
            ctx.mark_dirty(x)
            ctx.save_for_backward(out)  # the gradient is recoverable from the output: beta * exp(-y)
        else:
            ctx.save_for_backward(x)
        return out

    @staticmethod
    def backward(ctx, dy: Tensor):
        (t,) = ctx.saved_tensors
        dyc = dy.to(t.dtype)
        if dyc.stride() != t.stride():
            dyc = torch.empty_like(t).copy_(dyc)
        dx = torch.empty_like(t)
        fn = lib().hb_nl_relu_bwd_from_out if ctx.from_out else lib().hb_nl_relu_bwd
        check(fn(ptr(t), ptr(dyc), ptr(dx), t.numel(), _cf(ctx.beta), dtype_code(t), stream_ptr()), "hb_nl_relu_bwd")
        return dx, None, None


def nl_relu(x: Tensor, beta: float = 1.0, inplace: bool = False) -> Tensor:
    """Natural-logarithm ReLU ``log(1 + beta * max(0, x))`` — mirrors holocron/nn/functional.py:44-56.

    With ``inplace=True`` ``x`` is overwritten, so the backward pass computes the gradient from the output as
    ``beta * exp(-y)``. Two differences from the out-of-place gradient ``beta / (1 + beta * x)`` follow:

    - where ``0 < beta * x < 2**-24``, ``y`` rounds to 0 and the gradient is 0 instead of ``beta * dy``;
    - for bf16 / fp16 tensors ``y`` is stored rounded, so the gradient carries that rounding: a relative error of up to
      ``y * 2**-8`` (bf16) or ``y * 2**-11`` (fp16).
    """
    return _NLReluFn.apply(x, float(beta), inplace)


def concat_downsample2d(x: Tensor, scale_factor: int) -> Tensor:
    """Loss-less down-sampling of YOLOv2's pass-through route (reference nn/functional.py:116-136): every
    ``scale_factor x scale_factor`` pixel block is stacked on the channel axis, output channel order (row offset, column
    offset, channel). Pure data movement (one strided copy, any input layout; the reference's ``view`` needs a contiguous
    NCHW tensor), so it is the same code on every device."""
    b, c, h, w = x.shape
    if (h % scale_factor != 0) or (w % scale_factor != 0):
        raise AssertionError("Spatial size of input tensor must be multiples of `scale_factor`")
    x = x.reshape(b, c, h // scale_factor, scale_factor, w // scale_factor, scale_factor)
    return x.permute(0, 3, 5, 1, 2, 4).reshape(b, int(c * scale_factor**2), h // scale_factor, w // scale_factor)
