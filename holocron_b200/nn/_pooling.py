"""Pooling autograd bindings (holocron_b200/csrc/pooling.cu): the reference's ``BlurPool2d`` (ReflectionPad2d then a
depth-wise conv2d, holocron/nn/modules/downsample.py:106-151) without the padded copy, and the max / mean reductions of
``GlobalMaxPool2d`` (:80-99) and ``z_pool`` (holocron/nn/functional.py:139-147) with their backward passes writing the
input gradient once, without a zero-filled scatter target or a ``torch.cat``.

bf16 and fp32 tensors run natively, other float dtypes in fp32 (``_nhwc``). 4-D outputs are channels_last."""
import ctypes
from typing import Tuple

import torch
from torch import Tensor

from .._lib import check, dtype_code, lib, ptr, require_cuda, stream_ptr
from ._fused import _empty_cl
from ._nhwc import crop, nhwc, pitch as _pitch, require_4d, run_native

MAX_BLUR_KERNEL = 7
Z_POOL_DIMS = (1, 2, 3, -1, -2, -3)


def blur_padding(kernel_size: int, stride: int) -> int:
    """The reflection padding of the reference (get_padding with dilation 1, downsample.py:102-103)."""
    return ((stride - 1) + (kernel_size - 1)) // 2


def check_blurpool(channels: int, shape: Tuple[int, ...], kernel_size: int, stride: int) -> Tuple[int, int]:
    """Raises what the reference raises, before anything is launched, and returns the output grid (Ho, Wo).

    ReflectionPad2d refuses a padding that reaches the size of a side, and the depth-wise conv2d refuses a padded side
    shorter than the filter, an input whose channel count differs from ``channels`` (its groups check) or a
    non-positive stride: RuntimeError each.
    ``kernel_size`` above 7 has no kernel here: NotImplementedError."""
    if len(shape) != 4:
        raise NotImplementedError(f"BlurPool2d: 4-D (N, C, H, W) inputs only, got shape {tuple(shape)}")
    _, c, h, w = shape
    pad = blur_padding(kernel_size, stride)
    if pad >= h or pad >= w:
        raise RuntimeError(f"BlurPool2d: padding size {pad} must be less than the input sides {h}x{w}")
    if min(h, w) + 2 * pad < kernel_size:
        raise RuntimeError(f"BlurPool2d: padded input {h + 2 * pad}x{w + 2 * pad} is smaller than the kernel size "
                           f"{kernel_size}")
    if c != channels:
        raise RuntimeError(f"BlurPool2d: built for {channels} channels, got an input with {c}")
    if stride < 1:
        raise RuntimeError(f"BlurPool2d: non-positive stride {stride}")
    if kernel_size > MAX_BLUR_KERNEL:
        raise NotImplementedError(f"BlurPool2d: kernel_size {kernel_size} (supported: 2..{MAX_BLUR_KERNEL})")
    return (h + 2 * pad - kernel_size) // stride + 1, (w + 2 * pad - kernel_size) // stride + 1


def blur_taps(coeffs: Tensor, dtype: torch.dtype):
    """The 2-D filter as the reference builds it (the outer product of the float64 coefficients cast to the input
    dtype, downsample.py:140-142), as a host array of fp32 values for the kernel."""
    taps = (coeffs[:, None] * coeffs[None, :]).to(dtype).float().flatten().tolist()
    return (ctypes.c_float * len(taps))(*taps)


class _BlurPoolFn(torch.autograd.Function):
    """x [N, C, H, W] -> y [N, Cp, Ho, Wo] channels_last (the caller drops the padding channels)."""

    @staticmethod
    def forward(ctx, x: Tensor, taps, k: int, stride: int) -> Tensor:
        n, c, h, w = x.shape
        cp = _pitch(c, x.dtype)
        pad = blur_padding(k, stride)
        ho, wo = (h + 2 * pad - k) // stride + 1, (w + 2 * pad - k) // stride + 1
        xc = nhwc(x, cp)
        y = _empty_cl(n, cp, ho, wo, xc.device, xc.dtype)
        check(lib().hb_blurpool_fwd(ptr(xc), ptr(y), ctypes.cast(taps, ctypes.c_void_p), n, h, w, c, cp, k, stride,
                                    dtype_code(xc), stream_ptr()), "hb_blurpool_fwd")
        ctx.cfg = (taps, k, stride, c, h, w)
        return y

    @staticmethod
    def backward(ctx, dy: Tensor):
        taps, k, stride, c, h, w = ctx.cfg
        n, cp = dy.shape[:2]
        dyc = dy.contiguous(memory_format=torch.channels_last)
        dx = _empty_cl(n, cp, h, w, dyc.device, dyc.dtype)
        check(lib().hb_blurpool_bwd(ptr(dyc), ptr(dx), ctypes.cast(taps, ctypes.c_void_p), n, h, w, c, cp, k, stride,
                                    dtype_code(dyc), stream_ptr()), "hb_blurpool_bwd")
        return crop(dx, c), None, None, None


# Reduction modes: "hw" reduces H*W (global max pooling), 1 / 2 / 3 reduce that dim into (max, mean) (z_pool).
def _mid_view(mode, n: int, cp: int, h: int, w: int):
    """(A, L, M, output shape) of a middle-axis reduction of an NHWC tensor with row pitch cp."""
    if mode == "hw":
        return n, h * w, cp, (n, cp, 1, 1)
    if mode == 2:
        return n, h, w * cp, (n, cp, 2, w)
    return n * h, w, cp, (n, cp, h, 2)


class _ReduceFn(torch.autograd.Function):
    """x [N, C, H, W] -> the max (and mean) over ``mode``, channels_last; the channel-padded modes return Cp channels
    (the caller drops the padding channels). The int32 index of the max is kept for the backward pass."""

    @staticmethod
    def forward(ctx, x: Tensor, mode) -> Tensor:
        n, c, h, w = x.shape
        cp = _pitch(c, x.dtype)
        xc = nhwc(x, cp)
        L = lib()
        if mode == 1:
            y = _empty_cl(n, 2, h, w, xc.device, xc.dtype)
            idx = torch.empty(n * h * w, dtype=torch.int32, device=x.device)
            check(L.hb_pool_last_fwd(ptr(xc), ptr(y), ptr(idx), n * h * w, c, cp, dtype_code(xc), stream_ptr()),
                  "hb_pool_last_fwd")
        else:
            a, l, m, shape = _mid_view(mode, n, cp, h, w)
            y = _empty_cl(*shape, xc.device, xc.dtype)
            idx = torch.empty(a * m, dtype=torch.int32, device=x.device)
            check(L.hb_pool_mid_fwd(ptr(xc), ptr(y), ptr(idx), a, l, m, c, cp, int(mode != "hw"), dtype_code(xc),
                                    stream_ptr()), "hb_pool_mid_fwd")
        ctx.save_for_backward(idx)
        ctx.cfg = (mode, c, cp, h, w)
        return y

    @staticmethod
    def backward(ctx, dy: Tensor):
        (idx,) = ctx.saved_tensors
        mode, c, cp, h, w = ctx.cfg
        n = dy.shape[0]
        dyc = dy.contiguous(memory_format=torch.channels_last)
        dx = _empty_cl(n, cp, h, w, dyc.device, dyc.dtype)
        L = lib()
        if mode == 1:
            check(L.hb_pool_last_bwd(ptr(dyc), ptr(idx), ptr(dx), n * h * w, c, cp, dtype_code(dyc), stream_ptr()),
                  "hb_pool_last_bwd")
        else:
            a, l, m, _ = _mid_view(mode, n, cp, h, w)
            check(L.hb_pool_mid_bwd(ptr(dyc), ptr(idx), ptr(dx), a, l, m, c, cp, int(mode != "hw"), dtype_code(dyc),
                                    stream_ptr()), "hb_pool_mid_bwd")
        return crop(dx, c), None


def blur_pool2d(x: Tensor, coeffs: Tensor, channels: int, kernel_size: int, stride: int) -> Tensor:
    """BlurPool2d's forward (reference downsample.py:148-151): the reflection-padded depth-wise binomial filter."""
    check_blurpool(channels, tuple(x.shape), kernel_size, stride)
    require_cuda(x)
    return run_native(_BlurPoolFn, x, blur_taps(coeffs, x.dtype), int(kernel_size), int(stride))


def global_max_pool2d(x: Tensor) -> Tensor:
    """(N, C, H, W) -> (N, C, 1, 1): the max over space; its gradient goes to the element max(dim).indices names."""
    require_4d("GlobalMaxPool2d", x)
    require_cuda(x)
    return run_native(_ReduceFn, x, "hw")


def z_pool(x: Tensor, dim: int) -> Tensor:
    """cat([x.max(dim, keepdim=True).values, x.mean(dim, keepdim=True)], dim) of a 4-D tensor, dim in 1..3 (or its
    negative form)."""
    if x.ndim != 4 or dim not in Z_POOL_DIMS:
        raise NotImplementedError(f"z_pool: 4-D inputs with dim in {Z_POOL_DIMS} only, got shape {tuple(x.shape)} "
                                  f"and dim {dim}")
    require_cuda(x)
    dim = dim % 4
    return run_native(_ReduceFn, x, dim, crop_channels=dim != 1)
