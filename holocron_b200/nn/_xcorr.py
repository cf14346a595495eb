"""norm_conv2d / add2d (holocron/nn/functional.py:322-462).

``norm_conv2d`` is a dense contraction: it runs on the wgmma implicit-GEMM convolution (bf16 operands, fp32 accumulation)
with the per-patch standardisation folded algebraically into the epilogue,

    out[m, co] = rstd[m] * (conv(x, w)[m, co] - mean[m] * sum_k w[co, k]) + bias[co],

the patch statistics coming from one streaming pass over x (``hb_patch_stats_bf16``); nothing like the reference's
``N x L x Cin*k*k`` im2col tensor exists. ``HB_NORMCONV_FP32=1`` selects the fp32 CUDA-core kernel instead (bit-level
closeness to the fp32 reference, far slower). ``add2d`` has no multiplications (L1 distance): it stays on the fp32
CUDA-core tile kernel of ``csrc/xcorr.cu``; so do the weight gradients of both ops."""
import ctypes
import os
from typing import Optional, Tuple, Union

import torch
from torch import Tensor

from .._lib import check, lib, ptr, require_cuda, stream_ptr

_cf = ctypes.c_float


def _single(v: Union[int, Tuple[int, int]], what: str) -> int:
    if isinstance(v, (tuple, list)):
        if len(v) != 2 or v[0] != v[1]:
            raise NotImplementedError(f"only symmetric {what} is supported by the fused kernel")
        return int(v[0])
    return int(v)


def _out_size(h: int, w: int, kh: int, kw: int, stride: int, pad: int, dil: int) -> Tuple[int, int]:
    """(Ho, Wo) of the sliding windows, refused with the errors of F.unfold, which the reference's forward calls."""
    if stride <= 0:
        raise RuntimeError(f"stride should be greater than zero, but got stride_height: {stride} stride_width: {stride}")
    if dil <= 0:
        raise RuntimeError(f"dilation should be greater than zero, but got dilation_height: {dil} dilation_width: {dil}")
    if pad < 0:
        raise RuntimeError(f"padding should be non-negative, but got pad_height: {pad} pad_width: {pad}")
    span_h, span_w = h + 2 * pad - dil * (kh - 1) - 1, w + 2 * pad - dil * (kw - 1) - 1
    if span_h < 0 or span_w < 0:
        raise RuntimeError(f"Given input with spatial size ({h}, {w}), kernel_size=({kh}, {kw}), dilation=({dil}, {dil}), "
                           f"padding=({pad}, {pad}), calculated shape of the array of sliding blocks as "
                           f"({span_h // stride + 1}, {span_w // stride + 1}), but its components must be at least one.")
    return span_h // stride + 1, span_w // stride + 1


class _XcorrFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x: Tensor, weight: Tensor, bias: Optional[Tensor], stride: int, pad: int, dil: int, mode: int,
                normalize: bool, eps: float) -> Tensor:
        if x.ndim != 4 or weight.ndim != 4:
            raise ValueError("expected (N, C, H, W) input and (Cout, Cin, kh, kw) weight")
        n, cin, h, w = x.shape
        cout, cin_w, kh, kw = weight.shape
        ho, wo = _out_size(h, w, kh, kw, stride, pad, dil)
        require_cuda(x, weight)
        if cin_w != cin:
            # the reference ignores `groups`: a grouped weight makes its matmul fail with a shape error
            raise RuntimeError(f"weight expects {cin_w} input channels but the input has {cin} (groups are ignored)")
        x32 = x.detach().float().contiguous()
        w32 = weight.detach().float().contiguous()
        b32 = None if bias is None else bias.detach().float().contiguous()
        mean = torch.empty(n * ho * wo if normalize else 1, device=x.device, dtype=torch.float32)
        rstd = torch.empty_like(mean)
        if n == 0:
            # an empty batch has no windows (F.unfold gives an empty tensor); the kernels refuse an empty launch
            out = torch.empty((0, cout, ho, wo), device=x.device, dtype=torch.float32)
        elif mode == 0 and normalize and kh == kw and not os.environ.get("HB_NORMCONV_FP32"):
            out = _norm_conv_tensor_cores(x32, weight, b32, mean, rstd, stride, pad, dil, eps)
        else:
            out = torch.empty((n, cout, ho, wo), device=x.device, dtype=torch.float32)
            check(lib().hb_xcorr2d_fwd(ptr(x32), ptr(w32), ptr(b32), ptr(out), ptr(mean), ptr(rstd), n, cin, h, w, cout, kh,
                                       kw, stride, pad, dil, mode, int(normalize), _cf(eps), stream_ptr()), "hb_xcorr2d_fwd")
        ctx.save_for_backward(x32, w32, mean, rstd)
        ctx.cfg = (stride, pad, dil, mode, normalize, eps, bias is not None, x.dtype, weight.dtype)
        return out.to(x.dtype)

    @staticmethod
    def backward(ctx, gout: Tensor):
        x32, w32, mean, rstd = ctx.saved_tensors
        stride, pad, dil, mode, normalize, eps, has_bias, xdt, wdt = ctx.cfg
        n, cin, h, w = x32.shape
        cout, _, kh, kw = w32.shape
        g = gout.detach().float().contiguous()
        L = lib()
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            if normalize or mode == 0:
                # same situation as the reference, whose in-place slice normalisation makes autograd raise
                raise RuntimeError("the input gradient of a slice-normalised cross-correlation is not defined by the "
                                   "reference (its in-place normalisation breaks autograd); only add2d without "
                                   "normalize_slices propagates to the input")
            dx = torch.empty_like(x32)
            if n:
                check(L.hb_add2d_dgrad(ptr(x32), ptr(w32), ptr(g), ptr(dx), n, cin, h, w, cout, kh, kw, stride, pad, dil,
                                       stream_ptr()), "hb_add2d_dgrad")
            dx = dx.to(xdt)
        if ctx.needs_input_grad[1]:
            dw = torch.empty_like(w32) if n else torch.zeros_like(w32)    # the launcher zeroes dw itself
            if n:
                check(L.hb_xcorr2d_wgrad(ptr(x32), ptr(w32), ptr(g), ptr(mean), ptr(rstd), ptr(dw), n, cin, h, w, cout, kh,
                                         kw, stride, pad, dil, mode, int(normalize), _cf(eps), stream_ptr()),
                      "hb_xcorr2d_wgrad")
            dw = dw.to(wdt)
        if has_bias and ctx.needs_input_grad[2]:
            db = g.sum((0, 2, 3))
        return dx, dw, db, None, None, None, None, None, None


def _norm_conv_tensor_cores(x32: Tensor, weight: Tensor, b32: Optional[Tensor], mean: Tensor, rstd: Tensor, stride: int,
                            pad: int, dil: int, eps: float) -> Tensor:
    """Forward of norm_conv2d on the tensor-core kernel; fills ``mean`` / ``rstd`` (per output pixel) for the backward pass."""
    from . import _fused as K
    n, cin, h, w = x32.shape
    k = weight.shape[2]

    def patch_norm(xb: Tensor, pk):
        scratch = torch.empty(2 * n * h * w, device=x32.device, dtype=torch.float32)
        check(lib().hb_patch_stats_bf16(ptr(xb), ptr(mean), ptr(rstd), ptr(scratch), n, h, w, pk.cin_p, k, k, stride, pad,
                                        dil, cin * k * k, _cf(eps), stream_ptr()), "hb_patch_stats_bf16")
        return mean, rstd, pk.wf.float().sum((1, 2, 3))             # sum of the SAME bf16 filter values the MMAs read

    y, _, _ = K._packed_conv(x32, weight, b32, stride, pad, dil, norm=patch_norm)
    return y.float().contiguous()


def norm_conv2d(x: Tensor, weight: Tensor, bias: Optional[Tensor] = None, stride: Union[int, Tuple[int, int]] = 1,
                padding: Union[int, Tuple[int, int]] = 0, dilation: Union[int, Tuple[int, int]] = 1, groups: int = 1,
                eps: float = 1e-14) -> Tensor:
    """Normalised convolution — mirrors holocron/nn/functional.py:378-413: every im2col patch (the whole
    ``Cin*kh*kw`` vector, zero padding included) is standardised with its biased variance, then correlated with the
    filters. ``groups`` is accepted and ignored, as in the reference. No im2col tensor is materialised. Runs on the tensor
    cores (bf16 operands: ~3e-3 relative to the fp32 reference; see the module docstring for the fp32 switch)."""
    return _XcorrFn.apply(x, weight, bias, _single(stride, "stride"), _single(padding, "padding"),
                          _single(dilation, "dilation"), 0, True, float(eps))


def add2d(x: Tensor, weight: Tensor, bias: Optional[Tensor] = None, stride: Union[int, Tuple[int, int]] = 1,
          padding: Union[int, Tuple[int, int]] = 0, dilation: Union[int, Tuple[int, int]] = 1, groups: int = 1,
          normalize_slices: bool = False, eps: float = 1e-14) -> Tensor:
    """AdderNet layer ``-sum_k |patch_k - w_k|`` — mirrors holocron/nn/functional.py:426-462. The reference broadcasts
    an ``N x L x Cout x K`` tensor; here the L1 distances are accumulated tile by tile in shared memory."""
    return _XcorrFn.apply(x, weight, bias, _single(stride, "stride"), _single(padding, "padding"),
                          _single(dilation, "dilation"), 1, bool(normalize_slices), float(eps))
