"""Depth-wise convolution autograd binding + FReLU forward (holocron_b200/csrc/dwconv.cu)."""
from typing import Optional

import torch
from torch import Tensor, nn

from .._lib import check, lib, ptr, require_cuda, stream_ptr
from . import _fused as K


class _DwConvFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x: Tensor, weight: Tensor, bias: Optional[Tensor], stride: int, pad: int) -> Tensor:
        require_cuda(x, weight)
        c, one, k, k2 = weight.shape
        if one != 1 or k != k2:
            raise ValueError("depth-wise filter expected as (C, 1, k, k)")
        xb = K.to_channels_last_bf16(x)
        n, cx, h, w = xb.shape
        if cx != c or c % 8 != 0:
            raise NotImplementedError("depth-wise kernel needs channels % 8 == 0 and groups == channels")
        ho, wo = (h + 2 * pad - k) // stride + 1, (w + 2 * pad - k) // stride + 1
        w32 = weight.detach().float().contiguous()
        b32 = None if bias is None else bias.detach().float().contiguous()
        y = K._empty_cl(n, c, ho, wo, xb.device)
        if n > 0:       # an empty batch launches nothing: the C ABI refuses N < 1
            check(lib().hb_dwconv_fwd_bf16(ptr(xb), ptr(w32), ptr(b32), ptr(y), n, h, w, c, k, stride, pad, stream_ptr()),
                  "hb_dwconv_fwd_bf16")
        ctx.save_for_backward(xb, w32)
        ctx.cfg = (stride, pad, bias is not None)
        return y

    @staticmethod
    def backward(ctx, dy: Tensor):
        xb, w32 = ctx.saved_tensors
        stride, pad, has_bias = ctx.cfg
        n, c, h, w = xb.shape
        k = w32.shape[-1]
        dyb = K.to_channels_last_bf16(dy)
        L = lib()
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = K._empty_cl(n, c, h, w, dyb.device)
            if n > 0:
                check(L.hb_dwconv_bwd_data_bf16(ptr(dyb), ptr(w32), ptr(dx), n, h, w, c, k, stride, pad, stream_ptr()),
                      "hb_dwconv_bwd_data_bf16")
        if ctx.needs_input_grad[1] or (has_bias and ctx.needs_input_grad[2]):
            dw = torch.empty((c, 1, k, k), device=dyb.device, dtype=torch.float32)
            db = torch.empty(c, device=dyb.device, dtype=torch.float32) if has_bias else None
            if n == 0:
                dw.zero_()
                if db is not None:
                    db.zero_()
                return dx, dw, db, None, None
            sums = torch.empty(L.hb_dwconv_wgrad_scratch_doubles(c, k), device=dyb.device, dtype=torch.float64)
            check(L.hb_dwconv_bwd_weight_bf16(ptr(xb), ptr(dyb), ptr(dw), ptr(db), ptr(sums), n, h, w, c, k, stride, pad,
                                              stream_ptr()), "hb_dwconv_bwd_weight_bf16")
        return dx, dw, db, None, None


def dwconv2d(x: Tensor, weight: Tensor, bias: Optional[Tensor] = None, stride: int = 1, padding: int = 0) -> Tensor:
    """Depth-wise (groups == channels) convolution; bf16 channels_last in/out, fp32 filter."""
    return _DwConvFn.apply(x, weight, bias, int(stride), int(padding))


def frelu_forward(x: Tensor, conv: nn.Conv2d, bn: nn.BatchNorm2d) -> Tensor:
    """max(x, BN(dwconv(x) + bias)): depth-wise kernel, then ONE fused pass that normalises and takes the max with x
    (training: + one statistics pass). Reference: 3 kernels (cuDNN dw-conv, BatchNorm, max)."""
    t = dwconv2d(x, conv.weight, conv.bias, conv.stride[0], conv.padding[0])
    xb = K.to_channels_last_bf16(x)
    return K.bn_act([t], [bn], K.ACT_FRELU, 0.0, residual=xb)
