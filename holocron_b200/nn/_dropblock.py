"""dropblock2d on the fused CUDA kernels (holocron_b200/csrc/dropblock.cu)."""
import ctypes
from typing import Optional

import torch
from torch import Tensor

from .._lib import check, dtype_code, lib, ptr, require_cuda, stream_ptr


class _DropBlockFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x: Tensor, noise: Tensor, gamma: float, block_size: int, inplace: bool) -> Tensor:
        require_cuda(x)
        if x.ndim != 4:
            raise ValueError("dropblock2d expects (N, C, H, W) inputs")
        cl = x.is_contiguous(memory_format=torch.channels_last) and not x.is_contiguous()
        if not cl and not x.is_contiguous():
            if inplace:
                raise RuntimeError("dropblock2d(inplace=True) needs a dense (contiguous / channels_last) tensor")
            x = x.contiguous()
        n, c, h, w = x.shape
        L = lib()
        mask = torch.empty((n, h, w), device=x.device, dtype=torch.float32)
        kept = torch.empty(1, device=x.device, dtype=torch.int64)  # the kernels' 64-bit count of kept cells
        check(L.hb_dropblock_mask(ptr(noise), ptr(mask), ptr(kept), n, h, w, block_size, ctypes.c_float(gamma),
                                  stream_ptr()), "hb_dropblock_mask")
        out = x if inplace else torch.empty_like(x)
        check(L.hb_dropblock_apply(ptr(x), ptr(out), ptr(mask), ptr(kept), n, c, h, w, int(cl), dtype_code(x),
                                   stream_ptr()), "hb_dropblock_apply")
        if inplace:
            ctx.mark_dirty(x)
        ctx.save_for_backward(mask, kept)
        ctx.cl = cl
        return out

    @staticmethod
    def backward(ctx, dy: Tensor):
        mask, kept = ctx.saved_tensors
        n, c, h, w = dy.shape
        dyc = dy.contiguous(memory_format=torch.channels_last) if ctx.cl else dy.contiguous()
        dx = torch.empty_like(dyc)
        check(lib().hb_dropblock_apply(ptr(dyc), ptr(dx), ptr(mask), ptr(kept), n, c, h, w, int(ctx.cl), dtype_code(dyc),
                                       stream_ptr()), "hb_dropblock_apply[bwd]")
        return dx, None, None, None, None


def dropblock2d(x: Tensor, drop_prob: float, block_size: int, inplace: bool = False, training: bool = True,
                noise: Optional[Tensor] = None) -> Tensor:
    """DropBlock — mirrors holocron/nn/functional.py:465-500: seeds are drawn with probability
    ``drop_prob / block_size**2`` on an (N, H, W) grid shared by all channels, dilated to ``block_size`` squares, and
    the survivors are rescaled by ``mask.numel() / mask.sum()``. ``drop_prob == 0`` or ``training=False`` returns the
    input object itself. No host synchronisation (the reference syncs on ``mask.sum() > 0``).

    The kept cells are counted exactly, in an integer, and the scale is rounded as the reference rounds
    ``mask.numel() / one_count`` (``one_count.reciprocal() * numel``), so fp32 inputs give the reference's output bit
    for bit for the same noise. For bf16 / fp16 inputs the reference builds its mask in ``x.dtype``, so its count and
    scale are rounded to that type (a count of 6000 becomes 6016 in bf16); here the count stays exact and the scale
    fp32, and the output is ``x * numel / kept`` rounded once to ``x.dtype``.

    ``noise`` (not in the reference API) lets tests inject the uniform noise the reference would have drawn.
    """
    if not training or drop_prob == 0:
        return x
    gamma = drop_prob / block_size**2
    if noise is None:
        noise = torch.rand((x.shape[0], *x.shape[2:]), device=x.device)
    noise = noise.to(device=x.device, dtype=torch.float32).contiguous()
    return _DropBlockFn.apply(x, noise, float(gamma), int(block_size), inplace)
