"""Involution autograd binding (holocron_b200/csrc/involution.cu) - the unfold / multiply / sum of the reference's
``Involution2d.forward`` (holocron/nn/modules/conv.py:481-499) without the unfolded tensor."""
from torch import Tensor
import torch

from .._lib import check, lib, ptr, require_cuda, stream_ptr
from . import _fused as K
from ._nhwc import crop

SUPPORTED_KERNEL_SIZES = (1, 3, 5, 7)


def check_involution(in_channels: int, height: int, width: int, kernel_size: int, stride: int, padding: int,
                     dilation: int, groups: int):
    """Raises what the reference raises for shapes it cannot compute, before anything is launched, and returns the
    output grid (Ho, Wo).

    The reference reshapes the unfolded input onto the grid of the generated kernel, ``H // stride`` after the pooling;
    when the unfold grid differs (``padding=0`` with ``kernel_size=3``, an odd height with ``stride=2``) or the channels
    do not split into ``groups``, its reshape or product fails with a RuntimeError. ``kernel_size`` outside
    {1, 3, 5, 7} has no kernel here."""
    _check_groups_and_size(in_channels, kernel_size, groups)
    ho, wo = unfold_grid(height, width, kernel_size, stride, padding, dilation)
    if (ho, wo) != (height // stride, width // stride):
        raise RuntimeError(f"Involution2d: the unfold grid {ho}x{wo} differs from the kernel grid "
                           f"{height // stride}x{width // stride} of a {height}x{width} input")
    return ho, wo


def unfold_grid(height: int, width: int, kernel_size: int, stride: int, padding: int, dilation: int):
    return tuple((s + 2 * padding - dilation * (kernel_size - 1) - 1) // stride + 1 for s in (height, width))


def _check_groups_and_size(in_channels: int, kernel_size: int, groups: int) -> None:
    if in_channels % groups != 0:
        raise RuntimeError(f"Involution2d: {in_channels} channels do not split into {groups} groups")
    if kernel_size not in SUPPORTED_KERNEL_SIZES:
        raise NotImplementedError(f"Involution2d: kernel_size {kernel_size} (supported: {SUPPORTED_KERNEL_SIZES})")


class _InvolutionFn(torch.autograd.Function):
    """y = involution(x, kernel): x [N, C, H, W], kernel [N, Kp >= G*K*K, Ho, Wo] -> y [N, C, Ho, Wo], all bf16
    channels_last. Backward: the data gradient (gather form) and the kernel gradient (padding columns zero), each only
    when asked for."""

    @staticmethod
    def forward(ctx, x: Tensor, kernel: Tensor, k: int, stride: int, pad: int, dil: int, groups: int) -> Tensor:
        n, c, h, w = x.shape
        _check_groups_and_size(c, k, groups)
        ho, wo = unfold_grid(h, w, k, stride, pad, dil)
        if ho < 1 or wo < 1 or kernel.shape[0] != n or kernel.shape[1] < groups * k * k or tuple(kernel.shape[2:]) != (ho, wo):
            raise RuntimeError(f"Involution2d: kernel of shape {tuple(kernel.shape)} for a {n}x{c}x{h}x{w} input")
        cp = K.round_up(c, 8)
        xb = K.to_channels_last_bf16(x, cp)
        kb = K.to_channels_last_bf16(kernel)
        kp = kb.shape[1]
        y = K._empty_cl(n, cp, ho, wo, xb.device)
        check(lib().hb_involution_fwd_bf16(ptr(xb), ptr(kb), ptr(y), n, h, w, c, cp, kp, k, groups, stride, pad, dil,
                                           stream_ptr()), "hb_involution_fwd_bf16")
        ctx.save_for_backward(xb, kb)
        ctx.cfg = (c, k, stride, pad, dil, groups)
        return crop(y, c)

    @staticmethod
    def backward(ctx, dy: Tensor):
        xb, kb = ctx.saved_tensors
        c, k, stride, pad, dil, groups = ctx.cfg
        n, cp, h, w = xb.shape
        kp, ho, wo = kb.shape[1], kb.shape[2], kb.shape[3]
        dyb = K.to_channels_last_bf16(dy, cp)
        L = lib()
        dx = dker = None
        if ctx.needs_input_grad[0]:
            dxp = K._empty_cl(n, cp, h, w, dyb.device)
            check(L.hb_involution_bwd_data_bf16(ptr(dyb), ptr(kb), ptr(dxp), n, h, w, c, cp, kp, k, groups, stride, pad,
                                                dil, stream_ptr()), "hb_involution_bwd_data_bf16")
            dx = crop(dxp, c)
        if ctx.needs_input_grad[1]:
            dker = K._empty_cl(n, kp, ho, wo, dyb.device)
            check(L.hb_involution_bwd_kernel_bf16(ptr(xb), ptr(dyb), ptr(dker), n, h, w, c, cp, kp, k, groups, stride,
                                                  pad, dil, stream_ptr()), "hb_involution_bwd_kernel_bf16")
        return dx, dker, None, None, None, None, None


def involution2d(x: Tensor, kernel: Tensor, kernel_size: int, stride: int = 1, padding: int = 0, dilation: int = 1,
                 groups: int = 1) -> Tensor:
    """Involution of ``x`` [N, C, H, W] with the per-pixel kernel ``kernel`` [N, >= groups*K*K, Ho, Wo] (channel
    g*K*K + t: group g, tap t, extra columns ignored); bf16 channels_last in and out."""
    require_cuda(x, kernel)
    return _InvolutionFn.apply(x, kernel, int(kernel_size), int(stride), int(padding), int(dilation), int(groups))
