"""Execution of reference-shaped module stacks on the fused kernels.

The reference builds every backbone from ``conv_sequence`` lists ``[Conv2d, BatchNorm2d?, act?, DropBlock2d?]`` wrapped
in ``nn.Sequential`` (holocron/models/utils.py:28-86). The model files of this package keep exactly those module trees
(so ``state_dict`` keys and the init RNG order are unchanged) but use :class:`FusedSequential`, whose ``forward`` walks the
stack and maps every ``conv -> BN -> act`` run onto
  * the wgmma implicit-GEMM convolution (dense) or the depth-wise kernel (``groups == channels``), and
  * ONE fused normalise/(residual)/activate pass (+ one statistics pass in training),
instead of 3-4 separate library kernels. Anything it does not recognise is simply called.
"""
from typing import List, Optional, Sequence

import torch
import torch.nn.functional as TF
from torch import Tensor, nn

from ..nn import _fused as K

_ACTS = (nn.ReLU, nn.ReLU6, nn.SiLU, nn.LeakyReLU, nn.Mish, nn.Identity)


def _is_act(m: nn.Module) -> bool:
    return isinstance(m, _ACTS) or type(m).__name__ == "HardMish"


def _dense_ok(conv: nn.Conv2d) -> bool:
    return (conv.groups == 1 and conv.padding_mode == "zeros" and conv.kernel_size[0] == conv.kernel_size[1]
            and conv.stride[0] == conv.stride[1] and conv.padding[0] == conv.padding[1]
            and conv.dilation[0] == conv.dilation[1] == 1 and isinstance(conv.padding[0], int))


def _depthwise_ok(conv: nn.Conv2d) -> bool:
    return (conv.groups == conv.in_channels == conv.out_channels and conv.padding_mode == "zeros"
            and conv.kernel_size[0] == conv.kernel_size[1] and conv.stride[0] == conv.stride[1]
            and conv.padding[0] == conv.padding[1] and conv.dilation[0] == conv.dilation[1] == 1
            and conv.in_channels % 8 == 0)


def _patchify_ok(conv: nn.Conv2d, x: Tensor) -> bool:
    """Non-overlapping patch convolution (kernel == stride > 1, no padding: ConvNeXt's 4x4 stem and 2x2 stage transitions)."""
    k = conv.kernel_size[0]
    return k > 1 and conv.stride[0] == k and conv.padding[0] == 0 and x.shape[2] % k == 0 and x.shape[3] % k == 0


def _space_to_depth(x: Tensor, conv: nn.Conv2d):
    """A k x k stride-k convolution is a 1x1 convolution over k x k pixel blocks stacked on the channel axis: one NHWC
    re-tiling copy (N, H/k, W/k, [kh, kw, C]) and a filter view in the same (kh, kw, C) order, then the dense 1x1 GEMM path -
    forward, data gradient and weight gradient of which are the best-covered kernels of this package (the implicit-GEMM data
    gradient of an even-sized strided filter would need asymmetric padding)."""
    k = conv.kernel_size[0]
    cin = conv.in_channels
    xs = x if x.shape[1] == cin else x[:, :cin]
    n, _, h, w = xs.shape
    xr = xs.reshape(n, cin, h // k, k, w // k, k).permute(0, 2, 4, 3, 5, 1).reshape(n, h // k, w // k, k * k * cin)
    wr = conv.weight.permute(0, 2, 3, 1).reshape(conv.out_channels, k * k * cin, 1, 1)
    return xr.permute(0, 3, 1, 2), wr


def conv_bn_act(x: Tensor, conv: nn.Conv2d, bn: Optional[nn.BatchNorm2d], act: Optional[nn.Module],
                residual: Optional[Tensor] = None, res_after_act: bool = False, keep_padded: bool = False) -> Tensor:
    """One ``conv -> BN -> act`` unit (+ optional shortcut) on the fused kernels."""
    if type(conv).forward is not nn.Conv2d.forward:
        # a Conv2d subclass with its own forward (TridentConv2d: one filter shared by three channel chunks): the module decides
        # which kernels it runs on, the normalisation / activation pass below is the fused one
        y = conv(x)
    elif _dense_ok(conv):
        weight, stride, pad = conv.weight, conv.stride[0], conv.padding[0]
        if _patchify_ok(conv, x):
            x, weight, stride, pad = *_space_to_depth(x, conv), 1, 0
        if bn is None and residual is None:
            code, slope = K.act_code(act)
            return K.conv2d_bias_act(x, weight, conv.bias, stride, pad, code, slope)
        # training-mode BatchNorm next: the convolution's epilogue also produces the per-channel statistics of its output
        stats = bn is not None and (bn.training or bn.running_mean is None)
        y = K.conv2d(x, weight, conv.bias, stride, pad, keep_padded=keep_padded or bn is not None, want_stats=stats)
    elif _depthwise_ok(conv):
        from ..nn._dwconv import dwconv2d
        y = dwconv2d(x, conv.weight, conv.bias, conv.stride[0], conv.padding[0])
    else:
        # grouped (ResNeXt) / asymmetric / dilated convolutions are outside the hot path: library call on the activation's
        # dtype (the fused units hand over bf16 channels_last tensors, the parameters stay fp32 masters)
        xs = x if x.shape[1] == conv.in_channels else x[:, :conv.in_channels]
        w = conv.weight if conv.weight.dtype == xs.dtype else conv.weight.to(xs.dtype)
        b = conv.bias if conv.bias is None or conv.bias.dtype == xs.dtype else conv.bias.to(xs.dtype)
        if conv.padding_mode != "zeros":
            y = conv(xs.to(conv.weight.dtype))
        else:
            y = TF.conv2d(xs, w, b, conv.stride, conv.padding, conv.dilation, conv.groups)
    code, slope = K.act_code(act)
    if bn is not None:
        out = K.bn_act([y], [bn], code, slope, residual=residual, res_after_act=res_after_act)
        if out.shape[1] != bn.num_features and not keep_padded:      # == conv.out_channels (3x that behind a TridentConv2d)
            out = out[:, :bn.num_features]
        return out
    if residual is not None:
        cfg = ([], code, slope, False, True, res_after_act)
        raise NotImplementedError("shortcut without normalisation layer")
    return y if code == K.ACT_NONE else K.act_only(y, code, slope)


def run_fused(mods: Sequence[nn.Module], x: Tensor, residual: Optional[Tensor] = None,
              res_after_act: bool = False) -> Tensor:
    """Runs ``mods`` sequentially, fusing conv/BN/act runs. ``residual`` is fused into the LAST conv unit."""
    mods = list(mods)
    # index of the last convolution (the unit the shortcut is attached to)
    last_conv = max((i for i, m in enumerate(mods) if isinstance(m, nn.Conv2d)), default=-1)
    i = 0
    while i < len(mods):
        m = mods[i]
        if isinstance(m, nn.Conv2d):
            j = i + 1
            bn = act = None
            if j < len(mods) and K.is_batch_norm(mods[j]):
                bn = mods[j]; j += 1
            if j < len(mods) and _is_act(mods[j]):
                act = mods[j]; j += 1
            res = residual if i == last_conv else None
            x = conv_bn_act(x, m, bn, act, res, res_after_act)
            if res is not None:
                residual = None
            i = j
        elif isinstance(m, FusedSequential):
            x = m(x)
            i += 1
        elif K.is_batch_norm(m) and x.is_cuda and x.shape[1] % 8 != 0:
            # stand-alone BatchNorm on a width the fused pass cannot take (ReXNet-1.3x taps of DynamicUNet: 35, 61 ... channels;
            # behind a convolution the width is zero-padded instead): library call in the parameters' dtype
            x = m(x.to(m.weight.dtype if m.weight is not None else torch.float32)).to(x.dtype)
            i += 1
        elif K.is_batch_norm(m):
            act = None
            j = i + 1
            if j < len(mods) and _is_act(mods[j]):
                act = mods[j]; j += 1
            code, slope = K.act_code(act)
            x = K.bn_act([x], [m], code, slope)
            i = j
        elif _is_act(m) and x.is_cuda and x.ndim == 4 and x.shape[1] % 8 == 0 and not isinstance(m, nn.Identity):
            code, slope = K.act_code(m)
            x = K.act_only(x, code, slope)
            i += 1
        else:
            x = m(x)
            i += 1
    if residual is not None:
        x = x + residual
    return x


class FusedSequential(nn.Sequential):
    """Drop-in ``nn.Sequential`` (same children, same ``state_dict``) executed by :func:`run_fused`."""

    def forward(self, x: Tensor) -> Tensor:  # type: ignore[override]
        return run_fused(list(self), x)
