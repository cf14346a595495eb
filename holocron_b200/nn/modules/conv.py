"""Convolution-like modules on the hot path — mirrors holocron/nn/modules/conv.py (NormConv2d :55-147, Add2d :150-248,
SlimConv2d :251-370, PyConv2d :373-438, Involution2d :441-499). Parameter names/shapes are the reference's (state_dict contract)."""
import math
from typing import Any, List, Optional, Union

import torch
from torch import Tensor, nn
from torch.nn.functional import pad
from torch.nn.modules.conv import _ConvNd
from torch.nn.modules.utils import _pair

from .. import functional as F

__all__ = ["Add2d", "Involution2d", "NormConv2d", "PyConv2d", "SlimConv2d"]


class _NormConvNd(_ConvNd):
    def __init__(self, in_channels, out_channels, kernel_size, stride, padding, dilation, transposed, output_padding,
                 groups, bias, padding_mode, normalize_slices: bool = False, eps: float = 1e-14) -> None:
        super().__init__(in_channels, out_channels, kernel_size, stride, padding, dilation, transposed, output_padding,
                         groups, bias, padding_mode)
        self.normalize_slices = normalize_slices
        self.eps = eps

    def _padded(self, x: Tensor):
        """Non-zero padding modes pre-pad the input and run the kernel without padding (reference conv.py:127-137)."""
        if self.padding_mode != "zeros":
            return pad(x, self._reversed_padding_repeated_twice, mode=self.padding_mode), _pair(0)
        return x, self.padding


class NormConv2d(_NormConvNd):
    """Normalised convolution (https://arxiv.org/abs/2005.05274): patches are standardised before the correlation."""

    def __init__(self, in_channels: int, out_channels: int, kernel_size: int, stride: int = 1, padding: int = 0,
                 dilation: int = 1, groups: int = 1, bias: bool = True, padding_mode: str = "zeros",
                 eps: float = 1e-14) -> None:
        super().__init__(in_channels, out_channels, _pair(kernel_size), _pair(stride), _pair(padding), _pair(dilation),
                         False, _pair(0), groups, bias, padding_mode, False, eps)

    def forward(self, x: Tensor) -> Tensor:
        x, padding = self._padded(x)
        return F.norm_conv2d(x, self.weight, self.bias, self.stride, padding, self.dilation, self.groups, self.eps)


class Add2d(_NormConvNd):
    """AdderNet layer (https://arxiv.org/abs/1912.13200): L1 distance between patches and filters instead of products."""

    def __init__(self, in_channels: int, out_channels: int, kernel_size: int, stride: int = 1, padding: int = 0,
                 dilation: int = 1, groups: int = 1, bias: bool = True, padding_mode: str = "zeros",
                 normalize_slices: bool = False, eps: float = 1e-14) -> None:
        super().__init__(in_channels, out_channels, _pair(kernel_size), _pair(stride), _pair(padding), _pair(dilation),
                         False, _pair(0), groups, bias, padding_mode, normalize_slices, eps)

    def forward(self, x: Tensor) -> Tensor:
        x, padding = self._padded(x)
        return F.add2d(x, self.weight, self.bias, self.stride, padding, self.dilation, self.groups, self.normalize_slices,
                       self.eps)


class SlimConv2d(nn.Module):
    """SlimConv (https://arxiv.org/abs/2003.07469): channel attention w, two half-width pathways built from x*w and
    x*flip(w), a k x k conv on top and a 1x1 + k x k on the bottom, concatenated to 3C/4 channels.

    Children ``fc1, bn, fc2, conv_top, conv_bot1, conv_bot2`` as in the reference. The three spatial convolutions run on
    the wgmma implicit-GEMM kernel whenever their channel counts allow it (out_channels % 16 == 0), the squeeze path
    works on (N, C, 1, 1) tensors and stays in torch.
    """

    def __init__(self, in_channels: int, kernel_size: int, stride: int = 1, padding: int = 0, dilation: int = 1,
                 groups: int = 1, bias: bool = True, padding_mode: str = "zeros", r: int = 32, L: int = 2) -> None:  # noqa: N803
        super().__init__()
        self.fc1 = nn.Conv2d(in_channels, max(in_channels // r, L), 1)
        self.bn = nn.BatchNorm2d(max(in_channels // r, L))
        self.fc2 = nn.Conv2d(max(in_channels // r, L), in_channels, 1)
        self.conv_top = nn.Conv2d(in_channels // 2, in_channels // 2, kernel_size, stride, padding, dilation, groups, bias,
                                  padding_mode)
        self.conv_bot1 = nn.Conv2d(in_channels // 2, in_channels // 4, 1)
        self.conv_bot2 = nn.Conv2d(in_channels // 4, in_channels // 4, kernel_size, stride, padding, dilation, groups, bias,
                                   padding_mode)

    @staticmethod
    def _conv(mod: nn.Conv2d, x: Tensor) -> Tensor:
        from .. import _fused as K
        fast = (x.is_cuda and mod.groups == 1 and mod.padding_mode == "zeros" and mod.out_channels % 16 == 0
                and mod.in_channels % 8 == 0 and mod.dilation[0] == mod.dilation[1] == 1
                and mod.stride[0] == mod.stride[1] and mod.padding[0] == mod.padding[1])
        if fast:
            return K.conv2d(x, mod.weight, mod.bias, mod.stride[0], mod.padding[0]).to(x.dtype)
        return mod(x)

    def forward(self, x: Tensor) -> Tensor:
        half = x.shape[1] // 2
        z = x.mean(dim=(2, 3), keepdim=True)
        z = self.fc2(torch.relu(self.bn(self.fc1(z))))
        w = torch.sigmoid(z)
        xw = x * w
        x_top = xw[:, :half] + xw[:, half:]
        xw = x * w.flip(dims=(1,))
        x_bot = xw[:, :half] + xw[:, half:]
        x_top = self._conv(self.conv_top, x_top)
        x_bot = self._conv(self.conv_bot2, self._conv(self.conv_bot1, x_bot))
        return torch.cat((x_top, x_bot), dim=1)


class PyConv2d(nn.ModuleList):
    """Pyramidal convolution (https://arxiv.org/abs/2006.11538) — reference conv.py:373-438: ``num_levels`` parallel
    convolutions of growing kernel size (k, k + 2, ...) and group count over the same input, concatenated on the channel axis.
    Same children (``state_dict`` keys ``0.weight``, ``1.weight``, ...). The levels run through the conv unit executor: dense
    levels on the tensor-core kernel, grouped ones as a library call on the activation dtype."""

    def __init__(self, in_channels: int, out_channels: int, kernel_size: int, num_levels: int = 2, padding: int = 0,
                 groups: Optional[List[int]] = None, **kwargs: Any) -> None:
        if num_levels == 1:
            super().__init__([nn.Conv2d(in_channels, out_channels, kernel_size, padding=padding,
                                        groups=groups[0] if isinstance(groups, list) else 1, **kwargs)])
        else:
            exp2 = int(math.log2(num_levels))
            reminder = num_levels - 2**exp2
            out_chans = [out_channels // 2 ** (exp2 + 1)] * (2 * reminder) + [out_channels // 2**exp2] * (num_levels - 2 * reminder)
            k_sizes = [kernel_size + 2 * idx for idx in range(num_levels)]
            if groups is None:
                groups = [1] + [min(2 ** (2 + idx), out_chan) for idx, out_chan in zip(range(num_levels - 1), out_chans[1:])]
            elif not isinstance(groups, list) or len(groups) != num_levels:
                raise ValueError("The argument `group` is expected to be a list of integer of size `num_levels`.")
            paddings = [padding + idx for idx in range(num_levels)]
            super().__init__([nn.Conv2d(in_channels, out_chan, k_size, padding=pad_, groups=group, **kwargs)
                              for out_chan, k_size, pad_, group in zip(out_chans, k_sizes, paddings, groups)])
        self.num_levels = num_levels

    def forward(self, x: Tensor) -> Tensor:
        from ...models._blocks import conv_bn_act
        if self.num_levels == 1:
            return conv_bn_act(x, self[0], None, None)
        return torch.cat([conv_bn_act(x, conv, None, None) for conv in self], dim=1)


class Involution2d(nn.Module):
    """Involution (https://arxiv.org/abs/2103.06255): every output pixel applies its own K x K kernel, shared by the
    channels of a group and generated from the input by ``span(reduce(pool(x)))`` (two 1x1 convolutions with a bias and
    nothing in between; ``pool`` is an ``AvgPool2d(stride, stride)`` when ``stride > 1`` and ``None`` otherwise).

    Children ``pool, reduce, span, unfold`` as in the reference, created in its order (same seeded init and
    ``state_dict``); ``unfold`` only carries the configuration. The forward pass runs the average pooling as a library
    call, both 1x1 convolutions on the tensor-core kernel (``span`` keeps its zero-padded width) and the involution on its
    own kernels (:mod:`holocron_b200.nn._involution`), which read x once through a shared-memory halo instead of building
    the N*C*K^2*Ho*Wo unfolded tensor. A bf16 channels_last input takes no layout copy; other dtypes run in bf16 and the
    output is cast back. Shapes the reference cannot compute raise RuntimeError before any launch; ``kernel_size``
    outside {1, 3, 5, 7} raises NotImplementedError.
    """

    def __init__(self, in_channels: int, kernel_size: int, padding: int = 0, stride: int = 1, groups: int = 1,
                 dilation: int = 1, reduction_ratio: float = 1) -> None:
        super().__init__()
        self.groups = groups
        self.k_size = kernel_size
        self.pool = nn.AvgPool2d(stride, stride) if stride > 1 else None
        self.reduce = nn.Conv2d(in_channels, int(in_channels // reduction_ratio), 1)
        self.span = nn.Conv2d(int(in_channels // reduction_ratio), kernel_size**2 * groups, 1)
        self.unfold = nn.Unfold(kernel_size, dilation, padding, stride)

    def forward(self, x: Tensor) -> Tensor:
        from .. import _fused as K
        from .._involution import check_involution, involution2d
        u = self.unfold
        check_involution(x.shape[1], x.shape[2], x.shape[3], self.k_size, u.stride, u.padding, u.dilation, self.groups)
        xb = K.to_channels_last_bf16(x)
        kernel = self.pool(xb) if isinstance(self.pool, nn.Module) else xb
        kernel = K.conv2d(kernel, self.reduce.weight, self.reduce.bias)
        kernel = K.conv2d(kernel, self.span.weight, self.span.bias, keep_padded=True)
        y = involution2d(xb, kernel, self.k_size, u.stride, u.padding, u.dilation, self.groups)
        return y if x.dtype == torch.bfloat16 else y.to(x.dtype)
