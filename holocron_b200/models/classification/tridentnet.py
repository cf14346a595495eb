"""TridentNet on the fused kernels — API mirror of holocron/models/classification/tridentnet.py (TridentConv2d :27-59,
Tridentneck :62-134, _tridentnet :137-153, tridentnet50 :156-167).

The network carries three scale branches side by side on the channel axis (``ChannelRepeat(3)`` behind the stem); a
``TridentConv2d`` applies ONE filter to each third of the channels, with dilations 1 / 2 / 3 for the 3x3 layers, and the
BatchNorm that follows spans all ``3 x width`` channels. Here the dilation-1 chunks (all 1x1 layers and the first branch of
every 3x3 layer) run on the tensor-core convolution, the dilated chunks are library calls, and normalisation + activation
(+ shortcut) is one fused pass over the concatenated tensor."""
from typing import Any, Callable, List, Optional

import torch
import torch.nn.functional as TF
from torch import Tensor, nn

from ...nn import _fused as K
from ..utils import conv_sequence
from .resnet import ResNet, _ResBlock

__all__ = ["TridentConv2d", "Tridentneck", "tridentnet50"]


class TridentConv2d(nn.Conv2d):
    """Weight-shared convolution over ``num_branches`` channel chunks (reference tridentnet.py:27-59)."""

    num_branches: int = 3

    def __init__(self, *args: Any, **kwargs: Any) -> None:
        super().__init__(*args, **kwargs)
        if self.dilation[0] != 1 and self.dilation[0] != self.num_branches:
            raise ValueError(f"expected dilation to either be 1 or {self.num_branches}.")

    def forward(self, x: Tensor) -> Tensor:
        if x.shape[1] % self.num_branches != 0:
            raise ValueError("expected number of channels of input tensor to be a multiple of `num_branches`.")
        dilations = [1] * self.num_branches if self.dilation[0] == 1 else [1 + idx for idx in range(self.num_branches)]
        dense = self.groups == 1 and self.padding_mode == "zeros" and self.stride[0] == self.stride[1]
        outs = []
        for _x, dilation in zip(torch.chunk(x, self.num_branches, 1), dilations):
            if dense and dilation == 1:
                outs.append(K.conv2d(_x, self.weight, self.bias, self.stride[0], self.padding[0]))
            else:
                w = self.weight if self.weight.dtype == _x.dtype else self.weight.to(_x.dtype)
                b = self.bias if self.bias is None or self.bias.dtype == _x.dtype else self.bias.to(_x.dtype)
                outs.append(TF.conv2d(_x, w, b, self.stride, tuple(dilation * p for p in self.padding),
                                      (dilation,) * len(self.dilation), self.groups))
        return torch.cat(outs, 1)


class Tridentneck(_ResBlock):
    """Bottleneck of TridentConv2d layers with 3x-wide BatchNorms (reference tridentnet.py:62-134)."""

    expansion: int = 4

    def __init__(self, inplanes: int, planes: int, stride: int = 1, downsample: Optional[nn.Module] = None, groups: int = 1,
                 base_width: int = 64, dilation: int = 3, act_layer: Optional[nn.Module] = None,
                 norm_layer: Optional[Callable[[int], nn.Module]] = None,
                 drop_layer: Optional[Callable[..., nn.Module]] = None, **kwargs: Any) -> None:
        if norm_layer is None:
            norm_layer = nn.BatchNorm2d
        if act_layer is None:
            act_layer = nn.ReLU(inplace=True)
        width = int(planes * (base_width / 64.0)) * groups
        no_norm = norm_layer is None
        super().__init__(
            [*conv_sequence(inplanes, width, act_layer, norm_layer, drop_layer, TridentConv2d, bn_channels=3 * width,
                            kernel_size=1, stride=1, bias=no_norm, dilation=1, **kwargs),
             *conv_sequence(width, width, act_layer, norm_layer, drop_layer, TridentConv2d, bn_channels=3 * width,
                            kernel_size=3, stride=stride, padding=1, groups=groups, bias=no_norm, dilation=3, **kwargs),
             *conv_sequence(width, planes * self.expansion, None, norm_layer, drop_layer, TridentConv2d,
                            bn_channels=3 * planes * self.expansion, kernel_size=1, stride=1, bias=no_norm, dilation=1,
                            **kwargs)],
            downsample, act_layer)


def _tridentnet(pretrained: bool, num_blocks: List[int], out_chans: List[int], **kwargs: Any) -> ResNet:
    if pretrained:
        raise NotImplementedError("the released checkpoints need network access; load a reference state_dict instead "
                                  "(the module tree and parameter names are identical)")
    model = ResNet(Tridentneck, num_blocks, out_chans, num_repeats=3, **kwargs)  # type: ignore[arg-type]
    model.default_cfg = None
    return model


def tridentnet50(pretrained: bool = False, progress: bool = True, **kwargs: Any) -> ResNet:
    """TridentNet-50 (https://arxiv.org/abs/1901.01892) — reference tridentnet.py:156-167."""
    return _tridentnet(pretrained, [3, 4, 6, 3], [64, 128, 256, 512], **kwargs)
