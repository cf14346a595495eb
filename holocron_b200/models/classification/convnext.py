"""ConvNeXt on the fused kernels — API mirror of holocron/models/classification/convnext.py (LayerNorm2d :37-41,
LayerScale :44-52, Bottlenext :55-109, ConvNeXt :112-189, factories :223-401).

Block = 7x7 depth-wise conv (+bias) -> LayerNorm over channels -> 1x1 expand x4 (+bias) -> GELU -> 1x1 project (+bias) ->
per-channel LayerScale -> stochastic depth -> + identity. What runs where:
  * 7x7 depth-wise: the depth-wise CUDA kernels (`csrc/dwconv.cu`, channels % 8 == 0 - true for every factory);
  * the two 1x1 convolutions (all of the block's FLOPs) and the 4x4 / 2x2 patchify convolutions: wgmma implicit GEMM with
    the bias in the epilogue;
  * LayerNorm, GELU, LayerScale, the residual addition: library element-wise / row kernels on the NHWC tensor (LayerNorm over
    the innermost dimension of a channels_last tensor is a plain row normalisation, no permute copy).
The residual stream stays fp32 like under torch autocast (a block's contribution is scaled by 1e-6 at initialisation: adding
it to a bf16 stream would round it away); the block body works on bf16.
Module tree, parameter names and the truncated-normal init order are the reference's (``state_dict`` compatible)."""
from collections import OrderedDict
from functools import partial
from typing import Any, Callable, List, Optional

import torch
import torch.nn.functional as TF
from torch import Tensor, nn
from torchvision.ops.stochastic_depth import StochasticDepth

from ...nn import GlobalAvgPool2d
from .._blocks import FusedSequential
from ..utils import _configure_model, _requested_checkpoint, conv_sequence
from .resnet import _ResBlock

__all__ = ["ConvNeXt", "LayerNorm2d", "LayerScale", "Bottlenext", "convnext_atto", "convnext_femto", "convnext_pico",
           "convnext_nano", "convnext_tiny", "convnext_small", "convnext_base", "convnext_large", "convnext_xl"]


class LayerNorm2d(nn.LayerNorm):
    """LayerNorm over the channel axis of an NCHW-logical tensor (reference convnext.py:37-41). fp32 arithmetic whatever the
    activation dtype (the affine parameters are fp32 masters); the result comes back in the input's dtype and layout."""

    def forward(self, x: Tensor) -> Tensor:  # type: ignore[override]
        y = TF.layer_norm(x.permute(0, 2, 3, 1).float(), self.normalized_shape, self.weight, self.bias, self.eps)
        return y.to(x.dtype).permute(0, 3, 1, 2)


class LayerScale(nn.Module):
    """Learnable per-channel scale (reference convnext.py:44-52); the product is fp32 (the parameter's dtype)."""

    def __init__(self, chans: int, scale: float = 1e-6) -> None:
        super().__init__()
        self.register_parameter("weight", nn.Parameter(scale * torch.ones(chans)))

    def forward(self, x: Tensor) -> Tensor:
        return x.float() * self.weight.reshape(1, -1, *((1,) * (x.ndim - 2)))


class Bottlenext(_ResBlock):
    """ConvNeXt block (reference convnext.py:55-109)."""

    def __init__(self, inplanes: int, act_layer: Optional[nn.Module] = None,
                 norm_layer: Optional[Callable[[int], nn.Module]] = None,
                 drop_layer: Optional[Callable[..., nn.Module]] = None, chan_expansion: int = 4,
                 stochastic_depth_prob: float = 0.1, layer_scale: float = 1e-6) -> None:
        if norm_layer is None:
            norm_layer = partial(LayerNorm2d, eps=1e-6)
        if act_layer is None:
            act_layer = nn.GELU()
        super().__init__(
            [*conv_sequence(inplanes, inplanes, None, norm_layer, drop_layer, kernel_size=7, padding=3, stride=1, bias=True,
                            groups=inplanes),
             *conv_sequence(inplanes, inplanes * chan_expansion, act_layer, None, drop_layer, kernel_size=1, stride=1, bias=True),
             *conv_sequence(inplanes * chan_expansion, inplanes, None, None, drop_layer, kernel_size=1, stride=1, bias=True),
             LayerScale(inplanes, layer_scale),
             StochasticDepth(stochastic_depth_prob, "row")],
            None, None)

    def forward(self, x: Tensor) -> Tensor:
        # fp32 residual stream, bf16 block body (see the module docstring); `self.conv` is a FusedSequential: convolutions on the
        # CUDA kernels, everything else called as a module
        return x.float() + self.conv(x)


class ConvNeXt(nn.Sequential):
    """ConvNeXt (https://arxiv.org/abs/2201.03545) — reference convnext.py:112-189, same constructor."""

    def __init__(self, num_blocks: List[int], planes: List[int], num_classes: int = 10, in_channels: int = 3,
                 conv_layer: Optional[Callable[..., nn.Module]] = None, act_layer: Optional[nn.Module] = None,
                 norm_layer: Optional[Callable[[int], nn.Module]] = None,
                 drop_layer: Optional[Callable[..., nn.Module]] = None, stochastic_depth_prob: float = 0.0) -> None:
        if conv_layer is None:
            conv_layer = nn.Conv2d
        if norm_layer is None:
            norm_layer = partial(LayerNorm2d, eps=1e-6)
        if act_layer is None:
            act_layer = nn.GELU()
        self.dilation = 1
        # patchify stem: 4x4 stride-4 convolution + LayerNorm
        layers = conv_sequence(in_channels, planes[0], None, norm_layer, drop_layer, conv_layer, kernel_size=4, stride=4,
                               padding=0, bias=True)
        block_idx = 0
        tot_blocks = sum(num_blocks)
        for _num_blocks, _planes, _oplanes in zip(num_blocks, planes, planes[1:] + [planes[-1]]):
            # stochastic-depth probability grows linearly with the block's depth
            sd_probs = [stochastic_depth_prob * (block_idx + _idx) / (tot_blocks - 1.0) for _idx in range(_num_blocks)]
            stage: List[nn.Module] = [Bottlenext(_planes, act_layer, norm_layer, drop_layer, stochastic_depth_prob=sd_prob)
                                      for sd_prob in sd_probs]
            if _planes != _oplanes:
                stage.append(FusedSequential(LayerNorm2d(_planes), nn.Conv2d(_planes, _oplanes, kernel_size=2, stride=2)))
            layers.append(FusedSequential(*stage))
            block_idx += _num_blocks
        super().__init__(OrderedDict([
            ("features", FusedSequential(*layers)),
            ("pool", GlobalAvgPool2d(flatten=True)),
            ("head", nn.Sequential(nn.LayerNorm(planes[-1], eps=1e-6), nn.Linear(planes[-1], num_classes))),
        ]))
        for m in self.modules():
            if isinstance(m, (nn.Conv2d, nn.Linear)):
                nn.init.trunc_normal_(m.weight, std=0.02)
                if m.bias is not None:
                    nn.init.zeros_(m.bias)

    def forward(self, x: Tensor) -> Tensor:  # type: ignore[override]
        feats = self.pool(self.features(x)).float()
        return self.head(feats)


def _convnext(pretrained: bool, checkpoint: Any, num_blocks: List[int], out_chans: List[int], **kwargs: Any) -> ConvNeXt:
    checkpoint = _requested_checkpoint(pretrained, checkpoint)
    model = ConvNeXt(num_blocks, out_chans, **kwargs)
    return _configure_model(model, checkpoint)


def convnext_atto(pretrained: bool = False, checkpoint: Any = None, progress: bool = True, **kwargs: Any) -> ConvNeXt:
    """ConvNeXt-Atto (reference convnext.py:223-249)."""
    return _convnext(pretrained, checkpoint, [2, 2, 6, 2], [40, 80, 160, 320], **kwargs)


def convnext_femto(pretrained: bool = False, checkpoint: Any = None, progress: bool = True, **kwargs: Any) -> ConvNeXt:
    """ConvNeXt-Femto (reference convnext.py:252-268)."""
    return _convnext(pretrained, checkpoint, [2, 2, 6, 2], [48, 96, 192, 384], **kwargs)


def convnext_pico(pretrained: bool = False, checkpoint: Any = None, progress: bool = True, **kwargs: Any) -> ConvNeXt:
    """ConvNeXt-Pico (reference convnext.py:271-287)."""
    return _convnext(pretrained, checkpoint, [2, 2, 6, 2], [64, 128, 256, 512], **kwargs)


def convnext_nano(pretrained: bool = False, checkpoint: Any = None, progress: bool = True, **kwargs: Any) -> ConvNeXt:
    """ConvNeXt-Nano (reference convnext.py:290-306)."""
    return _convnext(pretrained, checkpoint, [2, 2, 8, 2], [80, 160, 320, 640], **kwargs)


def convnext_tiny(pretrained: bool = False, checkpoint: Any = None, progress: bool = True, **kwargs: Any) -> ConvNeXt:
    """ConvNeXt-Tiny (reference convnext.py:309-325)."""
    return _convnext(pretrained, checkpoint, [3, 3, 9, 3], [96, 192, 384, 768], **kwargs)


def convnext_small(pretrained: bool = False, checkpoint: Any = None, progress: bool = True, **kwargs: Any) -> ConvNeXt:
    """ConvNeXt-Small (reference convnext.py:328-344)."""
    return _convnext(pretrained, checkpoint, [3, 3, 27, 3], [96, 192, 384, 768], **kwargs)


def convnext_base(pretrained: bool = False, checkpoint: Any = None, progress: bool = True, **kwargs: Any) -> ConvNeXt:
    """ConvNeXt-Base (reference convnext.py:347-363)."""
    return _convnext(pretrained, checkpoint, [3, 3, 27, 3], [128, 256, 512, 1024], **kwargs)


def convnext_large(pretrained: bool = False, checkpoint: Any = None, progress: bool = True, **kwargs: Any) -> ConvNeXt:
    """ConvNeXt-Large (reference convnext.py:366-382)."""
    return _convnext(pretrained, checkpoint, [3, 3, 27, 3], [192, 384, 768, 1536], **kwargs)


def convnext_xl(pretrained: bool = False, checkpoint: Any = None, progress: bool = True, **kwargs: Any) -> ConvNeXt:
    """ConvNeXt-XL (reference convnext.py:385-401)."""
    return _convnext(pretrained, checkpoint, [3, 3, 27, 3], [256, 512, 1024, 2048], **kwargs)
