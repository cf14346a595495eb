"""ResNet / ResNeXt / ResNet-D on the fused kernels — API mirror of holocron/models/classification/resnet.py
(_ResBlock :59-87, BasicBlock :90-141, Bottleneck :144-210, ChannelRepeat :213-221, ResNet :224-443, factories :440-768).

Module tree, parameter names and init order are the reference's (``state_dict`` compatible). A block runs as fused
``conv -> BN -> act`` units (:mod:`holocron_b200.models._blocks`); the shortcut addition and the block's final activation are
folded into the last unit's normalisation pass, ``act(BN(conv(.)) + identity)`` - the reference's ``out += identity`` and
activation are two more tensor passes. Grouped 3x3 convolutions (ResNeXt) are a library call, everything else is on the
tensor-core kernels; the 7x7 stem takes the implicit-GEMM path, ResNet-D's 3x3 stem the im2col one."""
from collections import OrderedDict
from typing import Any, Callable, Dict, List, Optional, Type, Union

from torch import Tensor, nn

from ...nn import GlobalAvgPool2d, init
from ...nn import _fused as K
from .._blocks import FusedSequential, run_fused
from ..utils import _configure_model, _requested_checkpoint, conv_sequence

__all__ = ["BasicBlock", "Bottleneck", "ChannelRepeat", "ResNet", "resnet18", "resnet34", "resnet50", "resnet50d", "resnet101",
           "resnet152", "resnext50_32x4d", "resnext101_32x8d"]


class _ResBlock(nn.Module):
    """``act(conv(x) + shortcut(x))`` (reference resnet.py:59-87): ``conv`` is a stack of conv units whose last one has no
    activation, ``downsample`` the optional projection shortcut."""

    expansion: int = 1

    def __init__(self, convs: List[nn.Module], downsample: Optional[nn.Module] = None,
                 act_layer: Optional[nn.Module] = None) -> None:
        super().__init__()
        self.conv = FusedSequential(*convs)
        self.downsample = downsample
        if isinstance(act_layer, nn.Module):
            self.activation = act_layer

    def forward(self, x: Tensor) -> Tensor:
        identity = x if self.downsample is None else self.downsample(x)
        mods = list(self.conv)
        act = getattr(self, "activation", None)
        # fusable: the stack ends with [conv, BatchNorm] and the shortcut has the output's shape
        if K.is_batch_norm(mods[-1]) and isinstance(mods[-2], nn.Conv2d):
            return run_fused(mods + ([act] if act is not None else []), x, residual=identity, res_after_act=False)
        out = self.conv(x)
        out = out + identity
        return out if act is None else act(out)


class BasicBlock(_ResBlock):
    """Two 3x3 units (reference resnet.py:90-141)."""

    expansion: int = 1

    def __init__(self, inplanes: int, planes: int, stride: int = 1, downsample: Optional[nn.Module] = None, groups: int = 1,
                 base_width: int = 64, dilation: int = 1, act_layer: Optional[nn.Module] = None,
                 norm_layer: Optional[Callable[[int], nn.Module]] = None,
                 drop_layer: Optional[Callable[..., nn.Module]] = None,
                 conv_layer: Optional[Callable[..., nn.Module]] = None, **kwargs: Any) -> None:
        no_norm = norm_layer is None
        super().__init__(
            [*conv_sequence(inplanes, planes, act_layer, norm_layer, drop_layer, conv_layer, kernel_size=3, stride=stride,
                            padding=dilation, groups=groups, bias=no_norm, dilation=dilation, **kwargs),
             *conv_sequence(planes, planes, None, norm_layer, drop_layer, conv_layer, kernel_size=3, stride=1,
                            padding=dilation, groups=groups, bias=no_norm, dilation=dilation, **kwargs)],
            downsample, act_layer)


class Bottleneck(_ResBlock):
    """1x1 reduce, 3x3 (stride / groups / dilation), 1x1 expand x4 (reference resnet.py:144-210)."""

    expansion: int = 4

    def __init__(self, inplanes: int, planes: int, stride: int = 1, downsample: Optional[nn.Module] = None, groups: int = 1,
                 base_width: int = 64, dilation: int = 1, act_layer: Optional[nn.Module] = None,
                 norm_layer: Optional[Callable[[int], nn.Module]] = None,
                 drop_layer: Optional[Callable[..., nn.Module]] = None,
                 conv_layer: Optional[Callable[..., nn.Module]] = None, **kwargs: Any) -> None:
        width = int(planes * (base_width / 64.0)) * groups
        no_norm = norm_layer is None
        super().__init__(
            [*conv_sequence(inplanes, width, act_layer, norm_layer, drop_layer, conv_layer, kernel_size=1, stride=1,
                            bias=no_norm, **kwargs),
             *conv_sequence(width, width, act_layer, norm_layer, drop_layer, conv_layer, kernel_size=3, stride=stride,
                            padding=dilation, groups=groups, bias=no_norm, dilation=dilation, **kwargs),
             *conv_sequence(width, planes * self.expansion, None, norm_layer, drop_layer, conv_layer, kernel_size=1, stride=1,
                            bias=no_norm, **kwargs)],
            downsample, act_layer)


class ChannelRepeat(nn.Module):
    """Repeats the tensor along the channel axis (reference resnet.py:213-221, used by TridentNet)."""

    def __init__(self, chan_repeats: int = 1) -> None:
        super().__init__()
        self.chan_repeats = chan_repeats

    def forward(self, x: Tensor) -> Tensor:
        repeats = [1] * x.ndim
        repeats[1] = self.chan_repeats
        return x.repeat(*repeats)


class ResNet(nn.Sequential):
    """ResNet (https://arxiv.org/abs/1512.03385) — reference resnet.py:224-443, same constructor."""

    def __init__(self, block: Type[Union[BasicBlock, Bottleneck]], num_blocks: List[int], planes: List[int],
                 num_classes: int = 10, in_channels: int = 3, zero_init_residual: bool = False, width_per_group: int = 64,
                 conv_layer: Optional[Callable[..., nn.Module]] = None, act_layer: Optional[nn.Module] = None,
                 norm_layer: Optional[Callable[[int], nn.Module]] = None,
                 drop_layer: Optional[Callable[..., nn.Module]] = None, deep_stem: bool = False, stem_pool: bool = True,
                 avg_downsample: bool = False, num_repeats: int = 1,
                 block_args: Optional[Union[Dict[str, Any], List[Dict[str, Any]]]] = None) -> None:
        if conv_layer is None:
            conv_layer = nn.Conv2d
        if norm_layer is None:
            norm_layer = nn.BatchNorm2d
        if act_layer is None:
            act_layer = nn.ReLU(inplace=True)
        self.dilation = 1
        no_norm = norm_layer is None
        in_planes = 64
        if deep_stem:   # ResNet-C / -D stem: three 3x3 units
            stem = [(in_channels, in_planes // 2, 2), (in_planes // 2, in_planes // 2, 1), (in_planes // 2, in_planes, 1)]
            layers: List[nn.Module] = []
            for cin, cout, stride in stem:
                layers.extend(conv_sequence(cin, cout, act_layer, norm_layer, drop_layer, conv_layer, kernel_size=3,
                                            stride=stride, padding=1, bias=no_norm))
        else:
            layers = conv_sequence(in_channels, in_planes, act_layer, norm_layer, drop_layer, conv_layer, kernel_size=7,
                                   stride=2, padding=3, bias=no_norm)
        if stem_pool:
            layers.append(nn.MaxPool2d(kernel_size=3, stride=2, padding=1))
        if num_repeats > 1:
            layers.append(ChannelRepeat(num_repeats))
        if block_args is None:
            block_args = {"groups": 1}
        if not isinstance(block_args, list):
            block_args = [block_args] * len(num_blocks)
        stride = 1
        for nb, width, args in zip(num_blocks, planes, block_args):
            layers.append(self._make_layer(block, nb, in_planes, width, stride, width_per_group, act_layer=act_layer,
                                           norm_layer=norm_layer, drop_layer=drop_layer, avg_downsample=avg_downsample,
                                           num_repeats=num_repeats, block_args=args))
            in_planes = block.expansion * width
            stride = 2
        super().__init__(OrderedDict([
            ("features", FusedSequential(*layers)),
            ("pool", GlobalAvgPool2d(flatten=True)),
            ("head", nn.Linear(num_repeats * in_planes, num_classes)),
        ]))
        init.init_module(self, nonlinearity="relu")
        if zero_init_residual:
            # reference resnet.py:353-358 addresses `m.convs[..]`, an attribute its blocks do not have (they hold `conv`): the
            # option raises there as well; kept so that a config that fails on the reference does not silently pass here
            for m in self.modules():
                if isinstance(m, (Bottleneck, BasicBlock)):
                    m.convs[2 if isinstance(m, Bottleneck) else 1][1].weight.data.zero_()

    @staticmethod
    def _make_layer(block: Type[Union[BasicBlock, Bottleneck]], num_blocks: int, in_planes: int, planes: int, stride: int = 1,
                    width_per_group: int = 64, act_layer: Optional[nn.Module] = None,
                    norm_layer: Optional[Callable[[int], nn.Module]] = None,
                    drop_layer: Optional[Callable[..., nn.Module]] = None,
                    conv_layer: Optional[Callable[..., nn.Module]] = None, avg_downsample: bool = False,
                    num_repeats: int = 1, block_args: Optional[Dict[str, Any]] = None) -> nn.Sequential:
        downsample = None
        out_planes = planes * block.expansion
        if stride != 1 or in_planes != out_planes:
            pool = [nn.AvgPool2d(stride, ceil_mode=True, count_include_pad=False)] if avg_downsample else []   # ResNet-D
            downsample = FusedSequential(
                *pool,
                *conv_sequence(num_repeats * in_planes, num_repeats * out_planes, None, norm_layer, drop_layer, conv_layer,
                               kernel_size=1, stride=1 if avg_downsample else stride, bias=(norm_layer is None)))
        if block_args is None:
            block_args = {}
        common = dict(base_width=width_per_group, act_layer=act_layer, norm_layer=norm_layer, drop_layer=drop_layer, **block_args)
        blocks = [block(in_planes, planes, stride, downsample, **common)]
        blocks.extend(block(out_planes, planes, 1, None, **common) for _ in range(num_blocks - 1))
        return FusedSequential(*blocks)

    def forward(self, x: Tensor) -> Tensor:  # type: ignore[override]
        feats = self.pool(self.features(x))
        return K.head_linear(feats, self.head.weight, self.head.bias)


def _resnet(arch: str, pretrained: bool, checkpoint: Any, block: Type[Union[BasicBlock, Bottleneck]], num_blocks: List[int],
            out_chans: List[int], **kwargs: Any) -> ResNet:
    checkpoint = _requested_checkpoint(pretrained, checkpoint)
    model = ResNet(block, num_blocks, out_chans, **kwargs)
    return _configure_model(model, checkpoint)


def resnet18(pretrained: bool = False, checkpoint: Any = None, progress: bool = True, **kwargs: Any) -> ResNet:
    """ResNet-18 (reference resnet.py:472-498)."""
    return _resnet("resnet18", pretrained, checkpoint, BasicBlock, [2, 2, 2, 2], [64, 128, 256, 512], **kwargs)


def resnet34(pretrained: bool = False, checkpoint: Any = None, progress: bool = True, **kwargs: Any) -> ResNet:
    """ResNet-34 (reference resnet.py:520-541)."""
    return _resnet("resnet34", pretrained, checkpoint, BasicBlock, [3, 4, 6, 3], [64, 128, 256, 512], **kwargs)


def resnet50(pretrained: bool = False, checkpoint: Any = None, progress: bool = True, **kwargs: Any) -> ResNet:
    """ResNet-50 (reference resnet.py:563-589)."""
    return _resnet("resnet50", pretrained, checkpoint, Bottleneck, [3, 4, 6, 3], [64, 128, 256, 512], **kwargs)


def resnet50d(pretrained: bool = False, checkpoint: Any = None, progress: bool = True, **kwargs: Any) -> ResNet:
    """ResNet-50-D: deep 3x3 stem and average-pooled projection shortcuts (reference resnet.py:611-642)."""
    return _resnet("resnet50d", pretrained, checkpoint, Bottleneck, [3, 4, 6, 3], [64, 128, 256, 512], deep_stem=True,
                   avg_downsample=True, **kwargs)


def resnet101(pretrained: bool = False, checkpoint: Any = None, progress: bool = True, **kwargs: Any) -> ResNet:
    """ResNet-101 (reference resnet.py:645-663)."""
    return _resnet("resnet101", pretrained, checkpoint, Bottleneck, [3, 4, 23, 3], [64, 128, 256, 512], **kwargs)


def resnet152(pretrained: bool = False, checkpoint: Any = None, progress: bool = True, **kwargs: Any) -> ResNet:
    """ResNet-152 (reference resnet.py:666-684)."""
    return _resnet("resnet152", pretrained, checkpoint, Bottleneck, [3, 8, 86, 3], [64, 128, 256, 512], **kwargs)


def resnext50_32x4d(pretrained: bool = False, checkpoint: Any = None, progress: bool = True, **kwargs: Any) -> ResNet:
    """ResNeXt-50 32x4d (reference resnet.py:706-737): 32 groups of width 4 in the 3x3 units (library grouped convolution)."""
    kwargs["width_per_group"] = 4
    return _resnet("resnext50_32x4d", pretrained, checkpoint, Bottleneck, [3, 4, 6, 3], [64, 128, 256, 512],
                   block_args={"groups": 32}, **kwargs)


def resnext101_32x8d(pretrained: bool = False, checkpoint: Any = None, progress: bool = True, **kwargs: Any) -> ResNet:
    """ResNeXt-101 32x8d (reference resnet.py:740-768)."""
    kwargs["width_per_group"] = 8
    return _resnet("resnext101_32x8d", pretrained, checkpoint, Bottleneck, [3, 4, 23, 3], [64, 128, 256, 512],
                   block_args={"groups": 32}, **kwargs)
