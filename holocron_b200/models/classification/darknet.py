"""Darknet-53 (v3) and CSP-Darknet-53 (v4) on the fused kernels — API mirrors of
holocron/models/classification/darknetv3.py and darknetv4.py (+ the residual block base of resnet.py:59-87).

Module trees, parameter names and init order are the reference's; the conv/BN/activation runs execute through
:mod:`holocron_b200.models._blocks`. The residual shortcut of a ResBlock (``act(BN(conv)) + x``) is fused into the
second unit's normalisation pass."""
from collections import OrderedDict
from typing import Any, Callable, List, Optional, Tuple, Union

import torch
from torch import Tensor, nn

from ...nn import DropBlock2d, GlobalAvgPool2d
from ...nn import _fused as K
from ...nn.init import init_module
from .._blocks import FusedSequential, run_fused
from ..utils import _configure_model, _requested_checkpoint, conv_sequence

__all__ = ["CSPStage", "DarknetBodyV1", "DarknetBodyV2", "DarknetBodyV3", "DarknetBodyV4", "DarknetV1", "DarknetV2",
           "DarknetV3", "DarknetV4", "ResBlock", "cspdarknet53", "cspdarknet53_mish", "darknet19", "darknet24",
           "darknet53"]


class ResBlock(nn.Module):
    """1x1 (planes -> mid) then 3x3 (mid -> planes) conv units and an identity shortcut added after the activation
    (reference darknetv3.py:23-70, resnet.py:59-87)."""

    def __init__(self, planes: int, mid_planes: int, act_layer: Optional[nn.Module] = None,
                 norm_layer: Optional[Callable[[int], nn.Module]] = None,
                 drop_layer: Optional[Callable[..., nn.Module]] = None,
                 conv_layer: Optional[Callable[..., nn.Module]] = None) -> None:
        super().__init__()
        self.conv = FusedSequential(
            *conv_sequence(planes, mid_planes, act_layer, norm_layer, drop_layer, conv_layer, kernel_size=1,
                           bias=(norm_layer is None)),
            *conv_sequence(mid_planes, planes, act_layer, norm_layer, drop_layer, conv_layer, kernel_size=3, padding=1,
                           bias=(norm_layer is None)),
        )
        self.downsample = None
        if drop_layer is not None:
            self.dropblock = DropBlock2d(0.1, 7, inplace=True)
        # the reference switches the last activation to out-of-place for the shortcut; harmless here (fused pass)
        if hasattr(self.conv[-1], "inplace"):
            self.conv[-1].inplace = False

    def forward(self, x: Tensor) -> Tensor:
        mods = list(self.conv)
        # the shortcut can be fused when the stack ends with [conv, BN, act] (no drop layer behind the activation)
        fusable = isinstance(mods[-1], nn.Module) and not isinstance(mods[-1], (DropBlock2d, nn.Dropout)) and \
            any(K.is_batch_norm(m) for m in mods[-3:])
        if fusable and x.is_cuda:
            out = run_fused(mods, x, residual=x, res_after_act=True)
        else:
            out = self.conv(x)
            out = out + x
        if hasattr(self, "dropblock"):
            out = self.dropblock(out)
        return out


def _body_forward(stem: nn.Module, stages: nn.Sequential, x: Tensor, num_features: int):
    x = stem(x)
    if num_features == 1:
        return stages(x)
    feats = []
    for idx, stage in enumerate(stages):
        x = stage(x)
        if idx >= len(stages) - num_features:
            feats.append(x)
    return feats


class DarknetBodyV3(nn.Sequential):
    """reference darknetv3.py:73-166."""

    def __init__(self, layout: List[Tuple[int, int]], in_channels: int = 3, stem_channels: int = 32, num_features: int = 1,
                 act_layer: Optional[nn.Module] = None, norm_layer: Optional[Callable[[int], nn.Module]] = None,
                 drop_layer: Optional[Callable[..., nn.Module]] = None,
                 conv_layer: Optional[Callable[..., nn.Module]] = None) -> None:
        if act_layer is None:
            act_layer = nn.LeakyReLU(0.1, inplace=True)
        if norm_layer is None:
            norm_layer = nn.BatchNorm2d
        in_chans = [stem_channels] + [_layout[0] for _layout in layout[:-1]]
        super().__init__(OrderedDict([
            ("stem", FusedSequential(*conv_sequence(in_channels, stem_channels, act_layer, norm_layer, drop_layer, conv_layer,
                                                     kernel_size=3, padding=1, bias=(norm_layer is None)))),
            ("layers", nn.Sequential(*[
                self._make_layer(num_blocks, _in, out, act_layer, norm_layer, drop_layer, conv_layer)
                for _in, (out, num_blocks) in zip(in_chans, layout)])),
        ]))
        self.num_features = num_features

    @staticmethod
    def _make_layer(num_blocks: int, in_planes: int, out_planes: int, act_layer=None, norm_layer=None, drop_layer=None,
                    conv_layer=None) -> nn.Sequential:
        layers = conv_sequence(in_planes, out_planes, act_layer, norm_layer, drop_layer, conv_layer, kernel_size=3,
                               padding=1, stride=2, bias=(norm_layer is None))
        layers.extend([ResBlock(out_planes, out_planes // 2, act_layer, norm_layer, drop_layer, conv_layer)
                       for _ in range(num_blocks)])
        return FusedSequential(*layers)

    def forward(self, x: Tensor) -> Union[Tensor, List[Tensor]]:  # type: ignore[override]
        return _body_forward(self.stem, self.layers, x, self.num_features)


class _DarknetClassifier(nn.Sequential):
    def forward(self, x: Tensor) -> Tensor:  # type: ignore[override]
        feats = self.pool(self.features(x))
        lin = self.classifier
        return K.head_linear(feats, lin.weight, lin.bias)


class DarknetV3(_DarknetClassifier):
    """reference darknetv3.py:169-194."""

    def __init__(self, layout: List[Tuple[int, int]], num_classes: int = 10, in_channels: int = 3, stem_channels: int = 32,
                 act_layer=None, norm_layer=None, drop_layer=None, conv_layer=None) -> None:
        super().__init__(OrderedDict([
            ("features", DarknetBodyV3(layout, in_channels, stem_channels, 1, act_layer, norm_layer, drop_layer, conv_layer)),
            ("pool", GlobalAvgPool2d(flatten=True)),
            ("classifier", nn.Linear(layout[-1][0], num_classes)),
        ]))
        init_module(self, "leaky_relu")


class CSPStage(nn.Module):
    """Cross-stage-partial stage: stride-2 3x3 + 1x1 base, half of the channels through ``num_blocks`` ResBlocks,
    concat, 1x1 transition (reference darknetv4.py:38-115)."""

    def __init__(self, in_channels: int, out_channels: int, num_blocks: int = 1, act_layer=None, norm_layer=None,
                 drop_layer=None, conv_layer=None) -> None:
        super().__init__()
        compression = 2 if num_blocks > 1 else 1
        self.base_layer = FusedSequential(
            *conv_sequence(in_channels, out_channels, act_layer, norm_layer, drop_layer, conv_layer, kernel_size=3,
                           padding=1, stride=2, bias=(norm_layer is None)),
            *conv_sequence(out_channels, 2 * out_channels // compression, act_layer, norm_layer, drop_layer, conv_layer,
                           kernel_size=1, bias=(norm_layer is None)),
        )
        self.main = FusedSequential(
            *[ResBlock(out_channels // compression, out_channels // compression if num_blocks > 1 else in_channels,
                       act_layer, norm_layer, drop_layer, conv_layer) for _ in range(num_blocks)],
            *conv_sequence(out_channels // compression, out_channels // compression, act_layer, norm_layer, drop_layer,
                           conv_layer, kernel_size=1, bias=(norm_layer is None)),
        )
        self.transition = FusedSequential(
            *conv_sequence(2 * out_channels // compression, out_channels, act_layer, norm_layer, drop_layer, conv_layer,
                           kernel_size=1, bias=(norm_layer is None)))

    def forward(self, x: Tensor) -> Tensor:
        x = self.base_layer(x)
        x1, x2 = x.chunk(2, dim=1)
        return self.transition(torch.cat([x1, self.main(x2)], dim=1))


class DarknetBodyV4(nn.Sequential):
    """reference darknetv4.py:118-182."""

    def __init__(self, layout: List[Tuple[int, int]], in_channels: int = 3, stem_channels: int = 32, num_features: int = 1,
                 act_layer=None, norm_layer=None, drop_layer=None, conv_layer=None) -> None:
        if act_layer is None:
            act_layer = nn.LeakyReLU(inplace=True)
        if norm_layer is None:
            norm_layer = nn.BatchNorm2d
        in_chans = [stem_channels] + [_layout[0] for _layout in layout[:-1]]
        super().__init__(OrderedDict([
            ("stem", FusedSequential(*conv_sequence(in_channels, stem_channels, act_layer, norm_layer, drop_layer, conv_layer,
                                                     kernel_size=3, padding=1, bias=(norm_layer is None)))),
            ("stages", nn.Sequential(*[CSPStage(_in, out, nb, act_layer, norm_layer, drop_layer, conv_layer)
                                       for _in, (out, nb) in zip(in_chans, layout)])),
        ]))
        self.num_features = num_features

    def forward(self, x: Tensor) -> Union[Tensor, List[Tensor]]:  # type: ignore[override]
        return _body_forward(self.stem, self.stages, x, self.num_features)


class DarknetV4(_DarknetClassifier):
    """reference darknetv4.py:185-220."""

    def __init__(self, layout: List[Tuple[int, int]], num_classes: int = 10, in_channels: int = 3, stem_channels: int = 32,
                 num_features: int = 1, act_layer=None, norm_layer=None, drop_layer=None, conv_layer=None) -> None:
        super().__init__(OrderedDict([
            ("features", DarknetBodyV4(layout, in_channels, stem_channels, num_features, act_layer, norm_layer, drop_layer,
                                       conv_layer)),
            ("pool", GlobalAvgPool2d(flatten=True)),
            ("classifier", nn.Linear(layout[-1][0], num_classes)),
        ]))
        init_module(self, "leaky_relu")


class DarknetBodyV1(nn.Sequential):
    """YOLOv1 backbone: 7x7 stride-2 stem, then max-pool + alternating 1x1 / 3x3 units; no normalisation layer by
    default, so the convolutions carry a bias that is fused with the LeakyReLU in the conv epilogue pass
    (reference holocron/models/classification/darknet.py:29-105)."""

    def __init__(self, layout: List[List[int]], in_channels: int = 3, stem_channels: int = 64, act_layer=None,
                 norm_layer=None, drop_layer=None, conv_layer=None) -> None:
        if act_layer is None:
            act_layer = nn.LeakyReLU(0.1, inplace=True)
        in_chans = [stem_channels] + [_layout[-1] for _layout in layout[:-1]]
        super().__init__(OrderedDict([
            ("stem", FusedSequential(*conv_sequence(in_channels, stem_channels, act_layer, norm_layer, drop_layer, conv_layer,
                                                     kernel_size=7, padding=3, stride=2, bias=(norm_layer is None)))),
            ("layers", nn.Sequential(*[self._make_layer([_in, *planes], act_layer, norm_layer, drop_layer, conv_layer)
                                       for _in, planes in zip(in_chans, layout)])),
        ]))
        init_module(self, "leaky_relu")

    @staticmethod
    def _make_layer(planes: List[int], act_layer=None, norm_layer=None, drop_layer=None, conv_layer=None):
        layers: List[nn.Module] = [nn.MaxPool2d(2)]
        for in_planes, out_planes in zip(planes[:-1], planes[1:]):
            grow = out_planes > in_planes
            layers.extend(conv_sequence(in_planes, out_planes, act_layer, norm_layer, drop_layer, conv_layer,
                                        kernel_size=3 if grow else 1, padding=1 if grow else 0,
                                        bias=(norm_layer is None)))
        return FusedSequential(*layers)


class DarknetV1(_DarknetClassifier):
    """reference darknet.py:108-133."""

    def __init__(self, layout: List[List[int]], num_classes: int = 10, in_channels: int = 3, stem_channels: int = 64,
                 act_layer=None, norm_layer=None, drop_layer=None, conv_layer=None) -> None:
        super().__init__(OrderedDict([
            ("features", DarknetBodyV1(layout, in_channels, stem_channels, act_layer, norm_layer, drop_layer, conv_layer)),
            ("pool", GlobalAvgPool2d(flatten=True)),
            ("classifier", nn.Linear(layout[2][-1], num_classes)),
        ]))
        init_module(self, "leaky_relu")


class DarknetBodyV2(nn.Sequential):
    """YOLOv2 backbone (reference darknetv2.py:32-148): 3x3 stem, then per stage max-pool + 3x3 + n x (1x1, 3x3)."""

    def __init__(self, layout: List[Tuple[int, int]], in_channels: int = 3, stem_channels: int = 32, passthrough: bool = False,
                 act_layer=None, norm_layer=None, drop_layer=None, conv_layer=None) -> None:
        if act_layer is None:
            act_layer = nn.LeakyReLU(0.1, inplace=True)
        if norm_layer is None:
            norm_layer = nn.BatchNorm2d
        in_chans = [stem_channels] + [_layout[0] for _layout in layout[:-1]]
        super().__init__(OrderedDict([
            ("stem", FusedSequential(*conv_sequence(in_channels, stem_channels, act_layer, norm_layer, drop_layer, conv_layer,
                                                     kernel_size=3, padding=1, bias=(norm_layer is None)))),
            ("layers", nn.Sequential(*[self._make_layer(nb, _in, out, act_layer, norm_layer, drop_layer, conv_layer)
                                       for _in, (out, nb) in zip(in_chans, layout)])),
        ]))
        self.passthrough = passthrough

    @staticmethod
    def _make_layer(num_blocks: int, in_planes: int, out_planes: int, act_layer=None, norm_layer=None, drop_layer=None,
                    conv_layer=None):
        layers: List[nn.Module] = [nn.MaxPool2d(2)]
        layers.extend(conv_sequence(in_planes, out_planes, act_layer, norm_layer, drop_layer, conv_layer, kernel_size=3,
                                    padding=1, stride=1, bias=(norm_layer is None)))
        for _ in range(num_blocks):
            layers.extend(conv_sequence(out_planes, out_planes // 2, act_layer, norm_layer, drop_layer, conv_layer,
                                        kernel_size=1, padding=0, stride=1, bias=(norm_layer is None)))
            layers.extend(conv_sequence(out_planes // 2, out_planes, act_layer, norm_layer, drop_layer, conv_layer,
                                        kernel_size=3, padding=1, stride=1, bias=(norm_layer is None)))
        return FusedSequential(*layers)

    def forward(self, x: Tensor):  # type: ignore[override]
        x = self.stem(x)
        aux = None
        for idx, layer in enumerate(self.layers):
            x = layer(x)
            if self.passthrough and idx == len(self.layers) - 2:
                aux = x.clone()
        return (x, aux) if self.passthrough else x


class DarknetV2(nn.Sequential):
    """reference darknetv2.py:151-178 (1x1 convolution classifier followed by global average pooling)."""

    def __init__(self, layout: List[Tuple[int, int]], num_classes: int = 10, in_channels: int = 3, stem_channels: int = 32,
                 act_layer=None, norm_layer=None, drop_layer=None, conv_layer=None) -> None:
        super().__init__(OrderedDict([
            ("features", DarknetBodyV2(layout, in_channels, stem_channels, False, act_layer, norm_layer, drop_layer,
                                       conv_layer)),
            ("classifier", nn.Conv2d(layout[-1][0], num_classes, 1)),
            ("pool", GlobalAvgPool2d(flatten=True)),
        ]))
        init_module(self, "leaky_relu")

    def forward(self, x: Tensor) -> Tensor:  # type: ignore[override]
        from .._blocks import conv_bn_act
        feats = self.features(x)
        logits = conv_bn_act(feats, self.classifier, None, None, keep_padded=False)
        return logits.float().mean((2, 3))


def _no_pretrained(pretrained: bool, checkpoint: Any):
    """The factories' pretrained / checkpoint arguments -> the checkpoint to load (None: seeded initialisation)."""
    return _requested_checkpoint(pretrained, checkpoint)


def darknet24(pretrained: bool = False, progress: bool = True, **kwargs: Any) -> DarknetV1:
    """Darknet-24 / YOLOv1 backbone (reference darknet.py:143-159)."""
    ckpt = _no_pretrained(pretrained, None)
    return _configure_model(DarknetV1([[192], [128, 256, 256, 512], [*([256, 512] * 4), 512, 1024], [512, 1024] * 2], **kwargs), ckpt)


def darknet19(pretrained: bool = False, checkpoint: Any = None, progress: bool = True, **kwargs: Any) -> DarknetV2:
    """Darknet-19 / YOLOv2 backbone (reference darknetv2.py:211-237)."""
    ckpt = _no_pretrained(pretrained, checkpoint)
    return _configure_model(DarknetV2([(64, 0), (128, 1), (256, 1), (512, 2), (1024, 2)], **kwargs), ckpt)


def darknet53(pretrained: bool = False, checkpoint: Any = None, progress: bool = True, **kwargs: Any) -> DarknetV3:
    """Darknet-53 (reference darknetv3.py:218-244)."""
    ckpt = _no_pretrained(pretrained, checkpoint)
    return _configure_model(DarknetV3([(64, 1), (128, 2), (256, 8), (512, 8), (1024, 4)], **kwargs), ckpt)


def cspdarknet53(pretrained: bool = False, checkpoint: Any = None, progress: bool = True, **kwargs: Any) -> DarknetV4:
    """CSP-Darknet-53 (reference darknetv4.py:249-275)."""
    ckpt = _no_pretrained(pretrained, checkpoint)
    return _configure_model(DarknetV4([(64, 1), (128, 2), (256, 8), (512, 8), (1024, 4)], **kwargs), ckpt)


def cspdarknet53_mish(pretrained: bool = False, checkpoint: Any = None, progress: bool = True, **kwargs: Any) -> DarknetV4:
    """CSP-Darknet-53 with Mish activations and DropBlock regularisation (reference darknetv4.py:296-326)."""
    ckpt = _no_pretrained(pretrained, checkpoint)
    kwargs["act_layer"] = nn.Mish(inplace=True)
    kwargs["drop_layer"] = DropBlock2d
    return _configure_model(DarknetV4([(64, 1), (128, 2), (256, 8), (512, 8), (1024, 4)], **kwargs), ckpt)
