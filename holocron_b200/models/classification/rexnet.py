"""ReXNet on the fused kernels — API mirror of holocron/models/classification/rexnet.py (SEBlock :38-66, ReXBlock :69-143,
ReXNet :146-229, factories :275-534).

Module tree / ``state_dict`` / init order are the reference's. ReXNet's channel widths (27, 38, 50, 61, ... and their x6
expansions) are not multiples of the kernels' channel granularity, so activations are carried zero-padded to a multiple
of 16 channels *between* the fused ops (filters are packed with zero rows/columns, BatchNorm treats the padding as
``scale = shift = 0``): padded channels stay exactly zero through conv, BN, SiLU/ReLU6, the depth-wise conv and the
partial-channel shortcut, and gradients of the padding never reach a parameter.

Per block: 1x1 expand (tensor cores) -> fused BN+SiLU -> depth-wise 3x3 kernel -> fused BN -> [SE gate from the pooled map]
-> ReLU6 -> 1x1 project (tensor cores) -> fused BN (+ shortcut on the first ``in_channels`` channels, reference rexnet.py:141).
"""
import functools
import operator
from collections import OrderedDict
from math import ceil
from typing import Any, Callable, Optional

import torch
import torch.nn.functional as TF
from torch import Tensor, nn

from ...nn import GlobalAvgPool2d, init
from ...nn import _fused as K
from ...nn._dwconv import dwconv2d
from .._blocks import conv_bn_act
from ..utils import _configure_model, _requested_checkpoint, conv_sequence

__all__ = ["ReXBlock", "ReXNet", "SEBlock", "rexnet1_0x", "rexnet1_3x", "rexnet1_5x", "rexnet2_0x", "rexnet2_2x"]


def _pad_channels(x: Tensor, c: int) -> Tensor:
    return x if x.shape[1] == c else TF.pad(x, (0, 0, 0, 0, 0, c - x.shape[1]))


class SEBlock(nn.Module):
    """Squeeze-excite gate: GAP -> 1x1 -> BN -> act -> 1x1(+bias) -> sigmoid (reference rexnet.py:38-66)."""

    def __init__(self, channels: int, se_ratio: int = 12, act_layer: Optional[nn.Module] = None,
                 norm_layer: Optional[Callable[[int], nn.Module]] = None, drop_layer=None) -> None:
        super().__init__()
        self.pool = GlobalAvgPool2d(flatten=False)
        self.conv = nn.Sequential(
            *conv_sequence(channels, channels // se_ratio, act_layer, norm_layer, drop_layer, kernel_size=1, stride=1,
                           bias=(norm_layer is None)),
            *conv_sequence(channels // se_ratio, channels, nn.Sigmoid(), None, drop_layer, kernel_size=1, stride=1),
        )

    def gate(self, x: Tensor, channels: int) -> Tensor:
        """(N, C_padded, H, W) -> sigmoid gate (N, C_padded, 1, 1); the squeeze path works on (N, C, 1, 1) tensors."""
        y = self.pool(x)[:, :channels].float()
        y = self.conv(y)
        return _pad_channels(y, x.shape[1]).to(x.dtype)

    def forward(self, x: Tensor) -> Tensor:
        return x * self.gate(x, x.shape[1])


class ReXBlock(nn.Module):
    """Inverted-bottleneck block with a partial-channel shortcut (reference rexnet.py:69-143)."""

    def __init__(self, in_channels: int, channels: int, t: int, stride: int, use_se: bool = True, se_ratio: int = 12,
                 act_layer: Optional[nn.Module] = None, norm_layer: Optional[Callable[[int], nn.Module]] = None,
                 drop_layer=None) -> None:
        super().__init__()
        if act_layer is None:
            act_layer = nn.ReLU6(inplace=True)
        if norm_layer is None:
            norm_layer = nn.BatchNorm2d
        self.use_shortcut = stride == 1 and in_channels <= channels
        self.in_channels = in_channels
        self.out_channels = channels
        layers = []
        if t != 1:
            dw_channels = in_channels * t
            layers.extend(conv_sequence(in_channels, dw_channels, nn.SiLU(inplace=True), norm_layer, drop_layer,
                                        kernel_size=1, stride=1, bias=(norm_layer is None)))
        else:
            dw_channels = in_channels
        layers.extend(conv_sequence(dw_channels, dw_channels, None, norm_layer, drop_layer, kernel_size=3, stride=stride,
                                    padding=1, bias=(norm_layer is None), groups=dw_channels))
        if use_se:
            layers.append(SEBlock(dw_channels, se_ratio, act_layer, norm_layer, drop_layer))
        layers.append(act_layer)
        layers.extend(conv_sequence(dw_channels, channels, None, norm_layer, drop_layer, kernel_size=1, stride=1,
                                    bias=(norm_layer is None)))
        self.conv = nn.Sequential(*layers)
        self._dw_channels = dw_channels

    def forward(self, x: Tensor, keep_padded: bool = False) -> Tensor:
        mods = list(self.conv)
        if not all(isinstance(m, (nn.Conv2d, nn.SiLU, nn.ReLU6, SEBlock)) or K.is_batch_norm(m) for m in mods):
            raise NotImplementedError("fused ReXBlock expects the default BatchNorm2d (or SyncBatchNorm) / SiLU / ReLU6 layers")
        xin = K.to_channels_last_bf16(x, K.round_up(x.shape[1], 16))
        i = 0
        y = xin
        if isinstance(mods[0], nn.Conv2d) and mods[0].groups == 1:          # 1x1 expansion -> BN -> SiLU
            y = conv_bn_act(y, mods[0], mods[1], mods[2], keep_padded=True)
            i = 3
        dw, bn_dw = mods[i], mods[i + 1]                                     # depth-wise 3x3 -> BN
        cp = y.shape[1]
        w_dw = _pad_channels(dw.weight.permute(1, 0, 2, 3), cp).permute(1, 0, 2, 3) if cp != dw.weight.shape[0] else dw.weight
        b_dw = None if dw.bias is None else TF.pad(dw.bias, (0, cp - dw.bias.shape[0]))
        tdw = dwconv2d(y, w_dw, b_dw, dw.stride[0], dw.padding[0])
        tdw = K.bn_act([tdw], [bn_dw], K.ACT_NONE)
        i += 2
        if isinstance(mods[i], SEBlock):
            gate = mods[i].gate(tdw, self._dw_channels)
            u = K.gate_act(tdw, gate, *K.act_code(mods[i + 1]))                # x * gate -> ReLU6 in one pass
            i += 1
        else:
            u = K.act_only(tdw, *K.act_code(mods[i]))                        # ReLU6
        proj, bn_proj = mods[i + 1], mods[i + 2]                             # 1x1 projection -> BN (+ shortcut)
        out = K.conv2d(u, proj.weight, proj.bias, 1, 0, keep_padded=True, want_stats=bn_proj.training)
        res = _pad_channels(xin, out.shape[1]) if self.use_shortcut else None
        out = K.bn_act([out], [bn_proj], K.ACT_NONE, residual=res)
        return out if keep_padded else out[:, :self.out_channels]


class ReXNet(nn.Sequential):
    """ReXNet (https://arxiv.org/abs/2007.00992) — reference rexnet.py:146-229."""

    def __init__(self, width_mult: float = 1.0, depth_mult: float = 1.0, num_classes: int = 1000, in_channels: int = 3,
                 in_planes: int = 16, final_planes: int = 180, use_se: bool = True, se_ratio: int = 12,
                 dropout_ratio: float = 0.2, bn_momentum: float = 0.9, act_layer: Optional[nn.Module] = None,
                 norm_layer: Optional[Callable[[int], nn.Module]] = None, drop_layer=None) -> None:
        super().__init__()
        if act_layer is None:
            act_layer = nn.SiLU(inplace=True)
        if norm_layer is None:
            norm_layer = nn.BatchNorm2d
        num_blocks = [ceil(element * depth_mult) for element in [1, 2, 2, 3, 3, 5]]
        strides = functools.reduce(operator.iadd, [[element] + [1] * (num_blocks[idx] - 1)
                                                   for idx, element in enumerate([1, 2, 2, 2, 1, 2])], [])
        depth = sum(num_blocks)
        stem_channel = 32 / width_mult if width_mult < 1.0 else 32
        inplanes = in_planes / width_mult if width_mult < 1.0 else in_planes
        chans = [round(width_mult * stem_channel)]
        chans.extend([round(width_mult * (inplanes + idx * final_planes / depth)) for idx in range(depth)])
        ses = [False] * (num_blocks[0] + num_blocks[1]) + [use_se] * sum(num_blocks[2:])
        layers = conv_sequence(in_channels, chans[0], act_layer, norm_layer, drop_layer, kernel_size=3, stride=2, padding=1,
                               bias=(norm_layer is None))
        t = 1
        for in_c, c, s, se in zip(chans[:-1], chans[1:], strides, ses):
            # as in the reference, act/norm/drop layers are NOT forwarded to the blocks (rexnet.py:201-203)
            layers.append(ReXBlock(in_channels=in_c, channels=c, t=t, stride=s, use_se=se, se_ratio=se_ratio))
            t = 6
        pen_channels = int(width_mult * 1280)
        layers.extend(conv_sequence(chans[-1], pen_channels, act_layer, norm_layer, drop_layer, kernel_size=1, stride=1,
                                    padding=0, bias=(norm_layer is None)))
        super().__init__(OrderedDict([
            ("features", nn.Sequential(*layers)),
            ("pool", GlobalAvgPool2d(flatten=True)),
            ("head", nn.Sequential(nn.Dropout(dropout_ratio), nn.Linear(pen_channels, num_classes))),
        ]))
        init.init_module(self, nonlinearity="relu")

    def forward(self, x: Tensor) -> Tensor:  # type: ignore[override]
        mods = list(self.features)
        i = 0
        while i < len(mods):
            m = mods[i]
            if isinstance(m, ReXBlock):
                x = m(x, keep_padded=True)
                i += 1
            elif isinstance(m, nn.Conv2d):
                bn = mods[i + 1] if K.is_batch_norm(mods[i + 1]) else None
                j = i + (2 if bn is not None else 1)
                act = mods[j] if j < len(mods) and not isinstance(mods[j], (nn.Conv2d, ReXBlock)) else None
                x = conv_bn_act(x, m, bn, act, keep_padded=True)
                i = j + (1 if act is not None else 0)
            else:
                x = m(x)
                i += 1
        feats = self.pool(x)
        drop, lin = self.head[0], self.head[1]
        feats = drop(feats)[:, :lin.in_features]
        return K.head_linear(feats, lin.weight, lin.bias)


def _rexnet(width_mult: float, depth_mult: float, pretrained: bool, checkpoint: Any, **kwargs: Any) -> ReXNet:
    checkpoint = _requested_checkpoint(pretrained, checkpoint)
    return _configure_model(ReXNet(width_mult, depth_mult, **kwargs), checkpoint)


def rexnet1_0x(pretrained: bool = False, checkpoint: Any = None, progress: bool = True, **kwargs: Any) -> ReXNet:
    """ReXNet-1.0x (reference rexnet.py:275-301)."""
    return _rexnet(1, 1, pretrained, checkpoint, **kwargs)


def rexnet1_3x(pretrained: bool = False, checkpoint: Any = None, progress: bool = True, **kwargs: Any) -> ReXNet:
    """ReXNet-1.3x (reference rexnet.py:337-363)."""
    return _rexnet(1.3, 1, pretrained, checkpoint, **kwargs)


def rexnet1_5x(pretrained: bool = False, checkpoint: Any = None, progress: bool = True, **kwargs: Any) -> ReXNet:
    """ReXNet-1.5x (reference rexnet.py:399-425)."""
    return _rexnet(1.5, 1, pretrained, checkpoint, **kwargs)


def rexnet2_0x(pretrained: bool = False, checkpoint: Any = None, progress: bool = True, **kwargs: Any) -> ReXNet:
    """ReXNet-2.0x (reference rexnet.py:461-487)."""
    return _rexnet(2, 1, pretrained, checkpoint, **kwargs)


def rexnet2_2x(pretrained: bool = False, checkpoint: Any = None, progress: bool = True, **kwargs: Any) -> ReXNet:
    """ReXNet-2.2x (reference rexnet.py:508-534)."""
    return _rexnet(2.2, 1, pretrained, checkpoint, **kwargs)
