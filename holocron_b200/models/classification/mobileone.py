"""MobileOne on the fused kernels — API mirror of holocron/models/classification/mobileone.py (DepthConvBlock :27-91,
PointConvBlock :94-147, MobileOneBlock :150-177, MobileOne :180-230, factories :233-439).

The re-parametrisable sibling of RepVGG: a block is ``act(sum of BatchNorm'd depth-wise branches)`` followed by
``act(sum of BatchNorm'd 1x1 branches)`` - an identity BatchNorm (when shapes allow), a depth-wise 1x1 "scale" branch and
``overparam_factor`` 3x3 / 1x1 branches. Module tree, parameter names and init order are the reference's. Every branch
convolution runs on the depth-wise / tensor-core kernels and ALL BatchNorms of a branch sum plus the activation are folded into
fused passes of at most three branches each (the running sum of the previous pass enters the next one as its residual); the
reference issues one BatchNorm kernel per branch, ``len(branches) - 1`` additions and the activation.
``reparametrize()`` folds every branch into one convolution with a bias exactly like the reference (host-side, fp32)."""
from collections import OrderedDict
from typing import Any, Callable, List, Optional, Tuple

import torch
from torch import Tensor, nn

from ...nn import GlobalAvgPool2d, init
from ...nn import _fused as K
from .._blocks import _dense_ok, _depthwise_ok, conv_bn_act
from ..utils import _configure_model, _requested_checkpoint, conv_sequence, fuse_conv_bn

__all__ = ["DepthConvBlock", "MobileOne", "MobileOneBlock", "PointConvBlock", "mobileone_s0", "mobileone_s1", "mobileone_s2",
           "mobileone_s3"]


def _fused_branch_sum(branches: nn.ModuleList, x: Tensor, act: Optional[nn.Module]) -> Tensor:
    """act(sum_b BN_b(conv_b(x))) with the identity branch's conv_b = id; fused passes of <= 3 branches chained through the
    residual input of the next pass."""
    from ...nn._dwconv import dwconv2d
    pairs: List[Tuple[Tensor, nn.BatchNorm2d]] = []
    xb = None
    for mod in branches:
        if K.is_batch_norm(mod):
            xb = K.to_channels_last_bf16(x) if xb is None else xb
            pairs.append((xb, mod))
            continue
        conv, bn = mod[0], mod[1]
        if _depthwise_ok(conv):
            u = dwconv2d(x, conv.weight, conv.bias, conv.stride[0], conv.padding[0])
        else:
            u = K.conv2d(x, conv.weight, conv.bias, conv.stride[0], conv.padding[0], keep_padded=True,
                         want_stats=bn.training or bn.running_mean is None)
        pairs.append((u, bn))
    code, slope = K.act_code(act)
    out = None
    for i in range(0, len(pairs), 3):
        chunk = pairs[i:i + 3]
        last = i + 3 >= len(pairs)
        out = K.bn_act([u for u, _ in chunk], [bn for _, bn in chunk], code if last else K.ACT_NONE, slope if last else 0.0,
                       residual=out)
    return out


def _fusable(branches: nn.ModuleList, x: Tensor) -> bool:
    for mod in branches:
        if K.is_batch_norm(mod):
            if mod.num_features % 8 != 0:
                return False
        elif not (isinstance(mod, nn.Sequential) and len(mod) == 2 and isinstance(mod[0], nn.Conv2d)
                  and K.is_batch_norm(mod[1]) and mod[1].num_features % 8 == 0
                  and (_depthwise_ok(mod[0]) or _dense_ok(mod[0]))):
            return False
    return x.ndim == 4


class _BranchSum(nn.ModuleList):
    """Sum of parallel [BatchNorm] / [conv, BatchNorm] branches (the reference's ``sum(mod(x) for mod in self)``)."""

    def forward(self, x: Tensor, act: Optional[nn.Module] = None) -> Tensor:
        if _fusable(self, x):
            return _fused_branch_sum(self, x, act)
        # e.g. the 3-channel depth-wise branches of the first block: library modules on a tiny tensor
        out = sum(mod(x.float()) for mod in self)
        return out if act is None else act(out)


class DepthConvBlock(_BranchSum):
    """Re-parametrisable depth-wise block (reference mobileone.py:27-91): [BN (stride 1)] + dw1x1-BN + num_blocks x dw3x3-BN."""

    def __init__(self, channels: int, num_blocks: int, stride: int = 1,
                 norm_layer: Optional[Callable[[int], nn.Module]] = None) -> None:
        if norm_layer is None:
            norm_layer = nn.BatchNorm2d
        layers: List[nn.Module] = [norm_layer(channels)] if stride == 1 else []
        layers.append(nn.Sequential(*conv_sequence(channels, channels, kernel_size=1, stride=stride, norm_layer=norm_layer,
                                                   groups=channels)))
        layers.extend(nn.Sequential(*conv_sequence(channels, channels, kernel_size=3, padding=1, stride=stride,
                                                   norm_layer=norm_layer, groups=channels)) for _ in range(num_blocks))
        super().__init__(layers)

    def reparametrize(self) -> nn.Conv2d:
        """One depth-wise 3x3 convolution with bias equal to the (eval-mode) branch sum."""
        convs = [m for m in self if isinstance(m, nn.Sequential)]
        first = convs[0][0]
        chans = first.in_channels
        fused = nn.Conv2d(chans, chans, 3, padding=1, bias=True, stride=first.stride, groups=chans).to(first.weight.device)
        weight = torch.zeros_like(fused.weight.data)
        bias = torch.zeros_like(fused.bias.data)
        for mod in self:
            if K.is_batch_norm(mod):      # identity branch: a centre-tap filter
                scale = mod.weight.data / torch.sqrt(mod.running_var + mod.eps)
                bias += mod.bias.data - scale * mod.running_mean
                weight[..., 1, 1] += scale.unsqueeze(1)
                continue
            k, b = fuse_conv_bn(mod[0], mod[1])
            bias += b
            if k.shape[-1] == 1:                     # depth-wise 1x1 "scale" branch
                weight[..., 1:2, 1:2] += k
            else:
                weight += k
        fused.weight.data.copy_(weight)
        fused.bias.data.copy_(bias)
        return fused


class PointConvBlock(_BranchSum):
    """Re-parametrisable point-wise block (reference mobileone.py:94-147): [BN (in == out)] + num_blocks x conv1x1-BN."""

    def __init__(self, in_channels: int, out_channels: int, num_blocks: int,
                 norm_layer: Optional[Callable[[int], nn.Module]] = None) -> None:
        if norm_layer is None:
            norm_layer = nn.BatchNorm2d
        layers: List[nn.Module] = [norm_layer(out_channels)] if out_channels == in_channels else []
        layers.extend(nn.Sequential(*conv_sequence(in_channels, out_channels, kernel_size=1, norm_layer=norm_layer))
                      for _ in range(num_blocks))
        super().__init__(layers)

    def reparametrize(self) -> nn.Conv2d:
        """One 1x1 convolution with bias equal to the (eval-mode) branch sum."""
        convs = [m for m in self if isinstance(m, nn.Sequential)]
        first = convs[0][0]
        fused = nn.Conv2d(first.in_channels, first.out_channels, 1, bias=True).to(first.weight.device)
        weight = torch.zeros_like(fused.weight.data)
        bias = torch.zeros_like(fused.bias.data)
        for mod in self:
            if K.is_batch_norm(mod):      # identity branch: a diagonal filter
                scale = mod.weight.data / torch.sqrt(mod.running_var + mod.eps)
                bias += mod.bias.data - scale * mod.running_mean
                idx = torch.arange(weight.shape[0], device=weight.device)
                weight[idx, idx, 0, 0] += scale
                continue
            k, b = fuse_conv_bn(mod[0], mod[1])
            bias += b
            weight += k
        fused.weight.data.copy_(weight)
        fused.bias.data.copy_(bias)
        return fused


class MobileOneBlock(nn.Sequential):
    """Depth-wise block, activation, point-wise block, activation (reference mobileone.py:150-177)."""

    def __init__(self, in_channels: int, out_channels: int, overparam_factor: int = 1, stride: int = 1,
                 act_layer: Optional[nn.Module] = None, norm_layer: Optional[Callable[[int], nn.Module]] = None) -> None:
        if norm_layer is None:
            norm_layer = nn.BatchNorm2d
        if act_layer is None:
            act_layer = nn.ReLU(inplace=True)
        super().__init__(DepthConvBlock(in_channels, overparam_factor, stride, norm_layer), act_layer,
                         PointConvBlock(in_channels, out_channels, overparam_factor, norm_layer), act_layer)

    def forward(self, x: Tensor) -> Tensor:  # type: ignore[override]
        for idx in (0, 2):
            op, act = self[idx], self[idx + 1]
            if isinstance(op, _BranchSum):
                x = op(x, act)
            elif isinstance(op, nn.Conv2d) and (op.groups == 1 or op.in_channels % 8 == 0):
                x = conv_bn_act(x, op, None, act)      # re-parametrised form: one convolution + bias + activation
            else:
                x = act(op(x.float()))
        return x

    def reparametrize(self) -> None:
        """Replaces the two branch sums by their single-convolution equivalents."""
        self[0] = self[0].reparametrize()
        self[2] = self[2].reparametrize()


class MobileOne(nn.Sequential):
    """MobileOne (https://arxiv.org/abs/2206.04040) — reference mobileone.py:180-230, same constructor."""

    def __init__(self, num_blocks: List[int], width_multipliers: List[float], overparam_factor: int = 1, num_classes: int = 10,
                 in_channels: int = 3, act_layer: Optional[nn.Module] = None,
                 norm_layer: Optional[Callable[[int], nn.Module]] = None) -> None:
        if norm_layer is None:
            norm_layer = nn.BatchNorm2d
        if act_layer is None:
            act_layer = nn.ReLU(inplace=True)
        planes = [round(mult * chans) for mult, chans in zip(width_multipliers, [64, 128, 256, 512])]
        in_planes = min(64, planes[0])
        layers: List[nn.Module] = [MobileOneBlock(in_channels, in_planes, overparam_factor, 2, act_layer, norm_layer)]
        for nb, width in zip(num_blocks, planes):
            stage = [MobileOneBlock(in_planes, width, overparam_factor, 2, act_layer, norm_layer)]
            stage.extend(MobileOneBlock(width, width, overparam_factor, 1, act_layer, norm_layer) for _ in range(nb - 1))
            in_planes = width
            layers.append(nn.Sequential(*stage))
        super().__init__(OrderedDict([
            ("features", nn.Sequential(*layers)),
            ("pool", GlobalAvgPool2d(flatten=True)),
            ("head", nn.Linear(in_planes, num_classes)),
        ]))
        init.init_module(self, nonlinearity="relu")

    def forward(self, x: Tensor) -> Tensor:  # type: ignore[override]
        feats = self.pool(self.features(x))
        return K.head_linear(feats, self.head.weight, self.head.bias)

    def reparametrize(self) -> None:
        """Re-parametrises every block (inference form)."""
        self.features[0].reparametrize()
        for stage in self.features[1:]:
            for block in stage:
                block.reparametrize()


def _mobileone(pretrained: bool, checkpoint: Any, width_multipliers: List[float], overparam_factor: int, **kwargs: Any) -> MobileOne:
    checkpoint = _requested_checkpoint(pretrained, checkpoint)
    model = MobileOne([2, 8, 10, 1], width_multipliers, overparam_factor, **kwargs)
    return _configure_model(model, checkpoint)


def mobileone_s0(pretrained: bool = False, checkpoint: Any = None, progress: bool = True, **kwargs: Any) -> MobileOne:
    """MobileOne-S0 (reference mobileone.py:269-295): widths x(0.75, 1, 1, 2), over-parametrisation 4."""
    return _mobileone(pretrained, checkpoint, [0.75, 1.0, 1.0, 2.0], 4, **kwargs)


def mobileone_s1(pretrained: bool = False, checkpoint: Any = None, progress: bool = True, **kwargs: Any) -> MobileOne:
    """MobileOne-S1 (reference mobileone.py:317-343)."""
    return _mobileone(pretrained, checkpoint, [1.5, 1.5, 2.0, 2.5], 1, **kwargs)


def mobileone_s2(pretrained: bool = False, checkpoint: Any = None, progress: bool = True, **kwargs: Any) -> MobileOne:
    """MobileOne-S2 (reference mobileone.py:365-391)."""
    return _mobileone(pretrained, checkpoint, [1.5, 2.0, 2.5, 4.0], 1, **kwargs)


def mobileone_s3(pretrained: bool = False, checkpoint: Any = None, progress: bool = True, **kwargs: Any) -> MobileOne:
    """MobileOne-S3 (reference mobileone.py:413-439)."""
    return _mobileone(pretrained, checkpoint, [2.0, 2.5, 3.0, 4.0], 1, **kwargs)
