"""RepVGG on the H100 kernels — API mirror of holocron/models/classification/repvgg.py.

Same module tree / ``state_dict`` keys as the reference (``features.<stage>.<block>.branches.{0,1}.{0,1}.*``,
``features.<stage>.<block>.branches.2.*`` for the identity BN, ``head.*``; after ``reparametrize()``:
``...branches.weight/.bias``), same constructor arguments and the same RNG call order at init, so parameters are
interchangeable with the reference and ``torch.manual_seed(s)`` gives identical weights.

What differs is the execution: a train-form block is two wgmma implicit-GEMM convolutions (3x3 and 1x1) over
bf16 NHWC activations, one statistics pass and ONE fused pass that normalises the three branches, sums them and
applies the activation (reference: 2 cuDNN convs + 3 BatchNorm kernels + 2 adds + ReLU). A re-parametrised block
is a single convolution with bias and ReLU fused in its epilogue.
"""
from collections import OrderedDict
from typing import Any, Callable, List, Optional, Union, cast

import torch
import torch.nn.functional as TF
from torch import Tensor, nn

from ...nn import GlobalAvgPool2d, init
from ...nn import _fused as K
from ..utils import _configure_model, _requested_checkpoint, conv_sequence, fuse_conv_bn

__all__ = ["RepBlock", "RepVGG", "repvgg_a0", "repvgg_a1", "repvgg_a2", "repvgg_b0", "repvgg_b1", "repvgg_b2",
           "repvgg_b3"]


class RepBlock(nn.Module):
    """act(BN(conv3x3(x)) + BN(conv1x1(x)) [+ BN(x)]) — reference repvgg.py:38-107."""

    def __init__(
        self,
        inplanes: int,
        planes: int,
        stride: int = 1,
        identity: bool = True,
        act_layer: Optional[nn.Module] = None,
        norm_layer: Optional[Callable[[int], nn.Module]] = None,
    ) -> None:
        super().__init__()
        if norm_layer is None:
            norm_layer = nn.BatchNorm2d
        if act_layer is None:
            act_layer = nn.ReLU(inplace=True)
        self.branches: Union[nn.Conv2d, nn.ModuleList] = nn.ModuleList([
            nn.Sequential(*conv_sequence(inplanes, planes, None, norm_layer, kernel_size=3, padding=1, stride=stride)),
            nn.Sequential(*conv_sequence(inplanes, planes, None, norm_layer, kernel_size=1, padding=0, stride=stride)),
        ])
        self.activation = act_layer
        if identity:
            if inplanes != planes:
                raise ValueError("The number of input and output channels must be identical if identity is used")
            self.branches.append(norm_layer(planes))

    def _act(self):
        try:
            return K.act_code(self.activation) + (None,)
        except NotImplementedError:
            return K.ACT_NONE, 0.0, self.activation

    def forward(self, x: Tensor) -> Tensor:
        code, slope, post = self._act()
        if isinstance(self.branches, nn.Conv2d):
            out = K.conv2d_bias_act(x, self.branches.weight, self.branches.bias, self.branches.stride[0], 1, code, slope)
            return out if post is None else post(out)
        conv3, bn3 = cast(nn.Sequential, self.branches[0])
        conv1, bn1 = cast(nn.Sequential, self.branches[1])
        bns = [bn3, bn1] + ([self.branches[2]] if len(self.branches) == 3 else [])
        if not all(K.is_batch_norm(b) for b in bns):
            raise NotImplementedError("the fused RepBlock needs nn.BatchNorm2d or nn.SyncBatchNorm as norm_layer")
        if conv3.out_channels % 16 == 0 and all(b.eps == bn3.eps and b.momentum == bn3.momentum for b in bns) \
                and bn3.momentum is not None:
            # whole block as one autograd node (input-gradient contributions chained through the conv epilogues)
            # batch statistics iff the BatchNorm layers are in training mode (they may be frozen inside a training model)
            out = K.repblock(x, conv3.weight, conv1.weight, bns, conv3.stride[0], code, slope, bn3.training)
            return out if post is None else post(out)
        # generic composition: one bf16 NHWC copy of the input shared by both convolutions
        xb = K.to_channels_last_bf16(x, K.round_up(x.shape[1], 8))
        y3 = K.conv2d(xb, conv3.weight, None, conv3.stride[0], 1)
        y1 = K.conv2d(xb, conv1.weight, None, conv1.stride[0], 0)
        us = [y3, y1] + ([xb] if len(bns) == 3 else [])
        out = K.bn_act(us, bns, code, slope, training=bn3.training)
        return out if post is None else post(out)

    @torch.no_grad()
    def reparametrize(self) -> None:
        """Folds the three branches into one 3x3 convolution with bias (weight-sized fp32 arithmetic, same
        operation order as reference repvgg.py:75-107 so the folded weights match to the last bit)."""
        if not isinstance(self.branches, nn.ModuleList):
            raise AssertionError
        conv3 = cast(nn.Sequential, self.branches[0])[0]
        inplanes, planes = conv3.weight.data.shape[1], conv3.weight.data.shape[0]
        rep = nn.Conv2d(inplanes, planes, 3, padding=1, bias=True, stride=conv3.stride).to(conv3.weight.device)
        k3, b3 = fuse_conv_bn(*self.branches[0])
        k1, b1 = fuse_conv_bn(*self.branches[1])
        rep.weight.data = k3
        rep.bias.data = b3
        rep.weight.data[..., 1:2, 1:2] += k1
        rep.bias.data += b1
        if len(self.branches) == 3:
            bn = self.branches[2]
            scale = bn.weight.data / (bn.running_var + bn.eps).sqrt()
            rep.weight.data[range(planes), range(inplanes), 1, 1] += scale
            rep.bias.data += bn.bias.data
            rep.bias.data -= scale * bn.running_mean
        self.branches = rep


class RepVGG(nn.Sequential):
    """RepVGG — reference repvgg.py:110-171 (Holocron's layout: 5 stages of ``1 + num_blocks[i]`` blocks)."""

    def __init__(
        self,
        num_blocks: List[int],
        planes: List[int],
        width_multiplier: float,
        final_width_multiplier: float,
        num_classes: int = 10,
        in_channels: int = 3,
        act_layer: Optional[nn.Module] = None,
        norm_layer: Optional[Callable[[int], nn.Module]] = None,
    ) -> None:
        if norm_layer is None:
            norm_layer = nn.BatchNorm2d
        if act_layer is None:
            act_layer = nn.ReLU(inplace=True)
        if len(num_blocks) != len(planes):
            raise AssertionError("the length of `num_blocks` and `planes` are expected to be the same")
        chans = [in_channels, int(min(1, width_multiplier) * planes[0])]
        chans.extend([int(width_multiplier * chan) for chan in planes[1:-1]])
        chans.append(int(final_width_multiplier * planes[-1]))
        stages: List[nn.Sequential] = []
        for nb_blocks, in_chan, out_chan in zip(num_blocks, chans[:-1], chans[1:]):
            layers = [RepBlock(in_chan, out_chan, 2, False, act_layer, norm_layer)]
            layers.extend([RepBlock(out_chan, out_chan, 1, True, act_layer, norm_layer) for _ in range(nb_blocks)])
            stages.append(nn.Sequential(*layers))
        super().__init__(
            OrderedDict([
                ("features", nn.Sequential(*stages)),
                ("pool", GlobalAvgPool2d(flatten=True)),
                ("head", nn.Linear(chans[-1], num_classes)),
            ])
        )
        init.init_module(self, nonlinearity="relu")

    def forward(self, x: Tensor) -> Tensor:
        feats = self.pool(self.features(x))
        head = cast(nn.Linear, self.head)
        return K.head_linear(feats, head.weight, head.bias)

    def reparametrize(self) -> None:
        """Re-parametrises every block (inference form)."""
        self.features: nn.Sequential
        for stage in self.features:
            for block in stage:
                block.reparametrize()


def _repvgg(num_blocks: List[int], a: float, b: float, pretrained: bool, checkpoint: Any, **kwargs: Any) -> RepVGG:
    checkpoint = _requested_checkpoint(pretrained, checkpoint)
    return _configure_model(RepVGG(num_blocks, [64, 64, 128, 256, 512], a, b, **kwargs), checkpoint)


def repvgg_a0(pretrained: bool = False, checkpoint: Any = None, progress: bool = True, **kwargs: Any) -> RepVGG:
    """RepVGG-A0 (reference repvgg.py:206-232)."""
    return _repvgg([1, 2, 4, 14, 1], 0.75, 2.5, pretrained, checkpoint, **kwargs)


def repvgg_a1(pretrained: bool = False, checkpoint: Any = None, progress: bool = True, **kwargs: Any) -> RepVGG:
    """RepVGG-A1 (reference repvgg.py:253-279)."""
    return _repvgg([1, 2, 4, 14, 1], 1, 2.5, pretrained, checkpoint, **kwargs)


def repvgg_a2(pretrained: bool = False, checkpoint: Any = None, progress: bool = True, **kwargs: Any) -> RepVGG:
    """RepVGG-A2 (reference repvgg.py:300-326)."""
    return _repvgg([1, 2, 4, 14, 1], 1.5, 2.75, pretrained, checkpoint, **kwargs)


def repvgg_b0(pretrained: bool = False, checkpoint: Any = None, progress: bool = True, **kwargs: Any) -> RepVGG:
    """RepVGG-B0 (reference repvgg.py:347-373)."""
    return _repvgg([1, 4, 6, 16, 1], 1, 2.5, pretrained, checkpoint, **kwargs)


def repvgg_b1(pretrained: bool = False, checkpoint: Any = None, progress: bool = True, **kwargs: Any) -> RepVGG:
    """RepVGG-B1 (reference repvgg.py:394-420)."""
    return _repvgg([1, 4, 6, 16, 1], 2, 4, pretrained, checkpoint, **kwargs)


def repvgg_b2(pretrained: bool = False, checkpoint: Any = None, progress: bool = True, **kwargs: Any) -> RepVGG:
    """RepVGG-B2 (reference repvgg.py:441-467)."""
    return _repvgg([1, 4, 6, 16, 1], 2.5, 5, pretrained, checkpoint, **kwargs)


def repvgg_b3(pretrained: bool = False, checkpoint: Any = None, progress: bool = True, **kwargs: Any) -> RepVGG:
    """RepVGG-B3 (reference repvgg.py:476-498)."""
    return _repvgg([1, 4, 6, 16, 1], 3, 5, pretrained, checkpoint, **kwargs)
