"""UNet3+ on the fused kernels — API mirror of holocron/models/segmentation/unet3p.py (+ ``down_path`` of unet.py:36-55).

Same module tree / ``state_dict`` as the reference. Every 3x3 convolution (encoder conv-BN-ReLU pairs, the 64-channel
branch convolutions of each full-scale aggregation, the 320-channel fusion conv-BN-ReLU) runs on the tensor-core
implicit-GEMM kernel; max-pooling, bilinear up-sampling and channel concatenation are bandwidth-trivial resampling ops
left to torch (they operate on the same bf16 channels_last tensors, no layout changes)."""
from typing import Any, Callable, List, Optional

import torch
from torch import Tensor, nn

from ...nn.init import init_module
from .._blocks import FusedSequential, conv_bn_act
from ..utils import conv_sequence

__all__ = ["FSAggreg", "UNet3p", "unet3p"]


def down_path(in_chan: int, out_chan: int, downsample: bool = True, padding: int = 0, act_layer=None, norm_layer=None,
              drop_layer=None, conv_layer=None) -> FusedSequential:
    """[MaxPool2d(2)] + 2 x [conv3x3 -> BN -> act] (reference unet.py:36-55)."""
    layers: List[nn.Module] = [nn.MaxPool2d(2)] if downsample else []
    layers.extend([
        *conv_sequence(in_chan, out_chan, act_layer, norm_layer, drop_layer, conv_layer, kernel_size=3, padding=padding),
        *conv_sequence(out_chan, out_chan, act_layer, norm_layer, drop_layer, conv_layer, kernel_size=3, padding=padding),
    ])
    return FusedSequential(*layers)


class FSAggreg(nn.Module):
    """Full-scale aggregation (reference unet3p.py:24-86): every shallower map is max-pooled, every deeper map is
    bilinearly up-sampled (align_corners=True) to this scale, each goes through its own 3x3 conv to ``base_chan``
    channels, the results are concatenated and fused by a conv-BN-act."""

    def __init__(self, e_chans: List[int], skip_chan: int, d_chans: List[int], act_layer=None, norm_layer=None,
                 drop_layer=None, conv_layer=None) -> None:
        super().__init__()
        base_chan = e_chans[0] if len(e_chans) > 0 else skip_chan
        depth = len(e_chans) + 1 + len(d_chans)
        self.downsamples = nn.ModuleList([
            FusedSequential(nn.MaxPool2d(2 ** (len(e_chans) - idx)), nn.Conv2d(e_chan, base_chan, 3, padding=1))
            for idx, e_chan in enumerate(e_chans)
        ])
        self.skip = nn.Conv2d(skip_chan, base_chan, 3, padding=1) if len(e_chans) > 0 else nn.Identity()
        self.upsamples = nn.ModuleList([
            FusedSequential(nn.Upsample(scale_factor=2 ** (idx + 1), mode="bilinear", align_corners=True),
                            nn.Conv2d(d_chan, base_chan, 3, padding=1))
            for idx, d_chan in enumerate(d_chans)
        ])
        self.block = FusedSequential(*conv_sequence(depth * base_chan, depth * base_chan, act_layer, norm_layer, drop_layer,
                                                     conv_layer, kernel_size=3, padding=1))

    def forward(self, downfeats: List[Tensor], feat: Tensor, upfeats: List[Tensor]) -> Tensor:
        if len(downfeats) != len(self.downsamples) or len(upfeats) != len(self.upsamples):
            raise ValueError(f"Expected {len(self.downsamples)} encoding & {len(self.upsamples)} decoding features, "
                             f"received: {len(downfeats)} & {len(upfeats)}")
        skip = feat if isinstance(self.skip, nn.Identity) else conv_bn_act(feat, self.skip, None, None)
        x = torch.cat((*[d(f) for d, f in zip(self.downsamples, downfeats)], skip,
                       *[u(f) for u, f in zip(self.upsamples, upfeats)]), dim=1)
        return self.block(x)


class UNet3p(nn.Module):
    """UNet3+ (reference unet3p.py:89-158)."""

    def __init__(self, layout: List[int], in_channels: int = 3, num_classes: int = 10, act_layer: Optional[nn.Module] = None,
                 norm_layer: Optional[Callable[[int], nn.Module]] = None, drop_layer=None, conv_layer=None) -> None:
        super().__init__()
        if act_layer is None:
            act_layer = nn.ReLU(inplace=True)
        if norm_layer is None:
            norm_layer = nn.BatchNorm2d
        self.encoder = nn.ModuleList([])
        layout_ = [in_channels, *layout]
        pool = False
        for in_chan, out_chan in zip(layout_[:-1], layout_[1:]):
            self.encoder.append(down_path(in_chan, out_chan, pool, 1, act_layer, norm_layer, drop_layer, conv_layer))
            pool = True
        self.decoder = nn.ModuleList([])
        for row in range(len(layout) - 1):
            self.decoder.append(FSAggreg(layout[:row], layout[row],
                                         [len(layout) * layout[0]] * (len(layout) - 2 - row) + layout[-1:],
                                         act_layer, norm_layer, drop_layer, conv_layer))
        self.classifier = nn.Conv2d(len(layout) * layout[0], num_classes, 1)
        init_module(self, "relu")

    def forward(self, x: Tensor) -> Tensor:
        xs: List[Tensor] = []
        for encoder in self.encoder:
            xs.append(encoder(xs[-1] if len(xs) > 0 else x))
        for idx in range(len(self.decoder) - 1, -1, -1):
            xs[idx] = self.decoder[idx](xs[:idx], xs[idx], xs[idx + 1:])
        # per-pixel classifier = 1x1 convolution on the tensor cores (class count padded to 16 internally); fp32 logits
        return conv_bn_act(xs[0], self.classifier, None, None).float()


def unet3p(pretrained: bool = False, progress: bool = True, **kwargs: Any) -> UNet3p:
    """UNet3+ (https://arxiv.org/abs/2004.08790), layout [64, 128, 256, 512, 1024] (reference unet3p.py:171-186)."""
    if pretrained:
        raise NotImplementedError("pretrained checkpoints need network access; load a reference state_dict instead")
    return UNet3p([64, 128, 256, 512, 1024], **kwargs)
