"""UNet+ / UNet++ on the fused kernels — API mirror of holocron/models/segmentation/unetpp.py (UNetp :25-101, UNetpp :104-190,
factories :193-238).

Nested U-Nets (https://arxiv.org/abs/1912.05074): a triangular grid of ``UpPath`` cells; UNet+ feeds each cell the previous
cell of its row, UNet++ every previous cell of its row (dense skip connections). Same module trees / ``state_dict`` as the
reference; all conv units run on the tensor-core convolution + fused normalise / activate pass (see :mod:`.unet`)."""
from typing import Any, Callable, List, Optional

from torch import Tensor, nn

from ...nn.init import init_module
from .._blocks import FusedSequential
from ..utils import conv_sequence
from .unet import UpPath, _classify, _no_pretrained
from .unet3p import down_path

__all__ = ["UNetp", "UNetpp", "unetp", "unetpp"]


def _encoder_and_bridge(layout: List[int], in_channels: int, act_layer, norm_layer, drop_layer, conv_layer):
    encoder = nn.ModuleList([])
    layout_ = [in_channels, *layout]
    pool = False
    for in_chan, out_chan in zip(layout_[:-1], layout_[1:]):
        encoder.append(down_path(in_chan, out_chan, pool, 1, act_layer, norm_layer, drop_layer, conv_layer))
        pool = True
    bridge = FusedSequential(
        nn.MaxPool2d((2, 2)),
        *conv_sequence(layout[-1], 2 * layout[-1], act_layer, norm_layer, drop_layer, conv_layer, kernel_size=3, padding=1),
        *conv_sequence(2 * layout[-1], layout[-1], act_layer, norm_layer, drop_layer, conv_layer, kernel_size=3, padding=1),
    )
    return encoder, bridge


class UNetp(nn.Module):
    """UNet+ (reference unetpp.py:25-101), same constructor."""

    def __init__(self, layout: List[int], in_channels: int = 3, num_classes: int = 10, act_layer: Optional[nn.Module] = None,
                 norm_layer: Optional[Callable[[int], nn.Module]] = None,
                 drop_layer: Optional[Callable[..., nn.Module]] = None,
                 conv_layer: Optional[Callable[..., nn.Module]] = None) -> None:
        super().__init__()
        if act_layer is None:
            act_layer = nn.ReLU(inplace=True)
        self.encoder, self.bridge = _encoder_and_bridge(layout, in_channels, act_layer, norm_layer, drop_layer, conv_layer)
        self.decoder = nn.ModuleList([])
        layout_ = [layout[-1]] + layout[1:][::-1]
        for left_chan, up_chan, num_cells in zip(layout[::-1], layout_, range(1, len(layout) + 1)):
            self.decoder.append(nn.ModuleList([
                UpPath(left_chan + up_chan, left_chan, True, 1, act_layer, norm_layer, drop_layer, conv_layer)
                for _ in range(num_cells)
            ]))
        self.classifier = nn.Conv2d(layout[0], num_classes, 1)
        init_module(self, "relu")

    def forward(self, x: Tensor) -> Tensor:
        xs: List[Tensor] = []
        for encoder in self.encoder:
            xs.append(encoder(xs[-1] if len(xs) > 0 else x))
        xs.append(self.bridge(xs[-1]))
        # column j of the grid: every row that still has a deeper neighbour takes one more cell
        for j in range(len(self.decoder)):
            for i in range(len(xs) - 1):
                up_feat = xs[i + 1] if (i + 2) < len(xs) else xs.pop()
                xs[i] = self.decoder[-1 - i][j](xs[i], up_feat)  # type: ignore[index]
        return _classify(xs.pop(), self.classifier)


class UNetpp(nn.Module):
    """UNet++ (reference unetpp.py:104-190), same constructor."""

    def __init__(self, layout: List[int], in_channels: int = 3, num_classes: int = 10, act_layer: Optional[nn.Module] = None,
                 norm_layer: Optional[Callable[[int], nn.Module]] = None,
                 drop_layer: Optional[Callable[..., nn.Module]] = None,
                 conv_layer: Optional[Callable[..., nn.Module]] = None) -> None:
        super().__init__()
        if act_layer is None:
            act_layer = nn.ReLU(inplace=True)
        self.encoder, self.bridge = _encoder_and_bridge(layout, in_channels, act_layer, norm_layer, drop_layer, conv_layer)
        self.decoder = nn.ModuleList([])
        layout_ = [layout[-1]] + layout[1:][::-1]
        for left_chan, up_chan, num_cells in zip(layout[::-1], layout_, range(1, len(layout) + 1)):
            self.decoder.append(nn.ModuleList([
                UpPath(up_chan + (idx + 1) * left_chan, left_chan, True, 1, act_layer, norm_layer, drop_layer, conv_layer)
                for idx in range(num_cells)
            ]))
        self.classifier = nn.Conv2d(layout[0], num_classes, 1)
        init_module(self, "relu")

    def forward(self, x: Tensor) -> Tensor:
        xs: List[List[Tensor]] = []
        for encoder in self.encoder:
            xs.append([encoder(xs[-1][0] if len(xs) > 0 else x)])
        xs.append([self.bridge(xs[-1][-1])])
        # dense skips: cell (i, j) sees every earlier cell of row i plus the up-sampled cell (i + 1, j)
        for j in range(len(self.decoder)):
            for i in range(len(xs) - 1):
                up_feat = xs[i + 1][j] if (i + 2) < len(xs) else xs.pop()[-1]
                xs[i].append(self.decoder[-1 - i][j](list(xs[i]), up_feat))  # type: ignore[index]
        return _classify(xs.pop()[-1], self.classifier)


def unetp(pretrained: bool = False, progress: bool = True, **kwargs: Any) -> UNetp:
    """UNet+, layout [64, 128, 256, 512] (reference unetpp.py:205-220)."""
    _no_pretrained(pretrained)
    return UNetp([64, 128, 256, 512], **kwargs)


def unetpp(pretrained: bool = False, progress: bool = True, **kwargs: Any) -> UNetpp:
    """UNet++, layout [64, 128, 256, 512] (reference unetpp.py:223-238)."""
    _no_pretrained(pretrained)
    return UNetpp([64, 128, 256, 512], **kwargs)
