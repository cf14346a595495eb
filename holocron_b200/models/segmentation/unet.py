"""U-Net family on the fused kernels — API mirror of holocron/models/segmentation/unet.py (down_path :36-55, UpPath :58-101,
UNetBackbone :104-137, UNet :140-226, UBlock :229-279, DynamicUNet :282-370, factories :373-513).

Same module trees / ``state_dict`` as the reference. Every ``conv3x3 -> [norm] -> act`` unit of the contracting, bridge and
expansive paths runs on the wgmma implicit-GEMM kernel + the fused normalise / activate pass; max-pooling, bilinear / nearest
up-sampling, ``PixelShuffle``, transposed convolutions, cropping and channel concatenation are resampling / data-movement ops
left to the library (they act on the same bf16 channels_last tensors). ``DynamicUNet`` needs the channel counts of its encoder's
feature maps at construction time; the reference finds them by running the encoder on a CPU tensor - here the encoder is walked
over FAKE tensors (shape propagation through the export lowerings of :mod:`holocron_b200.onnx._lowering`, nothing is computed),
because the fused encoders have no CPU execution path."""
from collections import OrderedDict
from typing import Any, Callable, Dict, List, Optional, Tuple, Union

import torch
import torch.nn.functional as F
from torch import Tensor, nn
from torchvision.models._utils import IntermediateLayerGetter

from ...nn import GlobalAvgPool2d
from ...nn import _fused as K
from ...nn.init import init_module
from .._blocks import FusedSequential, conv_bn_act, run_fused
from ..utils import conv_sequence
from .unet3p import down_path

__all__ = ["DynamicUNet", "UBlock", "UNet", "UNetBackbone", "UpPath", "unet", "unet2", "unet_rexnet13", "unet_tvresnet34",
           "unet_tvvgg11"]


default_cfgs: Dict[str, Dict[str, Any]] = {
    "unet": {"encoder_layout": [64, 128, 256, 512], "url": None},
    "unet2": {"encoder_layout": [64, 128, 256, 512], "backbone_layers": ["0", "1", "2", "3"], "url": None},
    "unet_vgg11": {"backbone_layers": ["1", "4", "9", "14", "19"], "url": None},
    "unet_tvresnet34": {"backbone_layers": ["relu", "layer1", "layer2", "layer3", "layer4"], "url": None},
    "unet_rexnet13": {"backbone_layers": ["3", "5", "7", "13", "18"], "url": None},
}


def _in_dtype_of(module: nn.Module, x: Tensor) -> Tensor:
    """Library modules with fp32 master parameters (transposed convolution, a user-supplied norm layer) meet bf16 activations:
    run them in the parameters' dtype and hand the result back in the activation dtype."""
    p = next(module.parameters(), None)
    if p is None or p.dtype == x.dtype:
        return module(x)
    return module(x.to(p.dtype)).to(x.dtype)


def _classify(x: Tensor, classifier: nn.Conv2d) -> Tensor:
    # per-pixel classifier = 1x1 convolution on the tensor cores (class count padded to 16 internally); fp32 logits
    return conv_bn_act(x, classifier, None, None).float()


class UpPath(nn.Module):
    """Up-sample the expansive feature map (bilinear x2 or transposed convolution), centre-crop the contracting maps to it,
    concatenate, two conv units (reference unet.py:58-101)."""

    def __init__(self, in_chan: int, out_chan: int, bilinear_upsampling: bool = True, padding: int = 0,
                 act_layer: Optional[nn.Module] = None, norm_layer: Optional[Callable[[int], nn.Module]] = None,
                 drop_layer: Optional[Callable[..., nn.Module]] = None,
                 conv_layer: Optional[Callable[..., nn.Module]] = None) -> None:
        super().__init__()
        self.upsample: nn.Module
        if bilinear_upsampling:
            self.upsample = nn.Upsample(scale_factor=2, mode="bilinear", align_corners=True)
        else:
            self.upsample = nn.ConvTranspose2d(in_chan, out_chan, 2, stride=2)
        self.block = FusedSequential(
            *conv_sequence(in_chan, out_chan, act_layer, norm_layer, drop_layer, conv_layer, kernel_size=3, padding=padding),
            *conv_sequence(out_chan, out_chan, act_layer, norm_layer, drop_layer, conv_layer, kernel_size=3, padding=padding),
        )

    def forward(self, downfeats: Union[Tensor, List[Tensor]], upfeat: Tensor) -> Tensor:
        if not isinstance(downfeats, list):
            downfeats = [downfeats]
        upfeat_ = _in_dtype_of(self.upsample, upfeat)
        for idx, downfeat in enumerate(downfeats):      # valid-padding variants: centre crop of the contracting features
            if downfeat.shape != upfeat_.shape:
                delta_w = downfeat.shape[-1] - upfeat_.shape[-1]
                w_slice = slice(delta_w // 2, -(delta_w // 2) if delta_w > 0 else downfeat.shape[-1])
                delta_h = downfeat.shape[-2] - upfeat_.shape[-2]
                h_slice = slice(delta_h // 2, -(delta_h // 2) if delta_h > 0 else downfeat.shape[-2])
                downfeats[idx] = downfeat[..., h_slice, w_slice]
        dtype = upfeat_.dtype
        return self.block(torch.cat((*[d.to(dtype) for d in downfeats], upfeat_), dim=1))


class UNetBackbone(nn.Sequential):
    """The contracting path as a classifier (reference unet.py:104-137); its ``features`` are the encoder of ``unet2``."""

    def __init__(self, layout: List[int], in_channels: int = 3, num_classes: int = 10, act_layer: Optional[nn.Module] = None,
                 norm_layer: Optional[Callable[[int], nn.Module]] = None,
                 drop_layer: Optional[Callable[..., nn.Module]] = None,
                 conv_layer: Optional[Callable[..., nn.Module]] = None, same_padding: bool = True) -> None:
        if act_layer is None:
            act_layer = nn.ReLU(inplace=True)
        layers: List[nn.Module] = []
        layout_ = [in_channels, *layout]
        pool = False
        for in_chan, out_chan in zip(layout_[:-1], layout_[1:]):
            layers.append(down_path(in_chan, out_chan, pool, int(same_padding), act_layer, norm_layer, drop_layer, conv_layer))
            pool = True
        super().__init__(OrderedDict([
            ("features", FusedSequential(*layers)),
            ("pool", GlobalAvgPool2d(flatten=True)),
            ("head", nn.Linear(layout[-1], num_classes)),
        ]))
        init_module(self, "relu")

    def forward(self, x: Tensor) -> Tensor:  # type: ignore[override]
        return K.head_linear(self.pool(self.features(x)), self.head.weight, self.head.bias)


class UNet(nn.Module):
    """U-Net (https://arxiv.org/abs/1505.04597) — reference unet.py:140-226, same constructor."""

    def __init__(self, layout: List[int], in_channels: int = 3, num_classes: int = 10, act_layer: Optional[nn.Module] = None,
                 norm_layer: Optional[Callable[[int], nn.Module]] = None,
                 drop_layer: Optional[Callable[..., nn.Module]] = None,
                 conv_layer: Optional[Callable[..., nn.Module]] = None, same_padding: bool = True,
                 bilinear_upsampling: bool = True) -> None:
        super().__init__()
        if act_layer is None:
            act_layer = nn.ReLU(inplace=True)
        self.encoder = nn.ModuleList([])
        layout_ = [in_channels, *layout]
        pool = False
        for in_chan, out_chan in zip(layout_[:-1], layout_[1:]):
            self.encoder.append(down_path(in_chan, out_chan, pool, int(same_padding), act_layer, norm_layer, drop_layer,
                                          conv_layer))
            pool = True
        self.bridge = FusedSequential(
            nn.MaxPool2d((2, 2)),
            *conv_sequence(layout[-1], 2 * layout[-1], act_layer, norm_layer, drop_layer, conv_layer, kernel_size=3, padding=1),
            *conv_sequence(2 * layout[-1], layout[-1], act_layer, norm_layer, drop_layer, conv_layer, kernel_size=3, padding=1),
        )
        self.decoder = nn.ModuleList([])
        layout_ = [chan // 2 if bilinear_upsampling else chan for chan in layout[::-1][:-1]] + [layout[0]]
        for in_chan, out_chan in zip([2 * layout[-1]] + layout[::-1][:-1], layout_):
            self.decoder.append(UpPath(in_chan, out_chan, bilinear_upsampling, int(same_padding), act_layer, norm_layer,
                                       drop_layer, conv_layer))
        self.classifier = nn.Conv2d(layout[0], num_classes, 1)
        init_module(self, "relu")

    def forward(self, x: Tensor) -> Tensor:
        xs: List[Tensor] = []
        for encoder in self.encoder:
            xs.append(encoder(xs[-1] if len(xs) > 0 else x))
        x = self.bridge(xs[-1])
        for decoder in self.decoder:
            x = decoder(xs.pop(), x)
        return _classify(x, self.classifier)


class UBlock(nn.Module):
    """fastai-style decoder block (reference unet.py:229-279): 1x1 unit to 4x the channels + PixelShuffle up-sampling,
    BatchNorm of the skip features, activation, two conv units."""

    def __init__(self, left_chan: int, up_chan: int, out_chan: int, padding: int = 0, act_layer: Optional[nn.Module] = None,
                 norm_layer: Optional[Callable[[int], nn.Module]] = None,
                 drop_layer: Optional[Callable[..., nn.Module]] = None,
                 conv_layer: Optional[Callable[..., nn.Module]] = None) -> None:
        super().__init__()
        if act_layer is None:
            act_layer = nn.ReLU(inplace=True)
        self.upsample = FusedSequential(
            *conv_sequence(up_chan, up_chan * 2**2, act_layer, norm_layer, drop_layer, conv_layer, kernel_size=1),
            nn.PixelShuffle(upscale_factor=2),
        )
        self.bn = nn.BatchNorm2d(left_chan) if norm_layer is None else norm_layer(left_chan)
        self.block = FusedSequential(
            act_layer,
            *conv_sequence(left_chan + up_chan, out_chan, act_layer, norm_layer, drop_layer, conv_layer, kernel_size=3,
                           padding=padding),
            *conv_sequence(out_chan, out_chan, act_layer, norm_layer, drop_layer, conv_layer, kernel_size=3, padding=padding),
        )

    def forward(self, downfeat: Tensor, upfeat: Tensor) -> Tensor:
        upfeat_ = self.upsample(upfeat)
        if downfeat.shape[-2:] != upfeat_.shape[-2:]:
            upfeat_ = F.interpolate(upfeat_, downfeat.shape[-2:], mode="nearest")
        # skip features: BatchNorm alone (the activation follows the concatenation) - fused pass for nn.BatchNorm2d and
        # nn.SyncBatchNorm
        left = run_fused([self.bn], downfeat) if K.is_batch_norm(self.bn) else _in_dtype_of(self.bn, downfeat)
        if left.dtype != upfeat_.dtype and left.dtype == torch.float32:
            upfeat_ = upfeat_.float()          # fp32 skip features of a library encoder: keep their precision through the cat
        return self.block(torch.cat((left.to(upfeat_.dtype), upfeat_), dim=1))



def _feature_shapes(encoder: nn.Module, input_shape: Tuple[int, ...]) -> List[torch.Size]:
    """Shapes (C, H, W) of the encoder's feature maps for one input, by shape propagation over fake tensors."""
    from torch._subclasses.fake_tensor import FakeTensorMode

    from ...onnx._lowering import lowered
    training_mode = encoder.training
    encoder.eval()
    try:
        with lowered(), torch.no_grad(), FakeTensorMode(allow_non_fake_inputs=True):
            shapes = [v.shape[1:] for v in encoder(torch.zeros(1, *input_shape)).values()]
    finally:
        if training_mode:
            encoder.train()
    return shapes


class DynamicUNet(nn.Module):
    """U-Net decoder grown on any encoder (reference unet.py:282-370), same constructor."""

    def __init__(self, encoder: IntermediateLayerGetter, num_classes: int = 10, act_layer: Optional[nn.Module] = None,
                 norm_layer: Optional[Callable[[int], nn.Module]] = None,
                 drop_layer: Optional[Callable[..., nn.Module]] = None,
                 conv_layer: Optional[Callable[..., nn.Module]] = None, same_padding: bool = True,
                 input_shape: Optional[Tuple[int, int, int]] = None, final_upsampling: bool = False) -> None:
        super().__init__()
        if act_layer is None:
            act_layer = nn.ReLU(inplace=True)
        self.encoder = encoder
        input_shape = (3, 256, 256) if input_shape is None else input_shape
        chans = [s[0] for s in _feature_shapes(self.encoder, input_shape)]
        self.bridge = FusedSequential(
            nn.BatchNorm2d(chans[-1]) if norm_layer is None else norm_layer(chans[-1]),
            act_layer,
            *conv_sequence(chans[-1], 2 * chans[-1], act_layer, norm_layer, drop_layer, conv_layer, kernel_size=3, padding=1),
            *conv_sequence(2 * chans[-1], chans[-1], act_layer, norm_layer, drop_layer, conv_layer, kernel_size=3, padding=1),
        )
        self.decoder = nn.ModuleList([])
        layout = chans[::-1][1:] + [chans[0]]
        for up_chan, out_chan in zip(chans[::-1], layout):
            self.decoder.append(UBlock(up_chan, up_chan, out_chan, int(same_padding), act_layer, norm_layer, drop_layer,
                                       conv_layer))
        self.upsample: Optional[nn.Sequential] = None
        if final_upsampling:
            self.upsample = FusedSequential(
                *conv_sequence(chans[0], chans[0] * 2**2, act_layer, norm_layer, drop_layer, conv_layer, kernel_size=1),
                nn.PixelShuffle(upscale_factor=2),
            )
        self.classifier = nn.Conv2d(chans[0], num_classes, 1)
        init_module(self, "relu")

    def forward(self, x: Tensor) -> Tensor:
        xs: List[Tensor] = list(self.encoder(x).values())
        x = self.bridge(xs[-1])
        for decoder in self.decoder:
            x = decoder(xs.pop(), x)
        if self.upsample is not None:
            x = self.upsample(x)
        return _classify(x, self.classifier)


def _no_pretrained(pretrained: bool) -> None:
    if pretrained:
        raise NotImplementedError("pretrained checkpoints need network access; load a reference state_dict instead")


def unet(pretrained: bool = False, progress: bool = True, **kwargs: Any) -> UNet:
    """U-Net, layout [64, 128, 256, 512] (reference unet.py:383-398)."""
    _no_pretrained(pretrained)
    return UNet(default_cfgs["unet"]["encoder_layout"], **kwargs)


def _dynamic_unet(arch: str, backbone: nn.Module, pretrained: bool, num_classes: int = 21, **kwargs: Any) -> DynamicUNet:
    _no_pretrained(pretrained)
    encoder = IntermediateLayerGetter(backbone, {name: str(idx) for idx, name in enumerate(default_cfgs[arch]["backbone_layers"])})
    return DynamicUNet(encoder, num_classes=num_classes, **kwargs)


def unet2(pretrained: bool = False, progress: bool = True, in_channels: int = 3, **kwargs: Any) -> DynamicUNet:
    """U-Net with the fastai-style decoder on its own contracting path (reference unet.py:417-437)."""
    backbone = UNetBackbone(default_cfgs["unet2"]["encoder_layout"], in_channels=in_channels).features
    return _dynamic_unet("unet2", backbone, pretrained, **kwargs)


def unet_tvvgg11(pretrained: bool = False, pretrained_backbone: bool = False, progress: bool = True, **kwargs: Any) -> DynamicUNet:
    """DynamicUNet on torchvision's VGG-11 features (reference unet.py:440-459). The encoder consists of stock torch modules
    (library kernels); ``pretrained_backbone`` defaults to False here (the reference's True triggers a download)."""
    from torchvision.models import vgg11
    if pretrained_backbone:
        raise NotImplementedError("pretrained backbones need network access")
    return _dynamic_unet("unet_vgg11", vgg11(weights=None).features, pretrained, **kwargs)


def unet_tvresnet34(pretrained: bool = False, pretrained_backbone: bool = False, progress: bool = True,
                    **kwargs: Any) -> DynamicUNet:
    """DynamicUNet on torchvision's ResNet-34 (reference unet.py:462-482), with the final up-sampling stage."""
    from torchvision.models import resnet34
    if pretrained_backbone:
        raise NotImplementedError("pretrained backbones need network access")
    kwargs["final_upsampling"] = kwargs.get("final_upsampling", True)
    return _dynamic_unet("unet_tvresnet34", resnet34(weights=None), pretrained, **kwargs)


def unet_rexnet13(pretrained: bool = False, pretrained_backbone: bool = False, progress: bool = True, in_channels: int = 3,
                  **kwargs: Any) -> DynamicUNet:
    """DynamicUNet on this package's ReXNet-1.3x features (reference unet.py:485-513), with the final up-sampling stage."""
    from ..classification.rexnet import rexnet1_3x
    if pretrained_backbone:
        raise NotImplementedError("pretrained backbones need network access")
    backbone = rexnet1_3x(pretrained=False, in_channels=in_channels).features
    kwargs["final_upsampling"] = kwargs.get("final_upsampling", True)
    # the decoder's activation defaults to the encoder's (SiLU), like the reference
    kwargs["act_layer"] = kwargs.get("act_layer", nn.SiLU(inplace=True))
    backbone[21] = nn.SiLU(inplace=True)     # its own module instance at the last tap (reference: torchvision issue 3802)
    return _dynamic_unet("unet_rexnet13", backbone, pretrained, **kwargs)
