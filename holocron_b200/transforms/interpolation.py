"""``Resize`` and ``RandomZoomOut`` of holocron.transforms (reference holocron/transforms/interpolation.py) on one CUDA
launch per call (holocron_b200/csrc/resample.cu).

Both take a ``(C, H, W)`` CUDA tensor, as the reference does, or a list / tuple of ``(C, H_i, W_i)`` CUDA tensors of
different sizes, which they resize and place on their canvases together and return stacked as ``(N, C, h, w)``.
Squish-mode ``Resize`` also takes ``(..., H, W)`` tensors. Sources are read in place whatever their strides.

The output is what the reference computes on a CUDA tensor (torchvision's ``resize`` then ``pad``): uint8, fp16 and
bf16 interpolate in fp32 and are cast back (uint8 clamped and rounded half to even), fp64 stays fp64. Deviations: PIL
images and CPU tensors raise ``HolocronB200Error``, like every CUDA-only op of this package; dtypes other than uint8,
fp16, bf16, fp32 and fp64 raise ``TypeError``; an antialiased downscale needing more than 255 filter taps per axis
(about 1/127 bilinear, 1/63 bicubic) raises ``NotImplementedError``.
"""
from enum import Enum
from math import sqrt
from typing import Any, List, Tuple, Union

import torch
from PIL import Image
from torch import Tensor, nn
from torchvision.transforms import transforms as T
from torchvision.transforms.functional import InterpolationMode, _interpolation_modes_from_int

from .._lib import HolocronB200Error, require_cuda
from ._resample import resample

__all__ = ["RandomZoomOut", "Resize", "ResizeMethod"]

Images = Union[Tensor, List[Tensor], Tuple[Tensor, ...]]


class ResizeMethod(str, Enum):
    """How ``Resize`` fits an image to its target size: ``squish`` stretches it, ``pad`` keeps its aspect ratio and pads
    the rest."""

    SQUISH = "squish"
    PAD = "pad"


def _check_size(size) -> None:
    if not isinstance(size, (tuple, list)) or len(size) != 2 or any(s <= 0 for s in size):
        raise ValueError("size is expected to be a sequence of 2 positive integers")


def _image_hw(image) -> Tuple[int, int]:
    """(H, W) of a (C, H, W) tensor or a PIL image, with the reference's exceptions for anything else."""
    if isinstance(image, Tensor):
        if image.ndim != 3:
            raise ValueError("the input tensor is expected to be 3-dimensional")
        return int(image.shape[1]), int(image.shape[2])
    if isinstance(image, Image.Image):
        return image.size[1], image.size[0]
    raise TypeError("expected arg 'image' to be a PIL image or a torch.Tensor")


def _batch(images: Images, three_d: bool = True) -> List[Tensor]:
    """The CUDA tensors of one call. A list holds (C, H_i, W_i) images; a single tensor is (C, H, W), or any (..., H, W)
    when ``three_d`` is False."""
    items = list(images) if isinstance(images, (list, tuple)) else [images]
    if not items:
        raise ValueError("expected at least one image")
    for x in items:
        if isinstance(x, Image.Image):
            raise HolocronB200Error("holocron_b200 transforms run on CUDA tensors only: convert PIL images first "
                                    "(use the reference implementation for PIL images and CPU tensors)")
        if not isinstance(x, Tensor):
            raise TypeError("expected arg 'image' to be a PIL image or a torch.Tensor")
        require_cuda(x)
        if x.ndim != 3 and (three_d or isinstance(images, (list, tuple))):
            raise ValueError("the input tensor is expected to be 3-dimensional")
        if x.ndim < 2:
            raise TypeError("Tensor is not a torch image.")
    return items


def _planes(items: List[Tensor]) -> List[Tensor]:
    """The images of a call as [..., C, H, W] sources: a (H, W) tensor is one channel."""
    return [x if x.ndim >= 3 else x.unsqueeze(0) for x in items]


def _finish(images: Images, out: Tensor, size: Tuple[int, int]) -> Tensor:
    """The stacked canvases of a list, or the one canvas of a tensor in that tensor's leading shape."""
    if isinstance(images, (list, tuple)):
        return out
    return out.view(*images.shape[:-2], *size)


def _place(images: Images, items: List[Tensor], inner: List[Tuple[int, int]], size, interpolation, antialias,
           pad_mode: str) -> Tensor:
    out = resample(_planes(items), inner, (size[0], size[1]), interpolation, antialias, pad_mode)
    return _finish(images, out, (size[0], size[1]))


def _resize_options(interpolation=InterpolationMode.BILINEAR, max_size=None, antialias=True):
    """(interpolation, antialias) from the keyword arguments of torchvision's ``resize`` for a target size given as
    (h, w). ``antialias=None`` means off for tensors."""
    if isinstance(interpolation, int):
        interpolation = _interpolation_modes_from_int(interpolation)
    if max_size is not None:
        raise ValueError("max_size should only be passed if size specifies the length of the smaller edge, "
                         "i.e. size should be an int or a sequence of length 1 in torchscript mode.")
    return interpolation, bool(antialias)


class Resize(T.Resize):
    """Resizes images to ``size``, either stretching them (``mode=ResizeMethod.SQUISH``) or keeping their aspect ratio
    and padding the rest (``mode=ResizeMethod.PAD``, ``pad_mode`` one of constant (0), edge, reflect or symmetric).

    >>> import torch
    >>> from holocron_b200.transforms import Resize
    >>> from holocron_b200.transforms.interpolation import ResizeMethod
    >>> tf = Resize((224, 224), mode=ResizeMethod.PAD)
    >>> out = tf(torch.randint(0, 256, (3, 300, 500), dtype=torch.uint8, device="cuda"))

    Args:
        size: the target (height, width)
        mode: the resizing scheme
        pad_mode: how the canvas around the image is filled in pad mode
        kwargs: the keyword arguments of ``torchvision.transforms.Resize``; pad mode uses only ``interpolation`` (its
            resize keeps antialias on and takes no ``max_size``, as the reference's does)
    """

    def __init__(self, size: Tuple[int, int], mode: ResizeMethod = ResizeMethod.SQUISH, pad_mode: str = "constant",
                 **kwargs: Any) -> None:
        if not isinstance(mode, ResizeMethod):
            raise ValueError("mode is expected to be a ResizeMethod")
        _check_size(size)
        super().__init__(size, **kwargs)
        self.mode = mode
        self.pad_mode = pad_mode

    def get_params(self, image) -> Tuple[int, int]:
        """The (h, w) the image is resized to in pad mode: the largest size of its aspect ratio within ``size``, the
        rounded side computed on the host with Python's ``round``."""
        h, w = _image_hw(image)
        aspect = h / w
        th, tw = self.size
        if th / tw > aspect:
            return round(tw * aspect), tw
        return th, round(th / aspect)

    def forward(self, image: Images) -> Tensor:
        if self.mode == ResizeMethod.SQUISH:
            items = _batch(image, three_d=False)
            interpolation, antialias = _resize_options(self.interpolation, self.max_size, self.antialias)
            # torchvision hands back the input itself when it already has the target size
            if isinstance(image, Tensor) and tuple(image.shape[-2:]) == tuple(self.size):
                return image
            return _place(image, items, [tuple(self.size)] * len(items), self.size, interpolation, antialias,
                          "constant")
        items = _batch(image)
        inner = [self.get_params(x) for x in items]
        # the reference resizes with the interpolation alone: antialias stays at its default (on), max_size unused
        interpolation, _ = _resize_options(self.interpolation)
        return _place(image, items, inner, self.size, interpolation, True, self.pad_mode)


class RandomZoomOut(nn.Module):
    """Shrinks each image to a random share ``scale`` of the largest area its aspect ratio allows within ``size`` and
    centres it on a zero canvas of ``size``.

    >>> import torch
    >>> from holocron_b200.transforms import RandomZoomOut
    >>> tf = RandomZoomOut((224, 224), scale=(0.3, 1.0))
    >>> out = tf([torch.rand(3, 300, 400, device="cuda"), torch.rand(3, 500, 350, device="cuda")])

    Args:
        size: the canvas (height, width)
        scale: the range the area share is drawn from
        kwargs: the keyword arguments of ``torchvision.transforms.functional.resize``
    """

    def __init__(self, size: Tuple[int, int], scale: Tuple[float, float] = (0.5, 1.0), **kwargs: Any) -> None:
        _check_size(size)
        if len(scale) != 2 or scale[0] > scale[1]:
            raise ValueError("scale is expected to be a couple of floats, the first one being small than the second")
        super().__init__()
        self.size = size
        self.scale = scale
        self._kwargs = kwargs

    def get_params(self, image) -> Tuple[int, int]:
        """The (h, w) of the shrunk image. Draws one ``torch.rand(1)`` from the default CPU generator; the rounding
        (Python's ``round``) can give a side one pixel longer than ``size``, which the placement then crops."""
        h, w = _image_hw(image)
        share = (self.scale[1] - self.scale[0]) * torch.rand(1).item() + self.scale[0]
        aspect = h / w
        th, tw = self.size
        full = tw ** 2 * aspect if th / tw > aspect else th ** 2 / aspect
        area = full * share
        w_new = round(sqrt(area / aspect))
        return round(area / w_new), w_new

    def forward(self, image: Images) -> Images:
        if self.scale[0] == 1:
            return image
        items = _batch(image)
        interpolation, antialias = _resize_options(**self._kwargs)
        # one draw per image, in list order: a list call draws what calling the module image by image draws
        inner = [self.get_params(x) for x in items]
        return _place(image, items, inner, self.size, interpolation, antialias, "constant")
