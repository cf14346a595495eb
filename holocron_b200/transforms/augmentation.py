"""``RandomResizedCrop``, ``RandomHorizontalFlip``, ``TrivialAugmentWide`` and ``RandomErasing`` of torchvision, the
random transforms of the reference's classification training recipe (references/classification/train.py:101-107), and
``ColorJitter``, the photometric augmentation of its segmentation and detection recipes
(references/segmentation/train.py:133-140, references/detection/train.py:116-125), on one CUDA launch per call (two for
a ``TrivialAugmentWide`` batch where an image drew a histogram op, and for a ``ColorJitter`` batch where an image has a
contrast factor).

Each subclasses the torchvision class of the same name: constructor, validation, attributes and ``repr`` are
torchvision's, and the random draws are torchvision's own ``get_params`` (and ``torch.rand(1) < p``), called in
torchvision's order on the default CPU generator. Only ``forward`` differs, in what it takes:

- one tensor: what the torchvision class does to that tensor (one draw, leading dimensions carried along);
- a list or tuple of ``(C, H_i, W_i)`` CUDA tensors: one draw set per image, in list order, so a seeded list call draws
  exactly what calling the torchvision module image by image draws, and one launch for the whole list, which returns
  the stacked ``(N, C, h, w)`` result. ``RandomResizedCrop`` returns canvases of ``size``; the other transforms take
  images of one shape and raise ``ValueError`` otherwise, before any draw. Sources are read in place whatever their
  strides: pass a stacked batch as ``batch.unbind(0)``;
- ``RandomErasing(inplace=True)`` writes only the rectangles, into the given tensors, and returns the input as given.

A chain of batched calls does not draw what a per-image ``T.Compose`` of the same transforms draws: the chain makes
every image's crop draws, then every image's flip draw, and so on, where ``Compose`` goes image by image. Each single
call is draw-for-draw with its torchvision class.

Outputs are torchvision's on CUDA tensors: crops are resampled by the kernel of ``Resize`` (torchvision's filters with
torch's CUDA arithmetic), flips are exact copies, and erased pixels hold the fp32 values cast to the image dtype as
torch's copy casts them; ``TrivialAugmentWide`` and ``ColorJitter`` follow torchvision's fp32 arithmetic operation by
operation (their docstrings state where they may differ). Deviations: PIL images and CPU tensors raise
``HolocronB200Error``; dtypes other than uint8, fp16, bf16, fp32 and fp64 raise ``TypeError`` (other than uint8 for
``TrivialAugmentWide``, other than uint8 and fp32 for ``ColorJitter``); a crop needing more than 255 filter taps per
axis (antialiased downscales beyond about 1/127 bilinear, 1/63 bicubic) raises ``NotImplementedError``.
"""
from typing import Dict, List, Optional, Tuple

import torch
from torch import Tensor
from torchvision.transforms import autoaugment, transforms as T
from torchvision.transforms.functional import InterpolationMode

from . import _autoaugment, _color
from ._autoaugment import apply_ops, check_options
from ._color import jitter
from ._erase import Rect, erase
from ._resample import resample
from ._table import check_images
from .interpolation import Images, _batch, _finish, _planes, _resize_options

__all__ = ["ColorJitter", "RandomErasing", "RandomHorizontalFlip", "RandomResizedCrop", "TrivialAugmentWide"]


def _one_shape(images: Images, items: List[Tensor]) -> None:
    if isinstance(images, (list, tuple)) and any(x.shape != items[0].shape for x in items):
        raise ValueError(f"{type(images).__name__} of images of different shapes: this transform stacks images of one "
                         "shape (RandomResizedCrop resizes them to one)")


def _hw(items: List[Tensor]) -> Tuple[int, int]:
    return int(items[0].shape[-2]), int(items[0].shape[-1])


def erase_draw(t: T.RandomErasing, x: Tensor) -> Tuple[bool, Optional[Rect]]:
    """torchvision's ``RandomErasing.forward`` of ``t`` up to ``F.erase`` for one image (only x's shape is read):
    whether it erases, and the rectangle and values, None when get_params found no rectangle in its 10 attempts
    (torchvision then assigns the image to itself)."""
    if not torch.rand(1) < t.p:
        return False, None
    if isinstance(t.value, (int, float)):
        value = [float(t.value)]
    elif isinstance(t.value, str):
        value = None
    elif isinstance(t.value, (list, tuple)):
        value = [float(v) for v in t.value]
    else:
        value = t.value
    if value is not None and len(value) not in (1, x.shape[-3]):
        raise ValueError("If value is a sequence, it should have either a single value or "
                         f"{x.shape[-3]} (number of input channels)")
    i, j, h, w, v = t.get_params(x, scale=t.scale, ratio=t.ratio, value=value)
    return True, (None if v is x else (i, j, h, w, v))


def trivial_draw(op_meta: Dict[str, Tuple[Tensor, bool]]) -> Tuple[str, float]:
    """torchvision's ``TrivialAugmentWide.forward`` draws for one image, given its ``_augmentation_space``: the op,
    then its magnitude bin when it has several, then its sign when it is signed."""
    names = list(op_meta.keys())
    op_name = names[int(torch.randint(len(op_meta), (1,)).item())]
    magnitudes, signed = op_meta[op_name]
    magnitude = (float(magnitudes[torch.randint(len(magnitudes), (1,), dtype=torch.long)].item())
                 if magnitudes.ndim > 0 else 0.0)
    if signed and torch.randint(2, (1,)):
        magnitude *= -1.0
    return op_name, magnitude


class RandomResizedCrop(T.RandomResizedCrop):
    """torchvision's ``RandomResizedCrop`` on a batched CUDA resampling kernel: a random box of each image, resized to
    ``size``.

    >>> import torch
    >>> from holocron_b200.transforms import RandomResizedCrop
    >>> tf = RandomResizedCrop(176, scale=(0.3, 1.0))
    >>> out = tf([torch.randint(0, 256, (3, 300, 400), dtype=torch.uint8, device="cuda"),
    ...           torch.randint(0, 256, (3, 500, 350), dtype=torch.uint8, device="cuda")])
    """

    def forward(self, img: Images) -> Tensor:
        items = _batch(img, three_d=False)
        boxes = [self.get_params(x, self.scale, self.ratio) for x in items]
        size = (int(self.size[0]), int(self.size[1]))
        interpolation, antialias = _resize_options(self.interpolation, None, self.antialias)
        if isinstance(img, Tensor):
            if tuple(boxes[0][2:]) == size:
                # torchvision's resize hands back the crop itself when it already has the target size
                i, j, h, w = boxes[0]
                return img[..., i:i + h, j:j + w]
            if img.ndim == 2:  # torchvision's resize refuses what torch's interpolate refuses
                raise ValueError("Input and output must have the same number of spatial dimensions, but got input "
                                 f"with spatial dimensions of {[img.shape[-1]]} and output size of {list(size)}.")
        out = resample(_planes(items), [size] * len(items), size, interpolation, antialias, boxes=boxes)
        return _finish(img, out, size)


class RandomHorizontalFlip(T.RandomHorizontalFlip):
    """torchvision's ``RandomHorizontalFlip`` on a batched CUDA kernel: each image is mirrored left-right with
    probability ``p``.

    >>> import torch
    >>> from holocron_b200.transforms import RandomHorizontalFlip
    >>> batch = torch.rand(8, 3, 176, 176, device="cuda")
    >>> out = RandomHorizontalFlip()(batch.unbind(0))
    """

    def forward(self, img: Images) -> Images:
        items = _batch(img, three_d=False)
        _one_shape(img, items)
        flips = [bool(torch.rand(1) < self.p) for _ in items]
        if isinstance(img, Tensor) and not flips[0]:
            return img
        size = _hw(items)
        # a nearest resample at the image's own size is an exact copy; a flip reads the columns backwards
        out = resample(_planes(items), [size] * len(items), size, InterpolationMode.NEAREST, False, flips=flips)
        return _finish(img, out, size)


class RandomErasing(T.RandomErasing):
    """torchvision's ``RandomErasing`` on a batched CUDA kernel: with probability ``p``, a random rectangle of each
    image is filled with ``value`` (one number, one per channel, or ``"random"``: per-pixel standard normal draws, made
    on the host by torchvision's ``get_params``).

    >>> import torch
    >>> from holocron_b200.transforms import RandomErasing
    >>> batch = torch.rand(8, 3, 176, 176, device="cuda")
    >>> out = RandomErasing(p=1.0, scale=(0.02, 0.2), value="random")(batch.unbind(0))
    """

    def forward(self, img: Images) -> Images:
        items = _batch(img, three_d=False)
        _one_shape(img, items)
        draws = [erase_draw(self, x) for x in items]
        if isinstance(img, Tensor):
            chosen, rect = draws[0]
            # torchvision hands back the input unless it erases a copy
            if not chosen or (rect is None and self.inplace):
                return img
        out = erase(_planes(items), [rect for _, rect in draws], self.inplace)
        if self.inplace:
            return img
        return _finish(img, out, _hw(items))


class TrivialAugmentWide(autoaugment.TrivialAugmentWide):
    """torchvision's ``TrivialAugmentWide`` on batched CUDA kernels: each image gets one of fourteen ops, drawn at
    random with a random magnitude and sign, all images of a call in at most two launches.

    The draws are torchvision's (``torch.randint`` for the op, then for the magnitude bin when the op has several, then
    for the sign when the op is signed), one set per image in list order, on the default CPU generator; the magnitude
    table is built once per call. The output is torchvision's tensor path on CUDA, bit for bit for the per-channel value
    ops, Color and Sharpness. The affine ops (ShearX/Y, TranslateX/Y, Rotate) match it except where a sampling
    coordinate lies within fp32 rounding of a nearest-neighbour tie, or a bilinear value within it of a rounding tie:
    torch forms its sampling grid with a cuBLAS product whose summation order is not fixed. Images over 65,793 pixels
    may also take a Contrast value one lower or higher, where torch's own fp32 sum of the grayscale is inexact.

    Deviations: torchvision's PIL path (the one the reference recipe runs, on PIL images) gives different pixels; PIL
    images and CPU tensors raise ``HolocronB200Error``; dtypes other than uint8 raise ``TypeError`` whatever op is
    drawn; fill values outside [0, 255] raise ``ValueError``. A single tensor given the Identity op is handed back
    itself, as torchvision hands it back.

    >>> import torch
    >>> from torchvision.transforms import InterpolationMode
    >>> from holocron_b200.transforms import TrivialAugmentWide
    >>> batch = torch.randint(0, 256, (8, 3, 176, 176), dtype=torch.uint8, device="cuda")
    >>> out = TrivialAugmentWide(interpolation=InterpolationMode.BILINEAR)(batch.unbind(0))
    """

    def forward(self, img: Images) -> Tensor:
        items = _batch(img, three_d=False)
        _one_shape(img, items)
        check_options(self.interpolation, self.fill, check_images(items, _autoaugment.SUPPORTED))
        op_meta = self._augmentation_space(self.num_magnitude_bins)
        ops = [trivial_draw(op_meta) for _ in items]
        if isinstance(img, Tensor) and ops[0][0] == "Identity":
            return img
        out = apply_ops(items, ops, self.interpolation, self.fill)
        return _finish(img, out, _hw(items))


class ColorJitter(T.ColorJitter):
    """torchvision's ``ColorJitter`` on batched CUDA kernels: brightness, contrast, saturation and hue of each image,
    in a random order with random factors, all images of a call in at most two launches.

    The draws are torchvision's ``get_params`` (``torch.randperm(4)``, then one ``uniform_`` per factor that is not
    ``None``), one call per image of a list in list order, one for a single tensor and all its leading indices (each
    leading index still takes its own contrast mean). The output is torchvision's tensor path on CUDA: bit for bit on
    uint8 images, except that on images over 65,793 pixels a contrast value, and what the later ops make of it, may
    differ where torch's own fp32 sum of the grayscale is inexact; on fp32 images bit for bit for brightness,
    saturation and hue, and within the rounding of torch's fp32 sum for contrast and the ops after it (the mean here
    is an fp64 sum in a fixed order).

    Deviations: PIL images and CPU tensors raise ``HolocronB200Error``; dtypes other than uint8 and fp32 raise
    ``TypeError``, and so do channel counts other than 1 and 3 even when every factor is ``None``. A single tensor is
    handed back itself where torchvision hands it back: every factor ``None``, or one channel and only saturation and
    hue set.

    >>> import torch
    >>> from holocron_b200.transforms import ColorJitter
    >>> batch = torch.randint(0, 256, (8, 3, 256, 256), dtype=torch.uint8, device="cuda")
    >>> out = ColorJitter(brightness=0.3, contrast=0.3, saturation=0.1, hue=0.02)(batch.unbind(0))
    """

    def forward(self, img: Images) -> Tensor:
        items = _batch(img, three_d=False)
        _one_shape(img, items)
        C = check_images(items, _color.SUPPORTED)
        draws = [self.get_params(self.brightness, self.contrast, self.saturation, self.hue) for _ in items]
        if isinstance(img, Tensor):
            _, b, c, s, h = draws[0]
            # torchvision hands back the input when no op changes it
            if b is None and c is None and (C == 1 or (s is None and h is None)):
                return img
        out = jitter(items, draws)
        return _finish(img, out, _hw(items))
