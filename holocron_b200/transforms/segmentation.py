"""The paired image-and-mask transforms of the reference's segmentation recipe (references/segmentation/transforms.py:
``Compose``, ``Resize``, ``RandomResize``, ``RandomCrop``, ``RandomHorizontalFlip``, ``ToTensor``, ``ImageTransform``)
on the batched CUDA resampling kernel.

Each takes ``(image, target)``: a ``(C, H, W)`` CUDA image and an ``(H, W)`` or ``(1, H, W)`` uint8 CUDA mask of the
same size, or a list / tuple of each. Constructors and ``repr`` are the reference's. Images are resized with their
interpolation (antialiased) and padded with 0, masks are resized nearest and padded with 255, the ignore index.

``Compose`` folds each run of geometric steps (one ``Resize`` or ``RandomResize`` or none, then at most one
``RandomCrop`` and any number of ``RandomHorizontalFlip``; a resize or a second crop starts a new run) into one launch
for the images and one for the masks: only the output window is computed, the resized image is never built. A run
without a resize copies at the image's own size. The draws are the reference's on the default CPU generator, one image
at a time: image 0's draws for every step, then image 1's, which is what the reference's ``Compose`` draws applied
sample by sample. ``ImageTransform`` around a ``ColorJitter`` (torchvision's or this package's) makes that image's
``get_params`` draw at its place and runs the batched jitter on the stacked images; any other wrapped transform is called
once on the stacked image batch, so a random one draws once per call. ``ToTensor`` turns uint8 images into fp32 divided
by 255 (torchvision's ``to_tensor`` on a tensor) and masks into int64.

A list call returns stacked ``(N, C, S, S)`` images and ``(N, S, S)`` masks (``(N, 1, S, S)`` for ``(1, H, W)`` masks)
when its last run fixes the size (``RandomCrop``, ``Resize`` to a pair) or an ``ImageTransform`` or ``ToTensor``
stacked them, and otherwise lists of ``(C, h_i, w_i)`` / ``(h_i, w_i)`` views into one buffer. A single pair returns a
single pair.

The outputs are torchvision's tensor path for the same steps on CUDA (``resize`` with antialias, ``resize`` nearest,
``pad`` with 0 / 255 on the bottom and right, ``crop``, ``hflip``): masks bit for bit, images as this package's
``Resize``. Deviations: the reference runs on PIL images, whose pixels differ (PIL's nearest samples pixel centres where
torch's uses ``floor(dst * scale)``, and PIL's bilinear is fixed-point); its ``ToTensor`` turns a PIL image into float,
here it takes a uint8 CUDA tensor. PIL images and CPU tensors raise ``HolocronB200Error``; a mask that is not uint8 or
has more than one channel raises ``TypeError``; an image and mask of different sizes raise ``ValueError``, all before
any draw. An ``ImageTransform`` or ``ToTensor`` reached by images of different sizes raises ``ValueError`` after the
draws, before any launch.

>>> import torch
>>> from holocron_b200.transforms import ColorJitter
>>> from holocron_b200.transforms.segmentation import (Compose, ImageTransform, RandomCrop, RandomHorizontalFlip,
...                                                    RandomResize, ToTensor)
>>> tf = Compose([RandomResize(160, 640), RandomCrop(256), RandomHorizontalFlip(0.5),
...               ImageTransform(ColorJitter(0.3, 0.3, 0.1, 0.02)), ToTensor()])
>>> images = [torch.randint(0, 256, (3, 375, 500), dtype=torch.uint8, device="cuda") for _ in range(4)]
>>> masks = [torch.randint(0, 21, (375, 500), dtype=torch.uint8, device="cuda") for _ in range(4)]
>>> x, target = tf(images, masks)  # (4, 3, 256, 256) float32, (4, 256, 256) int64
"""
from dataclasses import dataclass
from typing import Any, List, Optional, Sequence, Tuple, Union

import torch
from PIL import Image
from torch import Tensor
from torchvision.transforms import transforms as T
from torchvision.transforms.functional import InterpolationMode, _compute_resized_output_size

from .._lib import HolocronB200Error, require_cuda
from ._color import jitter
from ._resample import resample
from ._table import check_images
from . import _color
from .interpolation import _resize_options

__all__ = ["Compose", "ImageTransform", "RandomCrop", "RandomHorizontalFlip", "RandomResize", "Resize", "ToTensor"]

IMAGE_FILL, MASK_FILL = 0.0, 255.0


class Resize:
    """Resizes the image with ``interpolation`` and the mask nearest to ``output_size``: an int sets the short side, a
    pair (h, w) both."""

    def __init__(self, output_size, interpolation=InterpolationMode.BILINEAR):
        self.output_size = output_size
        self.interpolation = interpolation

    def __call__(self, image, target):
        return Compose([self])(image, target)

    def __repr__(self):
        return f"{self.__class__.__name__}(output_size={self.output_size})"


class RandomResize:
    """Resizes the short side of the image (``interpolation``) and mask (nearest) to a size drawn from
    ``[min_size, max_size)`` (``torch.randint``; no draw when both are equal)."""

    def __init__(self, min_size, max_size=None, interpolation=InterpolationMode.BILINEAR):
        self.min_size = min_size
        if max_size is None:
            max_size = min_size
        self.max_size = max_size
        self.interpolation = interpolation

    def __call__(self, image, target):
        return Compose([self])(image, target)

    def __repr__(self):
        return f"{self.__class__.__name__}(min_size={self.min_size}, max_size={self.max_size})"


class RandomHorizontalFlip:
    """Mirrors the image and the mask left-right with probability ``prob`` (``torch.rand(1)``)."""

    def __init__(self, prob):
        self.prob = prob

    def __call__(self, image, target):
        return Compose([self])(image, target)

    def __repr__(self):
        return f"{self.__class__.__name__}(p={self.prob})"


class RandomCrop:
    """Pads the image with 0 and the mask with 255 on the bottom and right up to ``size`` where a side is shorter, then
    crops a random ``size`` x ``size`` window of both (``T.RandomCrop.get_params``)."""

    def __init__(self, size):
        self.size = size

    def __call__(self, image, target):
        return Compose([self])(image, target)

    def __repr__(self):
        return f"{self.__class__.__name__}(size={self.size})"


class ToTensor(T.ToTensor):
    """uint8 images to fp32 in [0, 1] (``x.to(float32).div(255)``, torchvision's ``to_tensor`` of a tensor), masks to
    int64."""

    def __call__(self, img, target):
        return Compose([self])(img, target)


class ImageTransform:
    """Applies ``transform`` to the images only."""

    def __init__(self, transform):
        self.transform = transform

    def __call__(self, image, target):
        return Compose([self])(image, target)

    def __repr__(self):
        return self.transform.__repr__()


_RESIZES = (Resize, RandomResize)
_GEOMETRIC = (Resize, RandomResize, RandomCrop, RandomHorizontalFlip)


@dataclass
class _Fold:
    """One image's run folded: its source resized to ``inner``, placed at (top, left) on a canvas of ``canvas``, the
    canvas mirrored when ``mirror``."""

    inner: Tuple[int, int]
    canvas: Tuple[int, int]
    top: int = 0
    left: int = 0
    mirror: bool = False

    def flip(self) -> None:
        self.mirror = not self.mirror

    def pad(self, bottom: int, right: int) -> None:
        """torchvision's pad of the bottom and right of the canvas: in a mirrored canvas the new columns are on the
        right of what is read, so the box moves right."""
        if self.mirror:
            self.left += right
        self.canvas = (self.canvas[0] + bottom, self.canvas[1] + right)

    def crop(self, i: int, j: int, h: int, w: int) -> None:
        self.top -= i
        self.left -= (self.canvas[1] - w - j) if self.mirror else j
        self.canvas = (h, w)


def fold_run(steps: Sequence[Any], size: Tuple[int, int]) -> _Fold:
    """One image's run (``steps``, the first possibly a resize) from an image of ``size`` = (H, W), folded; its draws
    are the reference's, in its order, on the default CPU generator."""
    f = _Fold(size, size)
    for t in steps:
        if isinstance(t, Resize):
            out = t.output_size
            f = _Fold(*(2 * [_resized(size, [out] if isinstance(out, int) else list(out))]))
        elif isinstance(t, RandomResize):
            s = t.min_size if t.min_size == t.max_size else torch.randint(t.min_size, t.max_size, (1,)).item()
            f = _Fold(*(2 * [_resized(size, [s])]))
        elif isinstance(t, RandomCrop):
            h, w = f.canvas
            if min(h, w) < t.size:
                f.pad(max(t.size - h, 0), max(t.size - w, 0))
            f.crop(*T.RandomCrop.get_params(torch.empty(0, *f.canvas, device="meta"), (t.size, t.size)))
        elif torch.rand(1).item() < t.prob:
            f.flip()
    return f


def _resized(size: Tuple[int, int], out: List[int]) -> Tuple[int, int]:
    h, w = _compute_resized_output_size(size, out)
    return int(h), int(w)


def _fixes_size(run: Sequence[Any]) -> bool:
    """Whether a run gives every image one output size whatever its input: it crops, or resizes to a pair."""
    return any(isinstance(t, RandomCrop) or
               (isinstance(t, Resize) and not isinstance(t.output_size, int) and len(t.output_size) == 2) for t in run)


def _segments(transforms: Sequence[Any]) -> List[Union[List[Any], Any]]:
    """The steps grouped: runs (lists of geometric steps) and the image-only steps between them."""
    segments: List[Union[List[Any], Any]] = []
    run: Optional[List[Any]] = None
    for t in transforms:
        if isinstance(t, _GEOMETRIC):
            if (run is None or isinstance(t, _RESIZES)
                    or (isinstance(t, RandomCrop) and any(isinstance(s, RandomCrop) for s in run))):
                run = []
                segments.append(run)
            run.append(t)
        elif isinstance(t, (ImageTransform, ToTensor)):
            run = None
            segments.append(t)
        else:
            raise TypeError(f"{type(t).__name__} is not a transform of holocron_b200.transforms.segmentation")
    return segments


def _inputs(image, target) -> Tuple[List[Tensor], List[Tensor], int]:
    """The images, the masks as (1, H, W) views, and the masks' dimension count; refuses what the module refuses."""
    single = not isinstance(image, (list, tuple))
    images = [image] if single else list(image)
    masks = [target] if single else list(target) if isinstance(target, (list, tuple)) else None
    if masks is None or len(masks) != len(images):
        raise ValueError("expected one mask per image")
    if not images:
        raise ValueError("expected at least one image")
    for x in images + masks:
        if isinstance(x, Image.Image):
            raise HolocronB200Error("holocron_b200 transforms run on CUDA tensors only: convert PIL images first "
                                    "(use the reference implementation for PIL images and CPU tensors)")
        if not isinstance(x, Tensor):
            raise TypeError("expected arg 'image' and 'target' to be torch.Tensor")
        require_cuda(x)
    ndim = masks[0].ndim
    for x, m in zip(images, masks):
        if x.ndim != 3:
            raise ValueError("the input image is expected to be 3-dimensional (C, H, W)")
        if m.dtype != torch.uint8 or m.ndim not in (2, 3) or (m.ndim == 3 and m.shape[0] != 1) or m.ndim != ndim:
            raise TypeError(f"masks must be uint8 (H, W) or (1, H, W) tensors of one layout, got {m.dtype} "
                            f"{tuple(m.shape)}")
        if m.shape[-2:] != x.shape[-2:]:
            raise ValueError(f"image {tuple(x.shape[-2:])} and mask {tuple(m.shape[-2:])} differ in size")
    return images, [m if m.ndim == 3 else m.unsqueeze(0) for m in masks], ndim


def _run(run: Sequence[Any], images: List[Tensor], masks: List[Tensor], folds: Sequence[_Fold], fixed: bool):
    """The two launches of a run: (images, masks) stacked when ``fixed``, else lists of views."""
    resize = run[0] if isinstance(run[0], _RESIZES) else None
    interpolation = _resize_options(resize.interpolation)[0] if resize is not None else InterpolationMode.NEAREST
    place = {"inner": [f.inner for f in folds], "offsets": [(f.top, f.left) for f in folds],
             "mirrors": [f.mirror for f in folds]}
    if fixed:
        place["canvas"] = folds[0].canvas
    else:
        place["canvas"], place["canvases"] = None, [f.canvas for f in folds]
    out_images = resample(images, interpolation=interpolation, antialias=resize is not None, fill=IMAGE_FILL,
                          **place)
    out_masks = resample(masks, interpolation=InterpolationMode.NEAREST, antialias=False, fill=MASK_FILL, **place)
    return out_images, out_masks


class Compose(T.Compose):
    """Applies ``transforms`` to ``(image, target)`` in order, folding each run of geometric steps into one launch for
    the images and one for the masks (see the module's documentation)."""

    def __init__(self, transforms):
        super(Compose, self).__init__(transforms)

    def __call__(self, image, target):
        images, masks, ndim = _inputs(image, target)
        segments = _segments(self.transforms)
        _check_order(segments, images[0].dtype)
        jitters = [s for s in segments if isinstance(s, ImageTransform) and isinstance(s.transform, T.ColorJitter)]
        if jitters:
            check_images(images, _color.SUPPORTED)
        # the draws, image by image as the reference's Compose applied sample by sample makes them
        plans = [_draw(segments, jitters, (int(x.shape[-2]), int(x.shape[-1]))) for x in images]
        _check_stackable(segments, plans, [tuple(x.shape[-2:]) for x in images])

        stacked_images: Optional[Tensor] = None
        stacked_masks: Optional[Tensor] = None
        for k, s in enumerate(segments):
            if isinstance(s, list):
                fixed = _fixes_size(s)
                images, masks = _run(s, images, masks, [p[k] for p in plans], fixed)
                stacked_images, stacked_masks = (images, masks) if fixed else (None, None)
            else:
                if stacked_images is None:
                    stacked_images, stacked_masks = torch.stack(images), torch.stack(masks)
                if isinstance(s, ToTensor):
                    stacked_images = stacked_images.to(torch.float32).div(255)
                    stacked_masks = stacked_masks.to(torch.int64)
                elif s in jitters:
                    stacked_images = jitter(stacked_images.unbind(0), [p[k] for p in plans])
                else:
                    stacked_images = s.transform(stacked_images)
            if stacked_images is not None:
                images, masks = list(stacked_images.unbind(0)), list(stacked_masks.unbind(0))
        if ndim == 2:
            masks = [m[0] for m in masks]
            stacked_masks = stacked_masks[:, 0] if stacked_masks is not None else None
        if not isinstance(image, (list, tuple)):
            return images[0], masks[0]
        if stacked_images is not None:
            return stacked_images, stacked_masks
        return images, masks


def _draw(segments: Sequence[Any], jitters: Sequence[Any], size: Tuple[int, int]) -> List[Any]:
    """One image's draws for every step: the fold of each run, the ``get_params`` of each ColorJitter, None for the
    other steps."""
    plan: List[Any] = []
    for s in segments:
        if isinstance(s, list):
            fold = fold_run(s, size)
            size = fold.canvas
            plan.append(fold)
        elif s in jitters:
            j = s.transform
            plan.append(j.get_params(j.brightness, j.contrast, j.saturation, j.hue))
        else:
            plan.append(None)
    return plan


def _check_order(segments: Sequence[Any], dtype: torch.dtype) -> None:
    """Refuses, before any draw, geometric steps after ``ToTensor`` (masks are int64 from there on) and ``ToTensor``
    of images known not to be uint8."""
    converted = False
    for s in segments:
        if isinstance(s, list) and converted:
            raise TypeError("geometric transforms take uint8 masks: place them before ToTensor")
        if isinstance(s, ToTensor):
            if dtype != torch.uint8:
                raise TypeError(f"ToTensor takes uint8 images, got {dtype}")
            converted = True
        if isinstance(s, ImageTransform) and not isinstance(s.transform, T.ColorJitter):
            dtype = None


def _check_stackable(segments: Sequence[Any], plans: Sequence[Sequence[Any]], sizes: List[Tuple[int, int]]) -> None:
    """Refuses an ``ImageTransform`` or ``ToTensor`` reached by images of different sizes."""
    for k, s in enumerate(segments):
        if isinstance(s, list):
            sizes = [p[k].canvas for p in plans]
        elif len(set(sizes)) > 1:
            raise ValueError(f"{s!r} takes images of one size, but the images reaching it have {len(set(sizes))} "
                             "sizes: crop or resize them to one size first")
