"""The image-and-box transforms of the reference's detection recipe (references/detection/transforms.py:
``Compose``, ``ImageTransform``, ``CenterCrop``, ``Resize``, ``RandomResizedCrop``, ``RandomHorizontalFlip``,
``convert_to_relative``, ``VOCTargetTransform``) on the batched CUDA resampling kernel and one box kernel.

Each takes ``(image, target)`` or lists of each: a ``(C, H, W)`` CUDA image and a dict holding ``boxes``, an fp32
``(n, 4)`` xyxy CUDA tensor with unit column stride (any row stride, n may be 0), and ``labels``, an int64 ``(n,)``
tensor on the same device; other keys pass through untouched. With ``VOCTargetTransform`` first in the chain, the
targets are VOC annotation dicts instead (``{"annotation": {"object": [{"name", "bndbox": {"xmin", ...}}]}}``): they
are parsed on the host and the boxes and labels of the whole batch are uploaded in one copy. Constructors and
``repr`` are the reference's (the classes subclass torchvision's as the reference's do).

``Compose`` folds each run of geometric steps (a ``Resize`` or ``RandomResizedCrop`` starts a run; a ``CenterCrop`` is
a placement on a canvas, a second one starts a new run; a flip mirrors the canvas) into one resampling launch for the
images, and the box steps of the whole chain into one launch for every box of the batch. The draws are the
reference's on the default CPU generator, one image at a time: image 0's draws for every step, then image 1's.
``ImageTransform`` around a ``ColorJitter`` (torchvision's or this package's) draws at its place and runs the batched
jitter; around ``T.PILToTensor()`` it is a no-op on uint8 images (``TypeError`` on other dtypes); around anything else
(``ConvertImageDtype``, ``Normalize``) it is called once on the stacked image batch.

A list call returns stacked ``(N, C, S, S)`` images when the last run fixes the size (``RandomResizedCrop``,
``CenterCrop``, ``Resize`` to a pair) or an ``ImageTransform`` stacked them, and otherwise a list of views into one
buffer; and a list of new target dicts whose ``boxes`` and ``labels`` are views into one buffer each. A single pair
returns a single pair. A chain with a ``RandomResizedCrop`` reads the survivors' counts back with one device-to-host
copy per call; other chains synchronise nothing.

Box arithmetic is the reference's, bit for bit: every step rounds to fp32 as its separate torch op does, with the
ratios formed in double and rounded to fp32. The reference's quirks are kept:

- ``RandomHorizontalFlip`` maps x to ``width - x`` where ``width`` is the reference's ``_, width = image.size``, i.e.
  the image's *height*;
- ``CenterCrop`` clamps the boxes to ``[x, x + size[0]]`` / ``[y, y + size[1]]`` with x and y computed from the
  cropped image (0 for a square crop), so the boxes are not shifted by the crop's offset;
- ``Resize`` with an int scales both axes by ``size / short side``; with a tuple it scales x by ``size[0] / W`` and y
  by ``size[1] / H``; with a list it leaves the boxes unscaled;
- ``RandomResizedCrop`` scales x by ``size[0] / w`` and y by ``size[1] / h`` of the crop.

None of them changes the recipe's chains (references/detection/train.py:116-125 and its validation chain), which see
square images. Deviations: the reference runs on PIL images, whose pixels differ (the images here are torchvision's
tensor ``resize`` with antialias, ``center_crop``, ``hflip``); it modifies the caller's boxes in place, here they are
read and new tensors are returned; with zero objects its ``VOCTargetTransform`` makes ``(0,)`` boxes, here ``(0, 4)``.
PIL images and CPU tensors raise ``HolocronB200Error``; wrong box or label dtypes or shapes raise ``TypeError``; a box
count that differs from the label count raises ``ValueError``; any other callable inside ``Compose`` (the recipe's
``lambda x, y: (x, y)`` is the identity: drop it) raises ``TypeError``, all before any draw.

>>> import torch
>>> from torchvision.transforms import transforms as T
>>> from holocron_b200.transforms.detection import (Compose, ImageTransform, RandomHorizontalFlip, Resize,
...                                                 convert_to_relative)
>>> tf = Compose([Resize((416, 416)), RandomHorizontalFlip(), convert_to_relative,
...               ImageTransform(T.ColorJitter(0.3, 0.3, 0.1, 0.02)), ImageTransform(T.ConvertImageDtype(torch.float32))])
>>> images = [torch.randint(0, 256, (3, 375, 500), dtype=torch.uint8, device="cuda") for _ in range(4)]
>>> targets = [{"boxes": torch.tensor([[10., 20., 110., 220.]], device="cuda"),
...             "labels": torch.tensor([3], device="cuda")} for _ in range(4)]
>>> x, target = tf(images, targets)  # (4, 3, 416, 416) float32, 4 dicts of (1, 4) boxes in [0, 1]
"""
from typing import Any, List, Optional, Sequence, Tuple

import numpy as np
import torch
from PIL import Image
from torch import Tensor
from torchvision.transforms import transforms as T
from torchvision.transforms.functional import InterpolationMode

from .._lib import HolocronB200Error, require_cuda
from . import _color
from ._boxes import CLAMP, DIV, FILTER, FLIP, SCALE, SUB, check_target, transform_boxes
from ._color import jitter
from ._fold import _Fold, check_stackable, draw, group, jitters_of, resized, sizes_of
from ._resample import resample
from ._table import check_images, upload

__all__ = ["CenterCrop", "Compose", "ImageTransform", "RandomHorizontalFlip", "RandomResizedCrop", "Resize",
           "VOCTargetTransform", "convert_to_relative"]


class VOCTargetTransform:
    """Parses a VOC annotation dict into fp32 ``boxes`` (the integer bounding boxes) and int64 ``labels`` (the index
    of each object's name in ``classes``)."""

    def __init__(self, classes):
        self.class_map = {label: idx for idx, label in enumerate(classes)}

    def __call__(self, image, target):
        return Compose([self])(image, target)

    def parse(self, target) -> Tuple[List[List[int]], List[int]]:
        objects = target["annotation"]["object"]
        boxes = [[int(o["bndbox"][k]) for k in ("xmin", "ymin", "xmax", "ymax")] for o in objects]
        return boxes, [self.class_map[o["name"]] for o in objects]


class Compose(T.Compose):
    """Applies ``transforms`` to ``(image, target)`` in order: one resampling launch per run of geometric steps, one
    launch for every box of the batch (see the module's documentation)."""

    def __call__(self, image, target):
        steps = list(self.transforms)
        voc = steps.pop(0) if steps and isinstance(steps[0], VOCTargetTransform) else None
        images, targets = _inputs(image, target)
        if voc is not None:
            parsed = [voc.parse(t) for t in targets]
        else:
            for t in targets:
                if not isinstance(t, dict) or "boxes" not in t or "labels" not in t:
                    raise TypeError("expected each target to be a dict with 'boxes' and 'labels'")
                check_target(t["boxes"], t["labels"], images[0].device)
        segments = group(steps, _kind, _starts_run, "detection")
        _check_steps(segments, images[0].dtype)
        ops = [op for s in segments for t in (s if isinstance(s, list) else [s]) for op in _box_ops(t)]
        jitters = jitters_of(segments, ImageTransform)
        if jitters:
            check_images(images, _color.SUPPORTED)
        # the draws, image by image as the reference's Compose applied sample by sample makes them
        plans, rows = zip(*[_draw(segments, jitters, size) for size in sizes_of(images)])
        check_stackable(segments, plans, sizes_of(images), _stacks)

        if voc is not None:
            targets = [{} for _ in targets]
            boxes, labels = _upload_voc(parsed, images[0].device)
        else:
            boxes, labels = [t["boxes"] for t in targets], [t["labels"] for t in targets]
        boxes, labels = transform_boxes(boxes, labels, ops, np.array(rows, dtype=np.float32))
        targets = [{**t, "boxes": b, "labels": lab} for t, b, lab in zip(targets, boxes, labels)]

        stacked: Optional[Tensor] = None
        for k, s in enumerate(segments):
            if isinstance(s, list):
                fixed = _fixes_size(s)
                out = _run(s, images, [p[k] for p in plans], fixed)
                stacked, images = (out, list(out.unbind(0))) if fixed else (None, out)
            elif _stacks(s):
                if stacked is None:
                    stacked = torch.stack(images)
                if s in jitters:
                    stacked = jitter(stacked.unbind(0), [p[k] for p in plans])
                else:
                    stacked = s.transform(stacked)
                images = list(stacked.unbind(0))
        if not isinstance(image, (list, tuple)):
            return images[0], targets[0]
        return (stacked if stacked is not None else images), targets


class ImageTransform:
    """Applies ``transform`` to the images only."""

    def __init__(self, transform):
        self.transform = transform

    def __call__(self, image, target):
        return Compose([self])(image, target)

    def __repr__(self):
        return self.transform.__repr__()


class CenterCrop(T.CenterCrop):
    """torchvision's ``center_crop`` of the image (padded with 0 where the crop is larger); the boxes clamped to
    ``[x, x + size[0]]`` / ``[y, y + size[1]]`` with ``x = int(W' / 2 - size[0] / 2)``, ``y = int(H' / 2 - size[1] /
    2)`` of the cropped image, then shifted by (-x, -y)."""

    def __call__(self, image, target):
        return Compose([self])(image, target)


class Resize(T.Resize):
    """torchvision's ``resize`` of the image; the boxes scaled by ``size / short side`` (int size), by ``size[0] / W``
    and ``size[1] / H`` (tuple), or not at all (list)."""

    def __call__(self, image, target):
        return Compose([self])(image, target)


class RandomResizedCrop(T.RandomResizedCrop):
    """torchvision's ``resized_crop`` of the image at ``get_params``; the boxes clamped to the crop, shifted to its
    origin, those with ``x1 == x2`` or ``y1 == y2`` dropped, then scaled by ``size[0] / w`` and ``size[1] / h``."""

    def __call__(self, image, target):
        return Compose([self])(image, target)


class RandomHorizontalFlip(T.RandomHorizontalFlip):
    """Mirrors the image left-right with probability ``p`` (``torch.rand(1)``); the boxes' x become ``H - x`` (the
    reference's width is the image's height) with x1 and x2 swapped."""

    def __call__(self, image, target):
        return Compose([self])(image, target)


def convert_to_relative(image, target):
    """Divides the boxes' x by the image width and y by its height, then clamps them to [0, 1]."""
    return Compose([convert_to_relative])(image, target)


_RESIZES = (Resize, RandomResizedCrop)
_GEOMETRIC = (Resize, RandomResizedCrop, CenterCrop, RandomHorizontalFlip)


def _kind(t: Any) -> Optional[str]:
    if isinstance(t, _GEOMETRIC):
        return "run"
    if t is convert_to_relative:
        return "join"
    return "step" if isinstance(t, (ImageTransform, VOCTargetTransform)) else None


def _starts_run(t: Any, run: List[Any]) -> bool:
    return isinstance(t, _RESIZES) or (isinstance(t, CenterCrop) and any(isinstance(s, CenterCrop) for s in run))


def _stacks(s: Any) -> bool:
    """Whether an image-only step takes the stacked batch: every ImageTransform but a PILToTensor, which is a no-op."""
    return isinstance(s, ImageTransform) and not isinstance(s.transform, T.PILToTensor)


def _box_ops(t: Any) -> List[int]:
    """The box kernel's ops for one step (the same for every image)."""
    if isinstance(t, Resize):
        return [SCALE] if isinstance(t.size, (int, tuple)) else []
    if isinstance(t, RandomResizedCrop):
        return [CLAMP, SUB, FILTER, SCALE]
    if isinstance(t, CenterCrop):
        return [CLAMP, SUB]
    if isinstance(t, RandomHorizontalFlip):
        return [FLIP]
    if t is convert_to_relative:
        return [DIV, CLAMP]
    return []


def _ratio(a: int, b: int) -> float:
    """a / b formed in double and rounded to fp32, as torch rounds a Python scalar for an fp32 tensor."""
    return float(np.float32(a / b))


def fold_run(steps: Sequence[Any], size: Tuple[int, int], row: List[float]) -> _Fold:
    """One image's run (``steps``) from an image of ``size`` = (H, W), folded; the operands of its box ops are
    appended to ``row``. Its draws are the reference's, in its order, on the default CPU generator."""
    f = _Fold(size, size)
    for t in steps:
        H, W = f.canvas
        if isinstance(t, Resize):
            s = t.size
            if isinstance(s, int):
                row += 2 * [_ratio(s, H if H < W else W)]
            elif isinstance(s, tuple):
                row += [_ratio(s[0], W), _ratio(s[1], H)]
            f = _Fold(*(2 * [resized((H, W), [s] if isinstance(s, int) else list(s), t.max_size)]))
        elif isinstance(t, RandomResizedCrop):
            i, j, h, w = T.RandomResizedCrop.get_params(torch.empty(0, H, W, device="meta"), t.scale, t.ratio)
            row += [j, j + w, i, i + h, j, i, _ratio(t.size[0], w), _ratio(t.size[1], h)]
            f = _Fold(*(2 * [(int(t.size[0]), int(t.size[1]))]), box=(i, j, h, w))
        elif isinstance(t, CenterCrop):
            ch, cw = t.size
            f.center_crop(ch, cw)
            x, y = int(cw / 2 - ch / 2), int(ch / 2 - cw / 2)
            row += [x, x + ch, y, y + cw, x, y]
        elif isinstance(t, RandomHorizontalFlip):
            flip = torch.rand(1).item() < t.p
            row += [float(flip), H]
            if flip:
                f.flip()
        else:  # convert_to_relative
            row += [W, H, 0, 1, 0, 1]
    return f


def _draw(segments: Sequence[Any], jitters: Sequence[Any], size: Tuple[int, int]) -> Tuple[List[Any], List[float]]:
    """One image's draws for every step: (the fold of each run, the ``get_params`` of each ColorJitter, None for the
    other steps; the image's box parameter row)."""
    row: List[float] = []

    def other(s, size):
        if s is convert_to_relative:
            row.extend([size[1], size[0], 0, 1, 0, 1])

    return draw(segments, jitters, size, lambda run, sz: fold_run(run, sz, row), other), row


def _fixes_size(run: Sequence[Any]) -> bool:
    """Whether a run gives every image one output size whatever its input."""
    return any(isinstance(t, (RandomResizedCrop, CenterCrop)) or
               (isinstance(t, Resize) and not isinstance(t.size, int) and len(t.size) == 2) for t in run)


def _run(run: Sequence[Any], images: List[Tensor], folds: Sequence[_Fold], fixed: bool):
    """The resampling launch of a run: the images stacked when ``fixed``, else a list of views."""
    resize = run[0] if isinstance(run[0], _RESIZES) else None
    place = {"inner": [f.inner for f in folds], "offsets": [(f.top, f.left) for f in folds],
             "mirrors": [f.mirror for f in folds]}
    if isinstance(resize, RandomResizedCrop):
        place["boxes"] = [f.box for f in folds]
    if fixed:
        place["canvas"] = folds[0].canvas
    else:
        place["canvas"], place["canvases"] = None, [f.canvas for f in folds]
    if resize is None:
        return resample(images, interpolation=InterpolationMode.NEAREST, antialias=False, **place)
    return resample(images, interpolation=resize.interpolation, antialias=bool(resize.antialias), **place)


def _inputs(image, target) -> Tuple[List[Tensor], List[Any]]:
    """The images and the targets as lists; refuses what the module refuses for images."""
    single = not isinstance(image, (list, tuple))
    images = [image] if single else list(image)
    targets = [target] if single else list(target) if isinstance(target, (list, tuple)) else None
    if targets is None or len(targets) != len(images):
        raise ValueError("expected one target per image")
    if not images:
        raise ValueError("expected at least one image")
    for x in images:
        if isinstance(x, Image.Image):
            raise HolocronB200Error("holocron_b200 transforms run on CUDA tensors only: convert PIL images first "
                                    "(use the reference implementation for PIL images and CPU tensors)")
        if not isinstance(x, Tensor):
            raise TypeError("expected arg 'image' to be torch.Tensor")
        require_cuda(x)
        if x.ndim != 3:
            raise ValueError("the input image is expected to be 3-dimensional (C, H, W)")
    return images, targets


def _check_steps(segments: Sequence[Any], dtype: Optional[torch.dtype]) -> None:
    """Refuses, before any draw, a ``PILToTensor`` of images known not to be uint8 and a ``Resize`` to a one-element
    tuple (the reference indexes its second element)."""
    for s in segments:
        for t in s if isinstance(s, list) else [s]:
            if isinstance(t, Resize) and isinstance(t.size, tuple) and len(t.size) != 2:
                raise IndexError(f"Resize({t.size}) scales boxes by size[0] and size[1]: give an int or a pair")
            if isinstance(t, VOCTargetTransform):
                raise TypeError("VOCTargetTransform parses the targets: place it first")
        if isinstance(s, ImageTransform):
            if isinstance(s.transform, T.PILToTensor):
                if dtype is not None and dtype != torch.uint8:
                    raise TypeError(f"PILToTensor takes uint8 images here, got {dtype}")
            elif not isinstance(s.transform, T.ColorJitter):
                dtype = None


def _upload_voc(parsed: Sequence[Tuple[List[List[int]], List[int]]], device: torch.device
                ) -> Tuple[List[Tensor], List[Tensor]]:
    """The parsed boxes and labels of the batch on ``device``, in one host-to-device copy: per-image views."""
    ns = [len(lab) for _, lab in parsed]
    boxes = np.array([b for bs, _ in parsed for b in bs], dtype=np.float32).reshape(-1, 4)
    labels = np.array([x for _, lab in parsed for x in lab], dtype=np.int64)
    dev, (pb, pl) = upload(device, boxes, labels)
    base = dev.data_ptr()
    all_boxes = dev[pb - base:pb - base + boxes.nbytes].view(torch.float32).view(-1, 4)
    all_labels = dev[pl - base:pl - base + labels.nbytes].view(torch.int64)
    starts = np.concatenate([[0], np.cumsum(ns)[:-1]]).astype(np.int64).tolist()
    return ([all_boxes[s:s + n] for s, n in zip(starts, ns)], [all_labels[s:s + n] for s, n in zip(starts, ns)])
