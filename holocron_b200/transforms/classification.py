"""The transform chains of the reference's classification recipe (references/classification/train.py:100-107 and
:115-121 for training, :162-168 and :175 for validation) as one batched ``Compose``, and ``Normalize`` on one CUDA
launch.

``Compose`` subclasses torchvision's (constructor and ``repr`` are torchvision's) and takes torchvision's
``RandomResizedCrop``, ``Resize``, ``CenterCrop``, ``RandomHorizontalFlip``, ``autoaugment.TrivialAugmentWide``,
``PILToTensor``, ``ConvertImageDtype(torch.float32)``, ``Normalize`` and ``RandomErasing``, or this package's
subclasses of them. A call takes one ``(C, H, W)`` CUDA tensor or a list / tuple of them, read in place whatever their
strides. Each image's draws are made for every step in chain order, image after image, on the default CPU generator,
before anything is launched: exactly what the recipe's ``T.Compose`` applied image by image draws. The chain then runs
in segments:

- a run (a ``RandomResizedCrop`` or ``Resize``, or neither, followed by any ``CenterCrop`` and flips) is one
  ``hb_resample_batch`` launch: the crop box is the row's source box, a ``CenterCrop`` a placement on the canvas
  (torchvision's ``center_crop``: zero padding where the crop is larger), a flip the row's mirror flag;
- ``TrivialAugmentWide`` is its one or two launches (two when an image drew a histogram op);
- a tail (a run of ``PILToTensor``, ``ConvertImageDtype``, ``Normalize`` and ``RandomErasing``, each at most once, in
  any order) is one ``hb_image_tail_batch`` launch that reads each image once and writes the finished fp32 batch.
  ``PILToTensor`` is a no-op on uint8 images. A tail that leaves the images uint8 (erasing before any conversion, or
  ``PILToTensor`` alone) is one ``hb_erase_batch`` copy instead.

So the recipe's ImageNette train chain takes 3 or 4 launches, its validation chain 2, the CIFAR train chain 3 or 4 and
the CIFAR validation chain 1, none of which synchronises the device with the host. A list returns the stacked
``(N, C, h, w)`` batch (what ``default_collate`` stacks), or a list of views when the last step is a run that leaves
the images at different sizes (a ``Resize`` to a short side); a single tensor returns what ``T.Compose`` returns.

Outputs are torchvision's on CUDA tensors: the runs are this package's ``Resize`` resampling, the tail is bit for bit
torchvision's ``image.to(float32) / 255``, ``sub_(mean).div_(std)`` and erasing, and ``TrivialAugmentWide`` is as its
class states. Deviations: PIL images and CPU tensors raise ``HolocronB200Error``; ``ConvertImageDtype`` to anything but
``torch.float32`` and ``Normalize`` of float images other than fp32 raise ``NotImplementedError``; ``Normalize`` of
uint8 images and ``PILToTensor`` of other than uint8 raise ``TypeError``, all before any draw; a ``std`` that is zero
after fp32 rounding raises torchvision's ``ValueError``, and so does a mean or std of a length other than 1 or C, both
before any draw; ``Normalize(inplace=True)`` and ``RandomErasing(inplace=True)`` never write the caller's images;
images of different sizes reaching ``TrivialAugmentWide`` or a tail raise ``ValueError`` before any launch;
``holocron_b200.transforms.Resize`` and ``RandomZoomOut`` (the reference's pad / squish resize) and any other callable
raise ``TypeError`` before any draw. ``RandomErasing(value="random")`` still draws one ``normal_()`` per erased image
on the host, as torchvision does; with the recipe's default ``--random-erase 0.0`` nothing is drawn.

>>> import torch
>>> from torchvision.transforms import autoaugment as A, transforms as T
>>> from holocron_b200.transforms.classification import Compose
>>> tf = Compose([T.RandomResizedCrop(176, scale=(0.3, 1.0)), T.RandomHorizontalFlip(),
...               A.TrivialAugmentWide(interpolation=T.InterpolationMode.BILINEAR), T.PILToTensor(),
...               T.ConvertImageDtype(torch.float32), T.Normalize((0.485, 0.456, 0.406), (0.229, 0.224, 0.225)),
...               T.RandomErasing(p=0.1, scale=(0.02, 0.2), value="random")])
>>> images = [torch.randint(0, 256, (3, 375, 500), dtype=torch.uint8, device="cuda") for _ in range(4)]
>>> x = tf(images)  # (4, 3, 176, 176) float32
"""
from typing import Any, Dict, List, Optional, Sequence, Tuple

import torch
from torch import Tensor
from torchvision.transforms import autoaugment, transforms as T
from torchvision.transforms.functional import InterpolationMode

from . import _autoaugment
from ._autoaugment import apply_ops, check_options
from ._erase import erase
from ._fold import _Fold, check_stackable, draw, group, resized, sizes_of
from ._resample import resample
from ._table import check_batch
from ._tail import norm_values, program, tail
from .augmentation import _hw, _one_shape, erase_draw, trivial_draw
from .interpolation import Images, RandomZoomOut, Resize, _batch, _finish

__all__ = ["Compose", "Normalize"]

_RESIZES = (T.RandomResizedCrop, T.Resize)
_GEOMETRIC = (T.RandomResizedCrop, T.Resize, T.CenterCrop, T.RandomHorizontalFlip)
_TAIL_STEPS = (T.PILToTensor, T.ConvertImageDtype, T.Normalize, T.RandomErasing)


class _Tail:
    """A run of tail steps, each kind at most once: one launch."""

    def __init__(self, step: Any):
        self.steps = [step]

    def takes(self, t: Any) -> bool:
        return all(_tail_kind(t) is not _tail_kind(s) for s in self.steps)

    def step(self, kind: type) -> Optional[Any]:
        return next((t for t in self.steps if isinstance(t, kind)), None)

    def __repr__(self):
        return f"{type(self).__name__}({self.steps!r})"


def _tail_kind(t: Any) -> type:
    return next(k for k in _TAIL_STEPS if isinstance(t, k))


def _kind(t: Any) -> Optional[str]:
    if isinstance(t, (Resize, RandomZoomOut)):  # the reference's pad / squish resize is not a torchvision resize
        return None
    if isinstance(t, _GEOMETRIC):
        return "run"
    return "step" if isinstance(t, (autoaugment.TrivialAugmentWide, *_TAIL_STEPS)) else None


def _segments(transforms: Sequence[Any]) -> List[Any]:
    """Runs (lists of geometric steps), TrivialAugmentWide steps and tails."""
    segments: List[Any] = []
    for s in group(transforms, _kind, lambda t, run: isinstance(t, _RESIZES), "classification"):
        if isinstance(s, _TAIL_STEPS):
            if segments and isinstance(segments[-1], _Tail) and segments[-1].takes(s):
                segments[-1].steps.append(s)
            else:
                segments.append(_Tail(s))
        else:
            segments.append(s)
    return segments


def fold_run(steps: Sequence[Any], size: Tuple[int, int]) -> _Fold:
    """One image's run from an image of ``size`` = (H, W), folded; its draws are torchvision's, in its order, on the
    default CPU generator (a meta tensor stands in for the image where ``get_params`` reads its shape)."""
    f = _Fold(size, size)
    for t in steps:
        H, W = f.canvas
        if isinstance(t, T.RandomResizedCrop):
            i, j, h, w = T.RandomResizedCrop.get_params(torch.empty(0, H, W, device="meta"), t.scale, t.ratio)
            f = _Fold(*(2 * [(int(t.size[0]), int(t.size[1]))]), box=(i, j, h, w))
        elif isinstance(t, T.Resize):
            f = _Fold(*(2 * [resized((H, W), [t.size] if isinstance(t.size, int) else list(t.size), t.max_size)]))
        elif isinstance(t, T.CenterCrop):
            f.center_crop(*t.size)
        elif torch.rand(1) < t.p:
            f.flip()
    return f


def _fixes_size(run: Sequence[Any]) -> bool:
    """Whether a run gives every image one output size whatever its input."""
    return any(isinstance(t, (T.RandomResizedCrop, T.CenterCrop)) or
               (isinstance(t, T.Resize) and not isinstance(t.size, int) and len(t.size) == 2) for t in run)


def _run(run: Sequence[Any], images: List[Tensor], folds: Sequence[_Fold], fixed: bool):
    """The resampling launch of a run: the images stacked when ``fixed``, else a list of views."""
    resize = run[0] if isinstance(run[0], _RESIZES) else None
    place = {"inner": [f.inner for f in folds], "offsets": [(f.top, f.left) for f in folds],
             "mirrors": [f.mirror for f in folds]}
    if isinstance(resize, T.RandomResizedCrop):
        place["boxes"] = [f.box for f in folds]
    if fixed:
        place["canvas"] = folds[0].canvas
    else:
        place["canvas"], place["canvases"] = None, [f.canvas for f in folds]
    if resize is None:  # flips and crops only: a nearest copy at the image's own size
        return resample(images, interpolation=InterpolationMode.NEAREST, antialias=False, **place)
    return resample(images, interpolation=resize.interpolation, antialias=bool(resize.antialias), **place)


def _check_steps(segments: Sequence[Any], dtype: torch.dtype, C: int) -> Dict[int, Any]:
    """Refuses, before any draw, what the steps refuse for images of ``dtype`` with C channels; returns each tail's
    (op program, output dtype, mean and std) by segment index."""
    programs: Dict[int, Any] = {}
    for k, s in enumerate(segments):
        if isinstance(s, autoaugment.TrivialAugmentWide):
            if dtype not in _autoaugment.SUPPORTED:
                raise TypeError(f"TrivialAugmentWide takes uint8 images here, got {dtype}")
            check_options(s.interpolation, s.fill, C)
        elif isinstance(s, _Tail):
            ops, out = program(s.steps, dtype)
            normalize = s.step(T.Normalize)
            norm = norm_values(normalize.mean, normalize.std, C) if normalize is not None else None
            programs[k] = (ops, out, norm)
            dtype = out
    return programs


def _apply_tail(s: _Tail, images: List[Tensor], rects: List[Any], ops: List[int], out_dtype: torch.dtype, norm):
    """The one launch of a tail."""
    if s.step(T.RandomErasing) is None:
        rects = None
    if out_dtype == torch.uint8:  # no conversion: at most an erase of the uint8 images, which hb_erase_batch copies
        return erase(images, rects if rects is not None else [None] * len(images), False)
    return tail(images, ops, rects, norm)


class Compose(T.Compose):
    """Applies ``transforms`` to a CUDA image or a list of them, draw for draw as torchvision's ``Compose`` applied
    image by image, in one launch per run, ``TrivialAugmentWide`` (two when an image drew a histogram op) and tail
    (see the module's documentation)."""

    def __call__(self, img: Images):
        images = _batch(img)
        check_batch(images, one_shape=False)
        segments = _segments(self.transforms)
        C = int(images[0].shape[-3])
        programs = _check_steps(segments, images[0].dtype, C)
        spaces = {id(s): s._augmentation_space(s.num_magnitude_bins) for s in segments
                  if isinstance(s, autoaugment.TrivialAugmentWide)}

        def other(s: Any, size: Tuple[int, int]) -> Any:
            if isinstance(s, autoaugment.TrivialAugmentWide):
                return trivial_draw(spaces[id(s)])
            erasing = s.step(T.RandomErasing)
            return erase_draw(erasing, torch.empty(C, *size, device="meta"))[1] if erasing is not None else None

        # the draws, image by image as torchvision's Compose applied to each image makes them
        plans = [draw(segments, [], size, fold_run, other) for size in sizes_of(images)]
        check_stackable(segments, plans, sizes_of(images))

        stacked: Optional[Tensor] = None
        for k, s in enumerate(segments):
            draws = [p[k] for p in plans]
            if isinstance(s, list):
                fixed = _fixes_size(s)
                out = _run(s, images, draws, fixed)
                stacked, images = (out, list(out.unbind(0))) if fixed else (None, out)
                continue
            if isinstance(s, autoaugment.TrivialAugmentWide):
                stacked = apply_ops(images, draws, s.interpolation, s.fill)
            else:
                stacked = _apply_tail(s, images, draws, *programs[k])
            images = list(stacked.unbind(0))
        if not isinstance(img, (list, tuple)):
            return images[0]
        if not segments:
            return img
        return stacked if stacked is not None else images


class Normalize(T.Normalize):
    """torchvision's ``Normalize`` on one CUDA launch: ``(v - mean[c]) / std[c]`` of every element of an fp32 image,
    bit for bit torchvision's ``sub_`` and ``div_`` on CUDA, without its three host synchronisations (the ``std == 0``
    test runs on the host, on the fp32-rounded values).

    It takes one ``(..., C, H, W)`` fp32 CUDA tensor, or a list / tuple of ``(C, H, W)`` ones of one shape, read in
    place whatever their strides, which it returns stacked as ``(N, C, H, W)``. Deviations: PIL images and CPU tensors
    raise ``HolocronB200Error``; float images other than fp32 raise ``NotImplementedError``; a mean or std of a length
    other than 1 or C raises ``ValueError``; ``inplace=True`` never writes the caller's images. So
    ``ImageTransform(Normalize(...))`` of the segmentation and detection chains normalises without a synchronisation.

    >>> import torch
    >>> from holocron_b200.transforms import Normalize
    >>> batch = torch.rand(8, 3, 224, 224, device="cuda")
    >>> out = Normalize((0.485, 0.456, 0.406), (0.229, 0.224, 0.225))(batch.unbind(0))
    """

    def forward(self, tensor: Images) -> Tensor:
        items = _batch(tensor, three_d=False)
        _one_shape(tensor, items)
        ops, _ = program([self], items[0].dtype)
        if items[0].ndim < 3:
            raise ValueError("Expected tensor to be a tensor image of size (..., C, H, W). Got tensor.size() = "
                             f"{items[0].size()}")
        out = tail(items, ops, norm=norm_values(self.mean, self.std, int(items[0].shape[-3])))
        return _finish(tensor, out, _hw(items))
