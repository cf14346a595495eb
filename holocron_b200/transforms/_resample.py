"""Host side of the batched resampling kernel (holocron_b200/csrc/resample.cu, ``hb_resample_batch``).

``resample`` takes a batch of images, each with the inner size it is resized to and the signed offset of that inner box
on a common canvas, validates what torchvision would refuse before anything is launched, writes one descriptor row per
image into pinned host memory, uploads the table asynchronously (no host synchronisation) and launches one kernel that
resizes every image and fills its canvas. An image may be cropped to a box first (its row then points at the box's
top-left pixel and has the box's size) and mirrored left-right (its row points at the last column with a negated column
stride): the kernel reads both as any other strided source."""
import math
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch
from torch import Tensor
from torchvision.transforms.functional import InterpolationMode

from .._lib import check, lib, require_cuda, stream_ptr
from ._table import INT32_MAX, batch_out, check_batch, dtype_code, planes, upload

# interpolation modes torchvision's tensor resize accepts, as the kernel's filter codes
FILTERS = {InterpolationMode.NEAREST: 0, InterpolationMode.NEAREST_EXACT: 1, InterpolationMode.BILINEAR: 2,
           InterpolationMode.BICUBIC: 3}
PAD_MODES = {"constant": 0, "edge": 1, "reflect": 2, "symmetric": 3}
# Taps per axis that fit the kernel's shared-memory weight tables for every dtype: antialiased downscales up to about
# 1/127 (bilinear) or 1/63 (bicubic).
MAX_TAPS = 255


def axis_taps(n_in: int, n_out: int, filter_code: int, antialias: bool, dtype: torch.dtype) -> int:
    """The most taps a filter from n_in to n_out samples has along one axis, computed as the kernel computes its
    support (in fp32, fp64 for fp64 images)."""
    if filter_code < 2:
        return 1
    if not antialias:
        return 2 if filter_code == 2 else 4
    acc = np.float64 if dtype == torch.float64 else np.float32
    scale = acc(n_in) / acc(n_out)
    half = 1.0 if filter_code == 2 else 2.0
    support = acc(half * float(scale)) if scale >= 1 else acc(half)
    return int(math.ceil(support)) * 2 + 1


def interpolation_code(interpolation) -> int:
    """The kernel's filter for a torchvision interpolation, refusing what torchvision refuses for tensors."""
    if not isinstance(interpolation, InterpolationMode):
        raise TypeError("Argument interpolation should be a InterpolationMode or a corresponding Pillow integer constant")
    if interpolation not in FILTERS:
        raise NotImplementedError(f"interpolation {interpolation.value!r} is not supported for tensors "
                                  f"(supported: {', '.join(m.value for m in FILTERS)})")
    return FILTERS[interpolation]


def _check_padding(pad_mode: str, pads: Tuple[int, int, int, int], h: int, w: int) -> None:
    """pads = (left, top, right, bottom). torch's reflection pad refuses a padding >= the side it mirrors; torchvision's
    symmetric pad indexes past the image for a padding > the side (IndexError on CPU tensors)."""
    left, top, right, bottom = pads
    if pad_mode == "reflect" and (max(left, right) >= w or max(top, bottom) >= h):
        raise RuntimeError(f"Padding size should be less than the corresponding input dimension, but got: padding "
                           f"({left}, {right}) at dimension 2 and ({top}, {bottom}) at dimension 1 of an image of "
                           f"{h}x{w}")
    if pad_mode == "symmetric" and (max(left, right) > w or max(top, bottom) > h):
        raise IndexError(f"symmetric padding ({left}, {top}, {right}, {bottom}) exceeds the image size {h}x{w}")


def descriptor_table(sources: Sequence[Tensor], inner: Sequence[Tuple[int, int]], canvas: Tuple[int, int],
                     filter_code: int, antialias: bool, pad_mode: str,
                     boxes: Optional[Sequence[Tuple[int, int, int, int]]] = None,
                     flips: Optional[Sequence[bool]] = None) -> Tuple[np.ndarray, int, int]:
    """(table, taps_y, taps_x): the int64 [N_total, 16] descriptor rows of hb_resample_batch, destination pointers left
    at 0, and the most filter taps per axis. Raises what torchvision would raise for these placements.

    ``boxes[i] = (top, left, height, width)`` crops source i to that box (inside the image) before it is resized;
    ``flips[i]`` mirrors it left-right."""
    check_batch(sources, one_shape=False)
    C = sources[0].shape[-3]
    Hc, Wc = canvas
    rows: List[List[int]] = []
    taps_y = taps_x = 1
    for k, (x, (h, w)) in enumerate(zip(sources, inner)):
        H, W = x.shape[-2:]
        sc, sh, sw = x.stride()[-3:]
        base = x.data_ptr()
        if boxes is not None:
            bi, bj, bh, bw = boxes[k]
            if bi < 0 or bj < 0 or bi + bh > H or bj + bw > W:
                raise ValueError(f"crop box {tuple(boxes[k])} is not inside the {H}x{W} image")
            base += (bi * sh + bj * sw) * x.element_size()
            H, W = bh, bw
        if flips is not None and flips[k]:
            base += (W - 1) * sw * x.element_size()
            sw = -sw
        if h <= 0 or w <= 0 or H <= 0 or W <= 0:
            raise RuntimeError(f"Input and output sizes should be greater than 0, but got input (H: {H}, W: {W}) "
                               f"output (H: {h}, W: {w})")
        dh, dw = Hc - h, Wc - w
        top, left = dh // 2, dw // 2
        _check_padding(pad_mode, (left, top, dw - left, dh - top), h, w)
        if (W - 1) * abs(sw) > INT32_MAX:
            raise ValueError("image rows span more than 2**31 elements")
        row = [base, 0, sc, sh, sw, C, H, W, h, w, top, left, Hc, Wc, PAD_MODES[pad_mode], 0]
        for o in planes(x):
            rows.append([row[0] + o * x.element_size()] + row[1:])
        taps_y = max(taps_y, axis_taps(H, h, filter_code, antialias, x.dtype))
        taps_x = max(taps_x, axis_taps(W, w, filter_code, antialias, x.dtype))
    if max(taps_y, taps_x) > MAX_TAPS:
        raise NotImplementedError(f"resampling needs {max(taps_y, taps_x)} filter taps per axis (at most {MAX_TAPS}: "
                                  "downscale in two steps)")
    return np.array(rows, dtype=np.int64), taps_y, taps_x


def resample(sources: Sequence[Tensor], inner: Sequence[Tuple[int, int]], canvas: Tuple[int, int],
             interpolation: InterpolationMode, antialias: bool, pad_mode: str = "constant",
             out: Optional[Tensor] = None, boxes: Optional[Sequence[Tuple[int, int, int, int]]] = None,
             flips: Optional[Sequence[bool]] = None) -> Tensor:
    """Resizes sources[i] ([..., C, H_i, W_i], CUDA, any strides) to inner[i] = (h_i, w_i) and centres it on a canvas
    of ``canvas`` = (Hc, Wc) the way torchvision's ``pad`` places it (left / top padding = floor(delta / 2), negative
    padding crops), filling the rest by ``pad_mode``. Returns ``out``, a contiguous tensor of shape
    (N_total, C, Hc, Wc) holding one canvas per source image (leading dimensions of a source count as images).
    ``boxes`` and ``flips`` (one entry per source) crop and mirror the sources first (``descriptor_table``)."""
    if pad_mode not in PAD_MODES:
        raise ValueError("Padding mode should be either constant, edge, reflect or symmetric")
    filter_code = interpolation_code(interpolation)
    antialias = bool(antialias) and filter_code >= 2
    ref = sources[0]
    require_cuda(*sources)
    dtype = dtype_code(ref)
    table, taps_y, taps_x = descriptor_table(sources, inner, canvas, filter_code, antialias, pad_mode, boxes, flips)
    n, C, (Hc, Wc) = table.shape[0], ref.shape[-3], canvas
    out = batch_out(sources, out, (C, Hc, Wc))
    table[:, 1] = out.data_ptr() + np.arange(n, dtype=np.int64) * (C * Hc * Wc * out.element_size())
    _dev, (descs,) = upload(ref.device, table)
    check(lib().hb_resample_batch(descs, n, Hc, Wc, filter_code, int(antialias), taps_y, taps_x, dtype, stream_ptr()),
          "hb_resample_batch")
    return out
