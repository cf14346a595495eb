"""Host side of the batched erasing kernel (holocron_b200/csrc/erase.cu, ``hb_erase_batch``).

``erase`` takes a batch of images of one shape and, per image, either nothing or the ``(i, j, h, w, v)`` that
torchvision's ``RandomErasing.get_params`` drew for it. It writes one descriptor row per image and the fp32 fill values
into one pinned host buffer, uploads both with one asynchronous copy (no host synchronisation) and launches one kernel
that copies every image with its rectangle filled, or fills the rectangles in place."""
from typing import List, Optional, Sequence, Tuple

import numpy as np
from torch import Tensor

from .._lib import check, lib, require_cuda, stream_ptr
from ._table import DESC_WORDS, INT32_MAX, batch_out, check_batch, dtype_code, planes, upload

# (top, left, height, width, values): values broadcast to the rectangle's [C, h, w], as torchvision assigns them
Rect = Tuple[int, int, int, int, Tensor]
FILL_NONE, FILL_CHANNEL, FILL_PIXEL = 0, 1, 2


def _fill(v: Tensor, C: int, h: int, w: int) -> Tuple[int, Tensor]:
    """(fill code, flat fp32 values) of the values torchvision assigns to a [C, h, w] rectangle."""
    if v.dim() != 3:
        raise ValueError(f"erasing values of shape {tuple(v.shape)}: expected [C, h, w] or [C or 1, 1, 1]")
    if tuple(v.shape[1:]) == (1, 1) and v.shape[0] in (1, C):
        return FILL_CHANNEL, v.reshape(-1).expand(C).float()
    if tuple(v.shape) != (C, h, w):
        raise ValueError(f"erasing values of shape {tuple(v.shape)} do not fit a rectangle of {(C, h, w)}")
    return FILL_PIXEL, v.reshape(-1).float()


def erase_table(sources: Sequence[Tensor], rects: Sequence[Optional[Rect]], inplace: bool,
                out: Optional[Tensor]) -> Tuple[np.ndarray, List[Tensor], int, int]:
    """(table, values, rows, row_len): the int64 [N_total, 16] rows of hb_erase_batch, the fp32 value tensors in the
    order of their offsets, and the grid extent (the most row segments an image writes, the longest segment).
    Destinations are the sources themselves in place, else consecutive images of the contiguous ``out`` (whose dtype
    may differ from the sources': hb_image_tail_batch writes fp32)."""
    check_batch(sources, one_shape=True)
    ref = sources[0]
    C, H, W = ref.shape[-3:]
    if C * H * W > INT32_MAX:
        raise ValueError("images of more than 2**31 - 1 elements")
    rows: List[List[int]] = []
    values: List[Tensor] = []
    voff = 0
    most_rows = C * H if not inplace else 0
    row_len = W if not inplace else 0
    es = ref.element_size()
    for x, rect in zip(sources, rects):
        fill, (i, j, h, w), off = FILL_NONE, (0, 0, 0, 0), 0
        if rect is not None:
            i, j, h, w, v = rect
            if i < 0 or j < 0 or h <= 0 or w <= 0 or i + h > H or j + w > W:
                raise ValueError(f"erasing rectangle {(i, j, h, w)} is not inside the {H}x{W} image")
            fill, flat = _fill(v, C, h, w)
            values.append(flat)
            off = voff
            voff += flat.numel()
            if inplace:
                most_rows, row_len = max(most_rows, C * h), max(row_len, w)
        sc, sh, sw = x.stride()[-3:]
        if (W - 1) * abs(sw) > INT32_MAX:
            raise ValueError("image rows span more than 2**31 elements")
        # leading dimensions of a source are erased alike
        for o in planes(x):
            src = x.data_ptr() + o * es
            dst = src if inplace else out.data_ptr() + len(rows) * C * H * W * out.element_size()
            rows.append([src, dst, sc, sh, sw, C, H, W, i, j, h, w, fill, off, 0, 0])
    return np.array(rows, dtype=np.int64).reshape(-1, DESC_WORDS), values, most_rows, row_len


def erase(sources: Sequence[Tensor], rects: Sequence[Optional[Rect]], inplace: bool,
          out: Optional[Tensor] = None) -> Optional[Tensor]:
    """Erases rects[i] (None: nothing) of sources[i] ([..., C, H, W], CUDA, any strides, one shape). In place, writes
    the rectangles into the sources and returns None; otherwise returns ``out``, a contiguous (N_total, C, H, W) tensor
    of the erased images (leading dimensions of a source count as images)."""
    ref = sources[0]
    require_cuda(*sources)
    dtype = dtype_code(ref)
    if not inplace:
        out = batch_out(sources, out, ref.shape[-3:])
    table, values, rows, row_len = erase_table(sources, rects, inplace, out)
    _dev, (descs, vals) = upload(ref.device, table, values)
    check(lib().hb_erase_batch(descs, vals, table.shape[0], rows, row_len, dtype, stream_ptr()), "hb_erase_batch")
    return out
