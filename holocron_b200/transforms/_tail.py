"""Host side of the batched classification tail kernel (holocron_b200/csrc/image_tail.cu, ``hb_image_tail_batch``).

A tail is a run of torchvision's ``PILToTensor``, ``ConvertImageDtype``, ``Normalize`` and ``RandomErasing``.
``program`` turns its steps into the kernel's op program for images of a given dtype, refusing what the steps refuse
before anything is drawn. ``tail`` writes hb_erase_batch's copy-mode rows (``_erase.erase_table``) and the fp32 fill
values, mean and std into one pinned host buffer, uploads it with one asynchronous copy (no host synchronisation) and
launches one kernel that writes the finished fp32 batch."""
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch
from torch import Tensor
from torchvision.transforms import transforms as T

from .._lib import check, lib, require_cuda, stream_ptr
from ._erase import Rect, erase_table
from ._table import DTYPES, upload

# op codes of the kernel
CONVERT, NORMALIZE, ERASE_U8, ERASE_F32 = 1, 2, 3, 4
SOURCES = (torch.uint8, torch.float32)


def program(steps: Sequence[object], dtype: torch.dtype) -> Tuple[List[int], torch.dtype]:
    """(op codes, the dtype the steps leave) of a tail's steps applied to images of ``dtype``."""
    if dtype.is_floating_point and dtype != torch.float32:
        raise NotImplementedError(f"{dtype} images: PILToTensor, ConvertImageDtype, Normalize and RandomErasing take "
                                  "uint8 or float32 images here")
    if dtype not in SOURCES:
        raise TypeError(f"PILToTensor, ConvertImageDtype, Normalize and RandomErasing take uint8 or float32 images "
                        f"here, got {dtype}")
    ops: List[int] = []
    for t in steps:
        if isinstance(t, T.PILToTensor):
            if dtype != torch.uint8:
                raise TypeError(f"PILToTensor takes uint8 images here, got {dtype}")
        elif isinstance(t, T.ConvertImageDtype):
            if t.dtype != torch.float32:
                raise NotImplementedError(f"ConvertImageDtype to {t.dtype}: only torch.float32 is supported")
            if dtype == torch.uint8:  # float32 to float32: torchvision returns the image itself
                ops.append(CONVERT)
                dtype = torch.float32
        elif isinstance(t, T.Normalize):
            if not dtype.is_floating_point:
                raise TypeError(f"Input tensor should be a float tensor. Got {dtype}.")
            ops.append(NORMALIZE)
        else:
            ops.append(ERASE_U8 if dtype == torch.uint8 else ERASE_F32)
    return ops, dtype


def norm_values(mean, std, C: int) -> np.ndarray:
    """fp32 [2 * C]: the mean then the std of each channel, as torchvision's ``normalize`` rounds them to fp32; raises
    its ValueError for a zero std, and ValueError for a length other than 1 or C."""
    m = torch.as_tensor(mean, dtype=torch.float32, device="cpu").reshape(-1)
    s = torch.as_tensor(std, dtype=torch.float32, device="cpu").reshape(-1)
    if (s == 0).any():
        raise ValueError(f"std evaluated to zero after conversion to {torch.float32}, leading to division by zero.")
    for name, v in (("mean", m), ("std", s)):
        if v.numel() not in (1, C):
            raise ValueError(f"{name} has {v.numel()} values: expected 1 or {C} (the image's channels)")
    return torch.cat([m.expand(C), s.expand(C)]).numpy()


def tail(sources: Sequence[Tensor], ops: Sequence[int], rects: Optional[Sequence[Optional[Rect]]] = None,
         norm: Optional[np.ndarray] = None) -> Tensor:
    """Runs the op program ``ops`` on sources[i] ([..., C, H, W] uint8 or fp32 CUDA tensors of one shape, any strides),
    erasing rects[i] (None: nothing) where the program erases and normalising with ``norm`` (``norm_values``). Returns
    a contiguous fp32 (N_total, C, H, W) tensor (leading dimensions of a source count as images)."""
    ref = sources[0]
    require_cuda(*sources)
    if ref.dtype not in SOURCES:
        raise TypeError(f"unsupported dtype {ref.dtype}: expected uint8 or float32")
    if len(ops) > 3:
        raise ValueError(f"a tail runs at most 3 ops, got {len(ops)}")
    n = sum(int(np.prod(x.shape[:-3])) for x in sources)
    out = torch.empty((n, *ref.shape[-3:]), dtype=torch.float32, device=ref.device)
    table, values, rows, row_len = erase_table(sources, rects if rects is not None else [None] * len(sources), False,
                                               out)
    noff = sum(v.numel() for v in values)
    if norm is not None:
        values.append(torch.from_numpy(norm))
    word = sum(op << (8 * i) for i, op in enumerate(ops))
    _dev, (descs, vals) = upload(ref.device, table, values)
    check(lib().hb_image_tail_batch(descs, vals, table.shape[0], rows, row_len, DTYPES[ref.dtype], word, noff,
                                    stream_ptr()), "hb_image_tail_batch")
    return out
