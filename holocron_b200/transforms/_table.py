"""Batch plumbing shared by the host sides of the transform kernels (``_resample``, ``_erase``, ``_autoaugment``,
``_color``): the checks on a batch of images, the images a source's leading dimensions hold, the contiguous output
batch, and the one asynchronous upload of a call's tables from pinned memory.

Every kernel takes one int64 descriptor row of ``DESC_WORDS`` words per image; the rows start with the same head
``[src, dst, sc, sh, sw, C, H, W]`` (addresses, strides in elements) and each module fills the tail its kernel reads."""
import math
from typing import List, Optional, Sequence, Tuple, Union

import numpy as np
import torch
from torch import Tensor

# the kernels' dtype codes: HB_DTYPE_* of holocron_b200/csrc/common.cuh
DTYPES = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2, torch.uint8: 3, torch.float64: 4}
INT32_MAX = 2 ** 31 - 1
DESC_WORDS = 16
# pixels one statistics CTA covers, and the most slices an (image, channel) is cut into
_SLICE_PIXELS = 4096
_MAX_SLICES = 64

Segment = Union[np.ndarray, Tensor, Sequence[Tensor]]


def dtype_code(x: Tensor) -> int:
    """The kernels' code of x's dtype, refusing the dtypes they do not take."""
    if x.dtype not in DTYPES:
        raise TypeError(f"unsupported dtype {x.dtype}: expected one of {', '.join(map(str, DTYPES))}")
    return DTYPES[x.dtype]


def check_images(items: Sequence[Tensor], dtypes: Sequence[torch.dtype]) -> int:
    """The channel count of a batch of images, refusing dtypes other than ``dtypes`` and what torchvision's colour ops
    refuse, with torchvision's messages."""
    ref = items[0]
    if ref.dtype not in dtypes:
        raise TypeError(f"Only {' and '.join(map(str, dtypes))} image tensors are supported, but found {ref.dtype}")
    if ref.ndim < 3:
        raise TypeError(f"Input image tensor should have at least 3 dimensions, but found {ref.ndim}")
    C = int(ref.shape[-3])
    if C not in (1, 3):
        raise TypeError(f"Input image tensor permitted channel values are [1, 3], but found {C}")
    return C


def check_batch(sources: Sequence[Tensor], one_shape: bool) -> None:
    """Refuses sources that do not match the first one: on dtype, device and channel count, and on the whole
    ``[C, H, W]`` when ``one_shape``."""
    dtype, device, shape = sources[0].dtype, sources[0].device, sources[0].shape[-3:]
    for x in sources:
        if (x.dtype != dtype or x.device != device or x.ndim < 3
                or (x.shape[-3:] != shape if one_shape else x.shape[-3] != shape[0])):
            raise ValueError("images of one call must share their shape, dtype and device" if one_shape else
                             "images of one call must share their dtype, device and channel count")


def planes(x: Tensor) -> List[int]:
    """The element offsets of the ``[C, H, W]`` images of x's leading dimensions, in index order: each is an image of
    its own."""
    offsets = [0]
    for n, s in zip(x.shape[:-3], x.stride()[:-3]):
        offsets = [o + k * s for o in offsets for k in range(n)]
    return offsets


def batch_out(sources: Sequence[Tensor], out: Optional[Tensor], shape: Tuple[int, int, int]) -> Tensor:
    """``out``, or a new tensor when it is None: one contiguous image of ``shape`` per image of the sources, in the
    sources' dtype and on their device."""
    ref = sources[0]
    full = (sum(math.prod(x.shape[:-3]) for x in sources), *shape)
    if out is None:
        return torch.empty(full, dtype=ref.dtype, device=ref.device)
    if out.shape != full or not out.is_contiguous() or out.dtype != ref.dtype or out.device != ref.device:
        raise ValueError(f"out must be a contiguous {ref.dtype} tensor of shape {full} on {ref.device}")
    return out


def upload(device: torch.device, *segments: Segment) -> Tuple[Tensor, List[int]]:
    """Packs the segments (numpy arrays, CPU tensors, or lists of CPU tensors laid end to end) into one pinned buffer,
    each segment starting 16-byte aligned, and copies it to ``device`` with one non-blocking copy on the current
    stream. Returns the device buffer and each segment's device address."""
    parts = [[p.numpy() if isinstance(p, Tensor) else p for p in (s if isinstance(s, (list, tuple)) else [s])]
             for s in segments]
    starts, total = [], 0
    for seg in parts:
        starts.append(total)
        total += -(-sum(p.nbytes for p in seg) // 16) * 16
    buf = torch.empty(total, dtype=torch.uint8, pin_memory=True)
    host = buf.numpy()
    for seg, at in zip(parts, starts):
        for p in seg:
            host[at:at + p.nbytes].view(p.dtype)[:] = p.reshape(-1)
            at += p.nbytes
    dev = buf.to(device, non_blocking=True)
    return dev, [dev.data_ptr() + at for at in starts]


def slices_for(H: int, W: int) -> int:
    """How many CTAs a statistics launch gives one (image, channel): enough that a large image is not one serial
    walk."""
    return max(1, min(_MAX_SLICES, -(-H * W // _SLICE_PIXELS)))
