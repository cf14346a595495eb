"""Host side of the batched ColorJitter kernels (holocron_b200/csrc/color_jitter.cu, ``hb_color_jitter_batch``).

``jitter`` takes a batch of uint8 or fp32 images of one shape and, per image, what torchvision's
``ColorJitter.get_params`` drew for it (``fn_idx`` and the four factors, ``None`` for an op that is off), and computes
what torchvision's ``ColorJitter.forward`` computes for each image on CUDA. It writes one descriptor row and 8 fp32
parameters per image, and the indices of the images with a contrast factor, into one pinned host buffer, uploads it
with one asynchronous copy (no host synchronisation) and makes one C call, which enqueues the statistics launch (only
when an image has a contrast factor) and the apply launch."""
import math
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch
from torch import Tensor

from .._lib import check, lib, require_cuda, stream_ptr
from ._table import DESC_WORDS, DTYPES, INT32_MAX, batch_out, check_batch, check_images, planes, slices_for, upload

# op codes of the kernel: torchvision's fn_idx values
OPS = ("brightness", "contrast", "saturation", "hue")
CONTRAST, HUE = 1, 3
MEAN = 7  # the parameter slot of the contrast mean's factor
SUPPORTED = (torch.uint8, torch.float32)
_PARAM_WORDS = 8

# (fn_idx, brightness, contrast, saturation, hue), as ColorJitter.get_params returns it
Draw = Tuple[Sequence[int], Optional[float], Optional[float], Optional[float], Optional[float]]


def chain(draw: Draw) -> Tuple[List[int], int, np.ndarray]:
    """(op codes in drawn order with the ``None`` ops dropped, the index of contrast among them or -1, the 8 fp32
    parameters but the mean factor) of one image's draw. A blend's ``1 - r`` is formed in double and then rounded, as
    torchvision's ``_blend`` forms it."""
    fn_idx, *factors = draw
    ops = [int(k) for k in fn_idx if factors[int(k)] is not None]
    params = np.zeros(_PARAM_WORDS, dtype=np.float32)
    for k in range(HUE):
        if factors[k] is not None:
            r = float(factors[k])
            params[2 * k], params[2 * k + 1] = r, 1.0 - r
    if factors[HUE] is not None:
        params[2 * HUE] = float(factors[HUE])
    return ops, (ops.index(CONTRAST) if CONTRAST in ops else -1), params


def mean_factor(images: int, H: int, W: int) -> np.float32:
    """The factor torch's CUDA mean multiplies its fp32 sum by, for the grayscale of a tensor holding ``images``
    images of H x W: the fp32 quotient of the output count by the input count."""
    return np.float32(images) / np.float32(images * H * W)


def jitter_table(sources: Sequence[Tensor], draws: Sequence[Draw],
                 out: Tensor) -> Tuple[np.ndarray, np.ndarray, List[int]]:
    """(table, params, stat_images): the int64 [N_total, 16] rows and fp32 [N_total, 8] parameters of
    hb_color_jitter_batch, and the images with a contrast op. Leading dimensions of a source are images of their own,
    given that source's draw; destinations are consecutive images of the contiguous ``out``."""
    check_batch(sources, one_shape=True)
    C, H, W = (int(s) for s in sources[0].shape[-3:])
    if C * H * W > INT32_MAX:
        raise ValueError("images of more than 2**31 - 1 elements")
    item = sources[0].element_size()
    rows: List[List[int]] = []
    params: List[np.ndarray] = []
    stat_images: List[int] = []
    for x, draw in zip(sources, draws):
        ops, at, p = chain(draw)
        p[MEAN] = mean_factor(math.prod(x.shape[:-3]), H, W)
        codes = ops + [-1] * (4 - len(ops))
        sc, sh, sw = x.stride()[-3:]
        for o in planes(x):
            stat = -1
            if at >= 0:
                stat = len(stat_images)
                stat_images.append(len(rows))
            dst = out.data_ptr() + len(rows) * C * H * W * item
            rows.append([x.data_ptr() + o * item, dst, sc, sh, sw, C, H, W, len(ops), *codes, at, stat, 0])
            params.append(p)
    return (np.array(rows, dtype=np.int64).reshape(-1, DESC_WORDS),
            np.stack(params).astype(np.float32).reshape(-1, _PARAM_WORDS), stat_images)


def jitter(sources: Sequence[Tensor], draws: Sequence[Draw], out: Optional[Tensor] = None) -> Tensor:
    """Applies draws[i] (what ``ColorJitter.get_params`` returned) to sources[i] ([..., C, H, W] uint8 or fp32 CUDA
    tensors of one shape, any strides) as torchvision's ``ColorJitter.forward`` does. Returns ``out``, a contiguous
    (N_total, C, H, W) tensor (leading dimensions of a source count as images)."""
    if len(sources) != len(draws):
        raise ValueError(f"{len(sources)} images and {len(draws)} draws")
    require_cuda(*sources)
    check_images(sources, SUPPORTED)
    ref = sources[0]
    out = batch_out(sources, out, ref.shape[-3:])
    table, params, stat_images = jitter_table(sources, draws, out)
    H, W = int(ref.shape[-2]), int(ref.shape[-1])
    slices = slices_for(H, W)
    # one int64 (uint8 images) or fp64 (fp32 images) partial sum per (image with contrast, slice)
    scratch = torch.empty(max(1, len(stat_images) * slices), dtype=torch.int64, device=ref.device)
    _dev, (descs, params_at, stats_at) = upload(ref.device, table, params, np.array(stat_images, dtype=np.int64))
    check(lib().hb_color_jitter_batch(descs, params_at, stats_at, scratch.data_ptr(), table.shape[0], len(stat_images),
                                      H, W, slices, DTYPES[ref.dtype], stream_ptr()), "hb_color_jitter_batch")
    return out
