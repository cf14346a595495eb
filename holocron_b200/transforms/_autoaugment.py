"""Host side of the batched TrivialAugmentWide kernels (holocron_b200/csrc/autoaugment.cu, ``hb_autoaugment_batch``).

``apply_ops`` takes a batch of uint8 images of one shape and, per image, the ``(op_name, magnitude)`` that
torchvision's ``TrivialAugmentWide`` drew for it, and computes what torchvision's ``autoaugment._apply_op`` computes for
each image on CUDA. It writes one descriptor row and 16 fp32 parameters per image, and the indices of the images whose
op needs a histogram (Contrast, AutoContrast, Equalize), into one pinned host buffer, uploads it with one asynchronous
copy (no host synchronisation) and makes one C call, which enqueues the histogram launch (only when such an image is
in the batch) and the apply launch."""
import math
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch
from torch import Tensor
from torchvision.transforms.functional import (InterpolationMode, _get_inverse_affine_matrix,
                                               _interpolation_modes_from_int)

from .._lib import check, lib, require_cuda, stream_ptr
from ._table import DESC_WORDS, INT32_MAX, batch_out, check_batch, check_images, planes, slices_for, upload

# op codes of the kernel: the order of torchvision's TrivialAugmentWide._augmentation_space
OPS = ("Identity", "ShearX", "ShearY", "TranslateX", "TranslateY", "Rotate", "Brightness", "Color", "Contrast",
       "Sharpness", "Posterize", "Solarize", "AutoContrast", "Equalize")
CODE = {name: i for i, name in enumerate(OPS)}
STAT_OPS = ("Contrast", "AutoContrast", "Equalize")
_BLEND_OPS = ("Brightness", "Color", "Contrast", "Sharpness")
_PARAM_WORDS = 16
R, Q, THRESHOLD, MATRIX, FILL = 0, 1, 2, 3, 9
SUPPORTED = (torch.uint8,)

Op = Tuple[str, float]


def check_options(interpolation, fill, C: int) -> Tuple[bool, Optional[List[float]]]:
    """(bilinear, fill as C fp values or None) from TrivialAugmentWide's ``interpolation`` and ``fill``."""
    if isinstance(interpolation, int):
        interpolation = _interpolation_modes_from_int(interpolation)
    if interpolation not in (InterpolationMode.NEAREST, InterpolationMode.BILINEAR):
        raise ValueError(f"Interpolation mode '{getattr(interpolation, 'value', interpolation)}' is unsupported with "
                         "Tensor input")
    if fill is None:
        return interpolation == InterpolationMode.BILINEAR, None
    values = [float(fill)] if isinstance(fill, (int, float)) else [float(f) for f in fill]
    if len(values) not in (1, C):
        raise ValueError(f"The number of elements in 'fill' cannot broadcast to match the number of channels of the "
                         f"image ({len(values)} != {C})")
    if any(not 0.0 <= v <= 255.0 for v in values):
        raise ValueError(f"fill values {values} are outside [0, 255], the range of a uint8 image")
    return interpolation == InterpolationMode.BILINEAR, values * (C // len(values))


def affine_matrix(op: str, magnitude: float, H: int, W: int) -> List[float]:
    """The inverse affine matrix torchvision's _apply_op has F.affine / F.rotate build for a geometric op, in
    double."""
    if op == "ShearX":  # center=[0, 0]: the top-left corner, relative to the image centre
        return _get_inverse_affine_matrix([-0.5 * W, -0.5 * H], 0.0, [0.0, 0.0], 1.0,
                                          [math.degrees(math.atan(magnitude)), 0.0])
    if op == "ShearY":
        return _get_inverse_affine_matrix([-0.5 * W, -0.5 * H], 0.0, [0.0, 0.0], 1.0,
                                          [0.0, math.degrees(math.atan(magnitude))])
    if op == "TranslateX":
        return _get_inverse_affine_matrix([0.0, 0.0], 0.0, [float(int(magnitude)), 0.0], 1.0, [0.0, 0.0])
    if op == "TranslateY":
        return _get_inverse_affine_matrix([0.0, 0.0], 0.0, [0.0, float(int(magnitude))], 1.0, [0.0, 0.0])
    return _get_inverse_affine_matrix([0.0, 0.0], -magnitude, [0.0, 0.0], 1.0, [0.0, 0.0])  # Rotate


def op_params(op: str, magnitude: float, H: int, W: int) -> Tuple[int, np.ndarray]:
    """(Posterize mask, the 16 fp32 parameters) of one op, raising what torchvision raises for it."""
    params = np.zeros(_PARAM_WORDS, dtype=np.float32)
    mask = 0xFF
    if op not in CODE:
        raise ValueError(f"The provided operator {op} is not recognized.")
    if op in _BLEND_OPS:
        ratio = 1.0 + magnitude  # in double, as torchvision forms the factor and _blend forms 1 - ratio
        params[R], params[Q] = ratio, 1.0 - ratio
    elif op == "Posterize":
        bits = int(magnitude)
        if not 0 <= bits <= 8:
            raise ValueError(f"The number if bits should be between 0 and 8. Got {bits}")
        mask = -int(2 ** (8 - bits)) & 0xFF
    elif op == "Solarize":
        params[THRESHOLD] = magnitude
    elif CODE[op] <= CODE["Rotate"] and op != "Identity":
        params[MATRIX:MATRIX + 6] = affine_matrix(op, magnitude, H, W)
    return mask, params


def op_table(sources: Sequence[Tensor], ops: Sequence[Op], bilinear: bool, fill: Optional[List[float]],
             out: Tensor) -> Tuple[np.ndarray, np.ndarray, List[int]]:
    """(table, params, stat_images): the int64 [N_total, 16] rows and fp32 [N_total, 16] parameters of
    hb_autoaugment_batch, and the images whose op needs a histogram. Leading dimensions of a source are images of their
    own, given that source's op; destinations are consecutive images of the contiguous ``out``."""
    check_batch(sources, one_shape=True)
    C, H, W = (int(s) for s in sources[0].shape[-3:])
    if C * H * W > INT32_MAX:
        raise ValueError("images of more than 2**31 - 1 elements")
    rows: List[List[int]] = []
    params: List[np.ndarray] = []
    stat_images: List[int] = []
    fill_flag = int(fill is not None)
    for x, (op, magnitude) in zip(sources, ops):
        mask, p = op_params(op, magnitude, H, W)
        if fill is not None:
            p[FILL:FILL + C] = fill
        sc, sh, sw = x.stride()[-3:]
        for o in planes(x):
            stat = -1
            if op in STAT_OPS:
                stat = len(stat_images)
                stat_images.append(len(rows))
            dst = out.data_ptr() + len(rows) * C * H * W
            rows.append([x.data_ptr() + o, dst, sc, sh, sw, C, H, W, CODE[op], stat, mask, fill_flag, int(bilinear),
                         0, 0, 0])
            params.append(p)
    return (np.array(rows, dtype=np.int64).reshape(-1, DESC_WORDS),
            np.stack(params).astype(np.float32).reshape(-1, _PARAM_WORDS), stat_images)


def apply_ops(sources: Sequence[Tensor], ops: Sequence[Op], interpolation, fill,
              out: Optional[Tensor] = None) -> Tensor:
    """Applies ops[i] = (op_name, magnitude) to sources[i] ([..., C, H, W] uint8 CUDA tensors of one shape, any
    strides) as torchvision's ``_apply_op`` does with this ``interpolation`` and ``fill``. Returns ``out``, a contiguous
    (N_total, C, H, W) tensor (leading dimensions of a source count as images)."""
    if len(sources) != len(ops):
        raise ValueError(f"{len(sources)} images and {len(ops)} ops")
    require_cuda(*sources)
    C = check_images(sources, SUPPORTED)
    bilinear, fill = check_options(interpolation, fill, C)
    ref = sources[0]
    out = batch_out(sources, out, ref.shape[-3:])
    table, params, stat_images = op_table(sources, ops, bilinear, fill, out)
    H, W = int(ref.shape[-2]), int(ref.shape[-1])
    slices = slices_for(H, W)
    scratch = torch.empty(max(1, 3 * len(stat_images) * slices * 256), dtype=torch.int32, device=ref.device)
    _dev, (descs, params_at, stats_at) = upload(ref.device, table, params, np.array(stat_images, dtype=np.int64))
    check(lib().hb_autoaugment_batch(descs, params_at, stats_at, scratch.data_ptr(), table.shape[0], len(stat_images),
                                     H, W, slices, stream_ptr()), "hb_autoaugment_batch")
    return out
