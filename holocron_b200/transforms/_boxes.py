"""Host side of the batched box-transform kernel (holocron_b200/csrc/boxes.cu, ``hb_box_transform_batch``).

``transform_boxes`` takes the boxes and labels of a batch of images, one op sequence for all of them and one fp32
parameter row per image, writes one descriptor row per image (pointers and strides: the boxes and labels are read in
place), uploads descriptors, parameters and ops in one asynchronous copy and launches one kernel for every box of the
batch. The survivors of each image are returned as views into one boxes buffer and one labels buffer."""
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch
from torch import Tensor

from .._lib import check, lib, stream_ptr
from ._table import upload

# the kernel's op codes (BoxOp of boxes.cu) and the operands each reads from the parameter row
SCALE, CLAMP, SUB, FILTER, FLIP, DIV = range(6)
OPERANDS = {SCALE: 2, CLAMP: 4, SUB: 2, FILTER: 0, FLIP: 2, DIV: 2}
DESC_WORDS = 8


def check_target(boxes, labels, device: torch.device) -> int:
    """The box count of one target, refusing what the kernel does not read: boxes must be an fp32 (n, 4) tensor with
    unit column stride and labels an int64 (n,) tensor, both on ``device``."""
    if not isinstance(boxes, Tensor) or not isinstance(labels, Tensor):
        raise TypeError("expected target['boxes'] and target['labels'] to be torch.Tensor")
    if boxes.dtype != torch.float32 or boxes.ndim != 2 or boxes.shape[1] != 4 or boxes.stride(1) != 1:
        raise TypeError(f"target['boxes'] must be a float32 (n, 4) tensor with unit column stride, got {boxes.dtype} "
                        f"{tuple(boxes.shape)} strides {boxes.stride()}")
    if labels.dtype != torch.int64 or labels.ndim != 1:
        raise TypeError(f"target['labels'] must be an int64 (n,) tensor, got {labels.dtype} {tuple(labels.shape)}")
    if labels.shape[0] != boxes.shape[0]:
        raise ValueError(f"{boxes.shape[0]} boxes but {labels.shape[0]} labels")
    if boxes.device != device or labels.device != device:
        raise ValueError(f"targets must be on the images' device {device}")
    return int(boxes.shape[0])


def transform_boxes(boxes: Sequence[Tensor], labels: Sequence[Tensor], ops: Sequence[int], params: np.ndarray,
                    out_boxes: Optional[Tensor] = None, out_labels: Optional[Tensor] = None
                    ) -> Tuple[List[Tensor], List[Tensor]]:
    """Applies ``ops`` to the boxes of each image with that image's row of ``params`` (fp32 [N, n_params]), in one
    launch. Image k's survivors go to rows [offset_k, offset_k + count_k) of the boxes (fp32 [total, 4]) and labels
    (int64 [total]) buffers, offset_k being its first box's index in the batch; ``out_boxes`` / ``out_labels`` give
    those buffers (contiguous, at least ``total`` rows). When ``ops`` drop boxes, the counts are read back with one
    device-to-host copy; otherwise nothing is synchronised. Returns the (count_k, 4) and (count_k,) views."""
    device = boxes[0].device
    ns = [int(b.shape[0]) for b in boxes]
    offsets = np.concatenate([[0], np.cumsum(ns)[:-1]]).astype(np.int64) if ns else np.zeros(0, np.int64)
    total = sum(ns)
    if out_boxes is None:
        out_boxes = torch.empty(total, 4, dtype=torch.float32, device=device)
    if out_labels is None:
        out_labels = torch.empty(total, dtype=torch.int64, device=device)
    if (out_boxes.dtype != torch.float32 or out_boxes.ndim != 2 or out_boxes.shape[0] < total
            or out_boxes.shape[1] != 4 or not out_boxes.is_contiguous() or out_labels.dtype != torch.int64
            or out_labels.ndim != 1 or out_labels.shape[0] < total or not out_labels.is_contiguous()):
        raise ValueError(f"out_boxes / out_labels must be contiguous float32 (>= {total}, 4) / int64 (>= {total},)")
    n_params = sum(OPERANDS[o] for o in ops)
    params = np.ascontiguousarray(params, dtype=np.float32).reshape(len(boxes), n_params)
    table = np.zeros((len(boxes), DESC_WORDS), dtype=np.int64)
    for k, (b, lab) in enumerate(zip(boxes, labels)):
        table[k, :6] = [b.data_ptr(), lab.data_ptr(), b.stride(0), lab.stride(0), ns[k], offsets[k]]
    counts = torch.empty(len(boxes), dtype=torch.int32, device=device)
    _dev, (descs, prm, opp) = upload(device, table, params, np.asarray(ops, dtype=np.int32))
    check(lib().hb_box_transform_batch(descs, prm, opp, len(ops), n_params, len(boxes), out_boxes.data_ptr(),
                                       out_labels.data_ptr(), counts.data_ptr(), stream_ptr()),
          "hb_box_transform_batch")
    kept = counts.tolist() if FILTER in ops else ns
    return ([out_boxes[o:o + c] for o, c in zip(offsets.tolist(), kept)],
            [out_labels[o:o + c] for o, c in zip(offsets.tolist(), kept)])
