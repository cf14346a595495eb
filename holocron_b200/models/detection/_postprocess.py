"""Host side of the batched YOLO post-processing kernels (holocron_b200/csrc/detect.cu, ``hb_detect``).

A *segment* is one set of decoded candidates for every image of a batch: boxes ``[B, M, 4]`` (xyxy, unclamped), objectness
``[B, M]`` and class scores ``[B, M, K]``, all fp32 probabilities, with its own score and NMS thresholds. YOLOv1/v2 have
one segment, YOLOv4 one per scale. :func:`detect_padded` runs select, order, suppress and emit for all images and
segments in one launch chain and returns padded outputs with per-image counts on the device; :func:`to_detections` turns
them into the reference's list of dicts with ONE device-to-host copy (the counts) per batch."""
import ctypes
from typing import Dict, List, Optional, Sequence, Tuple

import torch
from torch import Tensor

from ..._lib import check, lib, require_cuda, stream_ptr

__all__ = ["Segment", "detect_padded", "kernel_takes", "scratch_bytes", "to_detections"]

MAX_SEGMENTS = 4
MAX_CANDIDATES = 1 << 20      # per image and segment
_INT32_MAX = 2 ** 31 - 1

# (boxes [B, M, 4], objectness [B, M], class scores [B, M, K], box_score_thresh, rpn_nms_thresh)
Segment = Tuple[Tensor, Tensor, Tensor, float, float]
# dtypes that widen to fp32 exactly
_WIDENING = (torch.float32, torch.bfloat16, torch.float16)


def kernel_takes(boxes: Tensor, obj: Tensor, cls: Tensor) -> bool:
    """Whether the kernels compute exactly what the reference's loop computes on these decoded candidates: fp32 boxes
    (torchvision's nms then works in fp32, as the kernels do), and objectness and class scores that widen to fp32
    exactly and whose product the reference forms in fp32 (e.g. bf16 objectness with fp32 class scores, as a YOLOv1
    head gives under bf16 autocast). Other dtypes keep the reference's loop."""
    return (boxes.dtype == torch.float32 and obj.dtype in _WIDENING and cls.dtype in _WIDENING
            and torch.result_type(cls, obj) == torch.float32)


class _Seg(ctypes.Structure):
    """``hb_detect_seg`` of include/holocron_b200.h."""
    _fields_ = [("boxes", ctypes.c_void_p), ("obj", ctypes.c_void_p), ("cls", ctypes.c_void_p), ("M", ctypes.c_int),
                ("score_thresh", ctypes.c_float), ("iou_thresh", ctypes.c_float)]


def _table(segments: Sequence[Segment]) -> "ctypes.Array[_Seg]":
    table = (_Seg * len(segments))()
    for row, (boxes, obj, cls, score_thresh, iou_thresh) in zip(table, segments):
        row.boxes, row.obj, row.cls = boxes.data_ptr(), obj.data_ptr(), cls.data_ptr()
        row.M, row.score_thresh, row.iou_thresh = boxes.shape[1], float(score_thresh), float(iou_thresh)
    return table


def scratch_bytes(sizes: Sequence[int], batch: int, num_classes: int) -> int:
    """Device scratch of one hb_detect call for segments of ``sizes`` candidates per image (0 = refused table)."""
    table = (_Seg * len(sizes))()
    for row, m in zip(table, sizes):
        row.M = m
    return int(lib().hb_detect_scratch_bytes(table, len(sizes), batch, num_classes))


def _validate(segments: Sequence[Segment]) -> Tuple[int, int, torch.device]:
    """(B, K, device) of a segment list, or the error the launch would otherwise report as a CUDA error code."""
    if not 1 <= len(segments) <= MAX_SEGMENTS:
        raise ValueError(f"expected 1 to {MAX_SEGMENTS} segments, got {len(segments)}")
    ref = segments[0][0]
    if ref.ndim != 3 or ref.shape[-1] != 4:
        raise ValueError(f"boxes must have shape [B, M, 4], got {tuple(ref.shape)}")
    b = ref.shape[0]
    k = segments[0][2].shape[-1] if segments[0][2].ndim == 3 else -1
    cap = 0
    for boxes, obj, cls, _, _ in segments:
        for t in (boxes, obj, cls):
            if t.dtype != torch.float32:
                raise TypeError(f"YOLO post-processing kernels take float32 tensors, got {t.dtype}")
            if t.device != ref.device:
                raise ValueError("all candidate tensors of one call must be on the same device")
        m = boxes.shape[1] if boxes.ndim == 3 else -1
        if boxes.shape != (b, m, 4) or obj.shape != (b, m) or cls.shape != (b, m, k):
            raise ValueError(f"expected boxes [B, M, 4], objectness [B, M] and scores [B, M, K] with one B and K per "
                             f"call, got {tuple(boxes.shape)}, {tuple(obj.shape)} and {tuple(cls.shape)}")
        if m > MAX_CANDIDATES:
            raise ValueError(f"at most {MAX_CANDIDATES} candidates per image and segment, got {m}")
        cap += m
    if k < 1:
        raise ValueError("class scores need at least one class")
    if cap > _INT32_MAX or b * len(segments) > 65535:
        raise ValueError(f"batch too large for one call: {b} images x {cap} candidates")
    require_cuda(*(t for seg in segments for t in seg[:3]))
    return b, k, ref.device


def _aligned(boxes: Tensor) -> Tensor:
    """The kernels read a box as one 16-byte load."""
    return boxes if boxes.data_ptr() % 16 == 0 else boxes.clone()


def detect_padded(segments: Sequence[Segment]) -> Tuple[Tensor, Tensor, Tensor, Tensor]:
    """Post-processes every image of every segment on the device, without any host synchronisation.

    Returns ``boxes [B, cap, 4]`` (fp32, clamped to [0, 1]), ``scores [B, cap]`` (fp32), ``labels [B, cap]`` (int64) and
    ``counts [B]`` (int32) with ``cap = sum of M``: image b's detections are the first ``counts[b]`` rows, zeros after.
    Segments are suppressed independently and concatenated per image in segment order. Arguments are checked before
    anything is launched."""
    b, k, dev = _validate(segments)
    segments = [(_aligned(boxes.contiguous()), obj.contiguous(), cls.contiguous(), st, it)
                for boxes, obj, cls, st, it in segments]
    cap = sum(s[0].shape[1] for s in segments)
    boxes = torch.empty((b, cap, 4), dtype=torch.float32, device=dev)
    scores = torch.empty((b, cap), dtype=torch.float32, device=dev)
    labels = torch.empty((b, cap), dtype=torch.long, device=dev)
    counts = torch.empty((b,), dtype=torch.int32, device=dev)
    if b == 0:
        return boxes, scores, labels, counts
    table = _table(segments)
    nbytes = int(lib().hb_detect_scratch_bytes(table, len(segments), b, k))
    scratch = torch.empty((nbytes,), dtype=torch.uint8, device=dev)
    check(lib().hb_detect(table, len(segments), b, k, scratch.data_ptr(), boxes.data_ptr(), scores.data_ptr(),
                          labels.data_ptr(), counts.data_ptr(), stream_ptr()), "hb_detect")
    return boxes, scores, labels, counts


def to_detections(boxes: Tensor, scores: Tensor, labels: Tensor, counts: Tensor, no_candidate: Optional[Tensor] = None,
                  empty_dtype: Optional[torch.dtype] = None) -> List[Dict[str, Tensor]]:
    """The reference's per-image ``{"boxes", "scores", "labels"}`` dicts from padded outputs: one read-back of
    ``counts`` for the whole batch, then views of the first ``counts[b]`` rows of each image (the views share the
    batch's padded buffers). ``no_candidate`` (bool [B], read back in the same copy) marks the images the reference
    answers with empty boxes and scores of ``empty_dtype`` (YOLOv1/v2: objectness's dtype when no candidate passes
    objectness)."""
    if no_candidate is None:
        rows = [(n, False) for n in counts.tolist()]
    else:
        rows = list(zip(*torch.stack((counts, no_candidate.to(torch.int32))).tolist()))
    out = []
    for i, (n, empty) in enumerate(rows):
        if empty:
            out.append({"boxes": torch.zeros((0, 4), dtype=empty_dtype, device=boxes.device),
                        "scores": torch.zeros(0, dtype=empty_dtype, device=boxes.device), "labels": labels[i, :0]})
        else:
            out.append({"boxes": boxes[i, :n], "scores": scores[i, :n], "labels": labels[i, :n]})
    return out
