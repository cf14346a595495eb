"""The reference's YOLO post-processing, restated as it is today (holocron/models/detection/yolo.py:159-233 and
yolov4.py:303-335): a Python loop over images with boolean-mask gathers and torchvision's ``nms``."""
from fractions import Fraction

import numpy as np
import torch
from torchvision.ops.boxes import nms


def _ref_v12(pred_xyxy, b_o, b_scores, rpn_nms_thresh, box_score_thresh):
    """yolo.py:159-233 after to_isoboxes(..., clamp=True)."""
    detections = []
    for idx in range(b_o.shape[0]):
        coords = torch.zeros((0, 4), dtype=b_o.dtype, device=b_o.device)
        scores = torch.zeros(0, dtype=b_o.dtype, device=b_o.device)
        labels = torch.zeros(0, dtype=torch.long, device=b_o.device)
        obj_mask = b_o[idx] >= 0.5
        if torch.any(obj_mask):
            coords = pred_xyxy[idx, obj_mask]
            scores, labels = b_scores[idx, obj_mask].max(dim=-1)
            scores = scores * b_o[idx, obj_mask]
            keep = scores >= box_score_thresh
            coords, labels, scores = coords[keep], labels[keep], scores[keep]
            kept_idxs = nms(coords, scores, iou_threshold=rpn_nms_thresh)
            coords, scores, labels = coords[kept_idxs], scores[kept_idxs], labels[kept_idxs]
        detections.append({"boxes": coords, "scores": scores, "labels": labels})
    return detections


def _ref_v4(boxes, b_o, b_scores, rpn_nms_thresh, box_score_thresh):
    """yolov4.py:303-335."""
    b_o = torch.sigmoid(b_o)
    b_scores = torch.sigmoid(b_scores)
    boxes = boxes.clamp(0, 1)
    detections = []
    for idx in range(b_o.shape[0]):
        keep = b_o[idx] >= 0.5
        coords = boxes[idx][keep]
        if coords.shape[0] > 0:
            scores, labels = b_scores[idx][keep].max(dim=-1)
            scores = scores * b_o[idx][keep]
            sel = scores >= box_score_thresh
            coords, labels, scores = coords[sel].clamp(0, 1), labels[sel], scores[sel]
            kept = nms(coords, scores, iou_threshold=rpn_nms_thresh)
            coords, scores, labels = coords[kept], scores[kept], labels[kept]
        else:
            scores = torch.zeros(0, dtype=torch.float32, device=b_o.device)
            labels = torch.zeros(0, dtype=torch.long, device=b_o.device)
        detections.append({"boxes": coords, "scores": scores, "labels": labels})
    return detections


def _round_f32(x: Fraction) -> np.float32:
    """x rounded to the nearest fp32, ties to even."""
    r = np.float32(float(x))
    cands = [np.nextafter(r, np.float32(-np.inf)), r, np.nextafter(r, np.float32(np.inf))]
    return min(cands, key=lambda c: (abs(Fraction(float(c)) - x), int(np.float32(c).view(np.uint32)) & 1))


def iou_f32(a, b, fused: bool) -> np.float32:
    """fp32 IoU of box a (the higher-scored one) with box b, in torchvision's order of operations. fused: the area of b
    is added to the area of a in one fused multiply-add (how ptxas compiles torchvision's sm_90 nms kernel); otherwise
    every operation rounds on its own."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    area_a = (a[2] - a[0]) * (a[3] - a[1])
    wb, hb = b[2] - b[0], b[3] - b[1]
    if fused:
        total = _round_f32(Fraction(float(wb)) * Fraction(float(hb)) + Fraction(float(area_a)))
    else:
        total = np.float32(wb * hb) + area_a
    w = max(min(a[2], b[2]) - max(a[0], b[0]), np.float32(0))
    h = max(min(a[3], b[3]) - max(a[1], b[1]), np.float32(0))
    inter = np.float32(w * h)
    return np.float32(inter / np.float32(total - inter))


def fma_sensitive_pair(seed: int = 0):
    """(a, b, thr): two fp32 boxes in [0, 1] whose IoU rounds differently with and without the fused area sum, and a
    threshold between the two results, so that ``IoU > thr`` is True in exactly one of the two arithmetics."""
    rng = np.random.default_rng(seed)
    while True:
        a = np.sort(rng.random((2, 2), dtype=np.float32) * np.float32(0.6), axis=0).T.reshape(-1)[[0, 2, 1, 3]]
        b = a + (rng.random(4, dtype=np.float32) - np.float32(0.5)) * np.float32(0.1)
        if not (b[2] > b[0] and b[3] > b[1] and b.min() >= 0 and b.max() <= 1):   # the kernels clamp to [0, 1]
            continue
        f, u = iou_f32(a, b, True), iou_f32(a, b, False)
        if f != u and 0 < min(f, u):
            return a, b, float(min(f, u))
