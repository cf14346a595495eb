"""YOLOv1 on the fused kernels — API mirror of holocron/models/detection/yolo.py (_YOLO :28-233 with the losses :48-132,
YOLOv1 :236-380, yolov1 :411-478).

Module tree / ``state_dict`` / init order are the reference's (``backbone`` = ``DarknetBodyV1``, ``block4``, ``classifier``).
The conv-BN-LeakyReLU units run through :mod:`holocron_b200.models._blocks`; the two ``Linear`` layers of the classifier are
library GEMMs.

**Losses** (shared with YOLOv2). The reference walks the ground-truth boxes in a Python double loop, reading the predictions
of each box's cell one by one (4-5 tiny kernels and an index computation on the host per box). Here every ground-truth box
is one row of static-shape tensors: image index, cell, the IoUs of the box with the ``A`` predictions of its cell (ONE
launch of the pairwise IoU kernel of :mod:`holocron_b200.ops.boxes`, analytic backward), the best anchor, and from those the
four sums - no loop over boxes, no host synchronisation besides the reference's own input validation. Reference behaviour
kept on purpose:
  * the objectness target (the IoU) stays attached to the graph (yolo.py:103);
  * the width/height term subtracts the prediction from the square roots of ALL boxes of the image, not only the assigned one
    (``gt_wh.sqrt()`` is not indexed by the box at yolo.py:109): each box adds ``sum_g' |sqrt(wh_g') - sqrt(pred_wh)|^2``;
  * the classification term compares the one-hot label with the class scores of every anchor row of the cell
    (yolo.py:99-101; one row for YOLOv1, ``A`` rows for YOLOv2);
  * a (cell, anchor) slot claimed by several boxes is removed from the no-object term once, its other terms are counted once
    per box."""
from typing import Any, Callable, Dict, List, Optional, Tuple, Union

import torch
import torch.nn.functional as F
from torch import Tensor, nn
from torchvision.ops.boxes import nms

from ...nn.init import init_module
from ...ops.boxes import box_iou
from .._blocks import FusedSequential
from ..classification.darknet import DarknetBodyV1
from ..utils import conv_sequence
from ._postprocess import Segment, detect_padded, kernel_takes, to_detections

__all__ = ["YOLOv1", "yolov1"]


class _YOLO(nn.Module):
    """Loss, box conversion and post-processing shared by YOLOv1 / YOLOv2 (reference yolo.py:28-233)."""

    def __init__(self, num_classes: int = 20, rpn_nms_thresh: float = 0.7, box_score_thresh: float = 0.05,
                 lambda_obj: float = 1, lambda_noobj: float = 0.5, lambda_class: float = 1, lambda_coords: float = 5) -> None:
        super().__init__()
        self.num_classes = num_classes
        self.rpn_nms_thresh = rpn_nms_thresh
        self.box_score_thresh = box_score_thresh
        self.lambda_obj = lambda_obj
        self.lambda_noobj = lambda_noobj
        self.lambda_class = lambda_class
        self.lambda_coords = lambda_coords

    def _compute_losses(self, pred_boxes: Tensor, pred_o: Tensor, pred_scores: Tensor, target: List[Dict[str, Tensor]],
                        ignore_high_iou: bool = False) -> Dict[str, Tensor]:
        """pred_boxes (N, H, W, A, 4) relative (xc, yc, w, h); pred_o (N, H, W, A); pred_scores (N, H, W, A or 1, K)."""
        gt_boxes = [t["boxes"] for t in target]
        gt_labels = [t["labels"] for t in target]
        dev = pred_boxes.device
        capturing = dev.type == "cuda" and torch.cuda.is_current_stream_capturing()
        if not capturing and not all(torch.all(boxes >= 0) and torch.all(boxes <= 1) for boxes in gt_boxes):
            raise ValueError("Ground truth boxes are expected to have values between 0 and 1.")
        b, h, w, _, _ = pred_scores.shape
        na = pred_o.shape[3]
        pred_boxes, pred_o, pred_scores = pred_boxes.float(), pred_o.float(), pred_scores.float()
        pred_xyxy = self.to_isoboxes(pred_boxes, (h, w), clamp=False)
        pred_xy = (pred_xyxy[..., [0, 1]] + pred_xyxy[..., [2, 3]]) / 2
        n = pred_boxes.shape[0]
        is_noobj = torch.ones_like(pred_o)
        counts = tuple(int(bx.shape[0]) for bx in gt_boxes)
        num_gt = sum(counts)
        zero = pred_o.sum() * 0
        if num_gt == 0:
            obj = bbox = clf = zero
        else:
            cache = self.__dict__.setdefault("_img_index_cache", {})
            key = (counts, str(dev))
            if key not in cache:       # built once per box-count pattern (host -> device copy: not inside a graph capture)
                img_ = torch.repeat_interleave(torch.arange(b), torch.tensor(counts))
                cache[key] = (img_.to(dev), torch.arange(num_gt).to(dev))
            img, ar = cache[key]
            boxes = torch.cat(gt_boxes, dim=0).float()
            labels = torch.cat(gt_labels, dim=0)
            gt_xy = (boxes[:, :2] + boxes[:, 2:]) / 2
            gt_wh = boxes[:, 2:] - boxes[:, :2]
            cx = (boxes[:, [0, 2]].mean(dim=-1) * w).to(dtype=torch.long)
            cy = (boxes[:, [1, 3]].mean(dim=-1) * h).to(dtype=torch.long)
            cell_xyxy = pred_xyxy[img, cy, cx]                                       # [G, A, 4]
            # IoU of every box with the A predictions of ITS cell: the diagonal blocks of one (G*A) x G pairwise launch
            # (predictions first: the argument order whose data gradient YOLOv4's losses exercise as well)
            iou_cell = box_iou(cell_xyxy.reshape(-1, 4), boxes).view(num_gt, na, num_gt)[ar, :, ar]
            iou, anchor = iou_cell.max(dim=1)
            is_noobj = is_noobj.index_put((img, cy, cx, anchor), is_noobj.new_zeros(()))   # device-side value: graph-capturable
            onehot = F.one_hot(labels, self.num_classes).to(pred_scores.dtype)
            clf = (onehot[:, None, :] - pred_scores[img, cy, cx]).pow(2).sum()
            obj = (iou - pred_o[img, cy, cx, anchor]).pow(2).sum()
            bbox = (gt_xy - pred_xy[img, cy, cx, anchor]).pow(2).sum()
            same = (img[:, None] == img[None, :]).to(pred_boxes.dtype)               # [G(box), G(all boxes of its image)]
            d_wh = gt_wh.sqrt()[None, :, :] - pred_boxes[img, cy, cx, anchor, 2:].sqrt()[:, None, :]
            bbox = bbox + (d_wh.pow(2).sum(-1) * same).sum()
            if ignore_high_iou:
                for idx in range(b):
                    if counts[idx]:
                        iou_ = box_iou(pred_xyxy[idx].reshape(-1, 4), gt_boxes[idx].float()).max(dim=-1).values
                        is_noobj[idx] = is_noobj[idx] * (iou_.reshape(h, w, -1) < 0.5).to(is_noobj.dtype)
        noobj = (pred_o.pow(2) * is_noobj.detach()).sum()
        return {
            "obj_loss": (self.lambda_obj * obj / n).reshape(1),
            "noobj_loss": (self.lambda_noobj * noobj / n).reshape(1),
            "bbox_loss": (self.lambda_coords * bbox / n).reshape(1),
            "clf_loss": (self.lambda_class * clf / n).reshape(1),
        }

    @staticmethod
    def to_isoboxes(b_coords: Tensor, grid_shape: Tuple[int, int], clamp: bool = False) -> Tensor:
        """(..., H, W, A, 4) cell-relative (xc, yc) + image-relative (w, h) -> relative xyxy (reference yolo.py:134-158)."""
        c_x = torch.arange(grid_shape[1], dtype=torch.float, device=b_coords.device)
        c_y = torch.arange(grid_shape[0], dtype=torch.float, device=b_coords.device)
        b_x = (b_coords[..., 0] + c_x.reshape(1, 1, -1, 1)) / grid_shape[1]
        b_y = (b_coords[..., 1] + c_y.reshape(1, -1, 1, 1)) / grid_shape[0]
        xy = torch.stack((b_x, b_y), dim=-1)
        wh = b_coords[..., 2:]
        pred_xyxy = torch.cat((xy - wh / 2, xy + wh / 2), dim=-1).reshape(*b_coords.shape)
        if clamp:
            pred_xyxy = pred_xyxy.clamp(0, 1)
        return pred_xyxy

    def post_process(self, b_coords: Tensor, b_o: Tensor, b_scores: Tensor, grid_shape: Tuple[int, int],
                     rpn_nms_thresh: float = 0.7, box_score_thresh: float = 0.05) -> List[Dict[str, Tensor]]:
        """Objectness >= 0.5, class confidence x objectness >= ``box_score_thresh``, NMS (reference yolo.py:160-233).
        CUDA inputs go through the batched kernels of ``csrc/detect.cu`` when they reproduce the loop exactly (see
        :func:`~._postprocess.kernel_takes`): one launch chain for the batch and one device-to-host copy. Other inputs
        take the reference's per-image loop."""
        if b_o.is_cuda:
            seg = self._segment(b_coords, b_o, b_scores, grid_shape, rpn_nms_thresh, box_score_thresh)
            if kernel_takes(seg[0], b_o, b_scores):
                padded = detect_padded([seg])
                if b_o.dtype == torch.float32:
                    return to_detections(*padded)
                # an image without any candidate past objectness gets empty tensors of b_o's dtype in the reference
                return to_detections(*padded, no_candidate=~(b_o >= 0.5).any(dim=1), empty_dtype=b_o.dtype)
        pred_xyxy = self.to_isoboxes(b_coords.reshape(-1, *grid_shape, self.num_anchors, 4), grid_shape,
                                     clamp=True).reshape(b_o.shape[0], -1, 4)
        detections = []
        for idx in range(b_coords.shape[0]):
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

    def _segment(self, b_coords: Tensor, b_o: Tensor, b_scores: Tensor, grid_shape: Tuple[int, int],
                 rpn_nms_thresh: float, box_score_thresh: float) -> Segment:
        """post_process's inputs as one kernel segment: unclamped xyxy boxes [B, M, 4] (the kernel clamps them),
        objectness and class scores widened to fp32 (exact; the reference forms their product in fp32)."""
        pred_xyxy = self.to_isoboxes(b_coords.reshape(-1, *grid_shape, self.num_anchors, 4), grid_shape,
                                     clamp=False).reshape(b_o.shape[0], -1, 4)
        return pred_xyxy, b_o.float(), b_scores.float(), box_score_thresh, rpn_nms_thresh

    def detect_padded(self, x: Tensor) -> Tuple[Tensor, Tensor, Tensor, Tensor]:
        """The detections of the eval forward as padded device tensors, with no host synchronisation at all (an eval
        forward that can be captured in a CUDA graph): ``boxes [B, cap, 4]``, ``scores [B, cap]``, ``labels [B, cap]``
        (int64) and ``counts [B]`` (int32), cap = H * W * num_anchors. Image b's detections are the first
        ``counts[b]`` rows, equal to ``forward(x)[b]`` in the model's current mode (call it in eval mode)."""
        if isinstance(x, (list, tuple)):
            x = torch.stack(x, dim=0)
        b_coords, b_o, b_scores = self._format_outputs(self._forward(x))
        n, grid = b_coords.shape[0], (b_coords.shape[1], b_coords.shape[2])
        b_scores = b_scores.expand(*b_o.shape, self.num_classes).reshape(n, -1, self.num_classes)
        return detect_padded([self._segment(b_coords.reshape(n, -1, 4), b_o.reshape(n, -1), b_scores, grid,
                                            self.rpn_nms_thresh, self.box_score_thresh)])


class YOLOv1(_YOLO):
    """reference yolo.py:236-380, same constructor."""

    def __init__(self, layout: List[List[int]], num_classes: int = 20, in_channels: int = 3, stem_channels: int = 64,
                 num_anchors: int = 2, lambda_obj: float = 1, lambda_noobj: float = 0.5, lambda_class: float = 1,
                 lambda_coords: float = 5.0, rpn_nms_thresh: float = 0.7, box_score_thresh: float = 0.05,
                 head_hidden_nodes: int = 512, act_layer: Optional[nn.Module] = None,
                 norm_layer: Optional[Callable[[int], nn.Module]] = None,
                 drop_layer: Optional[Callable[..., nn.Module]] = None,
                 conv_layer: Optional[Callable[..., nn.Module]] = None,
                 backbone_norm_layer: Optional[Callable[[int], nn.Module]] = None) -> None:
        super().__init__(num_classes, rpn_nms_thresh, box_score_thresh, lambda_obj, lambda_noobj, lambda_class, lambda_coords)
        if act_layer is None:
            act_layer = nn.LeakyReLU(0.1, inplace=True)
        if backbone_norm_layer is None and norm_layer is not None:
            backbone_norm_layer = norm_layer
        self.backbone = DarknetBodyV1(layout, in_channels, stem_channels, act_layer, backbone_norm_layer)
        units = [dict(), dict(stride=2), dict(), dict()]
        self.block4 = FusedSequential(*[m for kw in units for m in conv_sequence(
            1024, 1024, act_layer, norm_layer, drop_layer, conv_layer, kernel_size=3, padding=1, bias=(norm_layer is None), **kw)])
        self.classifier = nn.Sequential(
            nn.Flatten(),
            nn.Linear(1024 * 7**2, head_hidden_nodes),
            act_layer,
            nn.Dropout(0.5),
            nn.Linear(head_hidden_nodes, 7**2 * (num_anchors * 5 + num_classes)),
        )
        self.num_anchors = num_anchors
        init_module(self.block4, "leaky_relu")
        init_module(self.classifier, "leaky_relu")

    def _format_outputs(self, x: Tensor) -> Tuple[Tensor, Tensor, Tensor]:
        """(N, 7*7*(A*5 + K)) -> boxes (N, 7, 7, A, 4) in (x, y, w, h), objectness (N, 7, 7, A), scores (N, 7, 7, 1, K)."""
        b, _ = x.shape
        h, w = 7, 7
        x = x.reshape(b, h, w, self.num_anchors * 5 + self.num_classes)
        b_scores = F.softmax(x[..., -self.num_classes:].unsqueeze(3), dim=-1)
        x = torch.sigmoid(x[..., : self.num_anchors * 5].reshape(b, h, w, self.num_anchors, 5))
        return x[..., :4], x[..., 4], b_scores

    def _forward(self, x: Tensor) -> Tensor:
        out = self.block4(self.backbone(x))
        # the classifier's Linear layers are fp32 library GEMMs on the flattened (NCHW-ordered, like the reference) map
        return self.classifier(out.float())

    def forward(self, x: Tensor, target: Optional[List[Dict[str, Tensor]]] = None
                ) -> Union[Dict[str, Tensor], List[Dict[str, Tensor]]]:
        if self.training and target is None:
            raise ValueError("`target` needs to be specified in training mode")
        if isinstance(x, (list, tuple)):
            x = torch.stack(x, dim=0)
        out = self._forward(x)
        b_coords, b_o, b_scores = self._format_outputs(out)
        if self.training:
            return self._compute_losses(b_coords, b_o, b_scores, target)  # type: ignore[arg-type]
        b_coords = b_coords.reshape(b_coords.shape[0], -1, 4)
        b_o = b_o.reshape(b_o.shape[0], -1)
        b_scores = b_scores.repeat_interleave(self.num_anchors, dim=3)
        b_scores = b_scores.contiguous().reshape(b_scores.shape[0], -1, self.num_classes)
        return self.post_process(b_coords, b_o, b_scores, (7, 7), self.rpn_nms_thresh, self.box_score_thresh)


def yolov1(pretrained: bool = False, progress: bool = True, pretrained_backbone: bool = False, **kwargs: Any) -> YOLOv1:
    """YOLO (https://pjreddie.com/media/files/papers/yolo_1.pdf) with a Darknet-24 backbone - reference yolo.py:411-478.
    ``pretrained_backbone`` defaults to False here (the reference's True triggers a download)."""
    if pretrained or pretrained_backbone:
        raise NotImplementedError("pretrained checkpoints need network access; load a reference state_dict instead")
    return YOLOv1([[192], [128, 256, 256, 512], [*([256, 512] * 4), 512, 1024], [512, 1024] * 2], **kwargs)
