"""YOLOv4 on the fused kernels — API mirror of holocron/models/detection/yolov4.py.

Module tree / ``state_dict`` / init order are the reference's (backbone = ``DarknetBodyV4``, ``neck.fpn/pan1/pan2``,
``head.head1 ... head.yolo3``). All conv-BN-Mish(-DropBlock) units run through :mod:`holocron_b200.models._blocks`
(tensor-core convolution + fused normalise/activate pass, DropBlock kernel without host sync); the 255-channel output
convolutions are padded to 256 channels inside the conv binding. The YOLO layer's box decoding, target assignment and
losses follow reference yolov4.py:269-420 using the fused pairwise box kernels of :mod:`holocron_b200.ops.boxes`
(``ciou_loss`` == DIoU loss, reference quirk; the "ignore" masking of yolov4.py:386 writes to a copy and is therefore
omitted)."""
from typing import Any, Callable, Dict, List, Optional, Tuple, Union

import torch
import torch.nn.functional as F
from torch import Tensor, nn
from torchvision.ops.boxes import nms

from ...nn import SPP, DropBlock2d
from ...nn.init import init_module
from ...ops.boxes import box_iou, ciou_loss
from .._blocks import FusedSequential
from ..classification.darknet import DarknetBodyV4
from ..utils import conv_sequence
from ._postprocess import Segment, detect_padded, kernel_takes, to_detections

__all__ = ["Neck", "PAN", "YOLOv4", "YoloLayer", "Yolov4Head", "yolov4"]


def _units(spec: List[Tuple[int, int, int]], act, norm, drop, conv, stride: int = 1) -> List[nn.Module]:
    """[(cin, cout, k), ...] -> concatenated conv_sequence units (k=3 -> padding 1)."""
    mods: List[nn.Module] = []
    for cin, cout, k in spec:
        kw: Dict[str, Any] = dict(kernel_size=k, bias=(norm is None))
        if k == 3:
            kw["padding"] = 1
        if stride != 1:
            kw["stride"] = stride
        mods.extend(conv_sequence(cin, cout, act, norm, drop, conv, **kw))
    return mods


class PAN(nn.Module):
    """Path-aggregation block (reference yolov4.py:31-139): 1x1 on the deep map + nearest x2 up-sampling, 1x1 on the
    lateral map, concat, five alternating 1x1 / 3x3 units."""

    def __init__(self, in_channels: int, act_layer=None, norm_layer=None, drop_layer=None, conv_layer=None) -> None:
        super().__init__()
        c, h = in_channels, in_channels // 2
        self.conv1 = FusedSequential(*_units([(c, h, 1)], act_layer, norm_layer, drop_layer, conv_layer))
        self.up = nn.Upsample(scale_factor=2, mode="nearest")
        self.conv2 = FusedSequential(*_units([(c, h, 1)], act_layer, norm_layer, drop_layer, conv_layer))
        self.convs = FusedSequential(*_units([(c, h, 1), (h, c, 3), (c, h, 1), (h, c, 3), (c, h, 1)], act_layer, norm_layer,
                                             drop_layer, conv_layer))

    def forward(self, x: Tensor, up: Tensor) -> Tensor:
        out = self.conv1(x)
        out = torch.cat([self.conv2(up), self.up(out)], dim=1)
        return self.convs(out)


class Neck(nn.Module):
    """SPP + two PAN blocks (reference yolov4.py:142-229)."""

    def __init__(self, in_planes: List[int], act_layer=None, norm_layer=None, drop_layer=None, conv_layer=None) -> None:
        super().__init__()
        c, h = in_planes[0], in_planes[0] // 2
        self.fpn = FusedSequential(
            *_units([(c, h, 1), (h, c, 3), (c, h, 1)], act_layer, norm_layer, drop_layer, conv_layer),
            SPP([5, 9, 13]),
            *_units([(4 * h, h, 1), (h, c, 3), (c, h, 1)], act_layer, norm_layer, drop_layer, conv_layer),
        )
        self.pan1 = PAN(in_planes[1], act_layer, norm_layer, drop_layer, conv_layer)
        self.pan2 = PAN(in_planes[2], act_layer, norm_layer, drop_layer, conv_layer)
        init_module(self, "leaky_relu")

    def forward(self, feats: List[Tensor]) -> Tuple[Tensor, Tensor, Tensor]:
        out = self.fpn(feats[2])
        aux1 = self.pan1(out, feats[1])
        aux2 = self.pan2(aux1, feats[0])
        return aux2, aux1, out


class YoloLayer(nn.Module):
    """Scale-specific decoding + loss (reference yolov4.py:232-442)."""

    def __init__(self, anchors: Tensor, num_classes: int = 80, scale_xy: float = 1.0, iou_thresh: float = 0.213,
                 lambda_obj: float = 1, lambda_noobj: float = 0.001, lambda_class: float = 0.1, lambda_coords: float = 1.0,
                 rpn_nms_thresh: float = 0.7, box_score_thresh: float = 0.05, ignore_thresh: float = 0.5) -> None:
        super().__init__()
        self.num_classes = num_classes
        self.register_buffer("anchors", anchors)
        self.rpn_nms_thresh = rpn_nms_thresh
        self.box_score_thresh = box_score_thresh
        self.ignore_thresh = ignore_thresh
        self.lambda_obj = lambda_obj
        self.lambda_noobj = lambda_noobj
        self.lambda_class = lambda_class
        self.lambda_coords = lambda_coords
        self.scale_xy = scale_xy
        self.iou_thresh = iou_thresh

    def extra_repr(self) -> str:
        return f"num_classes={self.num_classes}, scale_xy={self.scale_xy}"

    def _format_outputs(self, output: Tensor) -> Tuple[Tensor, Tensor, Tensor]:
        """(B, A*(5+K), H, W) raw map -> relative xyxy boxes (B,H,W,A,4), objectness logits, class logits (fp32)."""
        b, _, h, w = output.shape
        na = len(self.anchors)
        out = output.float().reshape(b, na, 5 + self.num_classes, h, w).permute(0, 3, 4, 1, 2)
        gx = torch.arange(w, dtype=torch.float32, device=out.device).reshape(1, 1, -1, 1)
        gy = torch.arange(h, dtype=torch.float32, device=out.device).reshape(1, -1, 1, 1)
        xy = self.scale_xy * torch.sigmoid(out[..., :2]) - 0.5 * (self.scale_xy - 1)
        cx = (xy[..., 0] + gx) / w
        cy = (xy[..., 1] + gy) / h
        wh = (torch.exp(out[..., 2:4]) * self.anchors.view(1, 1, 1, -1, 2)).clamp(0, 2)
        x1 = cx - 0.5 * wh[..., 0]
        y1 = cy - 0.5 * wh[..., 1]
        boxes = torch.stack((x1, y1, x1 + wh[..., 0], y1 + wh[..., 1]), dim=-1)
        return boxes, out[..., 4], out[..., 5:]

    @staticmethod
    def post_process(boxes: Tensor, b_o: Tensor, b_scores: Tensor, rpn_nms_thresh: float = 0.7,
                     box_score_thresh: float = 0.05) -> List[Dict[str, Tensor]]:
        """Reference yolov4.py:303-335. CUDA inputs go through the batched kernels of ``csrc/detect.cu`` when they
        reproduce the loop exactly (see :func:`~._postprocess.kernel_takes`): one launch chain for the batch and one
        device-to-host copy (the per-image counts). Other inputs take the reference's per-image loop."""
        if b_o.is_cuda and kernel_takes(boxes, b_o, b_scores):
            return to_detections(*detect_padded([YoloLayer._segment(boxes, b_o, b_scores, rpn_nms_thresh,
                                                                    box_score_thresh)]))
        return YoloLayer._post_process_per_image(boxes, b_o, b_scores, rpn_nms_thresh, box_score_thresh)

    @staticmethod
    def _post_process_per_image(boxes: Tensor, b_o: Tensor, b_scores: Tensor, rpn_nms_thresh: float,
                                box_score_thresh: float) -> List[Dict[str, Tensor]]:
        """The reference's loop over images (boolean-mask gathers, one torchvision nms per image)."""
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

    @staticmethod
    def _segment(boxes: Tensor, b_o: Tensor, b_scores: Tensor, rpn_nms_thresh: float, box_score_thresh: float) -> Segment:
        """post_process's inputs as one kernel segment: the (B, H, W, A) candidates flattened in the order of the
        reference's boolean masks, objectness and class probabilities through the same sigmoid, then widened to fp32."""
        n = b_o.shape[0]
        return (boxes.reshape(n, -1, 4), torch.sigmoid(b_o).float().reshape(n, -1),
                torch.sigmoid(b_scores).float().reshape(n, -1, b_scores.shape[-1]), box_score_thresh, rpn_nms_thresh)

    def _assignment(self, b: int, h: int, w: int, na: int, target: List[Dict[str, Tensor]], dev):
        """Per ground-truth box: image index, cell, best-shape anchor, linear index of its (image, cell, anchor) slot and
        the number of boxes sharing that slot (reference yolov4.py:338-388: cell = the one holding the box centre, anchor =
        best IoU between the box's and the anchors' shapes). Everything is a static-shape device tensor - the only host
        knowledge used is the number of boxes per image, which defines the shapes anyway."""
        counts = tuple(int(t["boxes"].shape[0]) for t in target)
        key = (counts, str(dev))
        cache = self.__dict__.setdefault("_img_index_cache", {})
        img = cache.get(key)
        if img is None:     # built once per box-count pattern (a pageable host->device copy: not inside a graph capture)
            img = torch.repeat_interleave(torch.arange(b), torch.tensor(counts)).to(dev)
            cache[key] = img
        boxes = torch.cat([t["boxes"] for t in target], dim=0).float()
        labels = torch.cat([t["labels"] for t in target], dim=0)
        cell_x = ((boxes[:, 0] + boxes[:, 2]) / 2 * w).to(torch.long)
        cell_y = ((boxes[:, 1] + boxes[:, 3]) / 2 * h).to(torch.long)
        gt_wh = boxes[:, 2:] - boxes[:, :2]
        anchor_idx = box_iou(torch.cat((-gt_wh, gt_wh), dim=-1),
                             torch.cat((-self.anchors, self.anchors), dim=-1)).argmax(dim=1)
        lin = ((img * h + cell_y) * w + cell_x) * na + anchor_idx
        cnt = torch.zeros(b * h * w * na, device=dev).index_put_((lin,), torch.ones_like(lin, dtype=torch.float32),
                                                                    accumulate=True)
        return img, cell_y, cell_x, anchor_idx, lin, cnt[lin], boxes, labels

    def _build_targets(self, pred_boxes: Tensor, b_o: Tensor, target: List[Dict[str, Tensor]]):
        """Dense objectness / class targets and the (obj, noobj) masks of reference yolov4.py:338-388, produced without any
        boolean-mask gather (no host synchronisation). Kept for introspection; the losses use the per-box form below."""
        b, h, w, na = b_o.shape
        dev = b_o.device
        target_o = torch.zeros((b, h, w, na), device=dev)
        target_scores = torch.zeros((b, h, w, na, self.num_classes), device=dev)
        obj_mask = torch.zeros((b, h, w, na), dtype=torch.bool, device=dev)
        noobj_mask = torch.ones((b, h, w, na), dtype=torch.bool, device=dev)
        if sum(t["boxes"].shape[0] for t in target) == 0:
            return target_o, target_scores, obj_mask, noobj_mask
        img, cy, cx, a, lin, mult, boxes, labels = self._assignment(b, h, w, na, target, dev)
        obj_mask[img, cy, cx, a] = True
        noobj_mask[img, cy, cx, :] = False
        ious, gt_idx = self._per_box_iou(pred_boxes[img, cy, cx, a], boxes, img)
        target_o[img, cy, cx, a] = ious
        target_scores[img, cy, cx, a, labels[gt_idx]] = 1.0
        return target_o, target_scores, obj_mask, noobj_mask

    @staticmethod
    def _per_box_iou(preds: Tensor, boxes: Tensor, img: Tensor) -> Tuple[Tensor, Tensor]:
        """For the prediction assigned to every ground-truth box: the best IoU with the boxes of ITS image and that box's
        index (reference: box_iou(pred_boxes[idx][obj_mask[idx]], gt_boxes[idx]).max(dim=1), one call per image)."""
        same = img[:, None] == img[None, :]
        iou = box_iou(preds, boxes)
        return torch.where(same, iou, torch.full_like(iou, -1.0)).max(dim=1)

    def _compute_losses(self, pred_boxes: Tensor, b_o: Tensor, b_scores: Tensor,
                        target: List[Dict[str, Tensor]]) -> Dict[str, Tensor]:
        """The four YOLOv4 losses of reference yolov4.py:390-420. The reference gathers the predictions of the assigned
        (cell, anchor) slots with boolean masks, image by image (data-dependent shapes, one host synchronisation per gather).
        Here every ground-truth box carries the prediction of its slot (static shapes); a slot shared by m boxes would be
        counted m times, so each row is weighted by 1/m - the rows of a shared slot are identical, hence the weighted sum
        equals the reference's sum over DISTINCT slots exactly. All pairs of one G x G box-op launch replace the per-image
        calls (pairs of different images masked out). No host synchronisation: the step can be CUDA-graph captured."""
        b, h, w, na = b_o.shape
        dev = b_o.device
        n = b
        prob_o = torch.sigmoid(b_o)
        if sum(t["boxes"].shape[0] for t in target) == 0:
            zero = torch.zeros((), device=dev) * prob_o.sum() * 0
            return {"obj_loss": zero, "noobj_loss": self.lambda_noobj * prob_o.pow(2).sum() / n,
                    "bbox_loss": torch.zeros(1, device=dev) + zero, "clf_loss": zero * b_scores.sum() * 0}
        img, cy, cx, a, lin, mult, boxes, labels = self._assignment(b, h, w, na, target, dev)
        wgt = 1.0 / mult
        preds = pred_boxes[img, cy, cx, a]                              # [G, 4], differentiable gather
        same = img[:, None] == img[None, :]
        ious, gt_idx = self._per_box_iou(preds, boxes, img)             # objectness target stays attached to the graph
        ciou = ciou_loss(preds, boxes)
        bbox = (torch.where(same, ciou, torch.full_like(ciou, float("inf"))).min(dim=1).values * wgt).sum()
        obj = ((prob_o[img, cy, cx, a] - ious).pow(2) * wgt).sum()
        noobj_w = torch.ones((b, h, w, na), device=dev)
        noobj_w.index_put_((img, cy, cx), noobj_w.new_zeros(()))    # device-side value: graph-capturable (no CPU scalar copy)
        onehot = F.one_hot(labels[gt_idx], self.num_classes).to(b_scores.dtype)
        clf = (F.binary_cross_entropy_with_logits(b_scores[img, cy, cx, a], onehot, reduction="none").mean(1) * wgt).sum()
        return {
            "obj_loss": self.lambda_obj * obj / n,
            "noobj_loss": self.lambda_noobj * (prob_o.pow(2) * noobj_w).sum() / n,
            "bbox_loss": (self.lambda_coords * bbox / n).reshape(1),
            "clf_loss": self.lambda_class * clf / n,
        }

    def forward(self, x: Tensor, target: Optional[List[Dict[str, Tensor]]] = None):
        if self.training and target is None:
            raise ValueError("`target` needs to be specified in training mode")
        pred_boxes, b_o, b_scores = self._format_outputs(x)
        if self.training:
            return self._compute_losses(pred_boxes, b_o, b_scores, target)  # type: ignore[arg-type]
        return self.post_process(pred_boxes, b_o, b_scores, self.rpn_nms_thresh, self.box_score_thresh)


class Yolov4Head(nn.Module):
    """Three detection heads with their down-sampling bridges (reference yolov4.py:445-640).

    In eval mode on CUDA, ``forward`` decodes the three scales with each YoloLayer's ``_format_outputs`` and thresholds
    and post-processes them in one kernel chain; it does not call ``yolo1`` / ``yolo2`` / ``yolo3`` as modules, so
    forward hooks registered on the YoloLayers do not fire on that path (they do in training and on CPU)."""

    def __init__(self, num_classes: int = 80, anchors: Optional[Tensor] = None, act_layer=None, norm_layer=None,
                 drop_layer=None, conv_layer=None) -> None:
        if anchors is None:
            anchors = torch.tensor([[[12, 16], [19, 36], [40, 28]], [[36, 75], [76, 55], [72, 146]],
                                    [[142, 110], [192, 243], [459, 401]]], dtype=torch.float32) / 608
        elif not isinstance(anchors, torch.Tensor):
            anchors = torch.tensor(anchors, dtype=torch.float32)
        if anchors.shape[0] != 3:
            raise AssertionError(f"The number of anchors is expected to be 3. received: {anchors.shape[0]}")
        super().__init__()
        out_ch = (5 + num_classes) * 3
        a, n, d, c = act_layer, norm_layer, drop_layer, conv_layer

        def out_conv(cin: int) -> List[nn.Module]:
            return conv_sequence(cin, out_ch, None, None, None, c, kernel_size=1, bias=True)

        self.head1 = FusedSequential(*_units([(128, 256, 3)], a, n, None, c), *out_conv(256))
        self.yolo1 = YoloLayer(anchors[0], num_classes=num_classes, scale_xy=1.2)
        self.pre_head2 = FusedSequential(*_units([(128, 256, 3)], a, n, d, c, stride=2))
        self.head2_1 = FusedSequential(*_units([(512, 256, 1), (256, 512, 3), (512, 256, 1), (256, 512, 3), (512, 256, 1)],
                                               a, n, d, c))
        self.head2_2 = FusedSequential(*_units([(256, 512, 3)], a, n, None, c), *out_conv(512))
        self.yolo2 = YoloLayer(anchors[1], num_classes=num_classes, scale_xy=1.1)
        self.pre_head3 = FusedSequential(*_units([(256, 512, 3)], a, n, d, c, stride=2))
        self.head3 = FusedSequential(*_units([(1024, 512, 1), (512, 1024, 3), (1024, 512, 1), (512, 1024, 3), (1024, 512, 1),
                                              (512, 1024, 3)], a, n, d, c), *out_conv(1024))
        self.yolo3 = YoloLayer(anchors[2], num_classes=num_classes, scale_xy=1.05)
        init_module(self, "leaky_relu")
        for head in (self.head1, self.head2_2, self.head3):   # zero-initialised output convolutions
            head[-1].weight.data.zero_()
            head[-1].bias.data.zero_()

    def _heads(self, feats: List[Tensor]) -> Tuple[Tensor, Tensor, Tensor]:
        o1 = self.head1(feats[0])
        h2 = self.head2_1(torch.cat([self.pre_head2(feats[0]), feats[1]], dim=1))
        o2 = self.head2_2(h2)
        o3 = self.head3(torch.cat([self.pre_head3(h2), feats[2]], dim=1))
        return o1, o2, o3

    def _detect(self, outs: Tuple[Tensor, Tensor, Tensor]) -> Tuple[Tensor, Tensor, Tensor, Tensor]:
        """The three scales as three segments of ONE kernel chain: suppressed per scale with each layer's thresholds,
        concatenated per image in scale order on the device."""
        return detect_padded([layer._segment(*layer._format_outputs(o), layer.rpn_nms_thresh, layer.box_score_thresh)
                              for layer, o in zip((self.yolo1, self.yolo2, self.yolo3), outs)])

    def detect_padded(self, feats: List[Tensor]) -> Tuple[Tensor, Tensor, Tensor, Tensor]:
        """See :meth:`YOLOv4.detect_padded`."""
        return self._detect(self._heads(feats))

    def forward(self, feats: List[Tensor], target: Optional[List[Dict[str, Tensor]]] = None):
        o1, o2, o3 = self._heads(feats)
        if not self.training and o1.is_cuda:     # one read-back for the batch, not one per scale
            return to_detections(*self._detect((o1, o2, o3)))
        y1, y2, y3 = self.yolo1(o1, target), self.yolo2(o2, target), self.yolo3(o3, target)
        if not self.training:
            return [{k: torch.cat((d1[k], d2[k], d3[k]), dim=0) for k in ("boxes", "scores", "labels")}
                    for d1, d2, d3 in zip(y1, y2, y3)]
        return {k: y1[k] + y2[k] + y3[k] for k in y1}


class YOLOv4(nn.Module):
    """reference yolov4.py:643-690."""

    def __init__(self, layout: List[Tuple[int, int]], num_classes: int = 80, in_channels: int = 3, stem_channels: int = 32,
                 anchors: Optional[Tensor] = None, act_layer: Optional[nn.Module] = None,
                 norm_layer: Optional[Callable[[int], nn.Module]] = None, drop_layer=None, conv_layer=None,
                 backbone_norm_layer: Optional[Callable[[int], nn.Module]] = None) -> None:
        super().__init__()
        if act_layer is None:
            act_layer = nn.Mish(inplace=True)
        if norm_layer is None:
            norm_layer = nn.BatchNorm2d
        if backbone_norm_layer is None:
            backbone_norm_layer = norm_layer
        if drop_layer is None:
            drop_layer = DropBlock2d
        self.backbone = DarknetBodyV4(layout, in_channels, stem_channels, 3, act_layer, backbone_norm_layer, drop_layer,
                                      conv_layer)
        self.neck = Neck([1024, 512, 256], act_layer, norm_layer, drop_layer, conv_layer)
        self.head = Yolov4Head(num_classes, anchors, act_layer, norm_layer, drop_layer, conv_layer)
        init_module(self.neck, "leaky_relu")
        init_module(self.head, "leaky_relu")

    def forward(self, x: Tensor, target: Optional[List[Dict[str, Tensor]]] = None):
        if not isinstance(x, torch.Tensor):
            x = torch.stack(x, dim=0)
        out = self.backbone(x)
        x20, x13, x6 = self.neck(out)
        return self.head((x20, x13, x6), target)

    def detect_padded(self, x: Tensor) -> Tuple[Tensor, Tensor, Tensor, Tensor]:
        """The detections of the eval forward as padded device tensors, with no host synchronisation at all (an eval
        forward that can be captured in a CUDA graph): ``boxes [B, cap, 4]``, ``scores [B, cap]``, ``labels [B, cap]``
        (int64) and ``counts [B]`` (int32), cap = the candidates of the three scales. Image b's detections are the first
        ``counts[b]`` rows, equal to ``forward(x)[b]`` in the model's current mode (call it in eval mode)."""
        if not isinstance(x, torch.Tensor):
            x = torch.stack(x, dim=0)
        return self.head.detect_padded(list(self.neck(self.backbone(x))))


def yolov4(pretrained: bool = False, progress: bool = True, pretrained_backbone: bool = False, **kwargs: Any) -> YOLOv4:
    """YOLOv4 (https://arxiv.org/abs/2004.10934) with a CSP-Darknet-53 backbone (reference yolov4.py:722-764).
    ``pretrained_backbone`` defaults to False here (the reference's True triggers a download)."""
    if pretrained or pretrained_backbone:
        raise NotImplementedError("pretrained checkpoints need network access; load a reference state_dict instead")
    return YOLOv4([(64, 1), (128, 2), (256, 8), (512, 8), (1024, 4)], **kwargs)
