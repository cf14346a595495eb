"""YOLOv2 on the fused kernels — API mirror of holocron/models/detection/yolov2.py (YOLOv2 :29-259, yolov2 :287-321).

Module tree / ``state_dict`` / init order are the reference's (``backbone`` = ``DarknetBodyV2`` with the pass-through route,
``block5``, ``passthrough_layer``, ``block6``, ``head``, buffer ``anchors``). The conv-BN-LeakyReLU units run on the tensor-core
convolution + fused normalise/activate pass; the 125-channel output convolution is zero-padded to 128 channels inside the
conv binding; the pass-through ``ConcatDownsample2d`` and the channel concatenation are pure data movement. The losses are
the sync-free per-box formulation of :class:`holocron_b200.models.detection.yolo._YOLO` (classification term over every
anchor row of the cell, like the reference)."""
from typing import Any, Callable, Dict, List, Optional, Tuple, Union

import torch
import torch.nn.functional as F
from torch import Tensor, nn

from ...nn import ConcatDownsample2d
from ...nn.init import init_module
from .._blocks import FusedSequential, conv_bn_act
from ..classification.darknet import DarknetBodyV2
from ..utils import conv_sequence
from .yolo import _YOLO

__all__ = ["YOLOv2", "yolov2"]


class YOLOv2(_YOLO):
    """reference yolov2.py:29-259, same constructor (including the ``stem_chanels`` spelling)."""

    def __init__(self, layout: List[Tuple[int, int]], num_classes: int = 20, in_channels: int = 3, stem_chanels: int = 32,
                 anchors: Optional[Tensor] = None, passthrough_ratio: int = 8, lambda_obj: float = 1, lambda_noobj: float = 0.5,
                 lambda_class: float = 1, lambda_coords: float = 5, rpn_nms_thresh: float = 0.7,
                 box_score_thresh: float = 0.05, act_layer: Optional[nn.Module] = None,
                 norm_layer: Optional[Callable[[int], nn.Module]] = None,
                 drop_layer: Optional[Callable[..., nn.Module]] = None,
                 conv_layer: Optional[Callable[..., nn.Module]] = None,
                 backbone_norm_layer: Optional[Callable[[int], nn.Module]] = None) -> None:
        super().__init__(num_classes, rpn_nms_thresh, box_score_thresh, lambda_obj, lambda_noobj, lambda_class, lambda_coords)
        if act_layer is None:
            act_layer = nn.LeakyReLU(0.1, inplace=True)
        if norm_layer is None:
            norm_layer = nn.BatchNorm2d
        if backbone_norm_layer is None:
            backbone_norm_layer = norm_layer
        if anchors is None:   # k-means priors of yolov2-voc.cfg, in units of the 13 x 13 grid
            anchors = torch.tensor([[1.3221, 1.73145], [3.19275, 4.00944], [5.05587, 8.09892], [9.47112, 4.84053],
                                    [11.2364, 10.0071]]) / 13
        self.backbone = DarknetBodyV2(layout, in_channels, stem_chanels, True, act_layer, backbone_norm_layer, drop_layer,
                                      conv_layer)
        c_last, c_route = layout[-1][0], layout[-2][0]

        def unit(cin: int, cout: int, **kw: Any) -> List[nn.Module]:
            return conv_sequence(cin, cout, act_layer, norm_layer, drop_layer, conv_layer, bias=(norm_layer is None), **kw)

        self.block5 = FusedSequential(*unit(c_last, c_last, kernel_size=3, padding=1), *unit(c_last, c_last, kernel_size=3, padding=1))
        self.passthrough_layer = FusedSequential(*unit(c_route, c_route // passthrough_ratio, kernel_size=1),
                                                 ConcatDownsample2d(scale_factor=2))
        self.block6 = FusedSequential(*unit(c_last + c_route // passthrough_ratio * 2**2, c_last, kernel_size=3, padding=1))
        # every box: objectness, 4 coordinates and one score per class
        self.head = nn.Conv2d(c_last, anchors.shape[0] * (5 + num_classes), 1)
        self.register_buffer("anchors", anchors)
        init_module(self.block5, "leaky_relu")
        init_module(self.passthrough_layer, "leaky_relu")
        init_module(self.block6, "leaky_relu")
        if self.head.bias is not None:
            self.head.bias.data.zero_()

    @property
    def num_anchors(self) -> int:
        return self.anchors.shape[0]

    @staticmethod
    def to_isoboxes(b_coords: Tensor, grid_shape: Tuple[int, int], clamp: bool = False) -> Tensor:
        """(..., 4) image-relative (xc, yc, w, h) -> xyxy (reference yolov2.py:145-163: no cell offsets here)."""
        xy = b_coords[..., :2]
        wh = b_coords[..., 2:]
        pred_xyxy = torch.cat((xy - wh / 2, xy + wh / 2), dim=-1).reshape(*b_coords.shape)
        if clamp:
            pred_xyxy = pred_xyxy.clamp(0, 1)
        return pred_xyxy

    def _format_outputs(self, x: Tensor) -> Tuple[Tensor, Tensor, Tensor]:
        """(N, A*(5+K), H, W) -> boxes (N, H, W, A, 4) in relative (xc, yc, w, h), objectness (N, H, W, A), class
        probabilities (N, H, W, A, K) - fp32 (reference yolov2.py:165-196)."""
        b, _, h, w = x.shape
        x = x.float().reshape(b, self.num_anchors, 5 + self.num_classes, h, w).permute(0, 3, 4, 1, 2)
        b_scores = F.softmax(x[..., -self.num_classes:], dim=-1)
        c_x = torch.arange(w, dtype=torch.float, device=x.device)
        c_y = torch.arange(h, dtype=torch.float, device=x.device)
        b_x = (torch.sigmoid(x[..., 0]) + c_x.reshape(1, 1, -1, 1)) / w
        b_y = (torch.sigmoid(x[..., 1]) + c_y.reshape(1, -1, 1, 1)) / h
        b_w = self.anchors[:, 0].reshape(1, 1, 1, -1) * torch.exp(x[..., 2])
        b_h = self.anchors[:, 1].reshape(1, 1, 1, -1) * torch.exp(x[..., 3])
        b_coords = torch.stack((b_x, b_y, b_w, b_h), dim=4)
        b_o = torch.sigmoid(x[..., 4])
        return b_coords, b_o, b_scores

    def _forward(self, x: Tensor) -> Tensor:
        out, passthrough = self.backbone(x)
        passthrough = self.passthrough_layer(passthrough)      # 1x1 unit, then 2x2 pixel blocks onto the channel axis
        out = self.block5(out)
        out = torch.cat((passthrough.to(out.dtype), out), 1)
        out = self.block6(out)
        return conv_bn_act(out, self.head, None, None)

    def forward(self, x: Union[Tensor, List[Tensor], Tuple[Tensor, ...]], target: Optional[List[Dict[str, Tensor]]] = None
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
        b_scores = b_scores.reshape(b_scores.shape[0], -1, self.num_classes)
        return self.post_process(b_coords, b_o, b_scores, tuple(out.shape[-2:]), self.rpn_nms_thresh,  # type: ignore[arg-type]
                                 self.box_score_thresh)


def yolov2(pretrained: bool = False, progress: bool = True, pretrained_backbone: bool = False, **kwargs: Any) -> YOLOv2:
    """YOLOv2 (https://pjreddie.com/media/files/papers/YOLO9000.pdf) with a Darknet-19 backbone - reference yolov2.py:287-321.
    ``pretrained_backbone`` defaults to False here (the reference's True triggers a download and freezes the backbone's
    BatchNorm layers)."""
    if pretrained or pretrained_backbone:
        raise NotImplementedError("pretrained checkpoints need network access; load a reference state_dict instead")
    return YOLOv2([(64, 0), (128, 1), (256, 1), (512, 2), (1024, 2)], **kwargs)
