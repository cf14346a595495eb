"""Host logic of the batched YOLO post-processing (models/detection/_postprocess.py, csrc/detect.cu) that needs no GPU:
scratch sizing and the refused tables of the C ABI, argument validation before any launch, YOLOv4's per-scale segments,
and CPU inputs keeping the reference's per-image loop."""
import importlib

import pytest
import torch

from _detect_oracle import _ref_v12, _ref_v4, fma_sensitive_pair, iou_f32
from holocron_b200 import _lib
from holocron_b200.models.detection import _postprocess as P
from holocron_b200.models.detection.yolov4 import YoloLayer, Yolov4Head

# the modules themselves (the package exports factory functions of the same names)
Y1 = importlib.import_module("holocron_b200.models.detection.yolo")
Y4 = importlib.import_module("holocron_b200.models.detection.yolov4")


def _align(x):
    return (x + 255) // 256 * 256


def _mirror_scratch(sizes, b):
    """csrc/detect.cu plan(): seven per-candidate arrays, two per-(image, segment) counters, the IoU bitmask (one
    64-bit word per survivor and 64-candidate block of its segment) and, above 16384 candidates, the global sort keys."""
    n = b * sum(sizes)
    total = sum(_align(n * w) for w in (4, 4, 4, 16, 4, 4, 4)) + 2 * _align(b * len(sizes) * 4)
    total += _align(8 * b * sum(m * ((m + 63) // 64) for m in sizes))
    pk = 1
    while pk < max(sizes):
        pk *= 2
    total += _align(8 * b * len(sizes) * pk) if pk > 16384 else 0
    return total


def _need_lib():
    if not _lib.lib_path().exists():
        pytest.skip("libholocron_b200.so has not been built")


@pytest.mark.parametrize("sizes,b", [([98], 1), ([845], 32), ([12288, 3072, 768], 16), ([17328, 4332, 1083], 2),
                                     ([0], 4), ([0, 5, 0], 3), ([1], 65535)])
def test_scratch_bytes_match_the_layout(sizes, b):
    _need_lib()
    assert P.scratch_bytes(sizes, b, 80) == max(_mirror_scratch(sizes, b), 1)


@pytest.mark.parametrize("sizes,b,k", [([], 1, 3), ([1] * 5, 1, 3), ([10], 1, 0), ([10], -1, 3), ([-1], 1, 3),
                                       ([(1 << 20) + 1], 1, 3), ([1, 1], 32768, 3)])
def test_scratch_query_refuses_bad_tables(sizes, b, k):
    _need_lib()
    assert P.scratch_bytes(sizes, b, k) == 0


def _seg(b=2, m=6, k=3, **over):
    seg = dict(boxes=torch.rand(b, m, 4), obj=torch.rand(b, m), cls=torch.rand(b, m, k))
    seg.update(over)
    return (seg["boxes"], seg["obj"], seg["cls"], 0.05, 0.7)


@pytest.mark.parametrize("segments,err", [
    ([], ValueError),
    ([_seg()] * 5, ValueError),
    ([_seg(boxes=torch.rand(2, 6, 5))], ValueError),
    ([_seg(obj=torch.rand(2, 7))], ValueError),
    ([_seg(), _seg(b=3)], ValueError),
    ([_seg(), _seg(k=4)], ValueError),
    ([_seg(k=0)], ValueError),
    ([_seg(boxes=torch.rand(2, 6, 4, dtype=torch.float64))], TypeError),
    ([_seg(cls=torch.rand(2, 6, 3).half())], TypeError),
    ([_seg(m=(1 << 20) + 1, k=1)], ValueError),
    ([_seg()], _lib.HolocronB200Error),          # well-formed, but not on a CUDA device
])
def test_arguments_are_checked_before_any_launch(segments, err, monkeypatch):
    def no_launch():
        raise AssertionError("the library was reached")
    monkeypatch.setattr(P, "lib", no_launch)
    with pytest.raises(err):
        P.detect_padded(segments)


def test_yolov4_segments_are_the_three_scales_in_order(monkeypatch):
    torch.manual_seed(0)
    head = Yolov4Head(num_classes=3)
    head.yolo2.rpn_nms_thresh, head.yolo3.box_score_thresh = 0.5, 0.2
    outs = tuple(torch.randn(2, 3 * 8, hw, hw) for hw in (8, 4, 2))
    seen = []
    monkeypatch.setattr(Y4, "detect_padded", lambda segments: seen.append(segments) or "padded")
    assert head._detect(outs) == "padded"
    (segments,) = seen
    assert [s[0].shape[1] for s in segments] == [3 * 64, 3 * 16, 3 * 4]
    assert [(s[3], s[4]) for s in segments] == [(0.05, 0.7), (0.05, 0.5), (0.2, 0.7)]
    for layer, o, (boxes, obj, cls, _, _) in zip((head.yolo1, head.yolo2, head.yolo3), outs, segments):
        ref_boxes, ref_o, ref_cls = layer._format_outputs(o)
        keep = torch.sigmoid(ref_o[1]) >= 0.5           # the reference's boolean mask of image 1 ...
        assert torch.equal(boxes[1][keep.flatten()], ref_boxes[1][keep])     # ... picks the same rows
        assert torch.equal(obj, torch.sigmoid(ref_o).reshape(2, -1))
        assert torch.equal(cls[1][keep.flatten()], torch.sigmoid(ref_cls)[1][keep])


def _no_kernels(monkeypatch):
    def refuse(*args, **kwargs):
        raise AssertionError("CPU inputs reached the CUDA post-processing")
    for mod in (Y1, Y4):
        monkeypatch.setattr(mod, "detect_padded", refuse)


def test_cpu_inputs_keep_the_per_image_loop_v1(monkeypatch):
    _no_kernels(monkeypatch)
    torch.manual_seed(0)
    model = Y1._YOLO(num_classes=4)
    model.num_anchors = 2
    b_coords, b_o, b_scores = torch.rand(3, 98, 4), torch.rand(3, 98), torch.rand(3, 98, 4).softmax(-1)
    got = model.post_process(b_coords, b_o, b_scores, (7, 7), 0.5, 0.1)
    xyxy = model.to_isoboxes(b_coords.reshape(-1, 7, 7, 2, 4), (7, 7), clamp=True).reshape(3, -1, 4)
    for g, w in zip(got, _ref_v12(xyxy, b_o, b_scores, 0.5, 0.1)):
        assert all(torch.equal(g[k], w[k]) for k in w)


def test_cpu_inputs_keep_the_per_image_loop_v4(monkeypatch):
    _no_kernels(monkeypatch)
    torch.manual_seed(0)
    boxes, b_o, b_scores = torch.rand(3, 4, 4, 3, 4), torch.randn(3, 4, 4, 3), torch.randn(3, 4, 4, 3, 5)
    got = YoloLayer.post_process(boxes, b_o, b_scores, 0.5, 0.1)
    for g, w in zip(got, _ref_v4(boxes, b_o, b_scores, 0.5, 0.1)):
        assert all(torch.equal(g[k], w[k]) for k in w)


@pytest.mark.parametrize("boxes,obj,cls,takes", [
    (torch.float32, torch.float32, torch.float32, True),
    (torch.float32, torch.bfloat16, torch.float32, True),      # YOLOv1 under bf16 autocast
    (torch.float32, torch.float32, torch.float16, True),
    (torch.float32, torch.bfloat16, torch.bfloat16, False),    # the reference's product is rounded to bf16
    (torch.float32, torch.float16, torch.float16, False),
    (torch.float16, torch.float32, torch.float32, False),      # torchvision's nms would work in fp16
    (torch.float64, torch.float64, torch.float64, False),
    (torch.float32, torch.float64, torch.float32, False),
])
def test_kernels_take_only_what_they_reproduce(boxes, obj, cls, takes):
    t = P.kernel_takes(torch.zeros(1, 1, 4, dtype=boxes), torch.zeros(1, 1, dtype=obj), torch.zeros(1, 1, 2, dtype=cls))
    assert t is takes


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_fma_sensitive_pairs_discriminate(seed):
    """The at-threshold GPU cases decide differently with and without the fused area sum."""
    a, b, thr = fma_sensitive_pair(seed)
    assert (iou_f32(a, b, True) > thr) != (iou_f32(a, b, False) > thr)
    assert 0 <= a.min() and a.max() <= 1 and 0 <= b.min() and b.max() <= 1
