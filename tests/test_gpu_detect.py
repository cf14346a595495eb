"""YOLO post-processing on the batched kernels (csrc/detect.cu) against the reference's per-image loop.

``_ref_v12`` and ``_ref_v4`` restate the reference's ``post_process`` (holocron/models/detection/yolo.py:159-233 and
yolov4.py:303-335: boolean-mask gathers and torchvision's ``nms`` image by image). The kernels must give exactly the
same boxes, scores, labels, dtypes and order."""
import numpy as np
import pytest
import torch
from torchvision.ops.boxes import nms

from _detect_oracle import _ref_v12, _ref_v4, fma_sensitive_pair, iou_f32
from holocron_b200.graphs import GraphedTrainStep
from holocron_b200.models.detection import yolov1, yolov2, yolov4
from holocron_b200.models.detection._postprocess import detect_padded, to_detections
from holocron_b200.models.detection.yolo import YOLOv1, _YOLO
from holocron_b200.models.detection.yolov2 import YOLOv2
from holocron_b200.models.detection.yolov4 import YoloLayer

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")


def _assert_same(got, want):
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        for k in ("boxes", "scores", "labels"):
            assert g[k].dtype == w[k].dtype and g[k].device == w[k].device, (i, k, g[k].dtype, w[k].dtype)
            assert g[k].shape == w[k].shape, (i, k, tuple(g[k].shape), tuple(w[k].shape))
            assert torch.equal(g[k], w[k]), (i, k)


# ---- light stand-ins holding only what post_process and _format_outputs read ----------------------------------------
class _V1(_YOLO):
    _format_outputs = YOLOv1._format_outputs

    def __init__(self, num_classes, num_anchors, **kw):
        super().__init__(num_classes, **kw)
        self.num_anchors = num_anchors


class _V2(_YOLO):
    _format_outputs = YOLOv2._format_outputs
    to_isoboxes = staticmethod(YOLOv2.to_isoboxes)
    num_anchors = property(lambda self: self.anchors.shape[0])

    def __init__(self, num_classes, anchors, **kw):
        super().__init__(num_classes, **kw)
        self.register_buffer("anchors", anchors)


def _v12_inputs(model, raw, v1):
    """The eval forward's tensors between _format_outputs and post_process (YOLOv1.forward / YOLOv2.forward)."""
    b_coords, b_o, b_scores = model._format_outputs(raw)
    grid = (b_coords.shape[1], b_coords.shape[2])
    n = b_coords.shape[0]
    if v1:
        b_scores = b_scores.repeat_interleave(model.num_anchors, dim=3)
    return b_coords.reshape(n, -1, 4), b_o.reshape(n, -1), b_scores.contiguous().reshape(n, -1, model.num_classes), grid


def _check_v12(model, raw, v1):
    b_coords, b_o, b_scores, grid = _v12_inputs(model, raw, v1)
    got = model.post_process(b_coords, b_o, b_scores, grid, model.rpn_nms_thresh, model.box_score_thresh)
    xyxy = model.to_isoboxes(b_coords.reshape(-1, *grid, model.num_anchors, 4), grid, clamp=True).reshape(
        b_o.shape[0], -1, 4)
    want = _ref_v12(xyxy, b_o, b_scores, model.rpn_nms_thresh, model.box_score_thresh)
    _assert_same(got, want)
    return got


def _v1_raw(b, k, a, gen, obj_bias=0.0):
    raw = torch.randn(b, 7, 7, a * 5 + k, generator=gen) * 2
    raw[..., 4:a * 5:5] += obj_bias
    return raw.reshape(b, -1).to(DEV)


def _v2_raw(b, k, a, h, gen, obj_bias=0.0):
    raw = torch.randn(b, a, 5 + k, h, h, generator=gen) * 2
    raw[:, :, 4] += obj_bias
    return raw.reshape(b, a * (5 + k), h, h).to(DEV)


_ANCHORS_V2 = torch.tensor([[1.08, 1.19], [3.42, 4.41], [6.63, 11.38], [9.42, 5.11], [16.62, 10.52]]) / 13
_ANCHORS_V4 = torch.tensor([[[12, 16], [19, 36], [40, 28]], [[36, 75], [76, 55], [72, 146]],
                            [[142, 110], [192, 243], [459, 401]]], dtype=torch.float32) / 608


def _layers(k, **kw):
    return [YoloLayer(_ANCHORS_V4[i], num_classes=k, scale_xy=s, **kw).to(DEV) for i, s in enumerate((1.2, 1.1, 1.05))]


def _v4_raw(b, k, hw, gen, obj_bias=0.0, scale=2.0):
    raw = torch.randn(b, 3, 5 + k, hw, hw, generator=gen) * scale
    raw[:, :, 4] += obj_bias
    return raw.reshape(b, 3 * (5 + k), hw, hw).to(DEV)


def _check_v4(layers, raws):
    """The head's merged path against the reference's three post_process calls concatenated per image."""
    segs = [layer._format_outputs(r) for layer, r in zip(layers, raws)]
    per_scale = [_ref_v4(*s, layer.rpn_nms_thresh, layer.box_score_thresh) for layer, s in zip(layers, segs)]
    want = [{k: torch.cat([d[k] for d in ds], dim=0) for k in ("boxes", "scores", "labels")} for ds in zip(*per_scale)]
    got = to_detections(*detect_padded([layer._segment(*s, layer.rpn_nms_thresh, layer.box_score_thresh)
                                        for layer, s in zip(layers, segs)]))
    _assert_same(got, want)
    for layer, s, w in zip(layers, segs, per_scale):      # each layer's own post_process (one segment)
        _assert_same(layer.post_process(*s, layer.rpn_nms_thresh, layer.box_score_thresh), w)
    return got


# ---- seeded head outputs -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("b", [1, 8, 32])
def test_v1_seeded(b):
    gen = torch.Generator().manual_seed(100 + b)
    model = _V1(20, 2).to(DEV)
    got = _check_v12(model, _v1_raw(b, 20, 2, gen), v1=True)
    assert sum(len(d["scores"]) for d in got) > 0


@pytest.mark.parametrize("b", [1, 8, 32])
def test_v2_seeded(b):
    gen = torch.Generator().manual_seed(200 + b)
    model = _V2(20, _ANCHORS_V2).to(DEV)
    got = _check_v12(model, _v2_raw(b, 20, 5, 13, gen), v1=False)
    assert sum(len(d["scores"]) for d in got) > 0


@pytest.mark.parametrize("b", [1, 8, 32])
def test_v4_seeded(b):
    gen = torch.Generator().manual_seed(300 + b)
    got = _check_v4(_layers(80), [_v4_raw(b, 80, hw, gen) for hw in (16, 8, 4)])
    assert sum(len(d["scores"]) for d in got) > 0


# ---- empty images --------------------------------------------------------------------------------------------------
def test_empty_images_mixed_with_full_ones():
    gen = torch.Generator().manual_seed(1)
    raw = _v2_raw(6, 4, 5, 13, gen)
    raw = raw.reshape(6, 5, 9, 13, 13)
    raw[1, :, 4] = -30.0           # image 1: no candidate passes objectness
    raw[4, :, 4] = -30.0
    raw[3, :, 5:] = 0.0            # image 3: uniform classes (score 0.25 * obj) ...
    model = _V2(4, _ANCHORS_V2, box_score_thresh=0.3).to(DEV)   # ... all under the score threshold
    got = _check_v12(model, raw.reshape(6, 45, 13, 13), v1=False)
    assert [len(d["scores"]) == 0 for d in got] == [False, True, False, True, True, False]


@pytest.mark.parametrize("which", ["v1", "v4"])
def test_every_image_empty(which):
    gen = torch.Generator().manual_seed(2)
    if which == "v1":
        got = _check_v12(_V1(5, 2).to(DEV), _v1_raw(4, 5, 2, gen, obj_bias=-40.0), v1=True)
    else:
        got = _check_v4(_layers(3), [_v4_raw(4, 3, hw, gen, obj_bias=-40.0) for hw in (8, 4, 2)])
    assert all(len(d["scores"]) == 0 and d["boxes"].shape == (0, 4) for d in got)


def test_all_under_score_threshold():
    gen = torch.Generator().manual_seed(3)
    got = _check_v4(_layers(3, box_score_thresh=1.5), [_v4_raw(3, 3, hw, gen, obj_bias=5.0) for hw in (8, 4, 2)])
    assert all(len(d["scores"]) == 0 for d in got)


# ---- many survivors: several bitmask blocks, the order kernel past shared memory, the capacity edge ------------------
def test_more_than_64_and_1024_survivors():
    gen = torch.Generator().manual_seed(4)
    raws = [_v4_raw(2, 6, hw, gen, obj_bias=8.0, scale=1.0) for hw in (64, 32, 16)]     # 12288 + 3072 + 768 per image
    layers = _layers(6)
    got = _check_v4(layers, raws)
    b_o = torch.sigmoid(layers[0]._format_outputs(raws[0])[1])
    assert int((b_o[0] >= 0.5).sum()) > 1024 and len(got[0]["scores"]) > 64


def test_segment_beyond_shared_memory_sort():
    """A segment of more than 16384 candidates (608x608 input, stride 8) sorts in global scratch."""
    gen = torch.Generator().manual_seed(5)
    layer = _layers(2, rpn_nms_thresh=1.0, box_score_thresh=0.0)[0]
    boxes, b_o, b_scores = layer._format_outputs(_v4_raw(2, 2, 76, gen, obj_bias=30.0))
    got = layer.post_process(boxes, b_o, b_scores, 1.0, 0.0)
    _assert_same(got, _ref_v4(boxes, b_o, b_scores, 1.0, 0.0))
    assert len(got[0]["scores"]) == 3 * 76 * 76       # rpn_nms_thresh = 1: nothing is suppressed


def test_every_candidate_kept_at_capacity():
    """Zero head outputs (the zero-initialised output convolutions): every candidate passes, all scores tie."""
    layers = _layers(3, rpn_nms_thresh=1.0, box_score_thresh=0.0)
    raws = [torch.zeros(2, 3 * 8, hw, hw, device=DEV) for hw in (16, 8, 4)]
    boxes, scores, labels, counts = detect_padded([
        layer._segment(*layer._format_outputs(r), 1.0, 0.0) for layer, r in zip(layers, raws)])
    assert counts.tolist() == [3 * (256 + 64 + 16)] * 2 and boxes.shape[1] == counts[0]
    _check_v4(layers, raws)


# ---- the threshold and the tie rule ----------------------------------------------------------------------------------
def _direct_v4(boxes, obj_logit, cls_logit, rpn, thr):
    """Hand-built candidates of one image as a (1, 1, 1, N) grid."""
    n = boxes.shape[0]
    args = (boxes.reshape(1, 1, 1, n, 4).to(DEV), obj_logit.reshape(1, 1, 1, n).to(DEV),
            cls_logit.reshape(1, 1, 1, n, -1).to(DEV))
    got = YoloLayer.post_process(*args, rpn, thr)
    _assert_same(got, _ref_v4(*args, rpn, thr))
    return got[0]


def test_iou_exactly_at_threshold():
    # IoU([0, 0, .5, .5], [0, 0, .5, .25]) = .125 / (.25 + .125 - .125) = 0.5 exactly in fp32
    boxes = torch.tensor([[0, 0, 0.5, 0.5], [0, 0, 0.5, 0.25], [0.5, 0.5, 1, 1], [0.5, 0.5, 1, 0.75]])
    obj = torch.full((4,), 4.0)
    cls = torch.tensor([[3.0, 0.0], [2.0, 0.0], [0.0, 3.0], [0.0, 2.0]])
    assert len(_direct_v4(boxes, obj, cls, 0.5, 0.05)["scores"]) == 4          # strict >: nothing suppressed at 0.5
    below = float(torch.nextafter(torch.tensor(0.5), torch.tensor(0.0)))
    assert len(_direct_v4(boxes, obj, cls, below, 0.05)["scores"]) == 2        # one ulp under: both pairs suppressed


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_iou_rounding_at_threshold_follows_torchvision(seed):
    """Box pairs whose fp32 IoU rounds differently with and without the fused area sum, with the threshold between the
    two values: only torchvision's exact arithmetic gives the reference's decision."""
    a, b, thr = fma_sensitive_pair(seed)
    fused = bool(iou_f32(a, b, True) > thr)
    assert fused != bool(iou_f32(a, b, False) > thr)
    boxes = torch.tensor(np.stack((a, b)))
    got = _direct_v4(boxes, torch.full((2,), 4.0), torch.tensor([[3.0], [2.0]]), thr, 0.05)
    assert len(got["scores"]) == (1 if fused else 2)


def test_torchvision_nms_keeps_equal_scores_in_candidate_order():
    """The tie rule the kernels reproduce: torchvision's CUDA nms sorts with a stable descending sort."""
    boxes = torch.tensor([[0.1 * i, 0, 0.1 * i + 0.05, 0.05] for i in range(300)], device=DEV)
    scores = torch.full((300,), 0.25, device=DEV)
    assert torch.equal(nms(boxes, scores, 0.5), torch.arange(300, device=DEV))


@pytest.mark.parametrize("mode", ["exact", "ulp"])
def test_equal_and_near_equal_scores(mode):
    """Class probabilities given directly (YOLOv2's post_process takes them as they are): all equal, or in groups one
    ulp apart."""
    gen = torch.Generator().manual_seed(6)
    n = 700
    model = _V2(4, torch.ones(1, 2) / 13, rpn_nms_thresh=0.3).to(DEV)
    b_coords = torch.cat((torch.rand(1, n, 2, generator=gen) * 0.8 + 0.1,
                          torch.rand(1, n, 2, generator=gen) * 0.2 + 0.05), dim=-1).to(DEV)
    b_o = torch.ones(1, n, device=DEV)
    b_scores = torch.full((1, n, 4), 0.1, device=DEV)
    b_scores[..., 1] = 0.5
    if mode == "ulp":
        up = torch.nextafter(torch.tensor(0.5), torch.tensor(1.0)).item()
        b_scores[0, ::3, 1] = up
    got = model.post_process(b_coords, b_o, b_scores, (1, n), model.rpn_nms_thresh, model.box_score_thresh)
    xyxy = model.to_isoboxes(b_coords, (1, n), clamp=True)
    _assert_same(got, _ref_v12(xyxy, b_o, b_scores, model.rpn_nms_thresh, model.box_score_thresh))
    assert 1 < len(got[0]["scores"]) < n


@pytest.mark.parametrize("b", [1, 8])
def test_zero_score_threshold_and_unit_nms_threshold(b):
    gen = torch.Generator().manual_seed(7)
    model = _V1(20, 2, rpn_nms_thresh=1.0, box_score_thresh=0.0).to(DEV)
    raw = _v1_raw(b, 20, 2, gen)
    got = _check_v12(model, raw, v1=True)
    b_o = model._format_outputs(raw)[1].reshape(b, -1)
    assert [len(d["scores"]) for d in got] == (b_o >= 0.5).sum(1).tolist()


# ---- models end to end -------------------------------------------------------------------------------------------
def _run_twice(model, x):
    with torch.no_grad():
        a, c = model(x), model(x)
    _assert_same(a, c)
    return a


def test_yolov1_end_to_end():
    torch.manual_seed(0)
    model = yolov1(num_classes=3).to(DEV).eval()
    x = torch.rand(2, 3, 448, 448, device=DEV)
    got = _run_twice(model, x)
    with torch.no_grad():
        b_coords, b_o, b_scores, grid = _v12_inputs(model, model._forward(x), v1=True)
        xyxy = model.to_isoboxes(b_coords.reshape(-1, *grid, 2, 4), grid, clamp=True).reshape(2, -1, 4)
        _assert_same(got, _ref_v12(xyxy, b_o, b_scores, model.rpn_nms_thresh, model.box_score_thresh))
        padded = model.detect_padded(x)
    _assert_same(to_detections(*padded), got)


def test_yolov2_end_to_end():
    torch.manual_seed(0)
    model = yolov2(num_classes=3).to(DEV).eval()
    x = torch.rand(2, 3, 416, 416, device=DEV)
    got = _run_twice(model, x)
    with torch.no_grad():
        b_coords, b_o, b_scores, grid = _v12_inputs(model, model._forward(x), v1=False)
        xyxy = model.to_isoboxes(b_coords, grid, clamp=True).reshape(2, -1, 4)
        _assert_same(got, _ref_v12(xyxy, b_o, b_scores, model.rpn_nms_thresh, model.box_score_thresh))
        padded = model.detect_padded(x)
    _assert_same(to_detections(*padded), got)


@pytest.mark.parametrize("perturb", [False, True])
def test_yolov4_end_to_end(perturb):
    torch.manual_seed(0)
    model = yolov4(num_classes=3).to(DEV).eval()
    if perturb:      # the output convolutions start at zero: give them weights so that scores differ
        for head in (model.head.head1, model.head.head2_2, model.head.head3):
            torch.nn.init.normal_(head[-1].weight, std=0.05)
            torch.nn.init.normal_(head[-1].bias, std=1.0)
    x = torch.rand(2, 3, 256, 256, device=DEV)
    got = _run_twice(model, x)
    layers = (model.head.yolo1, model.head.yolo2, model.head.yolo3)
    with torch.no_grad():
        outs = model.head._heads(list(model.neck(model.backbone(x))))
        per_scale = [_ref_v4(*layer._format_outputs(o), layer.rpn_nms_thresh, layer.box_score_thresh)
                     for layer, o in zip(layers, outs)]
        padded = model.detect_padded(x)
    want = [{k: torch.cat([d[k] for d in ds], dim=0) for k in ("boxes", "scores", "labels")} for ds in zip(*per_scale)]
    _assert_same(got, want)
    _assert_same(to_detections(*padded), got)


# ---- CUDA-graph capture --------------------------------------------------------------------------------------------
def test_detect_padded_kernels_capture_and_replay():
    gen = torch.Generator().manual_seed(8)
    layers = _layers(5)

    def step(*raws):
        return detect_padded([layer._segment(*layer._format_outputs(r), layer.rpn_nms_thresh, layer.box_score_thresh)
                              for layer, r in zip(layers, raws)])

    first = [_v4_raw(4, 5, hw, gen) for hw in (16, 8, 4)]
    graphed = GraphedTrainStep(step, first, warmup=2)
    for _ in range(2):
        raws = [_v4_raw(4, 5, hw, gen) for hw in (16, 8, 4)]
        replayed = [t.clone() for t in graphed(*raws)]
        eager = step(*raws)
        for r, e in zip(replayed, eager):
            assert torch.equal(r, e)
        _check_v4(layers, raws)


def test_yolov4_detect_padded_capture_and_replay():
    torch.manual_seed(1)
    model = yolov4(num_classes=3).to(DEV).eval()
    for head in (model.head.head1, model.head.head2_2, model.head.head3):
        torch.nn.init.normal_(head[-1].weight, std=0.05)
        torch.nn.init.normal_(head[-1].bias, std=1.0)

    def step(x):
        with torch.no_grad():
            return model.detect_padded(x)

    graphed = GraphedTrainStep(step, [torch.rand(2, 3, 256, 256, device=DEV)], warmup=2)
    x = torch.rand(2, 3, 256, 256, device=DEV)
    replayed = [t.clone() for t in graphed(x)]
    for r, e in zip(replayed, step(x)):
        assert torch.equal(r, e)
    with torch.no_grad():
        _assert_same(to_detections(*replayed), model(x))


# ---- dtypes other than fp32 ----------------------------------------------------------------------------------------
def test_yolov1_eval_under_bf16_autocast():
    """DetectionTrainer(amp=True).evaluate's forward: YOLOv1's head gives bf16 boxes and objectness, fp32 softmax."""
    torch.manual_seed(0)
    model = yolov1(num_classes=3).to(DEV).eval()
    x = torch.rand(2, 3, 448, 448, device=DEV)
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        got = model(x)
        b_coords, b_o, b_scores, grid = _v12_inputs(model, model._forward(x), v1=True)
        assert b_o.dtype == torch.bfloat16 and b_scores.dtype == torch.float32
        xyxy = model.to_isoboxes(b_coords.reshape(-1, *grid, 2, 4), grid, clamp=True).reshape(2, -1, 4)
        want = _ref_v12(xyxy, b_o, b_scores, model.rpn_nms_thresh, model.box_score_thresh)
    _assert_same(got, want)


@pytest.mark.parametrize("dtypes", [("bf16", "f32"), ("f32", "f16"), ("f16", "f16"), ("bf16", "bf16"), ("f64", "f64")])
def test_v1_post_process_dtypes(dtypes):
    """Objectness / class-score dtypes: the kernels where they reproduce the loop (widening to an fp32 product), the
    loop otherwise; images without any candidate past objectness keep the reference's empty dtype."""
    dt = {"f32": torch.float32, "bf16": torch.bfloat16, "f16": torch.float16, "f64": torch.float64}
    gen = torch.Generator().manual_seed(9)
    model = _V1(6, 2).to(DEV)
    b_coords, b_o, b_scores, grid = _v12_inputs(model, _v1_raw(4, 6, 2, gen), v1=True)
    b_o = b_o.clone()
    b_o[2] = 0.25                                    # image 2: nothing past objectness
    b_o, b_scores = b_o.to(dt[dtypes[0]]), b_scores.to(dt[dtypes[1]])
    b_coords = b_coords.to(torch.float64) if dtypes[0] == "f64" else b_coords
    got = model.post_process(b_coords, b_o, b_scores, grid, model.rpn_nms_thresh, model.box_score_thresh)
    xyxy = model.to_isoboxes(b_coords.reshape(-1, *grid, 2, 4), grid, clamp=True).reshape(4, -1, 4)
    want = _ref_v12(xyxy, b_o, b_scores, model.rpn_nms_thresh, model.box_score_thresh)
    _assert_same(got, want)
    assert got[2]["scores"].dtype == b_o.dtype and len(got[2]["scores"]) == 0


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float64])
def test_v4_post_process_dtypes(dtype):
    gen = torch.Generator().manual_seed(10)
    layer = _layers(4)[0]
    boxes, b_o, b_scores = layer._format_outputs(_v4_raw(3, 4, 8, gen))
    cases = [(boxes, b_o.to(dtype), b_scores), (boxes, b_o.to(dtype), b_scores.to(dtype))]
    if dtype != torch.bfloat16:                      # torchvision's nms takes no bf16 boxes
        cases.append((boxes.to(dtype), b_o.to(dtype), b_scores.to(dtype)))
    for args in cases:
        _assert_same(YoloLayer.post_process(*args, 0.7, 0.05), _ref_v4(*args, 0.7, 0.05))
