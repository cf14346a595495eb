"""Host side of the batched ground-truth matching (holocron_b200.trainer.assign_iou_batch, hb_assign_iou_batch in
csrc/boxes.cu), without a device: the descriptor rows, the fp32 rounding of the threshold, the refusals, and
DetectionTrainer.evaluate keeping the per-image loop for CPU batches. The kernel itself: tests/test_gpu_assign_batch.py."""
import ctypes
import math
import re
from pathlib import Path

import numpy as np
import pytest
import torch

import _trainer_cases as cases
from conftest import load_golden
from holocron_b200 import HolocronB200Error, _lib
from holocron_b200.trainer import DetectionTrainer, assign_iou_batch, trainers

BUILD = Path(__file__).resolve().parents[1] / "holocron_b200" / "csrc" / "build"


def test_descriptor_rows_read_boxes_and_labels_in_place():
    g0 = torch.rand(3, 6, dtype=torch.float64)[:, :4]         # [n, 6] view: row stride 6
    p0 = torch.rand(4, 4, dtype=torch.bfloat16).t()            # transposed: column stride 4
    g1 = torch.zeros(0, 4)
    p1 = torch.rand(5, 4, dtype=torch.float16)
    g2 = torch.rand(2, 4)
    p2 = torch.zeros(0, 4)
    gl = [torch.arange(6, dtype=torch.int32)[::2], torch.zeros(0, dtype=torch.int64), torch.tensor([1, 2])]
    pl = [torch.tensor([0, 1, 2, 3]), torch.arange(5, dtype=torch.int32), torch.zeros(0, dtype=torch.int32)]
    table, ns = trainers._match_table([g0, g1, g2], [p0, p1, p2], gl, pl)
    assert ns == [3, 0, 2]
    assert table.dtype == np.int64 and table.shape == (3, 16)
    want = [
        [g0.data_ptr(), p0.data_ptr(), gl[0].data_ptr(), pl[0].data_ptr(), 3, 4, 6, 1, 1, 4, 2, 1,
         4 | 1 << 8 | 1 << 16 | 0 << 24, 0],
        [g1.data_ptr(), p1.data_ptr(), gl[1].data_ptr(), pl[1].data_ptr(), 0, 5, 4, 1, 4, 1, 1, 1,
         0 | 2 << 8 | 0 << 16 | 1 << 24, 3],
        [g2.data_ptr(), p2.data_ptr(), gl[2].data_ptr(), pl[2].data_ptr(), 2, 0, 4, 1, 4, 1, 1, 1,
         0 | 0 << 8 | 0 << 16 | 1 << 24, 3],
    ]
    assert table[:, :14].tolist() == want
    assert not table[:, 14:].any()
    # without labels: no label addresses, strides or codes
    table, ns = trainers._match_table([g0, g1], [p0, p1], None, None)
    assert ns == [3, 0]
    assert not table[:, [2, 3, 10, 11]].any()
    assert table[:, 12].tolist() == [4 | 1 << 8, 0 | 2 << 8]
    assert table[:, 13].tolist() == [0, 3]


def test_threshold_is_rounded_to_fp32_as_torch_rounds_a_scalar():
    assert _lib.SIGNATURES["hb_assign_iou_batch"][2] == "f"
    v = float(np.float32(0.7))
    above = math.nextafter(v, 1.0)                             # rounds back to v in fp32
    for thr in (0.5, 0.7, 0.1, 1 / 3, v, above, 1e-45, 1e40, -0.0, float("inf"), float("nan")):
        f = ctypes.c_float(thr).value
        assert (math.isnan(f) and math.isnan(thr)) or f == float(torch.tensor(thr, dtype=torch.float32)), thr
    assert ctypes.c_float(above).value == v
    # an fp32 IoU equal to fp32(0.7) passes 0.7 although fp32(0.7) < 0.7, as in torch
    assert bool((torch.tensor([v]) >= 0.7).item()) and v < 0.7
    assert bool((torch.tensor([v]) >= above).item())


def _boxes(n, dtype=torch.float32):
    return torch.rand(n, 4, dtype=dtype)


@pytest.mark.parametrize("case", ["lengths", "shape", "width", "gt_labels", "pred_labels", "labels_one_side",
                                  "devices"])
def test_malformed_batches_are_refused(case):
    g, p = [_boxes(2)], [_boxes(3)]
    gl, pl = [torch.zeros(2, dtype=torch.int64)], [torch.zeros(3, dtype=torch.int64)]
    if case == "lengths":
        p = p + p
    elif case == "shape":
        g = [torch.rand(2, 4, 1)]
    elif case == "width":
        p = [torch.rand(3, 5)]
    elif case == "gt_labels":
        gl = [torch.zeros(3, dtype=torch.int64)]
    elif case == "pred_labels":
        pl = [torch.zeros(2, 1, dtype=torch.int64)]
    elif case == "labels_one_side":
        pl = None
    elif case == "devices":
        p = [torch.empty(3, 4, device="meta")]
    with pytest.raises(ValueError):
        trainers._match_table(g, p, gl, pl)


def test_unsupported_dtypes_are_refused():
    with pytest.raises(TypeError):
        trainers._match_table([torch.zeros(1, 4, dtype=torch.int32)], [_boxes(1)], None, None)
    with pytest.raises(TypeError):
        trainers._match_table([_boxes(1)], [_boxes(1)], [torch.zeros(1, dtype=torch.uint8)], [torch.zeros(1).long()])


def test_cpu_tensors_raise():
    with pytest.raises(HolocronB200Error):
        assign_iou_batch([_boxes(2)], [_boxes(3)])
    with pytest.raises(HolocronB200Error):
        trainers._assign_batch([_boxes(2)], [_boxes(3)], 0.5, [torch.zeros(2).long()], [torch.zeros(3).long()])
    assert assign_iou_batch([], []) == []


def test_matchable_needs_one_cuda_device_and_kernel_dtypes():
    loader, detections = cases.det_data()
    assert not trainers._matchable(loader[0][1], detections[:2], None)
    meta = lambda d: {k: torch.empty(v.shape, dtype=v.dtype, device="meta") for k, v in d.items()}   # noqa: E731
    assert not trainers._matchable([meta(t) for t in loader[0][1]], [meta(d) for d in detections[:2]], None)
    assert not trainers._matchable([], [], None)


def test_evaluate_keeps_the_per_image_loop_for_cpu_batches(monkeypatch):
    def refuse(*args, **kwargs):
        raise AssertionError("CPU batches must not reach the kernel path")

    monkeypatch.setattr(trainers, "_assign_batch", refuse)
    loader, detections = cases.det_data()
    model = cases.FixedDetector(detections)
    tr = DetectionTrainer(model, loader, loader, None, torch.optim.SGD(model.parameters(), lr=1e-2), gpu=None)
    got = tr.evaluate()
    want = load_golden("trainers")["detection"]["metrics"]
    assert set(got) == set(want)
    for k in want:
        assert math.isclose(got[k], want[k], rel_tol=1e-12, abs_tol=1e-12), (k, got[k], want[k])


def test_match_kernel_does_not_spill():
    log = BUILD / "boxes.log"
    if not log.exists():
        pytest.skip(f"{log.name} absent: build the library first (python -m holocron_b200.csrc.build)")
    text = log.read_text()
    m = re.search(r"Compiling entry function '(\w*match_kernel\w*)'.*?\n(.*?spill loads)", text, flags=re.S)
    assert m, "no ptxas -v output for match_kernel"
    assert "0 bytes spill stores, 0 bytes spill loads" in m.group(2)
