"""Batched ground-truth matching (hb_assign_iou_batch in csrc/boxes.cu, holocron_b200.trainer.assign_iou_batch) against
assign_iou, image by image: on CPU tensors (torchvision's box_iou on the fp32 boxes) and on CUDA tensors (the pairwise
IoU kernel). Every match vector must equal the one built from assign_iou's pairs, element for element, and the
{assigned, correct} counts the per-image loop of DetectionTrainer.evaluate would find. DetectionTrainer.evaluate on CUDA
batches must return the CPU run's dict bit for bit with one synchronisation per call."""
import math
import warnings

import pytest
import torch

import _trainer_cases as cases
from conftest import load_golden
from holocron_b200._lib import lib
from holocron_b200.trainer import DetectionTrainer, assign_iou, assign_iou_batch, trainers

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")


def _ref_match(g, p, thr):
    """The match vector of assign_iou's pairs: the prediction of each ground-truth box, or -1."""
    m = torch.full((g.shape[0],), -1, dtype=torch.int64)
    if g.shape[0] and p.shape[0]:
        gi, pi = assign_iou(g, p, thr)
        for a, b in zip(gi, pi):
            m[int(a)] = int(b)
    kept = m[m >= 0]
    assert kept.unique().numel() == kept.numel()           # one ground truth per prediction at most
    return m


def _check(gts, preds, thr):
    """gts / preds: device tensors (any box dtype and strides)."""
    got = assign_iou_batch(gts, preds, thr)
    assert len(got) == len(gts)
    for i, (g, p, m) in enumerate(zip(gts, preds, got)):
        assert m.dtype == torch.int64 and m.device == g.device and m.shape == (g.shape[0],), i
        m = m.cpu()
        want = _ref_match(g.float().cpu(), p.float().cpu(), thr)
        assert torch.equal(m, want), (i, "cpu", (m != want).nonzero().flatten()[:8].tolist())
        assert torch.equal(m, _ref_match(g, p, thr).cpu()), (i, "cuda")
    return got


def _check_counts(gts, preds, gl, pl, thr):
    """The {assigned, correct} counts, added twice into one accumulator, against the reference matches."""
    counts = torch.zeros(2, dtype=torch.int64, device=DEV)
    for _ in range(2):
        match, ns = trainers._assign_batch(gts, preds, thr, gl, pl, counts)
    assigned = correct = 0
    for g, p, a, b, m in zip(gts, preds, gl, pl, match.cpu().split(ns)):
        want = _ref_match(g.float().cpu(), p.float().cpu(), thr)
        assert torch.equal(m, want)
        k = want >= 0
        assigned += int(k.sum())
        correct += int((a.cpu().long()[k] == b.cpu().long()[want[k]]).sum())
    assert counts.tolist() == [2 * assigned, 2 * correct]


def _grid_boxes(n, g, dups=True):
    """Corners on a 1/8 grid (equal IoUs everywhere, zero-area boxes), a third of the rows duplicated."""
    c = torch.randint(0, 9, (n, 4), generator=g).float() / 8
    b = torch.stack([torch.minimum(c[:, 0], c[:, 2]), torch.minimum(c[:, 1], c[:, 3]),
                     torch.maximum(c[:, 0], c[:, 2]), torch.maximum(c[:, 1], c[:, 3])], 1)
    if dups and n > 1:
        b[torch.randint(0, n, (n // 3,), generator=g)] = b[torch.randint(0, n, (n // 3,), generator=g)]
    return b


def _voc_boxes(n, g):
    """Relative xyxy boxes of VOC-like sizes."""
    xy = torch.rand(n, 2, generator=g) * 0.8
    wh = 0.02 + torch.rand(n, 2, generator=g) * 0.5
    return torch.cat([xy, (xy + wh).clamp(max=1.0)], 1)


def _grid_batch(seed, n_img, max_gt=40, max_pred=300):
    g = torch.Generator().manual_seed(seed)
    gts, preds = [], []
    for _ in range(n_img):
        gts.append(_grid_boxes(int(torch.randint(0, max_gt + 1, (1,), generator=g)), g))
        preds.append(_grid_boxes(int(torch.randint(0, max_pred + 1, (1,), generator=g)), g))
    return gts, preds


def _dev(boxes, dtype=torch.float32):
    return [b.to(DEV, dtype) for b in boxes]


@pytest.mark.parametrize("thr", [0.5, 0.0, 0.3, 0.75, 1.0])
def test_grid_boxes_with_ties(thr):
    gts, preds = _grid_batch(1, 16)
    _check(_dev(gts), _dev(preds), thr)


def test_iou_exactly_at_the_threshold():
    g = torch.tensor([[0.0, 0.0, 1.0, 1.0], [0.0, 0.0, 1.0, 1.0], [2.0, 2.0, 3.0, 3.0]])
    p = torch.tensor([[0.0, 0.0, 1.0, 0.25], [0.0, 0.0, 1.0, 0.5], [2.0, 2.0, 3.0, 2.5], [0.0, 0.0, 1.0, 0.5]])
    got = _check(_dev([g]), _dev([p]), 0.5)
    assert got[0].tolist() == [1, -1, 2]                       # IoU 0.5 is kept; the lower target keeps the tie


def test_threshold_equal_to_an_iou_and_the_double_above_it():
    gts, preds = _grid_batch(2, 8, 30, 60)
    ious = torch.cat([trainers._pairwise_iou(a, b).flatten() for a, b in zip(gts, preds) if a.numel() and b.numel()])
    ious = ious[torch.isfinite(ious) & (ious > 0.2)]
    for v in ious.unique()[::7][:6].tolist():
        above = math.nextafter(v, 2.0)
        assert float(torch.tensor(above, dtype=torch.float32)) == v
        _check(_dev(gts), _dev(preds), v)
        _check(_dev(gts), _dev(preds), above)
    # fp32(0.7) < 0.7, and an IoU of fp32(0.7) passes 0.7 as it does in torch
    v = float(torch.tensor(0.7, dtype=torch.float32))
    g = torch.tensor([[0.0, 0.0, 1.0, 1.0]])
    p = torch.tensor([[0.0, 0.0, 1.0, v]])
    assert float(trainers._pairwise_iou(g, p)) == v
    assert _check(_dev([g]), _dev([p]), 0.7)[0].tolist() == [0]


def test_nan_inf_zero_area_and_inverted_boxes():
    nan, inf = float("nan"), float("inf")
    g = torch.tensor([[0.0, 0.0, 1.0, 1.0], [nan, 0.0, 1.0, 1.0], [0.5, 0.5, 0.5, 0.5], [0.0, 0.0, inf, 1.0],
                      [0.2, 0.2, 0.2, 0.6], [1.0, 1.0, 0.0, 0.0], [-inf, -inf, inf, inf], [0.0, 0.0, 1.0, 1.0],
                      [0.25, 0.25, 0.75, 0.75]])
    p = torch.tensor([[0.5, 0.5, 0.5, 0.5], [0.0, 0.0, 1.0, 1.0], [0.0, 0.0, 1.0, nan], [0.0, 0.0, inf, 1.0],
                      [1.0, 1.0, 0.0, 0.0], [0.25, 0.25, 0.75, 0.75], [inf, 0.0, inf, 1.0], [0.2, 0.2, 0.2, 0.6]])
    for thr in (0.5, 0.0, -1.0, float("-inf"), float("nan")):
        _check(_dev([g, p, g]), _dev([p, g, p[:1]]), thr)
    gts, preds = _grid_batch(3, 8, 20, 40)
    gen = torch.Generator().manual_seed(4)
    for b in gts + preds:
        if b.shape[0]:
            i = torch.randint(0, b.shape[0], (max(1, b.shape[0] // 5),), generator=gen)
            b[i, torch.randint(0, 4, (i.numel(),), generator=gen)] = torch.tensor([nan, inf, -inf, 0.0])[
                torch.randint(0, 4, (i.numel(),), generator=gen)]
    _check(_dev(gts), _dev(preds), 0.25)


def test_empty_images_and_empty_batches():
    gts, preds = _grid_batch(5, 6, 10, 20)
    gts[1] = torch.zeros(0, 4)
    preds[2] = torch.zeros(0, 4)
    gts[3], preds[3] = torch.zeros(0, 4), torch.zeros(0, 4)
    got = _check(_dev(gts), _dev(preds), 0.5)
    assert got[1].numel() == 0 and (got[2] == -1).all()
    got = _check(_dev([torch.zeros(0, 4)] * 3), _dev([torch.zeros(0, 4)] * 3), 0.5)
    assert [m.numel() for m in got] == [0, 0, 0]
    n = lib().hb_launch_count()
    assert assign_iou_batch([], []) == []
    assert lib().hb_launch_count() == n


def test_256_images_in_one_launch():
    gts, preds = _grid_batch(6, 256, 12, 40)
    n = lib().hb_launch_count()
    got = assign_iou_batch(_dev(gts), _dev(preds), 0.5)
    assert lib().hb_launch_count() - n == 1
    assert len(got) == 256
    _check(_dev(gts), _dev(preds), 0.5)


def test_one_image_with_1000_targets_and_10000_predictions():
    g = torch.Generator().manual_seed(7)
    gt = _voc_boxes(1000, g)
    pred = (gt[torch.randint(0, 1000, (10000,), generator=g)] + 0.03 * torch.randn(10000, 4, generator=g))
    pred = torch.round(pred * 64) / 64                          # ties among the jittered copies
    got = _check(_dev([gt]), _dev([pred]), 0.5)
    assert (got[0] >= 0).sum() > 500


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float64])
def test_prediction_and_target_dtypes(dtype):
    g = torch.Generator().manual_seed(8)
    gts = [_voc_boxes(int(n), g) for n in torch.randint(0, 30, (8,), generator=g)]
    preds = [torch.cat([a + 0.02 * torch.randn_like(a), _voc_boxes(20, g)]) for a in gts]
    _check(_dev(gts), _dev(preds, dtype), 0.5)
    _check(_dev(gts, dtype), _dev(preds), 0.5)
    _check(_dev(gts, torch.float64), _dev(preds, dtype), 0.5)


def test_strided_views():
    gts, preds = _grid_batch(9, 8, 20, 50)
    wide = lambda b: torch.cat([b, torch.rand(b.shape[0], 2)], 1).to(DEV)[:, :4]    # noqa: E731
    g6, p6 = [wide(b) for b in gts], [wide(b) for b in preds]
    assert g6[0].stride() == (6, 1)
    _check(g6, p6, 0.5)
    pt = [b.to(DEV).t().contiguous().t() for b in preds]       # column stride n
    _check(g6, pt, 0.5)


@pytest.mark.parametrize("label_dtypes", [(torch.int64, torch.int64), (torch.int32, torch.int64),
                                          (torch.int64, torch.int32), (torch.int32, torch.int32)])
def test_counts_with_int32_and_int64_labels(label_dtypes):
    gts, preds = _grid_batch(10, 32, 40, 120)
    g = torch.Generator().manual_seed(11)
    gl = [torch.randint(0, 3, (b.shape[0],), generator=g).to(DEV, label_dtypes[0]) for b in gts]
    pl = [torch.randint(0, 3, (b.shape[0],), generator=g).to(DEV, label_dtypes[1]) for b in preds]
    _check_counts(_dev(gts), _dev(preds), gl, pl, 0.25)
    pl = [torch.arange(0, 4 * b.shape[0], 2, device=DEV).to(label_dtypes[1])[::2] for b in preds]   # strided labels
    _check_counts(_dev(gts), _dev(preds), [torch.zeros_like(a) for a in gl], pl, 0.25)


def test_refusals_before_any_launch():
    g, p = _dev([torch.rand(3, 4)]), _dev([torch.rand(5, 4)])
    n = lib().hb_launch_count()
    with pytest.raises(ValueError):
        assign_iou_batch(g, _dev([torch.rand(5, 3)]))
    with pytest.raises(ValueError):
        assign_iou_batch(g, p + p)
    with pytest.raises(ValueError):
        trainers._assign_batch(g, p, 0.5, [torch.zeros(2, dtype=torch.int64, device=DEV)],
                               [torch.zeros(5, dtype=torch.int64, device=DEV)])
    if torch.cuda.device_count() > 1:
        with pytest.raises(ValueError):
            assign_iou_batch(g, [p[0].to("cuda:1")])
    assert lib().hb_launch_count() == n


def test_no_host_synchronisation():
    gts, preds = _grid_batch(12, 32, 40, 300)
    gts, preds = _dev(gts), _dev(preds)
    assign_iou_batch(gts, preds)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        got = assign_iou_batch(gts, preds)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    want = assign_iou_batch(gts, preds)
    assert all(torch.equal(a, b) for a, b in zip(got, want))


# ---- DetectionTrainer.evaluate ----------------------------------------------------------------------------------------
def _on(dev, loader, detections):
    return ([([x.to(dev) for x in xs], [{k: v.to(dev) for k, v in t.items()} for t in ts]) for xs, ts in loader],
            [{k: v.to(dev) for k, v in d.items()} for d in detections])


def _evaluate(loader, detections):
    """evaluate() with the number of synchronising calls it made."""
    model = cases.FixedDetector(detections)
    tr = DetectionTrainer(model, loader, loader, None, torch.optim.SGD(model.parameters(), lr=1e-2), gpu=None)
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            out = tr.evaluate()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    return out, sum("synchroniz" in str(w.message) for w in caught)


def _random_det_data(seed, n_batches=3, batch=4, classes=4):
    g = torch.Generator().manual_seed(seed)
    loader, detections = [], []
    for _ in range(n_batches):
        xs, ts = [], []
        for _ in range(batch):
            n = int(torch.randint(0, 12, (1,), generator=g))
            gt = _voc_boxes(n, g)
            k = int(torch.randint(0, 20, (1,), generator=g)) if n else 0
            near = gt[torch.randint(0, max(n, 1), (k,), generator=g)] + 0.04 * torch.randn(k, 4, generator=g)
            pred = torch.round(torch.cat([near, _voc_boxes(int(torch.randint(0, 6, (1,), generator=g)), g)]) * 32) / 32
            xs.append(torch.rand(3, 8, 8, generator=g))
            ts.append({"boxes": gt, "labels": torch.randint(0, classes, (n,), generator=g)})
            detections.append({"boxes": pred, "scores": torch.rand(pred.shape[0], generator=g),
                               "labels": torch.randint(0, classes, (pred.shape[0],), generator=g)})
        loader.append((xs, ts))
    return loader, detections


def test_evaluate_on_cuda_matches_cpu_and_golden_with_one_synchronisation():
    loader, detections = cases.det_data()
    want, _ = _evaluate(loader, detections)
    got, syncs = _evaluate(*_on(DEV, loader, detections))
    assert got == want
    assert syncs == 1
    golden = load_golden("trainers")["detection"]["metrics"]
    assert set(got) == set(golden)
    for k in golden:
        assert math.isclose(got[k], golden[k], rel_tol=1e-12, abs_tol=1e-12), (k, got[k], golden[k])


@pytest.mark.parametrize("seed", [0, 1])
def test_evaluate_on_random_cuda_batches(seed):
    loader, detections = _random_det_data(seed)
    want, _ = _evaluate(loader, detections)
    got, syncs = _evaluate(*_on(DEV, loader, detections))
    assert got == want
    assert syncs == 1
    assert want["clf_err"] is not None and 0 < want["loc_err"] < 1
