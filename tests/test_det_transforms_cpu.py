"""holocron_b200.transforms.detection without a GPU: signatures and ``repr`` against the reference's; the per-image
oracle (tests/_det_transforms_oracle.py) and this module's plan (draws, sizes, box ops and parameter rows run through
a CPU restatement of the box kernel) against the reference's record (tests/golden/det_transforms.pt, written by
make_golden_det_transforms.py from the unmodified reference), boxes and labels bit for bit; the fold of CenterCrop and
flips against torchvision on an index image; VOC parsing; the refusals before any draw; the result forms; and the
ptxas report of the box kernel."""
import inspect
import itertools
import re
from pathlib import Path

import numpy as np
import pytest
import torch
import torchvision.transforms.functional as TF
from PIL import Image
from torchvision.transforms import transforms as TT

import _det_transforms_oracle as DO
from holocron_b200 import HolocronB200Error
from holocron_b200.transforms import ColorJitter, _boxes
from holocron_b200.transforms import _fold
from holocron_b200.transforms import detection as D

ROOT = Path(__file__).resolve().parents[1]
G = torch.load(ROOT / "tests" / "golden" / "det_transforms.pt", weights_only=False)
LOG = ROOT / "holocron_b200" / "csrc" / "build" / "boxes.log"


def build(name, args):
    if name == "ImageTransform":
        inner, inner_args = args
        return D.ImageTransform(getattr(TT, inner)(*inner_args))
    if name == "convert_to_relative":
        return D.convert_to_relative
    return getattr(D, name)(*args)


def _signature(obj):
    out = []
    for name, p in inspect.signature(obj.__init__ if inspect.isclass(obj) else obj).parameters.items():
        if name != "self":
            out.append([name, p.kind.name, None if p.default is inspect.Parameter.empty else repr(p.default)])
    return out


@pytest.mark.parametrize("name", sorted(G["signatures"]))
def test_signatures(name):
    assert _signature(getattr(D, name)) == G["signatures"][name]


def test_reprs():
    for name, args, text in G["reprs"]:
        assert repr(build(name, args)) == text


class DrawLog:
    """Records torch.randint / torch.rand calls and RandomResizedCrop.get_params results as the golden generator
    records them."""

    def __init__(self, monkeypatch):
        self.calls = []
        randint, rand, get_params = torch.randint, torch.rand, TT.RandomResizedCrop.get_params

        def log_randint(*args, **kwargs):
            out = randint(*args, **kwargs)
            self.calls.append(("randint", tuple(int(a) if isinstance(a, int) else tuple(a) for a in args),
                               out.tolist()))
            return out

        def log_rand(*args, **kwargs):
            out = rand(*args, **kwargs)
            self.calls.append(("rand", tuple(tuple(a) if isinstance(a, (tuple, list)) else a for a in args),
                               out.tolist()))
            return out

        def log_get_params(img, scale, ratio):
            out = get_params(img, scale, ratio)
            self.calls.append(("get_params", (tuple(scale), tuple(ratio)), tuple(int(v) for v in out)))
            return out
        monkeypatch.setattr(torch, "randint", log_randint)
        monkeypatch.setattr(torch, "rand", log_rand)
        monkeypatch.setattr(TT.RandomResizedCrop, "get_params", staticmethod(log_get_params))


def _records():
    for name, records in G["chains"].items():
        for rec in records:
            yield f"{name}-{rec['seed']}", rec


KEYS = [k for k, _ in _records()]


def _target(t):
    return {"boxes": t["boxes"].clone(), "labels": t["labels"].clone()} if "boxes" in t else t


@pytest.mark.parametrize("key", KEYS)
def test_oracle_matches_reference(key, monkeypatch):
    """The oracle, image by image on CPU tensors: boxes and labels bit for bit, the draws, the image size after the
    chain and the generator state."""
    rec = dict(_records())[key]
    steps = [build(n, a) for n, a in rec["spec"]]
    torch.manual_seed(rec["seed"])
    for ((h, w), target), out in zip(rec["inputs"], rec["outputs"]):
        log = DrawLog(monkeypatch)
        image, got = DO.apply(steps, torch.zeros(3, h, w, dtype=torch.uint8), _target(target))
        monkeypatch.undo()
        assert log.calls == out["draws"]
        assert tuple(image.shape[-2:]) == out["after"][-1]
        assert got["boxes"].dtype == torch.float32 and got["labels"].dtype == torch.int64
        assert torch.equal(got["boxes"], out["boxes"].reshape(-1, 4)), (h, w)
        assert torch.equal(got["labels"], out["labels"])
    assert torch.equal(torch.get_rng_state(), rec["state"])


def emulate(boxes, labels, ops, row):
    """hb_box_transform_batch for one image, restated with torch fp32 ops on the CPU."""
    b, keep, q = boxes.clone(), torch.ones(len(boxes), dtype=torch.bool), 0
    for op in ops:
        p = row[q:q + _boxes.OPERANDS[op]]
        q += _boxes.OPERANDS[op]
        if op == _boxes.SCALE:
            b[:, [0, 2]] *= p[0]
            b[:, [1, 3]] *= p[1]
        elif op == _boxes.CLAMP:
            b[:, [0, 2]] = b[:, [0, 2]].clamp(p[0], p[1])
            b[:, [1, 3]] = b[:, [1, 3]].clamp(p[2], p[3])
        elif op == _boxes.SUB:
            b[:, [0, 2]] -= p[0]
            b[:, [1, 3]] -= p[1]
        elif op == _boxes.FILTER:
            keep &= (b[:, 0] != b[:, 2]) & (b[:, 1] != b[:, 3])
        elif op == _boxes.FLIP:
            if p[0] != 0:
                b = torch.stack([p[1] - b[:, 2], b[:, 1], p[1] - b[:, 0], b[:, 3]], 1)
        else:
            b[:, [0, 2]] /= p[0]
            b[:, [1, 3]] /= p[1]
    assert q == len(row)
    return b[keep], labels[keep]


def plan(steps, sizes):
    """This module's plan of a chain: (segments, ops, per-image (plan, row))."""
    if steps and isinstance(steps[0], D.VOCTargetTransform):
        steps = steps[1:]
    segments = _fold.group(steps, D._kind, D._starts_run, "detection")
    ops = [op for s in segments for t in (s if isinstance(s, list) else [s]) for op in D._box_ops(t)]
    jitters = _fold.jitters_of(segments, D.ImageTransform)
    return segments, ops, [D._draw(segments, jitters, size) for size in sizes]


@pytest.mark.parametrize("key", KEYS)
def test_plan_matches_reference(key, monkeypatch):
    """This module's draws (image by image), the size after each run, and the box kernel's ops and parameter rows run
    through the kernel's CPU restatement: boxes and labels bit for bit; then the generator state."""
    rec = dict(_records())[key]
    steps = [build(n, a) for n, a in rec["spec"]]
    voc = steps[0] if isinstance(steps[0], D.VOCTargetTransform) else None
    torch.manual_seed(rec["seed"])
    for ((h, w), target), out in zip(rec["inputs"], rec["outputs"]):
        log = DrawLog(monkeypatch)
        segments, ops, [(p, row)] = plan(steps, [(h, w)])
        monkeypatch.undo()
        assert log.calls == out["draws"], (h, w)
        ends = list(itertools.accumulate(len(s) if isinstance(s, list) else 1 for s in segments))
        for s, fold, end in zip(segments, p, ends):
            if isinstance(s, list):
                assert fold.canvas == out["after"][end - (0 if voc is None else -1) - 1]
        if voc is not None:
            bx, lab = voc.parse(target)
            boxes, labels = torch.tensor(bx, dtype=torch.float32).reshape(-1, 4), torch.tensor(lab)
        else:
            boxes, labels = target["boxes"], target["labels"]
        row = torch.tensor(row, dtype=torch.float64).tolist()
        assert all(np.float32(v) == v for v in row)  # operands are fp32 values
        b, lab = emulate(boxes, labels, ops, row)
        assert torch.equal(b, out["boxes"].reshape(-1, 4)) and torch.equal(lab, out["labels"])
    assert torch.equal(torch.get_rng_state(), rec["state"])


def test_quirks_on_record():
    """The reference's quirks as the record holds them, on a 400x300 (W x H) image."""
    flip = G["chains"]["flip"][0]
    (h, w), target = flip["inputs"][0]
    assert (h, w) == (300, 400)
    got = emulate(torch.tensor([[10., 20., 110., 220.]]), torch.tensor([0]), [_boxes.FLIP], [1.0, float(h)])[0]
    assert got.tolist() == [[190., 20., 290., 220.]]  # flipped around the height
    assert torch.equal(flip["outputs"][0]["boxes"][:, 0], h - target["boxes"][:, 2])
    _, ops, [(_, row)] = plan([D.CenterCrop(200)], [(300, 400)])
    assert ops == [_boxes.CLAMP, _boxes.SUB] and row == [0, 200, 0, 200, 0, 0]  # clamped, not shifted
    _, ops, [(_, row)] = plan([D.Resize([100, 200])], [(300, 400)])
    assert ops == [] and row == []
    _, ops, [(_, row)] = plan([D.Resize((100, 200))], [(300, 400)])
    assert ops == [_boxes.SCALE] and row == [0.25, float(np.float32(2 / 3))]


def _render(img, f):
    """A folded run without resize applied by indexing: the source (its ``box`` when given) placed at (top, left),
    the canvas mirrored when ``mirror``, 0 outside."""
    if f.box is not None:
        i, j, h, w = f.box
        img = img[..., i:i + h, j:j + w]
    Hc, Wc = f.canvas
    ys = torch.arange(Hc)[:, None] - f.top
    us = torch.arange(Wc)
    xs = ((Wc - 1 - us) if f.mirror else us)[None, :] - f.left
    live = (ys >= 0) & (ys < img.shape[-2]) & (xs >= 0) & (xs < img.shape[-1])
    out = img[..., ys.clamp(0, img.shape[-2] - 1), xs.clamp(0, img.shape[-1] - 1)]
    return torch.where(live, out, torch.zeros_like(out))


@pytest.mark.parametrize("order", [("crop",), ("flip", "crop"), ("crop", "flip"), ("flip", "crop", "flip")])
def test_center_crop_fold_matches_torchvision(order):
    """CenterCrop (larger, smaller, equal, odd differences) with flips around it: the fold applied by indexing equals
    torchvision's center_crop / hflip of an index image, with the same draws."""
    for (H, W), size, seed in itertools.product([(5, 7), (9, 4), (6, 6), (1, 8), (10, 12)],
                                                (1, 3, 6, 8, (4, 9), (11, 2)), range(3)):
        steps = [D.CenterCrop(size) if o == "crop" else D.RandomHorizontalFlip(0.5) for o in order]
        img = torch.arange(1, H * W + 1, dtype=torch.int64).view(1, H, W)
        torch.manual_seed(seed)
        fold = D.fold_run(steps, (H, W), [])
        state = torch.get_rng_state()
        torch.manual_seed(seed)
        want = img
        for t in steps:
            want = TF.center_crop(want, t.size) if isinstance(t, D.CenterCrop) else (
                TF.hflip(want) if torch.rand(1).item() < t.p else want)
        assert torch.equal(state, torch.get_rng_state())
        assert torch.equal(_render(img, fold), want), (H, W, size, seed, fold)


def test_fold_of_resizes():
    torch.manual_seed(3)
    fold = D.fold_run([D.RandomResizedCrop((40, 50)), D.RandomHorizontalFlip(1.0)], (300, 400), [])
    torch.manual_seed(3)
    i, j, h, w = TT.RandomResizedCrop.get_params(torch.empty(3, 300, 400), (0.08, 1.0), (3 / 4, 4 / 3))
    assert fold == _fold._Fold((40, 50), (40, 50), 0, 0, True, (i, j, h, w))
    assert D.fold_run([D.Resize(100)], (300, 400), []) == _fold._Fold((100, 133), (100, 133))
    assert D.fold_run([D.Resize([150])], (400, 300), []).canvas == (200, 150)


def test_segments():
    r, c, f, rc = D.Resize(8), D.CenterCrop(4), D.RandomHorizontalFlip(), D.RandomResizedCrop(6)
    rel, j = D.convert_to_relative, D.ImageTransform(ColorJitter(0.1))
    group = lambda ts: _fold.group(ts, D._kind, D._starts_run, "detection")  # noqa: E731
    assert group([r, f, rel, j]) == [[r, f, rel], j]
    assert group([rel, f, c, f, c, rc, f]) == [rel, [f, c, f], [c], [rc, f]]
    assert group([j, rel, f]) == [j, rel, [f]]
    for bad in (lambda x, y: (x, y), TT.ColorJitter(0.1)):
        with pytest.raises(TypeError):
            group([r, bad])


def _voc(objs):
    return {"annotation": {"object": [{"name": n, "bndbox": {"xmin": str(a), "ymin": str(b), "xmax": str(c),
                                                             "ymax": str(d)}} for n, (a, b, c, d) in objs]}}


def test_voc_parse():
    voc = D.VOCTargetTransform(["cat", "dog"])
    assert voc.parse(_voc([("dog", (1, 2, 30, 40)), ("cat", (0, 0, 5, 5))])) == ([[1, 2, 30, 40], [0, 0, 5, 5]],
                                                                                  [1, 0])
    assert voc.parse(_voc([])) == ([], [])
    with pytest.raises(KeyError):
        voc.parse(_voc([("bird", (1, 2, 3, 4))]))


@pytest.fixture
def planned(monkeypatch):
    """Runs Compose on CPU tensors, recording what each launch would be given; outputs are zeros of the launch's
    shape and the box kernel is its CPU restatement."""
    calls = []
    monkeypatch.setattr(D, "require_cuda", lambda *a: None)

    def fake_resample(sources, inner, canvas, interpolation, antialias, offsets, mirrors, canvases=None, boxes=None):
        calls.append({"resample": len(sources), "inner": inner, "canvas": canvas, "canvases": canvases,
                      "interpolation": interpolation, "antialias": antialias, "boxes": boxes})
        C, dtype = sources[0].shape[0], sources[0].dtype
        if canvas is not None:
            return torch.zeros(len(sources), C, *canvas, dtype=dtype)
        return [torch.zeros(C, *c, dtype=dtype) for c in canvases]

    def fake_boxes(boxes, labels, ops, params):
        calls.append({"boxes": len(boxes), "ops": ops})
        out = [emulate(b, lab, ops, row.tolist()) for b, lab, row in zip(boxes, labels, params)]
        return [o[0] for o in out], [o[1] for o in out]

    def fake_jitter(sources, draws):
        calls.append({"jitter": len(draws)})
        return torch.stack(list(sources))

    def fake_upload(device, boxes, labels):
        raise AssertionError("VOC targets are not uploaded by this fixture")

    monkeypatch.setattr(D, "resample", fake_resample)
    monkeypatch.setattr(D, "transform_boxes", fake_boxes)
    monkeypatch.setattr(D, "jitter", fake_jitter)
    monkeypatch.setattr(D, "_upload_voc", lambda parsed, device: (
        [torch.tensor(b, dtype=torch.float32).reshape(-1, 4) for b, _ in parsed],
        [torch.tensor(lab, dtype=torch.int64) for _, lab in parsed]))
    return calls


def _pairs(sizes, n=3, dtype=torch.uint8):
    images = [torch.zeros(3, h, w, dtype=dtype) for h, w in sizes]
    targets = [{"boxes": torch.tensor([[1., 2., 5., 6.]] * n), "labels": torch.arange(n), "image_id": k}
               for k in range(len(sizes))]
    return images, targets


def recipe(size=416):
    return D.Compose([D.VOCTargetTransform(["cat", "dog"]), D.Resize((size, size)), D.RandomHorizontalFlip(),
                      D.convert_to_relative, D.ImageTransform(TT.ColorJitter(0.3, 0.3, 0.1, 0.02)),
                      D.ImageTransform(TT.PILToTensor()), D.ImageTransform(TT.ConvertImageDtype(torch.float32)),
                      D.ImageTransform(TT.Normalize([0.485, 0.456, 0.406], [0.229, 0.224, 0.225]))])


def test_launch_plan_and_result_forms(planned):
    images = [torch.zeros(3, 30, 40, dtype=torch.uint8), torch.zeros(3, 50, 20, dtype=torch.uint8)]
    targets = [_voc([("dog", (1, 2, 30, 20))]), _voc([("cat", (0, 0, 5, 5)), ("dog", (3, 3, 9, 9))])]
    x, y = recipe(32)(images, targets)
    assert [list(c)[0] for c in planned] == ["boxes", "resample", "jitter"]
    assert planned[1]["inner"] == [(32, 32)] * 2 and planned[1]["canvas"] == (32, 32) and planned[1]["antialias"]
    assert x.shape == (2, 3, 32, 32) and x.dtype == torch.float32
    assert [set(t) for t in y] == [{"boxes", "labels"}] * 2 and y[1]["labels"].tolist() == [0, 1]
    planned.clear()
    images, targets = _pairs([(30, 40), (50, 20)])
    x, y = D.Compose([D.RandomResizedCrop(16), D.RandomHorizontalFlip(), D.CenterCrop(8)])(images, targets)
    assert [list(c)[0] for c in planned] == ["boxes", "resample"]
    assert planned[0]["ops"][:4] == [_boxes.CLAMP, _boxes.SUB, _boxes.FILTER, _boxes.SCALE]
    assert all(b is not None for b in planned[1]["boxes"]) and x.shape == (2, 3, 8, 8)
    assert y[1]["image_id"] == 1 and y[0]["boxes"] is not targets[0]["boxes"]
    for tf in (D.Resize(10), D.RandomHorizontalFlip(), D.Compose([D.CenterCrop(16), D.Resize([10])])):
        x, y = tf(images, targets)
        assert isinstance(x, list) and len(x) == len(y) == 2
    x, y = D.Compose([D.Resize((8, 12)), D.convert_to_relative])(images[0], targets[0])
    assert x.shape == (3, 8, 12) and y["boxes"].shape == (3, 4)
    planned.clear()
    D.convert_to_relative(images, targets)  # boxes only: no resampling launch
    assert [list(c)[0] for c in planned] == ["boxes"]


def test_refusals_before_any_draw(monkeypatch):
    chain = D.Compose([D.RandomResizedCrop(32), D.RandomHorizontalFlip()])
    pil = Image.fromarray(np.zeros((16, 32, 3), dtype=np.uint8))
    torch.manual_seed(0)
    state = torch.get_rng_state()
    images, targets = _pairs([(30, 40)])
    with pytest.raises(HolocronB200Error):
        chain(images, targets)  # CPU tensors
    with pytest.raises(HolocronB200Error):
        chain(pil, targets[0])
    monkeypatch.setattr(D, "require_cuda", lambda *a: None)

    def no_launch(*args, **kwargs):
        raise AssertionError("launched")
    for name in ("resample", "transform_boxes", "jitter", "_upload_voc"):
        monkeypatch.setattr(D, name, no_launch)
    bad = [
        (TypeError, {"boxes": torch.zeros(2, 4, dtype=torch.float64), "labels": torch.zeros(2, dtype=torch.int64)}),
        (TypeError, {"boxes": torch.zeros(2, 5), "labels": torch.zeros(2, dtype=torch.int64)}),
        (TypeError, {"boxes": torch.zeros(4, 2).t(), "labels": torch.zeros(4, dtype=torch.int64)}),
        (TypeError, {"boxes": torch.zeros(2, 4), "labels": torch.zeros(2, dtype=torch.int32)}),
        (TypeError, {"boxes": torch.zeros(2, 4), "labels": torch.zeros(2, 1, dtype=torch.int64)}),
        (ValueError, {"boxes": torch.zeros(2, 4), "labels": torch.zeros(3, dtype=torch.int64)}),
        (TypeError, {"boxes": torch.zeros(2, 4)}),
        (TypeError, [1., 2., 3., 4.]),
    ]
    for err, t in bad:
        with pytest.raises(err):
            chain(images, [t])
    with pytest.raises(ValueError):
        chain(images, targets * 2)
    for steps in ([D.Resize(8), lambda x, y: (x, y)], [D.Resize(8), D.VOCTargetTransform(["cat"])],
                  [TT.ColorJitter(0.1)], [D.ImageTransform(TT.PILToTensor())]):
        with pytest.raises(TypeError):
            D.Compose(steps)(*_pairs([(30, 40)], dtype=torch.float32))
    with pytest.raises(IndexError):
        D.Compose([D.Resize((8,)), D.RandomHorizontalFlip()])(images, targets)
    with pytest.raises(KeyError):  # an unknown class, while parsing
        recipe()(images, [_voc([("bird", (1, 2, 3, 4))])])
    with pytest.raises(TypeError):  # ColorJitter takes uint8 and fp32
        D.ImageTransform(ColorJitter(0.3))(*_pairs([(30, 40)], dtype=torch.float16))
    assert torch.equal(torch.get_rng_state(), state)
    # images of different sizes reaching an ImageTransform: refused after the draws, before any launch
    ragged = _pairs([(30, 40), (40, 30)])
    for tf in (D.Compose([D.Resize(10), D.ImageTransform(TT.ConvertImageDtype(torch.float32))]),
               D.ImageTransform(ColorJitter(0.3))):
        with pytest.raises(ValueError):
            tf(*ragged)


def test_header_and_binding_document_the_kernel():
    hdr = (ROOT / "include" / "holocron_b200.h").read_text()
    assert "references/detection/transforms.py:58-127" in hdr
    src = (ROOT / "holocron_b200" / "csrc" / "boxes.cu").read_text()
    ops = re.findall(r"B_(\w+) = (\d)", src)
    assert [(n, int(v)) for n, v in ops] == [(n, getattr(_boxes, n)) for n in ("SCALE", "CLAMP", "SUB", "FILTER",
                                                                                "FLIP", "DIV")]


def test_box_kernel_builds_without_spills():
    if not LOG.exists():
        pytest.skip(f"{LOG.name} absent: build the library first (python -m holocron_b200.csrc.build)")
    text = LOG.read_text()
    kernels = re.findall(r"Compiling entry function '(\w*box_transform_kernel\w*)'.*?(\d+) bytes stack frame, "
                         r"(\d+) bytes spill stores, (\d+) bytes spill loads", text, re.S)
    assert len(kernels) == 1
    for name, stack, stores, loads in kernels:
        assert (int(stack), int(stores), int(loads)) == (0, 0, 0), name
