"""The classification Compose and Normalize of holocron_b200.transforms without a GPU: the draws of the recipe's four
chains against torchvision's ``T.Compose`` applied image by image to CPU tensors (with the CUDA check and the launches
replaced by recorders, so only the host planning runs); the segments, folds, tail programs and descriptor rows of
known chains; the refusals, raised before any launch; the C ABI entry; and the tail kernel's ptxas report."""
import re
from pathlib import Path

import numpy as np
import pytest
import torch
import torchvision.transforms.functional as TF
from PIL import Image
from torchvision.transforms import autoaugment as TVA, transforms as TV

from holocron_b200 import HolocronB200Error, _lib
from holocron_b200 import transforms as HT
from holocron_b200.transforms import _erase, _fold, _tail, classification as C, interpolation

ROOT = Path(__file__).resolve().parents[1]
BILINEAR = TF.InterpolationMode.BILINEAR
MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


def imagenette_train(p):
    return [TV.RandomResizedCrop(24, scale=(0.3, 1.0), interpolation=BILINEAR), TV.RandomHorizontalFlip(),
            TVA.TrivialAugmentWide(interpolation=BILINEAR), TV.PILToTensor(), TV.ConvertImageDtype(torch.float32),
            TV.Normalize(MEAN, STD), TV.RandomErasing(p=p, scale=(0.02, 0.2), value="random")]


def imagenette_val():
    return [TV.Resize(28, interpolation=BILINEAR), TV.CenterCrop(24), TV.PILToTensor(),
            TV.ConvertImageDtype(torch.float32), TV.Normalize(MEAN, STD)]


def cifar_train(p):
    return [TV.RandomHorizontalFlip(), TVA.TrivialAugmentWide(interpolation=BILINEAR), TV.PILToTensor(),
            TV.ConvertImageDtype(torch.float32), TV.Normalize(MEAN, STD), TV.RandomErasing(p=p, value="random")]


def cifar_val():
    return [TV.PILToTensor(), TV.ConvertImageDtype(torch.float32), TV.Normalize(MEAN, STD)]


SIZES = [(30, 41), (52, 20), (17, 17), (40, 64)]


def _images(sizes, seed=0, dtype=torch.uint8):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, 256, (3, h, w), generator=g, dtype=torch.uint8).to(dtype) for h, w in sizes]


@pytest.fixture
def planned(monkeypatch):
    """Runs Compose on CPU tensors up to the launches: records what each launch would be given."""
    calls = []
    monkeypatch.setattr(interpolation, "require_cuda", lambda *a: None)

    def fake_resample(sources, inner, canvas, interpolation, antialias, offsets=None, mirrors=None, canvases=None,
                      boxes=None):
        calls.append(("resample", {"inner": inner, "canvas": canvas, "canvases": canvases, "offsets": offsets,
                                   "mirrors": mirrors, "boxes": boxes, "interpolation": interpolation,
                                   "antialias": antialias}))
        if canvas is None:
            return [torch.zeros(3, *c, dtype=sources[0].dtype) for c in canvases]
        return torch.zeros(len(sources), 3, *canvas, dtype=sources[0].dtype)

    def fake_apply_ops(sources, ops, interpolation, fill):
        calls.append(("autoaugment", list(ops)))
        return torch.zeros(len(sources), *sources[0].shape, dtype=sources[0].dtype)

    def fake_tail(sources, ops, rects=None, norm=None):
        calls.append(("tail", {"ops": list(ops), "rects": rects, "norm": norm}))
        return torch.zeros(len(sources), *sources[0].shape, dtype=torch.float32)

    def fake_erase(sources, rects, inplace):
        calls.append(("erase", {"rects": rects}))
        return torch.zeros(len(sources), *sources[0].shape, dtype=sources[0].dtype)

    for name, fn in (("resample", fake_resample), ("apply_ops", fake_apply_ops), ("tail", fake_tail),
                     ("erase", fake_erase)):
        monkeypatch.setattr(C, name, fn)
    return calls


def _torchvision_draws(chain, images, monkeypatch):
    """The draws torchvision's Compose makes applied image by image: per image, the events crop box, flip, op and
    erase rectangle, in order."""
    events = []
    real_rrc, real_flip = TV.RandomResizedCrop.get_params, TF.hflip
    real_op, real_erase = TVA._apply_op, TV.RandomErasing.get_params

    def rrc(img, scale, ratio):
        box = real_rrc(img, scale, ratio)
        events[-1].append(("crop", tuple(box)))
        return box

    def flip(img):
        events[-1].append(("flip",))
        return real_flip(img)

    def op(img, name, magnitude, interpolation, fill):
        events[-1].append(("op", name, magnitude))
        return real_op(img, name, magnitude, interpolation, fill)

    def erase_params(img, scale, ratio, value=None):
        i, j, h, w, v = real_erase(img, scale, ratio, value)
        events[-1].append(("erase", None) if v is img else ("erase", (i, j, h, w, v)))
        return i, j, h, w, v

    with monkeypatch.context() as m:
        m.setattr(TV.RandomResizedCrop, "get_params", staticmethod(rrc))
        m.setattr(TF, "hflip", flip)
        m.setattr(TVA, "_apply_op", op)
        m.setattr(TV.RandomErasing, "get_params", staticmethod(erase_params))
        tf = TV.Compose([t for t in chain if not isinstance(t, TV.PILToTensor)])  # PIL images only
        for x in images:
            events.append([])
            tf(x)
    return events


def _our_draws(chain, calls, n):
    """The same events from the recorded launches of our Compose."""
    events = [[] for _ in range(n)]
    erasing = next((t for t in chain if isinstance(t, TV.RandomErasing)), None)
    for kind, call in calls:
        for k in range(n):
            if kind == "resample":
                if call["boxes"] is not None:
                    events[k].append(("crop", tuple(call["boxes"][k])))
                if call["mirrors"][k]:
                    events[k].append(("flip",))
            elif kind == "autoaugment":
                events[k].append(("op", *call[k]))
    if erasing is not None:
        tail = next(c for kind, c in calls if kind == "tail")
        return events, tail["rects"]
    return events, None


@pytest.mark.parametrize("seed", [0, 1, 5])
@pytest.mark.parametrize("name, chain", [("imagenette_train_p0", imagenette_train(0.0)),
                                         ("imagenette_train_p05", imagenette_train(0.5)),
                                         ("imagenette_train_p1", imagenette_train(1.0)),
                                         ("imagenette_val", imagenette_val()),
                                         ("cifar_train_p0", cifar_train(0.0)), ("cifar_train_p1", cifar_train(1.0)),
                                         ("cifar_val", cifar_val())])
def test_draws_equal_torchvision_image_by_image(planned, monkeypatch, name, chain, seed):
    sizes = [(32, 32)] * 4 if name.startswith("cifar") else SIZES
    images = _images(sizes, seed)
    torch.manual_seed(seed)
    C.Compose(chain)(images)
    after_ours = torch.random.get_rng_state()
    torch.manual_seed(seed)
    want = _torchvision_draws(chain, images, monkeypatch)
    assert torch.equal(torch.random.get_rng_state(), after_ours)
    got, rects = _our_draws(chain, planned, len(images))
    for k in range(len(images)):
        want_k = [e for e in want[k] if e[0] != "erase"]
        assert got[k] == want_k, (k, got[k], want_k)
        erases = [e[1] for e in want[k] if e[0] == "erase"]
        if rects is not None:
            if not erases:
                assert rects[k] is None
            elif erases[0] is None:
                assert rects[k] is None
            else:
                assert rects[k][:4] == erases[0][:4] and torch.equal(rects[k][4], erases[0][4])


def test_erasing_without_a_rectangle_draws_as_torchvision(planned, monkeypatch):
    """A ratio no rectangle of the image satisfies: get_params gives up after its 10 attempts, erasing nothing."""
    chain = [TV.ConvertImageDtype(torch.float32), TV.RandomErasing(p=1.0, scale=(0.9, 1.0), ratio=(20.0, 30.0))]
    images = _images([(8, 8)] * 3, 2)
    torch.manual_seed(3)
    C.Compose(chain)(images)
    after = torch.random.get_rng_state()
    torch.manual_seed(3)
    want = _torchvision_draws(chain, images, monkeypatch)
    assert torch.equal(torch.random.get_rng_state(), after)
    assert all(w == [("erase", None)] for w in want)
    tail = planned[-1][1]
    assert tail["rects"] == [None] * 3 and tail["ops"] == [_tail.CONVERT, _tail.ERASE_F32]


# ---------------------------------------------------------------------------------------------------------------------
def test_segments_and_launch_plan(planned):
    segs = C._segments(imagenette_train(0.5))
    assert [type(s).__name__ for s in segs] == ["list", "TrivialAugmentWide", "_Tail"]
    assert [type(t).__name__ for t in segs[0]] == ["RandomResizedCrop", "RandomHorizontalFlip"]
    assert [type(t).__name__ for t in segs[2].steps] == ["PILToTensor", "ConvertImageDtype", "Normalize",
                                                         "RandomErasing"]
    # a kind seen twice starts a new tail; a resize starts a new run; this package's subclasses are accepted
    segs = C._segments([TV.Normalize(MEAN, STD), TV.RandomErasing(), HT.Normalize(MEAN, STD), TV.CenterCrop(4),
                        TV.RandomHorizontalFlip(), HT.RandomResizedCrop(3), TV.Resize(2)])
    assert [len(s.steps) if isinstance(s, C._Tail) else [type(t).__name__ for t in s] for s in segs] == \
        [2, 1, ["CenterCrop", "RandomHorizontalFlip"], ["RandomResizedCrop"], ["Resize"]]

    torch.manual_seed(0)
    out = C.Compose(imagenette_val())(_images(SIZES))
    assert [k for k, _ in planned] == ["resample", "tail"] and out.shape == (4, 3, 24, 24)
    res, tail = planned[0][1], planned[1][1]
    assert res["canvas"] == (24, 24) and res["boxes"] is None and res["antialias"] is True
    assert res["inner"] == [_fold.resized(s, [28]) for s in SIZES]
    assert tail["ops"] == [_tail.CONVERT, _tail.NORMALIZE]
    np.testing.assert_array_equal(tail["norm"], np.array(MEAN + STD, dtype=np.float32))
    planned.clear()
    assert C.Compose(cifar_val())(_images([(32, 32)] * 2)).shape == (2, 3, 32, 32)
    assert [k for k, _ in planned] == ["tail"]
    planned.clear()
    C.Compose(cifar_train(0.0))(_images([(32, 32)] * 2))
    assert [k for k, _ in planned] == ["resample", "autoaugment", "tail"]
    assert planned[0][1]["interpolation"] == TF.InterpolationMode.NEAREST
    assert planned[0][1]["canvases"] == [(32, 32)] * 2 and planned[2][1]["rects"] == [None, None]
    # a tail that leaves the images uint8 is an erase copy; one before conversion erases as uint8
    planned.clear()
    C.Compose([TV.RandomErasing(p=1.0, value=300.7)])(_images([(16, 16)] * 2))
    assert [k for k, _ in planned] == ["erase"]
    assert C._check_steps(C._segments([TV.RandomErasing(), TV.ConvertImageDtype(torch.float32)]), torch.uint8, 3) \
        == {0: ([_tail.ERASE_U8, _tail.CONVERT], torch.float32, None)}
    # a single tensor returns one image; a Resize to a short side returns views of different sizes
    planned.clear()
    assert C.Compose(cifar_val())(_images([(32, 32)])[0]).shape == (3, 32, 32)
    out = C.Compose([TV.Resize(10)])(_images(SIZES))
    assert [tuple(x.shape[-2:]) for x in out] == [_fold.resized(s, [10]) for s in SIZES]


@pytest.mark.parametrize("H, W", [(20, 26), (24, 24), (9, 30), (31, 7), (1, 1)])
@pytest.mark.parametrize("ch, cw", [(24, 24), (10, 13), (32, 9), (7, 40)])
def test_center_crop_fold_matches_torchvision(H, W, ch, cw):
    """The fold's placement of a CenterCrop, larger or smaller than the image, is torchvision's center_crop."""
    x = torch.arange(1, H * W + 1, dtype=torch.float32).view(1, H, W)
    want = TF.center_crop(x, [ch, cw])
    for mirror in (False, True):
        f = _fold._Fold((H, W), (H, W))
        if mirror:
            f.flip()
        f.center_crop(ch, cw)
        canvas = torch.zeros(1, ch, cw)
        src = x.flip(-1) if mirror else x
        for y in range(H):
            for xx in range(W):
                cy, cx = y + f.top, xx + f.left
                if 0 <= cy < ch and 0 <= cx < cw:
                    canvas[0, cy, cx] = x[0, y, xx]
        got = canvas.flip(-1) if mirror else canvas
        assert torch.equal(got, TF.center_crop(src, [ch, cw])), (H, W, ch, cw, mirror)
    assert want.shape == (1, ch, cw)


def test_tail_rows_and_program():
    images = [torch.zeros(3, 5, 7, dtype=torch.uint8), torch.zeros(3, 8, 10, dtype=torch.uint8)[:, 1:6, 2:9]]
    out = torch.empty(2, 3, 5, 7, dtype=torch.float32)
    rects = [None, (1, 2, 3, 4, torch.tensor([[[0.5]], [[1.5]], [[2.5]]]))]
    table, values, rows, row_len = _erase.erase_table(images, rects, False, out)
    assert (rows, row_len) == (15, 7)
    assert table[0].tolist() == [images[0].data_ptr(), out.data_ptr(), 35, 7, 1, 3, 5, 7] + [0] * 8
    assert table[1].tolist() == [images[1].data_ptr(), out.data_ptr() + 3 * 5 * 7 * 4, 80, 10, 1, 3, 5, 7, 1, 2, 3,
                                 4, _erase.FILL_CHANNEL, 0, 0, 0]
    assert [v.tolist() for v in values] == [[0.5, 1.5, 2.5]]
    steps = [TV.PILToTensor(), TV.RandomErasing(), TV.ConvertImageDtype(torch.float32), TV.Normalize(MEAN, STD)]
    assert _tail.program(steps, torch.uint8) == ([_tail.ERASE_U8, _tail.CONVERT, _tail.NORMALIZE], torch.float32)
    assert _tail.program(steps[2:], torch.float32) == ([_tail.NORMALIZE], torch.float32)
    np.testing.assert_array_equal(_tail.norm_values(0.5, [1.0, 2.0, 4.0], 3),
                                  np.array([0.5] * 3 + [1.0, 2.0, 4.0], dtype=np.float32))


# ---------------------------------------------------------------------------------------------------------------------
def test_refusals_before_any_launch(monkeypatch):
    lib = _lib.lib()
    lib.hb_launch_count_reset()
    cpu = _images([(16, 16)])
    pil = Image.fromarray(np.zeros((16, 16, 3), dtype=np.uint8))
    for img in (cpu, cpu[0], pil, [pil]):
        with pytest.raises(HolocronB200Error):
            C.Compose(cifar_val())(img)
        with pytest.raises(HolocronB200Error):
            HT.Normalize(MEAN, STD)(img)
    monkeypatch.setattr(interpolation, "require_cuda", lambda *a: None)
    u8 = _images(SIZES[:2])
    f32 = _images(SIZES[:2], dtype=torch.float32)
    before = torch.random.get_rng_state()
    refusals = [
        (TypeError, [TV.RandomHorizontalFlip(), HT.Resize((8, 8))], u8),
        (TypeError, [TV.RandomHorizontalFlip(), HT.RandomZoomOut((8, 8))], u8),
        (TypeError, [TV.RandomHorizontalFlip(), lambda x: x], u8),
        (TypeError, [TV.RandomHorizontalFlip(), TV.ColorJitter(0.1)], u8),
        (TypeError, [TV.RandomHorizontalFlip(), TV.Normalize(MEAN, STD)], u8),
        (TypeError, [TV.RandomHorizontalFlip(), TV.PILToTensor()], f32),
        (TypeError, [TV.RandomHorizontalFlip(), TVA.TrivialAugmentWide()], f32),
        (TypeError, [TV.ConvertImageDtype(torch.float32), TV.RandomResizedCrop(8), TVA.TrivialAugmentWide()], u8),
        (NotImplementedError, [TV.RandomHorizontalFlip(), TV.ConvertImageDtype(torch.float16)], u8),
        (NotImplementedError, [TV.RandomHorizontalFlip(), TV.Normalize(MEAN, STD)], [x.half() for x in f32]),
        (ValueError, [TV.RandomHorizontalFlip(), TV.ConvertImageDtype(torch.float32), TV.Normalize(MEAN, (1, 0, 1))],
         u8),
        (ValueError, [TV.RandomHorizontalFlip(), TV.ConvertImageDtype(torch.float32), TV.Normalize(MEAN, 1e-46)], u8),
        (ValueError, [TV.RandomHorizontalFlip(), TV.ConvertImageDtype(torch.float32), TV.Normalize((0, 1), STD)], u8),
        (ValueError, [TV.RandomHorizontalFlip(), TV.CenterCrop(8)], [u8[0], u8[1][:2]]),
    ]
    for exc, chain, images in refusals:
        with pytest.raises(exc):
            C.Compose(chain)(images)
        assert torch.equal(torch.random.get_rng_state(), before), chain
    # torchvision's std == 0 test, on the fp32-rounded values
    with pytest.raises(ValueError):
        TV.Normalize(MEAN, 1e-46)(torch.zeros(3, 4, 4))
    # images of different sizes reaching TrivialAugmentWide or a tail: after the draws, before any launch
    for chain in ([TV.RandomHorizontalFlip(), TVA.TrivialAugmentWide()], cifar_val()):
        with pytest.raises(ValueError):
            C.Compose(chain)(u8)
    with pytest.raises(ValueError):
        HT.Normalize(MEAN, STD)(f32)
    with pytest.raises(TypeError):
        HT.Normalize(MEAN, STD)(u8[:1])
    with pytest.raises(ValueError):
        HT.Normalize(MEAN, STD)(torch.zeros(4, 4))
    assert lib.hb_launch_count() == 0


def test_normalize_class():
    assert HT.Normalize.__mro__[1] is TV.Normalize and "Normalize" in HT.__all__
    a, b = HT.Normalize(MEAN, STD, inplace=True), TV.Normalize(MEAN, STD, inplace=True)
    assert repr(a) == repr(b) and vars(a) == vars(b) or \
        {k: v for k, v in vars(a).items() if not k.startswith("_")} == \
        {k: v for k, v in vars(b).items() if not k.startswith("_")}
    assert repr(C.Compose(cifar_val())) == repr(TV.Compose(cifar_val()))


def test_header_entry_and_binding():
    hdr = (ROOT / "include" / "holocron_b200.h").read_text()
    decl = re.search(r"int (hb_image_tail_batch)\((.*?)\);", hdr, flags=re.S)
    assert decl is not None and "references/classification/train.py:100-107, 162-168" in hdr
    assert len(decl.group(2).split(",")) == 9
    assert _lib.SIGNATURES["hb_image_tail_batch"] == "pp" + "i" * 6 + "p"


def test_tail_kernel_ptxas_clean():
    log = ROOT / "holocron_b200" / "csrc" / "build" / "image_tail.log"
    if not log.exists():
        pytest.skip(f"{log.name} absent: build the library first (python -m holocron_b200.csrc.build)")
    text = log.read_text()
    assert text.count("Compiling entry function") == 2  # uint8 and fp32 sources
    spills = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", text)
    assert len(spills) == 2 and all(s == ("0", "0", "0") for s in spills), spills
