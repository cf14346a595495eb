"""holocron_b200.transforms.segmentation without a GPU: signatures and ``repr`` against the reference's, the draws of
every chain and standalone transform and the generator state they leave against the reference's record
(tests/golden/seg_transforms.pt, written by make_golden_seg_transforms.py from the unmodified reference), the folding of
pad / crop / flip runs against torchvision on an index image, the descriptor rows of the new placement options, the
refusals before any draw, the result forms, and the ptxas report of the resampling kernel."""
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

from holocron_b200 import HolocronB200Error
from holocron_b200.transforms import ColorJitter, _resample
from holocron_b200.transforms import segmentation as S

ROOT = Path(__file__).resolve().parents[1]
G = torch.load(ROOT / "tests" / "golden" / "seg_transforms.pt", weights_only=False)
LOG = ROOT / "holocron_b200" / "csrc" / "build" / "resample.log"


def build(name, args):
    if name == "ImageTransform":
        inner, inner_args = args
        return S.ImageTransform(getattr(TT, inner)(*inner_args))
    return getattr(S, name)(*args)


def _signature(cls):
    out = []
    for name, p in inspect.signature(cls.__init__).parameters.items():
        if name != "self":
            out.append([name, p.kind.name, None if p.default is inspect.Parameter.empty else repr(p.default)])
    return out


@pytest.mark.parametrize("name", sorted(G["signatures"]))
def test_signatures(name):
    assert _signature(getattr(S, name)) == G["signatures"][name]


def test_reprs():
    for name, args, text in G["reprs"]:
        assert repr(build(name, args)) == text
    for name, records in G["chains"].items():
        assert repr(S.Compose([build(n, a) for n, a in records[0]["spec"]])) == G["compose_repr_" + name]


class DrawLog:
    """Records torch.randint / torch.rand calls as the golden generator records them."""

    def __init__(self, monkeypatch):
        self.calls = []
        randint, rand = torch.randint, torch.rand

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
        monkeypatch.setattr(torch, "randint", log_randint)
        monkeypatch.setattr(torch, "rand", log_rand)


def _records():
    for name, records in G["chains"].items():
        for rec in records:
            yield f"{name}-{rec['seed']}", rec
    for rec in G["standalone"]:
        yield f"{rec['spec'][0][0]}{rec['spec'][0][1]}-{rec['seed']}", rec


@pytest.mark.parametrize("key", [k for k, _ in _records()])
def test_draws_match_reference(key, monkeypatch):
    """Image by image: the draws (values and arguments), the size after each run and the generator state after the
    last image are the reference's."""
    rec = dict(_records())[key]
    steps = [build(n, a) for n, a in rec["spec"]]
    segments = S._segments(steps)
    jitters = [s for s in segments if isinstance(s, S.ImageTransform) and isinstance(s.transform, TT.ColorJitter)]
    # the step index that ends each segment
    ends = list(itertools.accumulate(len(s) if isinstance(s, list) else 1 for s in segments))
    torch.manual_seed(rec["seed"])
    for (h, w), sample in zip(rec["sizes"], rec["samples"]):
        log = DrawLog(monkeypatch)
        plan = S._draw(segments, jitters, (h, w))
        monkeypatch.undo()
        assert log.calls == sample["draws"], (h, w)
        for s, p, end in zip(segments, plan, ends):
            if isinstance(s, list):
                assert p.canvas == sample["after"][end - 1][0] == sample["after"][end - 1][1]
    assert torch.equal(torch.get_rng_state(), rec["state"])


def _render(inner, f, fill):
    """A folded run applied by indexing: canvas pixel (y, x) reads inner at (y - top, u - left), u the column before
    the mirror; outside the box it is ``fill``."""
    Hc, Wc = f.canvas
    ys = torch.arange(Hc)[:, None] - f.top
    us = torch.arange(Wc)
    xs = ((Wc - 1 - us) if f.mirror else us)[None, :] - f.left
    live = (ys >= 0) & (ys < inner.shape[-2]) & (xs >= 0) & (xs < inner.shape[-1])
    out = inner[..., ys.clamp(0, inner.shape[-2] - 1), xs.clamp(0, inner.shape[-1] - 1)]
    return torch.where(live, out, torch.full_like(out, fill))


def _torchvision_run(steps, img, fill):
    for t in steps:
        if isinstance(t, S.RandomCrop):
            h, w = img.shape[-2:]
            if min(h, w) < t.size:
                img = TF.pad(img, [0, 0, max(t.size - w, 0), max(t.size - h, 0)], fill=fill)
            img = TF.crop(img, *TT.RandomCrop.get_params(img, (t.size, t.size)))
        elif torch.rand(1).item() < t.prob:
            img = TF.hflip(img)
    return img


@pytest.mark.parametrize("order", list(itertools.permutations(["crop", "flip", "flip"]))[::2] +
                         [("crop",), ("flip",), ("crop", "flip"), ("flip", "crop")])
def test_fold_matches_torchvision(order):
    """Every order of crop and flips in a run, on sides below, equal to and above the crop: the fold applied by
    indexing equals torchvision's pad / crop / hflip of an index image, and draws the same."""
    for (H, W), size, seed in itertools.product([(5, 7), (9, 4), (6, 6), (1, 8), (10, 12), (1, 1)], (1, 3, 6, 8),
                                                range(4)):
        steps = [S.RandomCrop(size) if o == "crop" else S.RandomHorizontalFlip(0.5) for o in order]
        img = torch.arange(H * W, dtype=torch.int64).view(1, H, W)
        torch.manual_seed(seed)
        fold = S.fold_run(steps, (H, W))
        state = torch.get_rng_state()
        torch.manual_seed(seed)
        want = _torchvision_run(steps, img, -1)
        assert torch.equal(state, torch.get_rng_state())
        assert torch.equal(_render(img, fold, -1), want), (H, W, size, seed, fold)


def test_fold_with_resize():
    """A resized run places the resized box: inner is torchvision's output size, the crop's offset is negative."""
    torch.manual_seed(3)
    fold = S.fold_run([S.RandomResize(160, 640), S.RandomCrop(256), S.RandomHorizontalFlip(1.0)], (375, 500))
    torch.manual_seed(3)
    s = torch.randint(160, 640, (1,)).item()
    h, w = TF._compute_resized_output_size((375, 500), [s])
    assert fold.inner == (h, w) and fold.canvas == (256, 256) and fold.mirror
    assert fold.top <= 0 and fold.left <= 0
    assert S.fold_run([S.Resize((20, 30))], (7, 9)) == S._Fold((20, 30), (20, 30))
    assert S.fold_run([S.Resize(4)], (7, 9)).inner == (4, 5)
    assert S.fold_run([], (7, 9)) == S._Fold((7, 9), (7, 9))


def test_segments():
    r, c, f, t = S.RandomResize(5, 9), S.RandomCrop(4), S.RandomHorizontalFlip(0.5), S.ToTensor()
    j = S.ImageTransform(ColorJitter(0.1))
    assert S._segments([r, c, f, j, t]) == [[r, c, f], j, t]
    assert S._segments([f, c, f, c, f, r, f]) == [[f, c, f], [c, f], [r, f]]
    assert S._segments([c, j, f]) == [[c], j, [f]]
    with pytest.raises(TypeError):
        S._segments([TT.ColorJitter(0.1)])


def test_descriptor_rows():
    """offsets, canvases, mirrors and fill go into the row; rows built without them are unchanged."""
    a = torch.zeros(3, 40, 60)[:, ::2, 1::3]
    b = torch.zeros(3, 7, 9)
    plain, _, _ = _resample.descriptor_table([a], [(8, 8)], (8, 8), 2, True, "constant")
    same, _, _ = _resample.descriptor_table([a], [(8, 8)], (8, 8), 2, True, "constant", offsets=[(0, 0)],
                                            mirrors=[False], fill=0.0)
    assert plain[0, 15] == 0 and np.array_equal(plain, same)
    table, ty, tx = _resample.descriptor_table([a, b[None]], [(30, 40), (7, 9)], None, 2, True, "constant",
                                               offsets=[(-3, -5), (0, 2)], canvases=[(16, 16), (8, 12)],
                                               mirrors=[True, False], fill=255.0)
    fill = int(np.float32(255.0).view(np.uint32))
    assert fill == 0x437F0000
    assert table[0].tolist() == [a.data_ptr(), 0, 2400, 120, 3, 3, 20, 20, 30, 40, -3, -5, 16, 16, 0,
                                 fill | (1 << 32)]
    assert table[1].tolist() == [b.data_ptr(), 0, 63, 9, 1, 3, 7, 9, 7, 9, 0, 2, 8, 12, 0, fill]
    assert _resample.fill_word(-1.5, False) == int(np.float32(-1.5).view(np.uint32))
    with pytest.raises(ValueError):
        _resample.descriptor_table([a], [(8, 8)], None, 2, True, "constant", canvases=[(0, 4)])
    for canvas, canvases in (((8, 8), [(8, 8)]), (None, None)):
        with pytest.raises(ValueError):
            _resample.resample([a], [(8, 8)], canvas, _resample.InterpolationMode.BILINEAR, True, canvases=canvases)


def test_header_and_kernel_document_the_row():
    hdr = (ROOT / "include" / "holocron_b200.h").read_text()
    assert "pad_mode, fill | mirror << 32}" in hdr
    src = (ROOT / "holocron_b200" / "csrc" / "resample.cu").read_text()
    assert "unsigned int fill_bits, mirror;" in src


def _pairs(sizes, mask_ndim=2, dtype=torch.uint8):
    images = [torch.zeros(3, h, w, dtype=dtype) for h, w in sizes]
    masks = [torch.zeros(*([1] if mask_ndim == 3 else []), h, w, dtype=torch.uint8) for h, w in sizes]
    return images, masks


@pytest.fixture
def planned(monkeypatch):
    """Runs Compose on CPU tensors, recording what each resample launch would be given; outputs are zeros of the
    launch's shape."""
    calls = []
    monkeypatch.setattr(S, "require_cuda", lambda *a: None)

    def fake_resample(sources, inner, canvas, interpolation, antialias, fill, offsets, mirrors, canvases=None):
        calls.append({"sources": sources, "inner": inner, "canvas": canvas, "canvases": canvases,
                      "interpolation": interpolation, "antialias": antialias, "fill": fill, "offsets": offsets,
                      "mirrors": mirrors})
        C, dtype = sources[0].shape[0], sources[0].dtype
        if canvas is not None:
            return torch.zeros(len(sources), C, *canvas, dtype=dtype)
        return [torch.zeros(C, *c, dtype=dtype) for c in canvases]

    def fake_jitter(sources, draws):
        calls.append({"jitter": draws})
        return torch.stack(list(sources))

    monkeypatch.setattr(S, "resample", fake_resample)
    monkeypatch.setattr(S, "jitter", fake_jitter)
    return calls


def test_result_forms(planned):
    images, masks = _pairs([(30, 40), (50, 20)])
    x, y = S.RandomCrop(16)(images, masks)
    assert x.shape == (2, 3, 16, 16) and y.shape == (2, 16, 16)
    x, y = S.Resize((8, 12))(images, masks)
    assert x.shape == (2, 3, 8, 12) and y.shape == (2, 8, 12)
    for tf in (S.RandomResize(10, 20), S.Resize(10), S.RandomHorizontalFlip(0.5),
               S.Compose([S.RandomCrop(16), S.RandomResize(10)])):
        x, y = tf(images, masks)
        assert isinstance(x, list) and isinstance(y, list) and len(x) == len(y) == 2
        assert all(a.shape[-2:] == b.shape for a, b in zip(x, y))
    x, y = S.Compose([S.RandomCrop(16), S.RandomHorizontalFlip(0.5), S.ToTensor()])(images, masks)
    assert x.dtype == torch.float32 and y.dtype == torch.int64 and y.shape == (2, 16, 16)
    x, y = S.RandomCrop(16)(*_pairs([(30, 40), (50, 20)], mask_ndim=3))
    assert y.shape == (2, 1, 16, 16)
    x, y = S.Compose([S.RandomResize(10, 20), S.RandomCrop(8)])(images[0], masks[0])
    assert x.shape == (3, 8, 8) and y.shape == (8, 8)
    x, y = S.RandomHorizontalFlip(0.5)(images[0], masks[0][None])
    assert x.shape == (3, 30, 40) and y.shape == (1, 30, 40)


def test_launch_plan(planned):
    """One launch for the images and one for the masks per run: images with their interpolation (antialias on) and
    fill 0, masks nearest with fill 255; runs without a resize copy nearest at identity size."""
    images, masks = _pairs([(30, 40), (50, 20), (16, 16)])
    torch.manual_seed(0)
    S.Compose([S.RandomResize(10, 40, TT.InterpolationMode.BICUBIC), S.RandomCrop(16), S.RandomHorizontalFlip(0.5),
               S.RandomCrop(8), S.ImageTransform(ColorJitter(0.3, 0.3, 0.1, 0.02))])(images, masks)
    img1, mask1, img2, mask2, jit = planned
    assert img1["interpolation"] == TT.InterpolationMode.BICUBIC and img1["antialias"] and img1["fill"] == 0
    assert mask1["interpolation"] == TT.InterpolationMode.NEAREST and not mask1["antialias"] and mask1["fill"] == 255
    assert img1["canvas"] == mask1["canvas"] == (16, 16)
    for k in ("inner", "offsets", "mirrors"):
        assert img1[k] == mask1[k]
        assert img2[k] == mask2[k]
    assert img2["interpolation"] == TT.InterpolationMode.NEAREST and not img2["antialias"]
    assert img2["inner"] == [(16, 16)] * 3 and img2["canvas"] == (8, 8)
    assert all(m.shape[0] == 1 for m in mask1["sources"])
    assert len(jit["jitter"]) == 3


def test_refusals_before_any_draw(monkeypatch):
    recipe = S.Compose([S.RandomResize(160, 640), S.RandomCrop(256), S.RandomHorizontalFlip(0.5)])
    pil = Image.fromarray(np.zeros((16, 32, 3), dtype=np.uint8))
    torch.manual_seed(0)
    state = torch.get_rng_state()
    images, masks = _pairs([(30, 40)])
    with pytest.raises(HolocronB200Error):
        recipe(images, masks)  # CPU tensors
    with pytest.raises(HolocronB200Error):
        recipe(pil, Image.fromarray(np.zeros((16, 32), dtype=np.uint8)))
    monkeypatch.setattr(S, "require_cuda", lambda *a: None)

    def no_launch(*args, **kwargs):
        raise AssertionError("launched")
    monkeypatch.setattr(S, "resample", no_launch)
    bad_masks = [
        (TypeError, [torch.zeros(30, 40, dtype=torch.int64)]),
        (TypeError, [torch.zeros(2, 30, 40, dtype=torch.uint8)]),
        (TypeError, [torch.zeros(40, dtype=torch.uint8)]),
        (ValueError, [torch.zeros(30, 41, dtype=torch.uint8)]),
        (ValueError, []),
    ]
    for err, m in bad_masks:
        with pytest.raises(err):
            recipe(images, m)
    with pytest.raises(TypeError):  # masks of one call share their layout
        recipe(images * 2, [torch.zeros(30, 40, dtype=torch.uint8), torch.zeros(1, 30, 40, dtype=torch.uint8)])
    with pytest.raises(TypeError):  # geometric steps after ToTensor would get int64 masks
        S.Compose([S.ToTensor(), S.RandomCrop(8)])(images, masks)
    with pytest.raises(TypeError):
        S.ToTensor()(*_pairs([(30, 40)], dtype=torch.float32))
    with pytest.raises(TypeError):  # ColorJitter takes uint8 and fp32
        S.ImageTransform(ColorJitter(0.3))(*_pairs([(30, 40)], dtype=torch.float16))
    assert torch.equal(torch.get_rng_state(), state)
    # images of different sizes reaching an ImageTransform or ToTensor: refused after the draws, before any launch
    ragged = _pairs([(30, 40), (40, 30)])
    for tf in (S.Compose([S.RandomResize(10, 20), S.ToTensor()]), S.ToTensor(),
               S.ImageTransform(ColorJitter(0.3)), S.Compose([S.RandomHorizontalFlip(0.5), S.ToTensor()])):
        with pytest.raises(ValueError):
            tf(*ragged)


def test_resample_kernel_builds_without_spills():
    if not LOG.exists():
        pytest.skip(f"{LOG.name} absent: build the library first (python -m holocron_b200.csrc.build)")
    text = LOG.read_text()
    kernels = re.findall(r"Compiling entry function '(\w*resample_kernel\w*)'.*?(\d+) bytes stack frame, (\d+) bytes "
                         r"spill stores, (\d+) bytes spill loads\s+ptxas info\s+: Used (\d+) registers", text, re.S)
    assert len(kernels) == 5  # one per dtype
    for name, stack, stores, loads, regs in kernels:
        assert (int(stack), int(stores), int(loads)) == (0, 0, 0), name
        assert int(regs) <= 64, name  # __launch_bounds__(256, 4)
