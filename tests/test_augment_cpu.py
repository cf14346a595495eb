"""RandomResizedCrop, RandomHorizontalFlip and RandomErasing of holocron_b200.transforms without a GPU: signatures,
bases and repr against torchvision's classes; the draws of seeded list calls against torchvision's modules applied
image by image on CPU tensors (with the CUDA check and the launches replaced by recorders, so only the host planning
runs); the descriptor and erase rows; the refusals, raised before any launch; and the erase kernel's ptxas report."""
import inspect
import re
from pathlib import Path

import numpy as np
import pytest
import torch
import torchvision.transforms.functional as TF
from PIL import Image
from torchvision.transforms import transforms as TV

from holocron_b200 import HolocronB200Error, _lib
from holocron_b200 import transforms as T
from holocron_b200.transforms import _erase, _resample, augmentation, interpolation

ROOT = Path(__file__).resolve().parents[1]
NAMES = ["RandomResizedCrop", "RandomHorizontalFlip", "RandomErasing"]


def _count(sources):
    """Images in a list of sources, leading dimensions included."""
    return sum(x[..., 0, 0, 0].numel() for x in sources)


@pytest.fixture
def planned(monkeypatch):
    """Runs forward on CPU tensors up to the launch: records what resample / erase would be given."""
    calls = []
    monkeypatch.setattr(interpolation, "require_cuda", lambda *a: None)

    def fake_resample(sources, inner, canvas, interp, antialias, pad_mode="constant", out=None, boxes=None,
                      flips=None):
        calls.append({"sources": sources, "inner": inner, "canvas": canvas, "interpolation": interp,
                      "antialias": antialias, "boxes": boxes, "flips": flips})
        return torch.zeros(_count(sources), sources[0].shape[-3], *canvas, dtype=sources[0].dtype)

    def fake_erase(sources, rects, inplace, out=None):
        calls.append({"sources": sources, "rects": rects, "inplace": inplace})
        return None if inplace else torch.zeros(_count(sources), *sources[0].shape[-3:], dtype=sources[0].dtype)

    monkeypatch.setattr(augmentation, "resample", fake_resample)
    monkeypatch.setattr(augmentation, "erase", fake_erase)
    return calls


def _images(shapes, seed=0, dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    return [torch.rand(s, generator=g).to(dtype) for s in shapes]


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", NAMES)
def test_signature_bases_and_repr(name):
    ours, theirs = getattr(T, name), getattr(TV, name)
    assert ours.__mro__[1] is theirs
    assert inspect.signature(ours) == inspect.signature(theirs)
    assert name in T.__all__
    assert set(vars(ours)) - {"__module__", "__doc__", "__qualname__", "__firstlineno__", "__static_attributes__",
                              "__annotations__"} <= {"forward", "_draw"}
    for args, kwargs in {"RandomResizedCrop": [((176,), {"scale": (0.3, 1.0)}),
                                               (((32, 40),), {"interpolation": TF.InterpolationMode.BICUBIC,
                                                           "antialias": False})],
                         "RandomHorizontalFlip": [((), {}), ((0.25,), {})],
                         "RandomErasing": [((), {}), ((1.0, (0.02, 0.2)), {"value": "random", "inplace": True}),
                                           ((), {"value": (1, 2, 3)})]}[name]:
        a, b = ours(*args, **kwargs), theirs(*args, **kwargs)
        assert repr(a).replace("holocron_b200", "") == repr(b)
        assert {k: v for k, v in vars(a).items() if not k.startswith("_")} == \
            {k: v for k, v in vars(b).items() if not k.startswith("_")}


@pytest.mark.parametrize("scale, ratio", [((0.3, 1.0), (3 / 4, 4 / 3)), ((0.08, 1.0), (3 / 4, 4 / 3)),
                                          # every attempt too wide / too tall: the central-crop fallbacks
                                          ((0.9, 1.0), (8.0, 9.0)), ((0.9, 1.0), (0.1, 0.12)),
                                          ((1.0, 1.0), (1.0, 1.0))])
def test_crop_draws_equal_torchvision_image_by_image(planned, scale, ratio):
    imgs = _images([(3, 30, 41), (3, 52, 20), (3, 17, 17), (3, 9, 64), (3, 5, 6)], 1)
    size = (16, 12)
    torch.manual_seed(7)
    T.RandomResizedCrop(size, scale=scale, ratio=ratio)(imgs)
    after_ours = torch.random.get_rng_state()
    call = planned[-1]
    assert call["inner"] == [size] * len(imgs) and call["canvas"] == size
    tv = TV.RandomResizedCrop(size, scale=scale, ratio=ratio)
    torch.manual_seed(7)
    for x, box in zip(imgs, call["boxes"]):
        assert torch.equal(tv(x), TF.resized_crop(x, *box, list(size)))
    assert torch.equal(torch.random.get_rng_state(), after_ours)
    torch.manual_seed(7)
    assert call["boxes"] == [TV.RandomResizedCrop.get_params(x, scale, ratio) for x in imgs]


@pytest.mark.parametrize("p", [0.0, 0.5, 1.0])
def test_flip_draws_equal_torchvision_image_by_image(planned, p):
    imgs = _images([(3, 8, 11)] * 9, 2)
    torch.manual_seed(3)
    T.RandomHorizontalFlip(p)(imgs)
    after_ours = torch.random.get_rng_state()
    flips = planned[-1]["flips"]
    assert planned[-1]["interpolation"] == TF.InterpolationMode.NEAREST and planned[-1]["inner"] == [(8, 11)] * 9
    tv = TV.RandomHorizontalFlip(p)
    torch.manual_seed(3)
    for x, flip in zip(imgs, flips):
        assert torch.equal(tv(x), x.flip(-1) if flip else x)
    assert torch.equal(torch.random.get_rng_state(), after_ours)
    assert flips == {0.0: [False] * 9, 1.0: [True] * 9}.get(p, flips)
    assert p != 0.5 or 0 < sum(flips) < 9


@pytest.mark.parametrize("p", [0.0, 0.6, 1.0])
@pytest.mark.parametrize("value", [0, 0.25, (0.5, -1.5, 300.0), [7], "random"])
@pytest.mark.parametrize("scale, ratio", [((0.02, 0.33), (0.3, 3.3)), ((0.02, 0.2), (0.3, 3.3)),
                                          # no rectangle fits in 10 attempts: the image is left as it is
                                          ((0.95, 1.0), (0.3, 0.4))])
def test_erase_draws_equal_torchvision_image_by_image(planned, p, value, scale, ratio):
    imgs = _images([(3, 20, 31)] * 6, 4)
    kwargs = {"p": p, "scale": scale, "ratio": ratio, "value": value}
    torch.manual_seed(11)
    T.RandomErasing(**kwargs)(imgs)
    after_ours = torch.random.get_rng_state()
    rects = planned[-1]["rects"]
    tv = TV.RandomErasing(**kwargs)
    torch.manual_seed(11)
    for x, rect in zip(imgs, rects):
        want = x if rect is None else TF.erase(x, *rect)
        assert torch.equal(tv(x), want)
    assert torch.equal(torch.random.get_rng_state(), after_ours)
    if p == 0.0 or scale[0] == 0.95:
        assert rects == [None] * 6
    if p == 1.0 and scale[0] != 0.95:
        assert all(r is not None for r in rects)
        for (_, _, h, w, v) in rects:
            assert v.dtype == torch.float32
            assert tuple(v.shape) == ((3, h, w) if value == "random" else (1 if np.ndim(value) == 0 else len(value), 1, 1))


def test_single_tensor_semantics(planned):
    x = torch.rand(2, 3, 12, 10)
    torch.manual_seed(0)
    assert T.RandomHorizontalFlip(0.0)(x) is x
    assert T.RandomErasing(0.0)(x) is x
    # no rectangle found: torchvision assigns the image to itself, in place or on a copy
    assert T.RandomErasing(1.0, scale=(0.95, 1.0), ratio=(0.3, 0.4), inplace=True)(x) is x
    assert not planned
    out = T.RandomErasing(1.0, scale=(0.95, 1.0), ratio=(0.3, 0.4))(x)
    assert out.shape == x.shape and planned[-1]["rects"] == [None]
    assert T.RandomErasing(1.0, inplace=True)(x) is x and planned[-1]["inplace"]
    assert T.RandomHorizontalFlip(1.0)(x).shape == x.shape and planned[-1]["flips"] == [True]
    assert T.RandomResizedCrop((5, 7))(x).shape == (2, 3, 5, 7)
    with pytest.raises(ValueError):  # torchvision's resize of a 2-D tensor fails in torch's interpolate
        T.RandomResizedCrop((5, 7))(x[0, 0])
    # a crop already of the target size is handed back as torchvision's resize hands it back: the crop view itself
    n = len(planned)
    y = T.RandomResizedCrop((12, 10), scale=(1.0, 1.0), ratio=(10 / 12, 10 / 12))(x)
    assert len(planned) == n and y.data_ptr() == x.data_ptr() and y.shape == x.shape
    imgs = [torch.rand(3, 6, 6), torch.rand(3, 6, 6)]
    assert T.RandomErasing(1.0, inplace=True)(imgs) is imgs
    assert T.RandomErasing(1.0, inplace=True)(tuple(imgs)) == tuple(imgs)


def test_crop_and_flip_rows():
    base = torch.zeros(3, 40, 60)
    a = base[:, ::2, 1::3]  # strides (2400, 120, 3), 20 x 20
    b = torch.zeros(2, 3, 7, 9)
    table, ty, tx = _resample.descriptor_table([a, b], [(8, 8), (8, 8)], (8, 8), 2, True, "constant",
                                               boxes=[(3, 4, 10, 12), (1, 2, 5, 6)], flips=[True, False])
    es = 4
    # crop at (3, 4), then the last of its 12 columns, read backwards
    assert table[0].tolist() == [a.data_ptr() + (3 * 120 + 4 * 3 + 11 * 3) * es, 0, 2400, 120, -3, 3, 10, 12, 8, 8,
                                 0, 0, 8, 8, 0, 0]
    assert table[1].tolist() == [b.data_ptr() + (1 * 9 + 2) * es, 0, 63, 9, 1, 3, 5, 6, 8, 8, 0, 0, 8, 8, 0, 0]
    assert table[2, 0] == b.data_ptr() + (3 * 7 * 9 + 1 * 9 + 2) * es
    assert (ty, tx) == (5, 5)  # antialiased 10 -> 8 and 12 -> 8 (from the crop's size): 2 * ceil(1.25 or 1.5) + 1
    # flips alone: identity size, every column of a flipped row read from the right
    table, ty, tx = _resample.descriptor_table([b[0]], [(7, 9)], (7, 9), 0, False, "constant", flips=[True])
    assert table[0].tolist() == [b.data_ptr() + 8 * es, 0, 63, 9, -1, 3, 7, 9, 7, 9, 0, 0, 7, 9, 0, 0]
    assert (ty, tx) == (1, 1)
    # existing rows keep their meaning
    plain, _, _ = _resample.descriptor_table([a], [(8, 8)], (8, 8), 2, True, "constant")
    assert plain[0].tolist()[:8] == [a.data_ptr(), 0, 2400, 120, 3, 3, 20, 20]
    for box in [(-1, 0, 5, 5), (0, 0, 21, 5), (0, 16, 5, 5)]:
        with pytest.raises(ValueError):
            _resample.descriptor_table([a], [(8, 8)], (8, 8), 2, True, "constant", boxes=[box])
    with pytest.raises(RuntimeError):  # what torch's interpolate raises for an empty crop
        _resample.descriptor_table([a], [(8, 8)], (8, 8), 2, True, "constant", boxes=[(0, 0, 0, 5)])
    # the row-span check takes the magnitude of a negated stride
    wide = torch.zeros(1, 1, 2, device="meta").expand(3, 1, 2).as_strided((3, 1, 2), (1, 1, 2 ** 31))
    with pytest.raises(ValueError):
        _resample.descriptor_table([wide], [(1, 2)], (1, 2), 0, False, "constant", flips=[True])


def test_erase_rows():
    imgs = [torch.zeros(3, 10, 12, device="meta") for _ in range(3)]
    per_pixel = torch.arange(3 * 2 * 4, dtype=torch.float32).view(3, 2, 4)
    rects = [(1, 2, 2, 4, per_pixel), None, (5, 0, 4, 3, torch.tensor([0.5])[:, None, None])]
    out = torch.empty(3, 3, 10, 12, device="meta")
    table, values, rows, row_len = _erase.erase_table(imgs, rects, False, out)
    es = 4
    assert table.shape == (3, 16)
    assert table[0].tolist() == [imgs[0].data_ptr(), out.data_ptr(), 120, 12, 1, 3, 10, 12, 1, 2, 2, 4,
                                 _erase.FILL_PIXEL, 0, 0, 0]
    assert table[1].tolist() == [imgs[1].data_ptr(), out.data_ptr() + 360 * es, 120, 12, 1, 3, 10, 12, 0, 0, 0, 0,
                                 _erase.FILL_NONE, 0, 0, 0]
    assert table[2].tolist()[8:14] == [5, 0, 4, 3, _erase.FILL_CHANNEL, 24]
    assert torch.equal(values[0], per_pixel.view(-1)) and values[1].tolist() == [0.5] * 3
    assert (rows, row_len) == (30, 12)
    # in place: the destinations are the (strided) sources, the grid covers the rectangles only
    cl = torch.zeros(2, 3, 10, 12, device="meta").to(memory_format=torch.channels_last).unbind(0)
    table, _, rows, row_len = _erase.erase_table(cl, [rects[0], rects[2]], True, None)
    assert table[:, 0].tolist() == table[:, 1].tolist() == [cl[0].data_ptr(), cl[1].data_ptr()]
    assert table[0, 2:5].tolist() == [1, 36, 3]
    assert (rows, row_len) == (12, 4)
    # leading dimensions are images of their own, erased alike
    table, _, _, _ = _erase.erase_table([torch.zeros(2, 3, 10, 12, device="meta")], [rects[2]], False, out[:2])
    assert table[1, 0] == table[0, 0] + 360 * es and table[1, 1] == out.data_ptr() + 360 * es
    assert table[0, 8:14].tolist() == table[1, 8:14].tolist()
    for bad in [(0, 0, 11, 2, per_pixel), (9, 0, 2, 4, per_pixel), (1, 2, 2, 3, per_pixel),
                (1, 2, 2, 4, torch.zeros(2, 1, 1))]:
        with pytest.raises(ValueError):
            _erase.erase_table(imgs[:1], [bad], False, out[:1])
    with pytest.raises(ValueError):
        _erase.erase_table([imgs[0], torch.zeros(3, 10, 11, device="meta")], [None, None], False, out[:2])


def test_refusals_before_any_launch(monkeypatch):
    lib = _lib.lib()
    lib.hb_launch_count_reset()
    pil = Image.fromarray(np.zeros((16, 32, 3), dtype=np.uint8))
    cpu = torch.rand(3, 16, 32)
    for tf in (T.RandomResizedCrop(8), T.RandomHorizontalFlip(1.0), T.RandomErasing(1.0)):
        for img in (pil, cpu, [cpu]):
            with pytest.raises(HolocronB200Error):
                tf(img)
        with pytest.raises(TypeError):
            tf([np.zeros((3, 4, 4))])
    # past the CUDA check (meta tensors stand in for CUDA ones): the refusals torchvision and the kernels make
    for mod in (interpolation, _resample, _erase):
        monkeypatch.setattr(mod, "require_cuda", lambda *a: None)
    meta = [torch.zeros(3, 16, 32, device="meta"), torch.zeros(3, 16, 30, device="meta")]
    with pytest.raises(ValueError):
        T.RandomHorizontalFlip(1.0)(meta)
    with pytest.raises(ValueError):
        T.RandomErasing(1.0)(meta)
    with pytest.raises(ValueError):  # torchvision's: a value sequence of neither 1 nor C entries
        T.RandomErasing(1.0, value=(1.0, 2.0))(meta[:1])
    with pytest.raises(ValueError):
        TV.RandomErasing(1.0, value=(1.0, 2.0))(torch.zeros(3, 16, 32))
    with pytest.raises(IndexError):  # torchvision's get_params reads the channel count of a 2-D image
        T.RandomErasing(1.0)(torch.zeros(16, 32, device="meta"))
    ints = [torch.zeros(3, 16, 32, dtype=torch.int32, device="meta")]
    for tf in (T.RandomResizedCrop(8), T.RandomHorizontalFlip(1.0), T.RandomErasing(1.0)):
        with pytest.raises(TypeError):
            tf(ints)
    with pytest.raises(NotImplementedError):
        T.RandomResizedCrop(8, interpolation=TF.InterpolationMode.LANCZOS)(meta[:1])
    # torchvision's central-crop fallback rounds the width of a 1-row image to 0
    for tf, img in ((T.RandomResizedCrop(8, scale=(0.9, 1.0), ratio=(0.1, 0.12)), torch.zeros(3, 1, 5, device="meta")),
                    (TV.RandomResizedCrop(8, scale=(0.9, 1.0), ratio=(0.1, 0.12)), torch.zeros(3, 1, 5))):
        with pytest.raises(RuntimeError):
            tf([img] if img.is_meta else img)
    assert lib.hb_launch_count() == 0


def test_header_entry_and_binding():
    hdr = (ROOT / "include" / "holocron_b200.h").read_text()
    decl = re.search(r"int (hb_erase_batch)\((.*?)\);", hdr, flags=re.S)
    assert decl is not None and "RandomErasing" in hdr and "references/classification/train.py" in hdr
    assert len(decl.group(2).split(",")) == 7
    assert _lib.SIGNATURES["hb_erase_batch"] == "pp" + "i" * 4 + "p"


def test_erase_kernel_ptxas_clean():
    log = ROOT / "holocron_b200" / "csrc" / "build" / "erase.log"
    if not log.exists():
        pytest.skip(f"{log.name} absent: build the library first (python -m holocron_b200.csrc.build)")
    text = log.read_text()
    assert text.count("Compiling entry function") == 5  # one per dtype
    spills = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", text)
    assert spills and all(s == ("0", "0", "0") for s in spills), spills
