"""ColorJitter of holocron_b200.transforms without a GPU: signature, bases and repr against torchvision's class; the
draws of seeded list calls against torchvision's module applied image by image (with the CUDA check and the launch
replaced by recorders); the descriptor rows; the refusals, raised before any launch (and before any draw); the header
entry and its binding; and the kernels' ptxas report."""
import inspect
import re
from itertools import product
from pathlib import Path

import numpy as np
import pytest
import torch
from PIL import Image
from torchvision.transforms import transforms as TVT
from torchvision.transforms import functional as TVF

from holocron_b200 import HolocronB200Error, _lib
from holocron_b200 import transforms as T
from holocron_b200.transforms import _color, augmentation, interpolation

ROOT = Path(__file__).resolve().parents[1]
RECIPE = {"brightness": 0.3, "contrast": 0.3, "saturation": 0.1, "hue": 0.02}


@pytest.fixture
def planned(monkeypatch):
    """Runs forward on CPU tensors up to the launch: records the draws jitter would be given."""
    calls = []
    monkeypatch.setattr(interpolation, "require_cuda", lambda *a: None)

    def fake_jitter(sources, draws, out=None):
        calls.append({"sources": sources, "draws": list(draws)})
        n = sum(x[..., 0, 0, 0].numel() for x in sources)
        return torch.zeros(n, *sources[0].shape[-3:], dtype=sources[0].dtype)

    monkeypatch.setattr(augmentation, "jitter", fake_jitter)
    return calls


def _as_plain(draw):
    fn_idx, *factors = draw
    return [int(k) for k in fn_idx], factors


def test_signature_bases_and_repr():
    ours, theirs = T.ColorJitter, TVT.ColorJitter
    assert ours.__mro__[1] is theirs and "ColorJitter" in T.__all__
    assert inspect.signature(ours) == inspect.signature(theirs)
    assert set(vars(ours)) - {"__module__", "__doc__", "__qualname__", "__firstlineno__", "__static_attributes__",
                              "__annotations__"} <= {"forward"}
    for kwargs in ({}, RECIPE, {"brightness": (0.5, 1.5), "hue": (-0.5, 0.5)}, {"contrast": 0.0, "saturation": 2}):
        a, b = ours(**kwargs), theirs(**kwargs)
        assert repr(a) == repr(b)
        assert vars(a).keys() == vars(b).keys()
        assert {k: v for k, v in vars(a).items() if not k.startswith("_")} == \
            {k: v for k, v in vars(b).items() if not k.startswith("_")}


# every subset of the four factors, with scalar and tuple ranges
SUBSETS = [dict(zip(RECIPE, vals)) for vals in product(*[(0, RECIPE[k]) for k in RECIPE])]
TUPLES = [{"brightness": (0.0, 2.0), "contrast": (0.0, 1.0), "saturation": (0.5, 0.5), "hue": (-0.5, 0.5)},
          {"brightness": (1.0, 1.0), "hue": (-0.02, 0.0)}]


@pytest.mark.parametrize("kwargs", SUBSETS + TUPLES)
def test_draws_equal_torchvision_image_by_image(planned, monkeypatch, kwargs):
    g = torch.Generator().manual_seed(1)
    imgs = [torch.randint(0, 256, (3, 6, 7), generator=g, dtype=torch.uint8) for _ in range(50)]
    torch.manual_seed(5)
    T.ColorJitter(**kwargs)(imgs)
    after_ours = torch.random.get_rng_state()
    ours = [_as_plain(d) for d in planned[-1]["draws"]]
    theirs = []
    for name in ("adjust_brightness", "adjust_contrast", "adjust_saturation", "adjust_hue"):
        monkeypatch.setattr(TVF, name, lambda img, f, name=name: theirs[-1][1].append((name, f)) or img)
    tv = TVT.ColorJitter(**kwargs)
    real = tv.get_params

    def recording(*a):
        draw = real(*a)
        theirs.append((draw, []))
        return draw

    monkeypatch.setattr(tv, "get_params", recording)
    torch.manual_seed(5)
    for x in imgs:
        tv(x)
    assert torch.equal(torch.random.get_rng_state(), after_ours)
    assert ours == [_as_plain(d) for d, _ in theirs]
    # the ops torchvision applied are the rows' ops, in their order, with their factors
    for (draw, applied) in theirs:
        ops, at, p = _color.chain(draw)
        assert [_color.OPS[k] for k in ops] == [name[len("adjust_"):] for name, _ in applied]
        assert at == (ops.index(1) if 1 in ops else -1)
        for k, (_, f) in zip(ops, applied):
            assert p[2 * k] == np.float32(f) and (k == 3 or p[2 * k + 1] == np.float32(1.0 - f))


def test_single_tensor_draws_once(planned):
    x = torch.zeros(2, 4, 3, 6, 7, dtype=torch.uint8)
    tf = T.ColorJitter(**RECIPE)
    torch.manual_seed(0)
    y = tf(x)
    after = torch.random.get_rng_state()
    assert y.shape == x.shape and len(planned[-1]["draws"]) == 1
    torch.manual_seed(0)
    tf.get_params(tf.brightness, tf.contrast, tf.saturation, tf.hue)
    assert torch.equal(torch.random.get_rng_state(), after)


def test_hands_back_input_where_torchvision_does(planned):
    for C, kwargs, same in ((3, {}, True), (1, {}, True), (1, {"saturation": 0.5, "hue": 0.1}, True),
                            (1, {"saturation": 0.5}, True), (1, {"hue": 0.1, "contrast": 0.2}, False),
                            (3, {"hue": 0.1}, False), (1, {"brightness": 0.2}, False)):
        x = torch.zeros(C, 5, 6, dtype=torch.float32)
        torch.manual_seed(0)
        state = torch.random.get_rng_state()
        y = T.ColorJitter(**kwargs)(x)
        assert (y is x) == same, (C, kwargs)
        ours = torch.random.get_rng_state()
        torch.random.set_rng_state(state)
        z = TVT.ColorJitter(**kwargs)(x)
        assert (z is x) == same and torch.equal(torch.random.get_rng_state(), ours)
    # a list always comes back stacked, even when nothing changes it
    x = [torch.zeros(3, 5, 6, dtype=torch.uint8)] * 2
    assert T.ColorJitter()(x).shape == (2, 3, 5, 6)


def _rows(sources, draws, dtype=torch.uint8):
    n = sum(x[..., 0, 0, 0].numel() for x in sources)
    out = torch.empty(n, *sources[0].shape[-3:], dtype=dtype, device="meta")
    return out, *_color.jitter_table(sources, draws, out)


def test_descriptor_rows():
    img = torch.zeros(3, 10, 12, dtype=torch.uint8, device="meta")
    draw = (torch.tensor([2, 1, 3, 0]), 1.25, 0.7, None, -0.01)
    out, table, params, stats = _rows([img], [draw])
    assert table[0].tolist() == [img.data_ptr(), out.data_ptr(), 120, 12, 1, 3, 10, 12, 3, 1, 3, 0, -1, 0, 0, 0]
    assert stats == [0]
    assert params[0].tolist() == [np.float32(1.25), np.float32(1.0 - 1.25), np.float32(0.7), np.float32(1.0 - 0.7),
                                  0.0, 0.0, np.float32(-0.01), np.float32(1.0) / np.float32(120)]
    # the prefix length of contrast: where it sits among the ops that are on
    for order in ([1, 0, 2, 3], [0, 1, 2, 3], [3, 2, 0, 1], [0, 2, 3, 1]):
        for factors in ((1.1, 0.9, 1.0, 0.01), (None, 0.9, 1.0, None), (1.1, None, 1.0, 0.01)):
            _, table, _, stats = _rows([img], [(torch.tensor(order), *factors)])
            on = [k for k in order if factors[k] is not None]
            assert table[0, 8] == len(on) and table[0, 9:9 + len(on)].tolist() == on
            assert (table[0, 9 + len(on):13] == -1).all()
            assert table[0, 13] == (on.index(1) if 1 in on else -1)
            assert table[0, 14] == (0 if 1 in on else -1) and stats == ([0] if 1 in on else [])
    # no factor: a copy
    _, table, params, stats = _rows([img], [(torch.tensor([0, 1, 2, 3]), None, None, None, None)])
    assert table[0, 8:15].tolist() == [0, -1, -1, -1, -1, -1, -1] and not params[0, :7].any() and stats == []
    # fp32: byte addresses, element strides; leading dimensions, channels_last, cropped and unbound sources
    x = torch.zeros(2, 3, 10, 12, dtype=torch.float32, device="meta").to(memory_format=torch.channels_last)
    full = torch.zeros(3, 20, 30, dtype=torch.float32, device="meta")
    crop = full[:, 4:14, 7:19]
    assert crop.data_ptr() == full.data_ptr() + (4 * 30 + 7) * 4
    base = torch.zeros(4, 3, 10, 12, dtype=torch.float32, device="meta")
    on = (torch.tensor([0, 1, 2, 3]), 1.1, 0.9, None, None)
    off = (torch.tensor([3, 2, 1, 0]), 1.1, None, 1.2, None)
    out, table, _, stats = _rows([x, crop, base.unbind(0)[2]], [on, off, on], torch.float32)
    assert table[:, 0].tolist() == [x.data_ptr(), x.data_ptr() + 360 * 4, crop.data_ptr(),
                                    base.data_ptr() + 2 * 360 * 4]
    assert table[:, 1].tolist() == [out.data_ptr() + k * 360 * 4 for k in range(4)]
    assert table[0, 2:5].tolist() == [1, 36, 3] and table[2, 2:5].tolist() == [600, 30, 1]
    assert table[3, 2:5].tolist() == [120, 12, 1]
    assert table[:, 14].tolist() == [0, 1, -1, 2] and stats == [0, 1, 3]
    with pytest.raises(ValueError):
        _rows([img, torch.zeros(3, 10, 13, dtype=torch.uint8, device="meta")], [draw, draw])


def test_refusals(monkeypatch):
    lib = _lib.lib()
    lib.hb_launch_count_reset()
    tf = T.ColorJitter(**RECIPE)
    pil = Image.fromarray(np.zeros((16, 32, 3), dtype=np.uint8))
    cpu = torch.zeros(3, 16, 32, dtype=torch.uint8)
    for img in (pil, cpu, [cpu]):
        state = torch.random.get_rng_state()
        with pytest.raises(HolocronB200Error):
            tf(img)
        assert torch.equal(torch.random.get_rng_state(), state)
    monkeypatch.setattr(interpolation, "require_cuda", lambda *a: None)
    monkeypatch.setattr(_color, "require_cuda", lambda *a: None)
    meta = torch.zeros(3, 16, 32, dtype=torch.uint8, device="meta")
    cases = [([meta, torch.zeros(3, 16, 30, dtype=torch.uint8, device="meta")], ValueError),
             ([meta.half()], TypeError), (meta.double(), TypeError), ([meta.to(torch.int16)], TypeError),
             ([torch.zeros(2, 16, 32, dtype=torch.uint8, device="meta")], TypeError),
             (torch.zeros(4, 16, 32, dtype=torch.float32, device="meta"), TypeError),
             (torch.zeros(16, 32, dtype=torch.uint8, device="meta"), TypeError)]
    for module in (tf, T.ColorJitter()):
        for img, exc in cases:
            state = torch.random.get_rng_state()
            with pytest.raises(exc):
                module(img)
            assert torch.equal(torch.random.get_rng_state(), state)  # refused before any draw
    with pytest.raises(TypeError, match=r"permitted channel values are \[1, 3\], but found 2"):
        tf([torch.zeros(2, 16, 32, dtype=torch.uint8, device="meta")])
    # torchvision's message lists [1, 3] or, when contrast runs first, [3, 1]
    with pytest.raises(TypeError, match=r"permitted channel values are \[(1, 3|3, 1)\], but found 2"):
        TVT.ColorJitter(**RECIPE)(torch.zeros(2, 16, 32, dtype=torch.uint8))
    with pytest.raises(ValueError):
        _color.jitter([meta], [])
    assert lib.hb_launch_count() == 0


def test_header_entry_and_binding():
    hdr = (ROOT / "include" / "holocron_b200.h").read_text()
    decl = re.search(r"int (hb_color_jitter_batch)\((.*?)\);", hdr, flags=re.S)
    assert decl is not None and "ColorJitter" in hdr and "references/segmentation/train.py:133-140" in hdr
    assert len(decl.group(2).split(",")) == 11
    assert _lib.SIGNATURES["hb_color_jitter_batch"] == "pppp" + "i" * 6 + "p"


def test_kernel_ptxas_clean():
    log = ROOT / "holocron_b200" / "csrc" / "build" / "color_jitter.log"
    if not log.exists():
        pytest.skip(f"{log.name} absent: build the library first (python -m holocron_b200.csrc.build)")
    text = log.read_text()
    assert text.count("Compiling entry function") == 2  # the statistics and apply kernels
    spills = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", text)
    assert len(spills) == 2 and all(s == ("0", "0", "0") for s in spills), spills
