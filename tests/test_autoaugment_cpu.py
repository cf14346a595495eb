"""TrivialAugmentWide of holocron_b200.transforms without a GPU: signature, bases and repr against torchvision's class;
the draws of seeded list calls against torchvision's module applied image by image (with the CUDA check and the
launch replaced by recorders); the descriptor rows; the refusals, raised before any launch (and before any draw where
they do not depend on it); the fp64 oracle against torchvision's CPU ``_apply_op``; and the kernels' ptxas report."""
import inspect
import math
import re
from pathlib import Path

import numpy as np
import pytest
import torch
from PIL import Image
from torchvision.transforms import InterpolationMode
from torchvision.transforms import autoaugment as TVA
from torchvision.transforms.functional import _get_inverse_affine_matrix

from holocron_b200 import HolocronB200Error, _lib
from holocron_b200 import transforms as T
from holocron_b200.transforms import _autoaugment, augmentation, interpolation

from _autoaugment_oracle import apply_op as oracle_op

ROOT = Path(__file__).resolve().parents[1]
GEOMETRIC = ("ShearX", "ShearY", "TranslateX", "TranslateY", "Rotate")


def _every_op(num_bins=31):
    """(op, magnitude) for every op, magnitude bin and sign of the augmentation space."""
    for op, (mags, signed) in TVA.TrivialAugmentWide()._augmentation_space(num_bins).items():
        for m in ([0.0] if mags.ndim == 0 else [float(v) for v in mags]):
            for sign in ((1.0, -1.0) if signed else (1.0,)):
                yield op, m * sign


@pytest.fixture
def planned(monkeypatch):
    """Runs forward on CPU tensors up to the launch: records the ops apply_ops would be given."""
    calls = []
    monkeypatch.setattr(interpolation, "require_cuda", lambda *a: None)

    def fake_apply_ops(sources, ops, interp, fill, out=None):
        calls.append({"sources": sources, "ops": list(ops), "interpolation": interp, "fill": fill})
        n = sum(x[..., 0, 0, 0].numel() for x in sources)
        return torch.zeros(n, *sources[0].shape[-3:], dtype=sources[0].dtype)

    monkeypatch.setattr(augmentation, "apply_ops", fake_apply_ops)
    return calls


def test_signature_bases_and_repr():
    ours, theirs = T.TrivialAugmentWide, TVA.TrivialAugmentWide
    assert ours.__mro__[1] is theirs and "TrivialAugmentWide" in T.__all__
    assert inspect.signature(ours) == inspect.signature(theirs)
    assert set(vars(ours)) - {"__module__", "__doc__", "__qualname__", "__firstlineno__", "__static_attributes__",
                              "__annotations__"} <= {"forward"}
    for kwargs in ({}, {"num_magnitude_bins": 5, "interpolation": InterpolationMode.BILINEAR, "fill": [1, 2, 3]},
                   {"fill": 7}):
        a, b = ours(**kwargs), theirs(**kwargs)
        assert repr(a) == repr(b)
        assert vars(a).keys() == vars(b).keys()
        assert {k: v for k, v in vars(a).items() if not k.startswith("_")} == \
            {k: v for k, v in vars(b).items() if not k.startswith("_")}


@pytest.mark.parametrize("num_bins", [31, 5])
def test_draws_equal_torchvision_image_by_image(planned, monkeypatch, num_bins):
    g = torch.Generator().manual_seed(1)
    imgs = [torch.randint(0, 256, (3, 6, 7), generator=g, dtype=torch.uint8) for _ in range(300)]
    torch.manual_seed(5)
    T.TrivialAugmentWide(num_bins)(imgs)
    after_ours = torch.random.get_rng_state()
    ours = planned[-1]["ops"]
    theirs = []
    monkeypatch.setattr(TVA, "_apply_op", lambda img, op, m, interpolation, fill: theirs.append((op, m)) or img)
    tv = TVA.TrivialAugmentWide(num_bins)
    torch.manual_seed(5)
    for x in imgs:
        tv(x)
    assert ours == theirs
    assert torch.equal(torch.random.get_rng_state(), after_ours)
    assert {op for op, _ in ours} == set(_autoaugment.OPS)
    assert any(m < 0 for _, m in ours)


def test_single_tensor_draws_once(planned):
    x = torch.zeros(2, 4, 3, 6, 7, dtype=torch.uint8)
    torch.manual_seed(0)
    for _ in range(40):
        y = T.TrivialAugmentWide()(x)
        if y is x:  # Identity hands the tensor back, as torchvision does
            continue
        assert y.shape == x.shape and len(planned[-1]["ops"]) == 1


def _row_of(op, magnitude, C=3, H=10, W=12, fill=None, bilinear=False):
    img = torch.zeros(C, H, W, dtype=torch.uint8, device="meta")
    out = torch.empty(1, C, H, W, dtype=torch.uint8, device="meta")
    table, params, stats = _autoaugment.op_table([img], [(op, magnitude)], bilinear, fill, out)
    return img, out, table[0], params[0], stats


def test_descriptor_rows():
    img, out, row, p, stats = _row_of("Brightness", -0.33)
    assert row.tolist() == [img.data_ptr(), out.data_ptr(), 120, 12, 1, 3, 10, 12, 6, -1, 255, 0, 0, 0, 0, 0]
    assert p[0] == np.float32(1.0 + -0.33) and p[1] == np.float32(1.0 - (1.0 + -0.33)) and stats == []
    for op, magnitude in _every_op():
        _, _, row, p, stats = _row_of(op, magnitude, H=37, W=53)
        assert row[8] == _autoaugment.OPS.index(op)
        assert (row[9] == 0) == (op in ("Contrast", "AutoContrast", "Equalize"))
        assert stats == ([0] if row[9] == 0 else [])
        if op in ("Brightness", "Color", "Contrast", "Sharpness"):
            r = 1.0 + magnitude
            assert (p[0], p[1]) == (np.float32(r), np.float32(1.0 - r))
        if op == "Posterize":
            assert row[10] == (-int(2 ** (8 - int(magnitude)))) & 0xFF
        if op == "Solarize":
            assert p[2] == np.float32(magnitude)
        if op in GEOMETRIC:
            if op.startswith("Shear"):
                shear = [math.degrees(math.atan(magnitude)), 0.0][::1 if op == "ShearX" else -1]
                want = _get_inverse_affine_matrix([-26.5, -18.5], 0.0, [0.0, 0.0], 1.0, shear)
            elif op.startswith("Translate"):
                t = [float(int(magnitude)), 0.0][::1 if op == "TranslateX" else -1]
                want = _get_inverse_affine_matrix([0.0, 0.0], 0.0, t, 1.0, [0.0, 0.0])
            else:
                want = _get_inverse_affine_matrix([0.0, 0.0], -magnitude, [0.0, 0.0], 1.0, [0.0, 0.0])
            assert torch.equal(torch.from_numpy(p[3:9].copy()), torch.tensor(want, dtype=torch.float32))
    # fills: broadcast to C values, flagged
    _, _, row, p, _ = _row_of("Rotate", 45.0, fill=[7.0, 8.0, 9.0], bilinear=True)
    assert row[11] == 1 and row[12] == 1 and p[9:12].tolist() == [7.0, 8.0, 9.0]
    assert _autoaugment.check_options(InterpolationMode.NEAREST, 5, 3) == (False, [5.0] * 3)
    assert _autoaugment.check_options(2, [4], 3) == (True, [4.0] * 3)
    assert _autoaugment.check_options(0, None, 1) == (False, None)
    # leading dimensions and strided sources: one row per image, the same op, consecutive destinations
    x = torch.zeros(2, 3, 10, 12, dtype=torch.uint8, device="meta").to(memory_format=torch.channels_last)
    out = torch.empty(3, 3, 10, 12, dtype=torch.uint8, device="meta")
    table, _, stats = _autoaugment.op_table([x, x[0]], [("Equalize", 0.0), ("Solarize", 3.0)], False, None, out)
    assert table[:, 0].tolist() == [x.data_ptr(), x.data_ptr() + 360, x.data_ptr()]
    assert table[:, 1].tolist() == [out.data_ptr() + k * 360 for k in range(3)]
    assert table[0, 2:5].tolist() == [1, 36, 3] and table[:, 9].tolist() == [0, 1, -1] and stats == [0, 1]


def _draws_posterize_first(seed):
    """Whether torchvision's one-bin module draws Posterize first under this seed (it then raises ValueError)."""
    torch.manual_seed(seed)
    try:
        TVA.TrivialAugmentWide(num_magnitude_bins=1)(torch.zeros(3, 4, 4, dtype=torch.uint8))
    except ValueError:
        return True
    return False


def test_refusals(monkeypatch):
    lib = _lib.lib()
    lib.hb_launch_count_reset()
    tf = T.TrivialAugmentWide()
    pil = Image.fromarray(np.zeros((16, 32, 3), dtype=np.uint8))
    cpu = torch.zeros(3, 16, 32, dtype=torch.uint8)
    for img in (pil, cpu, [cpu]):
        with pytest.raises(HolocronB200Error):
            tf(img)
    monkeypatch.setattr(interpolation, "require_cuda", lambda *a: None)
    monkeypatch.setattr(_autoaugment, "require_cuda", lambda *a: None)
    meta = torch.zeros(3, 16, 32, dtype=torch.uint8, device="meta")
    cases = [(tf, [meta, torch.zeros(3, 16, 30, dtype=torch.uint8, device="meta")], ValueError),
             (tf, [meta.float()], TypeError),
             (tf, meta.float(), TypeError),
             (tf, [torch.zeros(2, 16, 32, dtype=torch.uint8, device="meta")], TypeError),
             (tf, torch.zeros(16, 32, dtype=torch.uint8, device="meta"), TypeError),
             (T.TrivialAugmentWide(interpolation=InterpolationMode.BICUBIC), [meta], ValueError),
             (T.TrivialAugmentWide(fill=[1.0, 2.0]), [meta], ValueError),
             (T.TrivialAugmentWide(fill=[]), [meta], ValueError),
             (T.TrivialAugmentWide(fill=256), [meta], ValueError),
             (T.TrivialAugmentWide(fill=[0, -1, 0]), [meta], ValueError)]
    for module, img, exc in cases:
        state = torch.random.get_rng_state()
        with pytest.raises(exc):
            module(img)
        assert torch.equal(torch.random.get_rng_state(), state)  # refused before any draw
    with pytest.raises(ValueError):  # torchvision's own type for this mode
        TVA.TrivialAugmentWide(interpolation=InterpolationMode.BICUBIC)(torch.zeros(3, 4, 4, dtype=torch.uint8))
    # after the draws: what torchvision raises for the drawn op (one bin: Posterize gets a bit count outside [0, 8])
    seed = next(s for s in range(200) if _draws_posterize_first(s))
    torch.manual_seed(seed)
    with pytest.raises(ValueError):
        T.TrivialAugmentWide(num_magnitude_bins=1)([meta])
    with pytest.raises(ValueError):
        _autoaugment.apply_ops([meta], [("Posterize", 9.0)], InterpolationMode.NEAREST, None)
    with pytest.raises(ValueError):
        _autoaugment.apply_ops([meta], [("Invert", 0.0)], InterpolationMode.NEAREST, None)
    assert lib.hb_launch_count() == 0


@pytest.mark.parametrize("C", [1, 3])
@pytest.mark.parametrize("interp", [InterpolationMode.NEAREST, InterpolationMode.BILINEAR])
def test_oracle_equals_torchvision_cpu(C, interp):
    g = torch.Generator().manual_seed(C)
    imgs = [torch.randint(0, 256, (C, 37, 53), generator=g, dtype=torch.uint8),
            torch.randint(0, 256, (C, 3, 3), generator=g, dtype=torch.uint8),
            torch.full((C, 6, 5), 77, dtype=torch.uint8),
            (torch.randint(0, 2, (C, 9, 11), generator=g, dtype=torch.uint8) * 200 + 20)]
    for img in imgs:
        for fill in (None, [128.0], [float(40 * c + 5) for c in range(C)]):
            for op, magnitude in _every_op():
                if fill is not None and op not in GEOMETRIC:
                    continue
                want = TVA._apply_op(img, op, magnitude, interp, fill).numpy()
                got, amb = oracle_op(img.numpy(), op, magnitude, interp == InterpolationMode.BILINEAR, fill, "cpu")
                bad = (got != want) & ~amb[None]
                assert not bad.any(), (op, magnitude, tuple(img.shape), fill, int(bad.sum()))
                if op not in GEOMETRIC:
                    assert not amb.any()


def test_header_entry_and_binding():
    hdr = (ROOT / "include" / "holocron_b200.h").read_text()
    decl = re.search(r"int (hb_autoaugment_batch)\((.*?)\);", hdr, flags=re.S)
    assert decl is not None and "TrivialAugmentWide" in hdr and "references/classification/train.py:103" in hdr
    assert len(decl.group(2).split(",")) == 10
    assert _lib.SIGNATURES["hb_autoaugment_batch"] == "pppp" + "i" * 5 + "p"


def test_kernel_ptxas_clean():
    log = ROOT / "holocron_b200" / "csrc" / "build" / "autoaugment.log"
    if not log.exists():
        pytest.skip(f"{log.name} absent: build the library first (python -m holocron_b200.csrc.build)")
    text = log.read_text()
    assert text.count("Compiling entry function") == 2  # the histogram and apply kernels
    spills = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", text)
    assert len(spills) == 2 and all(s == ("0", "0", "0") for s in spills), spills
