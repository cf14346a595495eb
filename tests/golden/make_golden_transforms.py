"""Generates tests/golden/transforms.pt by running the UNMODIFIED reference (frgfm/Holocron, a checkout named by the
HOLOCRON_REFERENCE environment variable) on seeded CPU inputs:

    HOLOCRON_REFERENCE=/path/to/Holocron python tests/golden/make_golden_transforms.py

It records holocron.transforms: the constructors' signatures, bases and refusals, ``get_params`` of Resize over a
table of image shapes and target sizes, seeded ``RandomZoomOut`` draws (including the shapes whose rounding gives a
box one pixel larger than the canvas), and the outputs of both transforms on small uint8 and fp32 CPU tensors for
every mode, pad mode, interpolation and antialias setting.
"""
import importlib
import sys
from pathlib import Path

import torch
from torchvision.transforms import InterpolationMode

sys.path.insert(0, str(Path(__file__).resolve().parent))
from make_golden import OUT, describe_signature  # noqa: E402  (loads the reference)

TF = importlib.import_module("holocron.transforms.interpolation")

INTERPOLATIONS = ("nearest", "nearest-exact", "bilinear", "bicubic")
PAD_MODES = ("constant", "edge", "reflect", "symmetric")
PARAM_SHAPES = [(1, 1), (1, 7), (7, 1), (3, 5), (16, 32), (32, 16), (299, 500), (500, 299), (375, 500), (224, 224),
                (481, 353), (2, 1000)]
SIZES = [(224, 224), (32, 32), (17, 23), (64, 48), (1, 5)]
SCALES = [(0.5, 1.0), (0.3, 0.99), (0.99, 0.999), (0.1, 0.2)]
# (C, H, W) inputs and target sizes of the output records: down- and upscales, odd sides, 1-pixel sides
OUTPUT_CASES = [((3, 13, 21), (16, 16)), ((3, 40, 30), (12, 18)), ((2, 9, 9), (20, 14)), ((1, 1, 6), (5, 5)),
                ((3, 24, 7), (8, 8))]
ERRORS = [("Resize", (16,), {}), ("Resize", ((16, 16),), {"mode": "stretch"}), ("Resize", ((16, 16),), {"mode": "pad"}),
          ("Resize", ((16, 16), (1, 0.5)), {}), ("Resize", ((16, 0),), {}), ("Resize", ((16, 16, 16),), {}),
          ("Resize", ([16, -1],), {}), ("RandomZoomOut", (224,), {}), ("RandomZoomOut", ((16, 16),), {"scale": (1, 0.5)}),
          ("RandomZoomOut", ((16, 16),), {"scale": (0.5,)}), ("RandomZoomOut", ((0, 16),), {})]


def _inputs(shape, seed):
    g = torch.Generator().manual_seed(seed)
    u8 = torch.randint(0, 256, shape, generator=g, dtype=torch.uint8)
    f32 = torch.rand(shape, generator=g, dtype=torch.float32) * 2 - 0.5
    return {"uint8": u8, "float32": f32}


def _zoom_draws():
    """Seeded RandomZoomOut.get_params draws (5 per case) over shapes x sizes x scales, in draw order."""
    out = []
    for (h, w) in PARAM_SHAPES:
        img = torch.empty(3, h, w)
        for size in SIZES:
            for scale in SCALES:
                tf = TF.RandomZoomOut(size, scale=scale)
                torch.manual_seed(h * 1000 + w)
                draws = []
                for _ in range(5):
                    try:
                        draws.append(tf.get_params(img))
                    except ZeroDivisionError:
                        draws.append(None)
                out.append({"shape": (h, w), "size": size, "scale": scale, "seed": h * 1000 + w, "draws": draws})
    return out


def _negative_padding_cases():
    """(shape, size, scale, seed) whose first draw gives a box larger than the canvas on some side."""
    found = []
    for h in range(20, 60):
        for w in (17, 23, 31, 44):
            tf = TF.RandomZoomOut((32, 32), scale=(0.995, 1.0))
            torch.manual_seed(h)
            bh, bw = tf.get_params(torch.empty(1, h, w))
            if bh > 32 or bw > 32:
                found.append(((3, h, w), (32, 32), (0.995, 1.0), h))
    return found[:6]


def main():
    rec = {"signatures": {name: describe_signature(getattr(TF, name)) for name in ("Resize", "RandomZoomOut")},
           "bases": {name: [f"{c.__module__}.{c.__qualname__}" for c in getattr(TF, name).__mro__[1:]]
                     for name in ("Resize", "RandomZoomOut")},
           "resize_method": [(m.name, m.value) for m in TF.ResizeMethod]}
    errors = []
    for cls, args, kwargs in ERRORS:
        try:
            getattr(TF, cls)(*args, **kwargs)
            errors.append((cls, args, kwargs, None))
        except Exception as e:  # noqa: BLE001  (the exception type is the record)
            errors.append((cls, args, kwargs, type(e).__name__))
    rec["errors"] = errors
    rec["resize_params"] = [{"shape": s, "size": z, "hw": TF.Resize(z, mode=TF.ResizeMethod.PAD).get_params(
        torch.empty(3, *s))} for s in PARAM_SHAPES for z in SIZES]
    rec["zoom_draws"] = _zoom_draws()

    outputs = []
    for k, (shape, size) in enumerate(OUTPUT_CASES):
        for dtype, x in _inputs(shape, k).items():
            for interp in INTERPOLATIONS:
                mode_i = InterpolationMode(interp)
                for aa in (True, False):
                    y = TF.Resize(size, mode=TF.ResizeMethod.SQUISH, interpolation=mode_i, antialias=aa)(x)
                    outputs.append({"kind": "squish", "x": x, "size": size, "interpolation": interp, "antialias": aa,
                                    "pad_mode": "constant", "y": y})
                for pad_mode in PAD_MODES:
                    try:
                        y = TF.Resize(size, mode=TF.ResizeMethod.PAD, pad_mode=pad_mode, interpolation=mode_i)(x)
                        err = None
                    except Exception as e:  # noqa: BLE001
                        y, err = None, type(e).__name__
                    outputs.append({"kind": "pad", "x": x, "size": size, "interpolation": interp, "antialias": True,
                                    "pad_mode": pad_mode, "y": y, "error": err})
    zooms = []
    cases = [((3, 30, 40), (16, 16), (0.3, 0.9), 0), ((3, 11, 5), (20, 24), (0.5, 1.0), 1)]
    cases += _negative_padding_cases()
    for k, (shape, size, scale, seed) in enumerate(cases):
        for dtype, x in _inputs(shape, 100 + k).items():
            for interp, aa in (("bilinear", True), ("nearest", False), ("bicubic", False)):
                tf = TF.RandomZoomOut(size, scale=scale, interpolation=InterpolationMode(interp), antialias=aa)
                torch.manual_seed(seed)
                y = tf(x)
                torch.manual_seed(seed)
                hw = tf.get_params(x)
                zooms.append({"x": x, "size": size, "scale": scale, "seed": seed, "interpolation": interp,
                              "antialias": aa, "hw": hw, "y": y})
    rec["outputs"] = outputs
    rec["zoom_outputs"] = zooms
    torch.save(rec, OUT / "transforms.pt")
    print(f"wrote {OUT / 'transforms.pt'}: {len(outputs)} resize outputs, {len(zooms)} zoom outputs, "
          f"{len(cases) - 2} negative-padding cases")


if __name__ == "__main__":
    main()
