"""holocron_b200.transforms without a GPU: constructors, signatures and refusals against the reference's records,
get_params and seeded RandomZoomOut draws equal to the reference's, the fp64 oracle against the reference's CPU outputs,
the C-ABI entry point, and the refusal of PIL images and CPU tensors (tests/golden/transforms.pt, written by
make_golden_transforms.py from the unmodified reference)."""
import inspect
import re
from pathlib import Path

import numpy as np
import pytest
import torch
from PIL import Image

import _transforms_oracle as O
from holocron_b200 import HolocronB200Error, _lib
from holocron_b200 import transforms as T
from holocron_b200.transforms import _resample, _table
from holocron_b200.transforms.interpolation import ResizeMethod

ROOT = Path(__file__).resolve().parents[1]
G = torch.load(ROOT / "tests" / "golden" / "transforms.pt", weights_only=False)
# a uint8 output may differ from the oracle's rounding only where the fp64 value lies this close to a .5 tie (or within
# the float bound below, when that is wider)
TIE = 1e-4
# fp32 outputs of the reference against the oracle, relative to the sum of absolute terms: nearest copies exactly, the
# bilinear filters stay within 1e-6; the bicubic ones reach 5.7e-6 (about 48 fp32 ulps: the reference's CPU kernel
# evaluates its cancelling cubic polynomials and positions in fp32) on the fixture's upscales
REL = {"nearest": 0.0, "nearest-exact": 0.0, "bilinear": 1e-6, "bicubic": 8e-6}


def _signature(cls):
    out = []
    for name, p in inspect.signature(cls.__init__).parameters.items():
        if name != "self":
            out.append([name, p.kind.name, None if p.default is inspect.Parameter.empty else repr(p.default)])
    return out


@pytest.mark.parametrize("name", ["Resize", "RandomZoomOut"])
def test_signature_and_bases(name):
    cls = getattr(T, name)
    assert _signature(cls) == G["signatures"][name]
    assert [f"{c.__module__}.{c.__qualname__}" for c in cls.__mro__[1:]] == G["bases"][name]


def test_resize_method():
    assert [(m.name, m.value) for m in ResizeMethod] == G["resize_method"]
    assert issubclass(ResizeMethod, str)


def test_constructor_refusals():
    for cls, args, kwargs, err in G["errors"]:
        if err is None:
            getattr(T, cls)(*args, **kwargs)
        else:
            with pytest.raises(Exception) as info:
                getattr(T, cls)(*args, **kwargs)
            assert type(info.value).__name__ == err, (cls, args, kwargs)


def test_resize_get_params():
    for r in G["resize_params"]:
        tf = T.Resize(r["size"], mode=ResizeMethod.PAD)
        assert tf.get_params(torch.empty(3, *r["shape"])) == r["hw"], r


def test_zoom_draws():
    for r in G["zoom_draws"]:
        tf = T.RandomZoomOut(r["size"], scale=r["scale"])
        torch.manual_seed(r["seed"])
        img = torch.empty(3, *r["shape"])
        for want in r["draws"]:
            if want is None:
                with pytest.raises(ZeroDivisionError):
                    tf.get_params(img)
            else:
                assert tf.get_params(img) == want, r


def test_zoom_negative_padding_recorded():
    """The fixture holds boxes one pixel larger than the canvas, which the placement crops."""
    assert any(r["hw"][0] > r["size"][0] or r["hw"][1] > r["size"][1] for r in G["zoom_outputs"])


def _check_against(want: torch.Tensor, value: np.ndarray, mag: np.ndarray, interpolation: str, what):
    if want.dtype == torch.uint8:
        got = O.to_uint8(value)
        diff = got.astype(np.int64) != want.numpy().astype(np.int64)
        near_tie = O.tie_distance(np.clip(value, 0, 255)) < np.maximum(TIE, REL[interpolation] * mag)
        assert not (diff & ~near_tie).any(), what
        assert (np.abs(got.astype(np.int64) - want.numpy()) <= 1).all(), what
        return int(diff.sum())
    err = np.abs(want.double().numpy() - value)
    assert (err <= REL[interpolation] * mag).all(), (what, err.max())
    return 0


def test_oracle_reproduces_reference_resize():
    ties = 0
    n = 0
    for r in G["outputs"]:
        x = r["x"]
        if r["kind"] == "squish":
            inner = r["size"]
        else:
            inner = T.Resize(r["size"], mode=ResizeMethod.PAD).get_params(x)
            if r["error"] is not None:
                top, left = O.placement(inner, r["size"])
                pads = (left, top, r["size"][1] - inner[1] - left, r["size"][0] - inner[0] - top)
                with pytest.raises(Exception) as info:
                    _resample._check_padding(r["pad_mode"], pads, *inner)
                assert type(info.value).__name__ == r["error"]
                continue
        value, mag = O.resize_pad(x, inner, r["size"], r["interpolation"], r["antialias"], r["pad_mode"])
        assert tuple(r["y"].shape) == value.shape
        ties += _check_against(r["y"], value, mag, r["interpolation"],
                               {k: r[k] for k in ("kind", "size", "antialias", "pad_mode")})
        n += value.size
    assert ties <= 1e-3 * n


def test_oracle_reproduces_reference_zoom_out():
    for r in G["zoom_outputs"]:
        value, mag = O.resize_pad(r["x"], r["hw"], r["size"], r["interpolation"], r["antialias"])
        assert tuple(r["y"].shape) == value.shape
        _check_against(r["y"], value, mag, r["interpolation"], r["hw"])


def test_host_tap_bound_covers_every_filter():
    """The tap counts the host sizes the kernel's tables with bound every row of the oracle's filters."""
    for n_in, n_out in [(400, 224), (1600, 200), (56, 224), (7, 1), (1, 9), (333, 41)]:
        for code, name in enumerate(O.FILTERS):
            for aa in (False, True):
                m = O.axis_matrix(n_in, n_out, name, aa and code >= 2)
                nz = np.nonzero(m)
                span = max((nz[1][nz[0] == r].max() - nz[1][nz[0] == r].min() + 1) for r in range(n_out))
                assert span <= _resample.axis_taps(n_in, n_out, code, aa and code >= 2, torch.float32)


def test_header_entry_and_binding():
    hdr = (ROOT / "include" / "holocron_b200.h").read_text()
    assert "holocron/transforms/interpolation.py:87-96" in hdr
    decl = re.search(r"int (hb_resample_batch)\((.*?)\);", hdr, flags=re.S)
    assert decl is not None
    assert _lib.SIGNATURES["hb_resample_batch"] == "p" + "i" * 8 + "p"
    assert len(decl.group(2).split(",")) == 10


def test_dtype_codes_match_the_kernels():
    text = (ROOT / "holocron_b200" / "csrc" / "common.cuh").read_text()
    codes = {name: int(v) for name, v in re.findall(r"#define HB_DTYPE_(\w+) (\d+)", text)}
    names = {torch.float32: "F32", torch.bfloat16: "BF16", torch.float16: "F16", torch.uint8: "U8",
             torch.float64: "F64"}
    assert codes == {names[dt]: code for dt, code in _table.DTYPES.items()}


def test_pil_and_cpu_tensors_refused():
    pil = Image.fromarray(np.full((16, 32, 3), 255, dtype=np.uint8))
    cpu = torch.rand(3, 16, 32)
    for tf in (T.Resize((32, 32), mode=ResizeMethod.PAD), T.Resize((32, 32)), T.Resize((16, 32)),
               T.RandomZoomOut((32, 32), scale=(0.5, 0.99))):
        for img in (pil, cpu, [cpu]):
            with pytest.raises(HolocronB200Error):
                tf(img)


def test_zoom_identity_returns_input():
    """scale[0] == 1 hands the input back unchanged, as the reference does, without a draw."""
    tf = T.RandomZoomOut((32, 32), scale=(1.0, 1.0))
    x = torch.rand(3, 16, 16)
    torch.manual_seed(0)
    first = torch.rand(1)
    torch.manual_seed(0)
    assert tf(x) is x
    assert torch.equal(torch.rand(1), first)


def test_inputs_the_reference_refuses():
    with pytest.raises(ValueError):
        T.Resize((8, 8), mode=ResizeMethod.PAD).get_params(torch.rand(1, 3, 8, 8))
    with pytest.raises(ValueError):
        T.RandomZoomOut((8, 8)).get_params(torch.rand(1, 3, 8, 8))
    with pytest.raises(TypeError):
        T.Resize((8, 8), mode=ResizeMethod.PAD).get_params(np.zeros((3, 8, 8)))
    with pytest.raises(NotImplementedError):
        _resample.interpolation_code(_resample.InterpolationMode.LANCZOS)
    with pytest.raises(ValueError):
        _resample.resample([torch.rand(3, 4, 4)], [(4, 4)], (4, 4), _resample.InterpolationMode.BILINEAR, True,
                           pad_mode="wrap")


def test_descriptor_table():
    """The descriptor rows of a list with a strided view, a box larger than its canvas and a 4-D source."""
    a = torch.zeros(3, 40, 60)[:, ::2, 1::3]
    b = torch.zeros(2, 3, 7, 9, dtype=torch.float32)
    table, ty, tx = _resample.descriptor_table([a, b], [(34, 30), (15, 16)], (33, 32), 2, True, "edge")
    assert table.shape == (3, 16)
    assert table[0].tolist() == [a.data_ptr(), 0, 2400, 120, 3, 3, 20, 20, 34, 30, -1, 1, 33, 32, 1, 0]
    assert table[1].tolist() == [b.data_ptr(), 0, 63, 9, 1, 3, 7, 9, 15, 16, 9, 8, 33, 32, 1, 0]
    assert table[2, 0] == b.data_ptr() + 3 * 7 * 9 * 4
    assert (ty, tx) == (3, 3)  # upscales: the triangle's support of 1 on each side
    with pytest.raises(RuntimeError):
        _resample.descriptor_table([a], [(4, 30)], (33, 32), 2, True, "reflect")
    with pytest.raises(IndexError):
        _resample.descriptor_table([a], [(4, 30)], (33, 32), 2, True, "symmetric")
    with pytest.raises(NotImplementedError):
        _resample.descriptor_table([torch.zeros(1, 2, 4000)], [(2, 10)], (2, 10), 3, True, "constant")
