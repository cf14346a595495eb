"""holocron_b200.transforms on the GPU: per element against the fp64 oracle (tests/_transforms_oracle.py), against
torchvision's resize + pad run on the same CUDA tensor (what the reference executes), against the reference's CPU
outputs (tests/golden/transforms.pt), and the batching, placement, refusal and determinism properties of the one-launch
kernel.

Bounds. Float outputs: |out - oracle| <= REL[filter] * sum|terms|, plus one ulp of the output dtype for fp16 / bf16,
whose fp32 result is rounded once more, plus a position term. Every implementation computes its sample positions
scale * (i + 0.5) - 0.5 in fp32 (fp64 for fp64 images), and one that contracts them into a fused multiply-add moves a
position by an ulp of the coordinate, which moves the value by that ulp times the step between neighbouring source
values: the position term is eps * (longest side) * 2 axes * 2 max|x| (x1.5 for bicubic). REL covers the rounding of
the weights and sums (fp32: about 80 ulps of sum|terms| for bilinear, 170 for bicubic, whose filters have negative
lobes). uint8 outputs equal the oracle's clamped, half-to-even rounding except where the fp64 value lies within
max(1e-4, REL * sum|terms| + position term) of a .5 tie; those ties are counted and bounded."""
from pathlib import Path

import numpy as np
import pytest
import torch
import torchvision.transforms.functional as TF
from torchvision.transforms.functional import InterpolationMode

import _transforms_oracle as O
from holocron_b200 import _lib
from holocron_b200 import transforms as T
from holocron_b200.transforms import _resample
from holocron_b200.transforms.interpolation import ResizeMethod

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
ROOT = Path(__file__).resolve().parents[1]
DTYPES = (torch.uint8, torch.float16, torch.bfloat16, torch.float32, torch.float64)
INTERP = {name: InterpolationMode(name) for name in O.FILTERS}
TIE = 1e-4
REL32 = {"nearest": 0.0, "nearest-exact": 0.0, "bilinear": 1e-5, "bicubic": 2e-5}
REL64 = {"nearest": 0.0, "nearest-exact": 0.0, "bilinear": 1e-12, "bicubic": 1e-12}


def _image(shape, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    if dtype == torch.uint8:
        return torch.randint(0, 256, shape, generator=g, dtype=torch.uint8).to(DEV)
    return (torch.rand(shape, generator=g, dtype=torch.float64) * 4 - 1).to(dtype).to(DEV)


def _position_term(x, interp):
    """One rounding of a sample coordinate (an ulp of the longest side) times the largest step between neighbouring
    source values, per axis: what a position computed with or without a fused multiply-add can move a value by."""
    if interp.startswith("nearest"):
        return 0.0
    eps = torch.finfo(torch.float64 if x.dtype == torch.float64 else torch.float32).eps
    return eps * max(x.shape[-2:]) * 2 * 2 * float(x.double().abs().max()) * (1.5 if interp == "bicubic" else 1.0)


def _bound(dtype, interp, value, mag, pos=0.0):
    rel = (REL64 if dtype == torch.float64 else REL32)[interp]
    b = rel * mag + pos
    if dtype in (torch.float16, torch.bfloat16):
        b = b + torch.finfo(dtype).eps * np.exp2(np.floor(np.log2(np.maximum(np.abs(value), 1e-30))))
    return b


def check_oracle(out, value, mag, interp, x=None):
    """Asserts the per-element bound (with the position term of source x); returns the number of uint8 elements rounded
    the other way at a tie."""
    pos = 0.0 if x is None else _position_term(x, interp)
    got = out.detach().cpu()
    assert tuple(got.shape) == value.shape
    if got.dtype == torch.uint8:
        want = O.to_uint8(value)
        diff = got.numpy().astype(np.int64) - want
        window = np.maximum(TIE, REL32[interp] * mag + pos)
        assert (np.abs(diff) <= 1).all()
        assert not ((diff != 0) & (O.tie_distance(np.clip(value, 0, 255)) >= window)).any()
        return int((diff != 0).sum())
    err = np.abs(got.double().numpy() - value)
    bound = _bound(got.dtype, interp, value, mag, pos)
    assert (err <= bound).all(), (float(err.max()), float((err - bound).max()))
    return 0


def check_pair(a, b, value, mag, interp, x=None):
    """Two executions of the same resize (ours, torchvision's): each within the bound of the fp64 value."""
    check_oracle(a, value, mag, interp, x)
    check_oracle(b, value, mag, interp, x)


def torchvision_chain(x, inner, canvas, interp, antialias, pad_mode="constant"):
    """The reference's execution on a CUDA tensor: torchvision resize, then pad (negative padding crops)."""
    y = TF.resize(x, list(inner), INTERP[interp], antialias=antialias)
    dh, dw = canvas[0] - inner[0], canvas[1] - inner[1]
    return TF.pad(y, [dw // 2, dh // 2, dw - dw // 2, dh - dh // 2], padding_mode=pad_mode)


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=str)
@pytest.mark.parametrize("interp", O.FILTERS)
@pytest.mark.parametrize("antialias", [True, False])
def test_squish_every_dtype_filter(dtype, interp, antialias):
    x = _image((3, 37, 53), dtype, 1)
    ties = 0
    for size in [(24, 32), (61, 70), (37, 20)]:
        out = T.Resize(size, interpolation=INTERP[interp], antialias=antialias)(x)
        value, mag = O.resize_pad(x, size, size, interp, antialias)
        ties += check_oracle(out, value, mag, interp, x)
        check_pair(out, TF.resize(x, list(size), INTERP[interp], antialias=antialias), value, mag, interp, x)
    assert ties <= 1e-3 * 3 * (24 * 32 + 61 * 70 + 37 * 20)


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
@pytest.mark.parametrize("interp", O.FILTERS)
@pytest.mark.parametrize("pad_mode", O.PAD_MODES)
def test_pad_every_dtype_filter_pad_mode(dtype, interp, pad_mode):
    tf = T.Resize((48, 40), mode=ResizeMethod.PAD, pad_mode=pad_mode, interpolation=INTERP[interp])
    for shape in [(3, 50, 23), (3, 30, 45)]:
        x = _image(shape, dtype, 2)
        inner = tf.get_params(x)
        out = tf(x)
        value, mag = O.resize_pad(x, inner, (48, 40), interp, True, pad_mode)
        check_pair(out, torchvision_chain(x, inner, (48, 40), interp, True, pad_mode), value, mag, interp, x)


@pytest.mark.parametrize("interp", O.FILTERS)
@pytest.mark.parametrize("antialias", [True, False])
@pytest.mark.parametrize("case", [((3, 256, 200), (32, 25)), ((3, 12, 10), (48, 40)), ((2, 801, 9), (100, 36)),
                                  ((3, 1, 7), (1, 28)), ((1, 1, 1), (3, 4)), ((3, 9, 1), (2, 1))])
def test_heavy_scales_and_one_pixel_sides(interp, antialias, case):
    """Downscales to 1/8, upscales to 4x, and 1-pixel sides, in fp32 and uint8."""
    shape, size = case
    for dtype in (torch.float32, torch.uint8):
        x = _image(shape, dtype, 3)
        out = T.Resize(size, interpolation=INTERP[interp], antialias=antialias)(x)
        value, mag = O.resize_pad(x, size, size, interp, antialias)
        check_pair(out, TF.resize(x, list(size), INTERP[interp], antialias=antialias), value, mag, interp, x)


def test_one_pixel_box_in_every_pad_mode():
    x = _image((3, 1, 7), torch.float32, 4)
    for pad_mode in O.PAD_MODES:
        tf = T.Resize((5, 5), mode=ResizeMethod.PAD, pad_mode=pad_mode)
        inner = tf.get_params(x)
        assert inner == (1, 5)
        if pad_mode == "reflect":
            with pytest.raises(RuntimeError):
                tf(x)
            continue
        if pad_mode == "symmetric":  # torchvision indexes past the 1-row image (IndexError on CPU tensors)
            with pytest.raises(IndexError):
                tf(x)
            continue
        value, mag = O.resize_pad(x, inner, (5, 5), "bilinear", True, pad_mode)
        out = tf(x)
        check_pair(out, torchvision_chain(x, inner, (5, 5), "bilinear", True, pad_mode), value, mag, "bilinear", x)


def test_reflect_refused_before_any_launch():
    tf = T.Resize((40, 40), mode=ResizeMethod.PAD, pad_mode="reflect")
    x = _image((3, 4, 40), torch.float32, 5)  # inner (4, 40): 18 rows of padding above a 4-row image
    _lib.lib().hb_launch_count_reset()
    with pytest.raises(RuntimeError):
        tf(x)
    with pytest.raises(RuntimeError):
        tf([_image((3, 40, 40), torch.float32, 6), x])
    assert _lib.lib().hb_launch_count() == 0
    with pytest.raises(RuntimeError):
        torchvision_chain(x, tf.get_params(x), (40, 40), "bilinear", True, "reflect")


def test_negative_padding_crops():
    """RandomZoomOut boxes one pixel larger than the canvas: the box is cropped like torchvision's negative pad."""
    G = torch.load(ROOT / "tests" / "golden" / "transforms.pt", weights_only=False)
    seen = 0
    for r in G["zoom_outputs"]:
        if r["hw"][0] <= r["size"][0] and r["hw"][1] <= r["size"][1]:
            continue
        seen += 1
        x = r["x"].to(DEV)
        tf = T.RandomZoomOut(r["size"], scale=r["scale"], interpolation=INTERP[r["interpolation"]],
                             antialias=r["antialias"])
        torch.manual_seed(r["seed"])
        out = tf(x)
        value, mag = O.resize_pad(x, r["hw"], r["size"], r["interpolation"], r["antialias"])
        tv = torchvision_chain(x, r["hw"], r["size"], r["interpolation"], r["antialias"])
        check_pair(out, tv, value, mag, r["interpolation"], x)
    assert seen >= 6


def test_golden_reference_outputs():
    G = torch.load(ROOT / "tests" / "golden" / "transforms.pt", weights_only=False)
    for r in G["outputs"]:
        x = r["x"].to(DEV)
        mode = ResizeMethod.SQUISH if r["kind"] == "squish" else ResizeMethod.PAD
        tf = T.Resize(r["size"], mode=mode, pad_mode=r["pad_mode"], interpolation=INTERP[r["interpolation"]],
                      antialias=r["antialias"])
        if r.get("error") is not None:
            with pytest.raises(Exception) as info:
                tf(x)
            assert type(info.value).__name__ == r["error"]
            continue
        out = tf(x)
        inner = r["size"] if r["kind"] == "squish" else tf.get_params(x)
        value, mag = O.resize_pad(x, inner, r["size"], r["interpolation"], r["antialias"], r["pad_mode"])
        check_pair(out, r["y"], value, mag, r["interpolation"], r["x"])
    for r in G["zoom_outputs"]:
        tf = T.RandomZoomOut(r["size"], scale=r["scale"], interpolation=INTERP[r["interpolation"]],
                             antialias=r["antialias"])
        torch.manual_seed(r["seed"])
        out = tf(r["x"].to(DEV))
        value, mag = O.resize_pad(r["x"], r["hw"], r["size"], r["interpolation"], r["antialias"])
        check_pair(out, r["y"], value, mag, r["interpolation"], r["x"])


@pytest.mark.parametrize("dtype", [torch.uint8, torch.float32, torch.bfloat16])
def test_strided_views_read_in_place(dtype):
    base = _image((3, 90, 121), dtype, 7)
    hwc = _image((67, 45, 3), dtype, 8)
    views = [base[:, ::2, 1::3], hwc.permute(2, 0, 1), base[1:, 5:70, :].transpose(1, 2)]
    for tf in (T.Resize((30, 30), mode=ResizeMethod.PAD, pad_mode="reflect"), T.Resize((21, 50)),
               T.Resize((30, 30), mode=ResizeMethod.PAD, interpolation=InterpolationMode.BICUBIC)):
        for v in views:
            assert not v.is_contiguous()
            assert torch.equal(tf(v), tf(v.contiguous()))


def test_list_equals_per_image_calls():
    imgs = [_image((3, h, w), torch.uint8, 10 + k) for k, (h, w) in enumerate([(300, 451), (500, 333), (224, 224),
                                                                                (60, 90), (480, 480)])]
    for tf in (T.Resize((224, 224), mode=ResizeMethod.PAD), T.Resize((224, 224), mode=ResizeMethod.PAD,
                                                                     pad_mode="symmetric"),
               T.Resize((64, 96), interpolation=InterpolationMode.BICUBIC)):
        batch = tf(imgs)
        assert batch.shape == (5, 3, *tf.size)
        singles = torch.stack([tf(x) if tuple(x.shape[-2:]) != tuple(tf.size) else tf(x).clone() for x in imgs])
        assert torch.equal(batch, singles)
        assert torch.equal(tf(tuple(imgs)), batch)


def test_zoom_out_list_equals_seeded_image_by_image():
    imgs = [_image((3, h, w), torch.float32, 20 + k) for k, (h, w) in enumerate([(300, 451), (500, 333), (31, 40),
                                                                                 (90, 17)])]
    tf = T.RandomZoomOut((64, 64), scale=(0.2, 0.999))
    torch.manual_seed(123)
    batch = tf(imgs)
    after_list = torch.rand(1)
    torch.manual_seed(123)
    singles = torch.stack([tf(x) for x in imgs])
    after_singles = torch.rand(1)
    assert torch.equal(batch, singles)
    assert torch.equal(after_list, after_singles)
    torch.manual_seed(123)
    for x, y in zip(imgs, batch):
        inner = tf.get_params(x)
        value, mag = O.resize_pad(x, inner, (64, 64), "bilinear", True)
        check_oracle(y, value, mag, "bilinear", x)


def test_squish_leading_dims_and_identity():
    x = _image((2, 3, 40, 50), torch.float16, 30)
    out = T.Resize((20, 60))(x)
    assert out.shape == (2, 3, 20, 60)
    assert torch.equal(out, torch.stack([T.Resize((20, 60))(x[i]) for i in range(2)]))
    y = _image((40, 50), torch.float32, 31)
    assert torch.equal(T.Resize((20, 60))(y), T.Resize((20, 60))(y[None])[0])
    z = _image((3, 20, 60), torch.uint8, 32)
    assert T.Resize((20, 60))(z) is z  # torchvision returns the input itself at the target size
    with pytest.raises(ValueError):
        T.Resize((8, 8), mode=ResizeMethod.PAD)(x)
    with pytest.raises(ValueError):
        T.RandomZoomOut((8, 8))(x)


def test_sentinels_around_the_output_stay_untouched():
    imgs = [_image((3, 33, 47), torch.uint8, 40), _image((3, 60, 20), torch.uint8, 41)]
    n = 2 * 3 * 24 * 24
    buf = torch.full((n + 2048,), 0xA5, dtype=torch.uint8, device=DEV)
    out = buf[1024:1024 + n].view(2, 3, 24, 24)
    # boxes larger than the canvas on both axes: nothing outside the canvas may be written
    _resample.resample(imgs, [(26, 27), (25, 26)], (24, 24), InterpolationMode.BILINEAR, True, "constant", out=out)
    torch.cuda.synchronize()
    assert (buf[:1024] == 0xA5).all() and (buf[1024 + n:] == 0xA5).all()
    for x, inner, y in zip(imgs, [(26, 27), (25, 26)], out):
        value, mag = O.resize_pad(x, inner, (24, 24), "bilinear", True)
        check_oracle(y, value, mag, "bilinear", x)


def test_two_runs_bit_identical_and_one_launch():
    imgs = [_image((3, 300 + 7 * k, 500 - 11 * k), torch.float32, 50 + k) for k in range(8)]
    tf = T.Resize((224, 224), mode=ResizeMethod.PAD, interpolation=InterpolationMode.BICUBIC)
    a = tf(imgs)
    _lib.lib().hb_launch_count_reset()
    b = tf(imgs)
    assert _lib.lib().hb_launch_count() == 1
    assert torch.equal(a, b)


def test_reference_test_cases_on_cuda():
    """The tensor cases of the reference's tests/test_transforms.py, on CUDA tensors."""
    img1 = np.full((16, 32, 3), 255, dtype=np.uint8)
    img2 = np.full((32, 16, 3), 255, dtype=np.uint8)
    tf = T.Resize((32, 32), mode=ResizeMethod.PAD)
    assert isinstance(tf, torch.nn.Module)
    out = tf(torch.from_numpy(img1).to(dtype=torch.float32).permute(2, 0, 1).to(DEV) / 255)
    assert isinstance(out, torch.Tensor) and out.shape == (3, 32, 32)
    np_out = out.cpu().numpy()
    assert np.all(np.abs(np_out[:, 8:-8] - 1) <= 2 * np.finfo(np.float32).eps)
    assert np.all(np_out[:, :8] == 0)
    out = tf(torch.from_numpy(img2).to(dtype=torch.float32).permute(2, 0, 1).to(DEV) / 255)
    assert out.shape == (3, 32, 32)
    np_out = out.cpu().numpy()
    assert np.all(np.abs(np_out[:, :, 8:-8] - 1) <= 2 * np.finfo(np.float32).eps)
    assert np.all(np_out[:, :, :8] == 0)

    torch_img = torch.ones((3, 64, 64), dtype=torch.float32, device=DEV)
    tf = T.RandomZoomOut((32, 32), scale=(0.5, 0.99))
    out = tf(torch_img)
    assert isinstance(out, torch.Tensor) and out.shape == (3, 32, 32)
    np_out = out.cpu().numpy()
    # the box is an antialiased downscale of ones: its fp32 weights, normalised by an fp32 division, sum to 1 within
    # an ulp or two (the reference asserts == 1 on the CPU)
    assert np.all(np.abs(np_out[:, 16, 16] - 1) <= 2 * np.finfo(np.float32).eps)
    assert np_out.mean() < 1
