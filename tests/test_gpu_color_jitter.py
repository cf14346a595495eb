"""ColorJitter of holocron_b200.transforms on the GPU, against torchvision's ``ColorJitter`` chain
(``adjust_brightness``, ``adjust_contrast``, ``adjust_saturation``, ``adjust_hue`` in the drawn order) on the same
CUDA images: every one of the 24 op orders and orders with one to three ops off, both channel counts, uint8 and fp32,
at the segmentation recipe's 256x256 crop, odd and degenerate sizes and 16-pixel tails; every uint8 colour through hue
and saturation; constant, gray and two-valued content; strided sources; a recipe batch through the module; single
tensors; launches, determinism, sentinels and synchronisation.

Bars. uint8 is bit-identical, except that on images over 65,793 pixels (where torch's fp32 sum of a uint8 grayscale can
be inexact) a contrast value may be one off where its exact value lies within reach of that sum of an integer; those
images are tested with contrast last. fp32 is bit-identical for brightness, saturation and hue. For contrast, and every
op after it, the mean here is an fp64 sum in a fixed order rounded to fp32, and torch's is an fp32 tree reduction:
with d = |torch's mean - this mean| measured on the image (plus one ulp of the mean for the rounding of the fp64 sum),
contrast's output moves by at most |1 - r| * d, and each later op multiplies that difference by at most its Lipschitz
constant in the max norm over channels: r for brightness, |r| + |1 - r| for saturation (the grayscale weights sum to
0.9999), and 3 for hue (the shifted middle channel is min +- (mid - min) + c * (max - min) with |c| <= 2 on each piece
of the piecewise-linear map, a row sum of at most 3; max and min pass through, and sorting is 1-Lipschitz). Each op
after contrast also rounds on its own: 2^-18 (32 ulps of 1.0) per op covers the fp32 roundings of the longest op,
hue."""
import itertools

import numpy as np
import pytest
import torch
from torchvision.transforms import functional as TVF
from torchvision.transforms import transforms as TVT

from holocron_b200 import _lib
from holocron_b200 import transforms as T
from holocron_b200.transforms import _color, augmentation

pytestmark = pytest.mark.gpu

EXACT_SUM = 2 ** 24 // 255  # 65,793: below it the fp32 sum of a uint8 grayscale is exact in any order
ROUNDING = 2.0 ** -18
RECIPE = {"brightness": 0.3, "contrast": 0.3, "saturation": 0.1, "hue": 0.02}
ORDERS = list(itertools.permutations(range(4)))
# (brightness, contrast, saturation, hue) factors: the recipe's range, and the edges (0 blends, hue +-0.5 and 0)
FACTORS = [(1.21, 0.77, 1.08, 0.013), (0.0, 0.0, 0.0, 0.5), (0.5, 1.8, 0.0, -0.5), (1.7, 0.0, 2.0, 0.0),
           (0.9, 1.3, 0.6, -0.02)]
ADJUST = (TVF.adjust_brightness, TVF.adjust_contrast, TVF.adjust_saturation, TVF.adjust_hue)


def _draw(order, factors, off=()):
    return (torch.tensor(order), *[None if k in off else f for k, f in enumerate(factors)])


def _torchvision(img, draw, upto=None):
    """torchvision's ColorJitter.forward for this draw; with ``upto``, only the ops before the op ``upto``."""
    fn_idx, *factors = draw
    for k in fn_idx.tolist():
        if k == upto:
            break
        if factors[k] is not None:
            img = ADJUST[k](img, factors[k])
    return img


def _fp32_tolerance(img, draw):
    """The bound of the module docstring for one fp32 image (0 when it has no contrast op)."""
    fn_idx, *factors = draw
    ops = [k for k in fn_idx.tolist() if factors[k] is not None]
    if 1 not in ops:
        return 0.0
    prefix = _torchvision(img, draw, upto=1)
    gray = TVF.rgb_to_grayscale(prefix) if img.shape[-3] == 3 else prefix
    theirs = torch.mean(gray, dim=(-3, -2, -1)).item()
    n = gray.shape[-1] * gray.shape[-2]
    ours = float(np.float32(gray.double().sum().item()) * (np.float32(1.0) / np.float32(n)))
    d = abs(theirs - ours) + float(np.spacing(np.float32(max(abs(ours), 1e-30))))
    c = factors[1]
    tol = abs(1.0 - c) * d + ROUNDING
    rgb = img.shape[-3] == 3
    for k in ops[ops.index(1) + 1:]:
        f = factors[k]
        lip = {0: abs(f), 2: abs(f) + abs(1.0 - f) if rgb else 1.0, 3: 3.0 if rgb else 1.0}[k]
        tol = tol * lip + ROUNDING
    return tol


def _check(got, want, img, draw):
    if img.dtype == torch.uint8:
        assert torch.equal(got, want), (tuple(img.shape), draw, int((got != want).sum()))
        return
    tol = _fp32_tolerance(img, draw)
    if tol == 0.0:
        assert torch.equal(got, want), (tuple(img.shape), draw, int((got != want).sum()),
                                        (got - want).abs().max().item())
    else:
        err = (got.double() - want.double()).abs().max().item()
        assert err <= tol, (tuple(img.shape), draw, err, tol)


def _image(kind, C, H, W, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    if kind == "random":
        x = torch.randint(0, 256, (C, H, W), generator=g, dtype=torch.uint8)
        if dtype == torch.float32:
            return torch.rand(C, H, W, generator=g).cuda()
    elif kind == "constant":
        x = torch.full((C, H, W), 93, dtype=torch.uint8)
    elif kind == "gray":  # r == g == b: the maxc == minc branch of _rgb2hsv
        x = torch.randint(0, 256, (1, H, W), generator=g, dtype=torch.uint8).expand(C, H, W).contiguous()
    else:  # two-valued
        x = torch.randint(0, 2, (C, H, W), generator=g, dtype=torch.uint8) * 170 + 40
    return (x if dtype == torch.uint8 else x.float() / 255).cuda()


def _draws():
    """Every order with all four factors (at every factor set), and every subset of one to three ops off."""
    draws = [_draw(o, f) for f in FACTORS for o in ORDERS]
    for r in (1, 2, 3):
        for i, off in enumerate(itertools.combinations(range(4), r)):
            for j, f in enumerate(FACTORS):
                draws.append(_draw(ORDERS[(7 * i + 5 * j + r) % 24], f, off))
    return draws


def _sweep(img, draws):
    out = _color.jitter([img] * len(draws), draws)
    for got, draw in zip(out, draws):
        _check(got, _torchvision(img, draw), img, draw)


SHAPES = [(256, 256), (37, 53), (1, 19), (19, 1), (2, 2), (1, 1), (21, 35), (5, 100), (3, 33), (4, 47)]


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("C", [1, 3])
@pytest.mark.parametrize("dtype", [torch.uint8, torch.float32])
def test_every_order_matches_torchvision(shape, C, dtype):
    _sweep(_image("random", C, *shape, dtype, seed=shape[0] * 7 + shape[1] + C), _draws())


@pytest.mark.parametrize("kind", ["constant", "gray", "two-valued"])
@pytest.mark.parametrize("C", [1, 3])
@pytest.mark.parametrize("dtype", [torch.uint8, torch.float32])
def test_degenerate_content(kind, C, dtype):
    draws = [_draw(o, f) for f in FACTORS[:3] for o in ORDERS]
    for shape in ((64, 64), (9, 14)):
        _sweep(_image(kind, C, *shape, dtype, seed=3), draws)


def test_fp32_edge_values():
    below_one = float(np.nextafter(np.float32(1.0), np.float32(0.0)))
    g = torch.Generator().manual_seed(8)
    idx = torch.randint(0, 3, (3, 40, 50), generator=g)
    img = torch.tensor([0.0, 1.0, below_one])[idx].cuda()
    for C in (1, 3):
        _sweep(img[:C].contiguous(), [_draw(o, f) for f in FACTORS for o in ORDERS])


def test_large_uint8_contrast():
    """Over 65,793 pixels: contrast last (alone or after the others), one off at most, and only where torch's inexact
    fp32 sum can reach the rounding of its exact value."""
    img = _image("random", 3, 512, 640, torch.uint8, seed=5)
    assert 512 * 640 > EXACT_SUM
    img[:, :200] //= 4  # skewed content: a mean away from 127.5
    draws = [_draw(o, f, off) for f in FACTORS for o, off in (((1, 0, 2, 3), (0, 2, 3)), ((0, 2, 3, 1), ()),
                                                              ((3, 0, 2, 1), ()))]
    for C in (1, 3):
        x = img[:C].contiguous()
        out = _color.jitter([x] * len(draws), draws)
        for got, draw in zip(out, draws):
            prefix = _torchvision(x, draw, upto=1)
            want = _torchvision(x, draw)
            diff = (got.int() - want.int()).abs().cpu()
            gray = TVF.rgb_to_grayscale(prefix) if C == 3 else prefix
            mean = gray.double().mean().item()
            r = draw[2]
            v = r * prefix.double().cpu() + (1 - r) * mean
            near = (v - v.round()).abs() < abs(1 - r) * mean * 2.0 ** -16 + 2.0 ** -20
            assert diff.max() <= 1 and not (diff.bool() & ~near).any(), draw


def _every_colour():
    idx = torch.arange(2 ** 24, dtype=torch.int32, device="cuda")
    return torch.stack([idx >> 16, (idx >> 8) & 255, idx & 255]).to(torch.uint8).view(3, 4096, 4096)


def test_every_uint8_colour_through_hue_and_saturation():
    img = _every_colour()
    g = torch.Generator().manual_seed(9)
    hues = [0.5, -0.5, 0.02, -0.02, 0.0] + [float(v) for v in torch.rand(3, generator=g) - 0.5]
    for h in hues:
        got = _color.jitter([img], [_draw((3, 0, 1, 2), (0, 0, 0, h), (0, 1, 2))])[0]
        assert torch.equal(got, TVF.adjust_hue(img, h)), h
    for s in (0.0, 0.3, 1.1, 2.0):
        got = _color.jitter([img], [_draw((2, 0, 1, 3), (0, 0, s, 0), (0, 1, 3))])[0]
        assert torch.equal(got, TVF.adjust_saturation(img, s)), s
    # the same colours as fp32 images
    x = img.float() / 255
    for h in hues[:4]:
        got = _color.jitter([x], [_draw((3, 0, 1, 2), (0, 0, 0, h), (0, 1, 2))])[0]
        assert torch.equal(got, TVF.adjust_hue(x, h)), h


@pytest.mark.parametrize("layout", ["channels_last", "cropped", "unbind"])
@pytest.mark.parametrize("dtype", [torch.uint8, torch.float32])
def test_strided_sources(layout, dtype):
    g = torch.Generator().manual_seed(11)
    batch = torch.randint(0, 256, (4, 3, 40, 61), generator=g, dtype=torch.uint8).cuda()
    if dtype == torch.float32:
        batch = batch.float() / 255
    if layout == "channels_last":
        sources = batch.to(memory_format=torch.channels_last).unbind(0)
    elif layout == "cropped":
        sources = [b[:, 3:36, 5:58] for b in batch]
    else:
        sources = batch.unbind(0)
    draws = _draws()
    for i, x in enumerate(sources):
        chosen = draws[i::len(sources)]
        out = _color.jitter([x] * len(chosen), chosen)
        for got, draw in zip(out, chosen):
            _check(got, _torchvision(x, draw), x, draw)


@pytest.mark.parametrize("dtype", [torch.uint8, torch.float32])
def test_recipe_batch_matches_module_image_by_image(monkeypatch, dtype):
    g = torch.Generator().manual_seed(2)
    batch = torch.randint(0, 256, (256, 3, 256, 256), generator=g, dtype=torch.uint8).cuda()
    if dtype == torch.float32:
        batch = batch.float() / 255
    batch = batch.to(memory_format=torch.channels_last)
    recorded = []
    real = augmentation.jitter
    monkeypatch.setattr(augmentation, "jitter", lambda s, draws: recorded.extend(draws) or real(s, draws))
    torch.manual_seed(123)
    out = T.ColorJitter(**RECIPE)(batch.unbind(0))
    after = torch.random.get_rng_state()
    assert out.shape == batch.shape and out.is_contiguous()
    tv = TVT.ColorJitter(**RECIPE)
    torch.manual_seed(123)
    want = [tv(x) for x in batch.unbind(0)]
    assert torch.equal(torch.random.get_rng_state(), after)
    for x, got, w, draw in zip(batch.unbind(0), out, want, recorded):
        _check(got, w, x, draw)


def test_single_tensor_matches_module():
    g = torch.Generator().manual_seed(4)
    x8 = torch.randint(0, 256, (4, 3, 37, 53), generator=g, dtype=torch.uint8).cuda()
    for x in (x8, x8.float() / 255, x8[:, :1], x8.view(2, 2, 3, 37, 53)):
        for seed in range(12):
            torch.manual_seed(seed)
            got = T.ColorJitter(0.4, 0.4, 0.4, 0.2)(x)
            after = torch.random.get_rng_state()
            tf = TVT.ColorJitter(0.4, 0.4, 0.4, 0.2)
            torch.manual_seed(seed)
            want = tf(x)
            assert torch.equal(torch.random.get_rng_state(), after)
            assert got.shape == x.shape
            torch.manual_seed(seed)
            draw = tf.get_params(tf.brightness, tf.contrast, tf.saturation, tf.hue)
            if x.dtype == torch.uint8:
                assert torch.equal(got, want), seed
            else:
                for i in range(x.shape[0]):
                    _check(got[i], want[i], x[i], draw)


def test_launches_determinism_sentinels_and_no_sync():
    lib = _lib.lib()
    g = torch.Generator().manual_seed(6)
    imgs = torch.randint(0, 256, (16, 3, 29, 45), generator=g, dtype=torch.uint8).cuda().unbind(0)
    with_contrast = [_draw(ORDERS[k], FACTORS[0]) for k in range(16)]
    without = [_draw(ORDERS[k], FACTORS[0], (1,)) for k in range(16)]
    C, H, W = 3, 29, 45
    n = C * H * W
    for dtype in (torch.uint8, torch.float32):
        xs = [x if dtype == torch.uint8 else x.float() / 255 for x in imgs]
        for chosen, launches in ((with_contrast, 2), (without, 1)):
            buf = torch.full(((len(xs) + 2) * n,), 0xA5 if dtype == torch.uint8 else -7.0, dtype=dtype,
                             device="cuda")
            out = buf[n:-n].view(len(xs), C, H, W)
            lib.hb_launch_count_reset()
            _color.jitter(xs, chosen, out=out)
            assert lib.hb_launch_count() == launches
            assert bool((buf[:n] == buf[0]).all()) and bool((buf[-n:] == buf[0]).all())
            again = _color.jitter(xs, chosen)
            assert torch.equal(out, again)
    tf = T.ColorJitter(**RECIPE)
    tf(list(imgs))  # warm-up: first launches load modules
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(8):
            lib.hb_launch_count_reset()
            tf(list(imgs))
            assert lib.hb_launch_count() == 2
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
