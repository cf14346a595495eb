"""TrivialAugmentWide of holocron_b200.transforms on the GPU, against torchvision's ``autoaugment._apply_op`` on the
same CUDA images: every op, magnitude bin and sign, both channel counts and interpolations, every fill kind, at the
recipe's size, odd and degenerate sizes, vector tails, one large image, constant and two-valued content, and strided
sources. The value-map, blend and stencil ops must be bit-identical (Contrast on images over 65,793 pixels may be one
off where its exact value is within fp32 reach of an integer); the affine ops must be bit-identical outside the pixels
the oracle of ``_autoaugment_oracle.py`` marks as ambiguous (its docstring derives the band)."""
import numpy as np
import pytest
import torch
from torchvision.transforms import InterpolationMode
from torchvision.transforms import autoaugment as TVA

from _autoaugment_oracle import apply_op as oracle_op, gray
from holocron_b200 import _lib
from holocron_b200 import transforms as T
from holocron_b200.transforms import _autoaugment, augmentation

pytestmark = pytest.mark.gpu

GEOMETRIC = ("ShearX", "ShearY", "TranslateX", "TranslateY", "Rotate")
NEAREST, BILINEAR = InterpolationMode.NEAREST, InterpolationMode.BILINEAR
EXACT_SUM = 2 ** 24 // 255  # 65,793: below it the fp32 sum of a uint8 grayscale is exact in any order
STATS = {"geometric": 0, "ambiguous": 0, "mismatched": 0}


def _every_op(num_bins=31):
    for op, (mags, signed) in TVA.TrivialAugmentWide()._augmentation_space(num_bins).items():
        for m in ([0.0] if mags.ndim == 0 else [float(v) for v in mags]):
            for sign in ((1.0, -1.0) if signed else (1.0,)):
                yield op, m * sign


def _image(kind, C, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    if kind == "random":
        x = torch.randint(0, 256, (C, H, W), generator=g, dtype=torch.uint8)
    elif kind == "constant":
        x = torch.full((C, H, W), 93, dtype=torch.uint8)
    else:  # two-valued
        x = torch.randint(0, 2, (C, H, W), generator=g, dtype=torch.uint8) * 170 + 40
    return x.cuda()


def _contrast_near_integer(img, magnitude):
    """Pixels whose exact Contrast blend r*v + (1 - r)*mean lies within the reach of torch's inexact fp32 sum of an
    integer (a relative sum error of up to 2^-16, far above what a tree reduction of 2^20 terms makes)."""
    x = img.double().cpu()
    mean = (x if x.shape[0] == 1 else torch.from_numpy(gray(img.cpu().numpy()).astype(np.float64))).mean().item()
    r = 1.0 + magnitude
    v = r * x + (1 - r) * mean
    bound = abs(1 - r) * mean * 2.0 ** -16 + 2.0 ** -20
    return (v - v.round()).abs() < bound


def _check(got, want, img, op, magnitude, interp, fill):
    """Asserts the bar of this op; returns nothing."""
    if op not in GEOMETRIC:
        if op == "Contrast" and img.shape[-1] * img.shape[-2] > EXACT_SUM:
            diff = (got.int() - want.int()).abs().cpu()
            assert diff.max() <= 1 and not (diff.bool() & ~_contrast_near_integer(img, magnitude)).any()
            return
        assert torch.equal(got, want), (op, magnitude, tuple(img.shape), int((got != want).sum()))
        return
    mism = (got != want).cpu().numpy()
    _, amb = oracle_op(img.cpu().numpy(), op, magnitude, interp == BILINEAR, fill)
    bad = mism & ~amb[None]
    assert not bad.any(), (op, magnitude, tuple(img.shape), interp, fill, int(bad.sum()), np.argwhere(bad)[:5])
    STATS["geometric"] += amb.size
    STATS["ambiguous"] += int(amb.sum())
    STATS["mismatched"] += int(mism.any(0).sum())


def _sweep(img, interp, fill, ops=None):
    ops = list(_every_op()) if ops is None else ops
    if fill is not None:
        ops = [o for o in ops if o[0] in GEOMETRIC]
    out = _autoaugment.apply_ops([img] * len(ops), ops, interp, fill)
    for (op, m), got in zip(ops, out):
        want = TVA._apply_op(img, op, m, interp, fill)
        _check(got, want, img, op, m, interp, fill)


SHAPES = [(176, 176), (37, 53), (1, 19), (19, 1), (2, 2), (3, 3), (21, 35), (5, 100)]


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("C", [1, 3])
@pytest.mark.parametrize("interp", [NEAREST, BILINEAR])
def test_every_op_matches_torchvision(shape, C, interp):
    img = _image("random", C, *shape, seed=shape[0] * 7 + C)
    for fill in (None, [128.0], [float(60 * c + 7) for c in range(C)]):
        _sweep(img, interp, fill)


@pytest.mark.parametrize("kind", ["constant", "two-valued"])
@pytest.mark.parametrize("C", [1, 3])
def test_degenerate_content(kind, C):
    for shape in ((176, 176), (9, 14)):
        img = _image(kind, C, *shape, seed=3)
        for interp in (NEAREST, BILINEAR):
            _sweep(img, interp, None if interp == NEAREST else [200.0])


def test_large_image():
    img = _image("random", 3, 768, 1024, seed=5)
    # skewed content: large, uneven Equalize counts
    img[:, :300] //= 8
    ops = [o for o in _every_op(7)]
    _sweep(img, BILINEAR, None, ops)
    _sweep(img[:1].contiguous(), NEAREST, None, [o for o in ops if o[0] not in GEOMETRIC])


@pytest.mark.parametrize("layout", ["channels_last", "cropped", "unbind"])
def test_strided_sources(layout):
    g = torch.Generator().manual_seed(11)
    batch = torch.randint(0, 256, (4, 3, 40, 61), generator=g, dtype=torch.uint8).cuda()
    if layout == "channels_last":
        sources = batch.to(memory_format=torch.channels_last).unbind(0)
    elif layout == "cropped":
        sources = [b[:, 3:36, 5:58] for b in batch]
    else:
        sources = batch.unbind(0)
    ops = list(_every_op(5))
    for i, x in enumerate(sources):
        chosen = ops[i::len(sources)]
        out = _autoaugment.apply_ops([x] * len(chosen), chosen, BILINEAR, [9.0, 99.0, 199.0])
        for (op, m), got in zip(chosen, out):
            _check(got, TVA._apply_op(x.contiguous(), op, m, BILINEAR, [9.0, 99.0, 199.0]), x, op, m, BILINEAR,
                   [9.0, 99.0, 199.0])


def test_mixed_batch_matches_module_image_by_image(monkeypatch):
    g = torch.Generator().manual_seed(2)
    batch = torch.randint(0, 256, (256, 3, 176, 176), generator=g, dtype=torch.uint8).cuda()
    batch = batch.to(memory_format=torch.channels_last)
    recorded = []
    real = augmentation.apply_ops
    monkeypatch.setattr(augmentation, "apply_ops", lambda s, ops, *a: recorded.extend(ops) or real(s, ops, *a))
    fill = [10.0, 20.0, 30.0]
    torch.manual_seed(123)
    out = T.TrivialAugmentWide(interpolation=BILINEAR, fill=fill)(batch.unbind(0))
    assert out.shape == batch.shape and out.is_contiguous()
    assert {op for op, _ in recorded} == set(_autoaugment.OPS)
    tv = TVA.TrivialAugmentWide(interpolation=BILINEAR, fill=fill)
    torch.manual_seed(123)
    for x, got, (op, m) in zip(batch.unbind(0), out, recorded):
        _check(got, tv(x), x, op, m, BILINEAR, fill)


def test_single_tensor_matches_module():
    g = torch.Generator().manual_seed(4)
    x = torch.randint(0, 256, (4, 3, 37, 53), generator=g, dtype=torch.uint8).cuda()
    for seed in range(40):
        torch.manual_seed(seed)
        got = T.TrivialAugmentWide(interpolation=BILINEAR)(x)
        after = torch.random.get_rng_state()
        torch.manual_seed(seed)
        want = TVA.TrivialAugmentWide(interpolation=BILINEAR)(x)
        assert torch.equal(torch.random.get_rng_state(), after)
        assert got.shape == x.shape
        torch.manual_seed(seed)
        op, m = _draw_one()
        for i in range(4):
            _check(got[i], want[i], x[i], op, m, BILINEAR, None)


def _draw_one():
    """The (op, magnitude) torchvision's module draws next, for a 31-bin space."""
    space = TVA.TrivialAugmentWide()._augmentation_space(31)
    op = list(space)[int(torch.randint(len(space), (1,)).item())]
    mags, signed = space[op]
    m = float(mags[torch.randint(len(mags), (1,), dtype=torch.long)].item()) if mags.ndim > 0 else 0.0
    if signed and torch.randint(2, (1,)):
        m *= -1.0
    return op, m


def test_launches_determinism_sentinels_and_no_sync():
    lib = _lib.lib()
    g = torch.Generator().manual_seed(6)
    imgs = torch.randint(0, 256, (16, 3, 29, 45), generator=g, dtype=torch.uint8).cuda().unbind(0)
    ops = [("Rotate", 30.0), ("Equalize", 0.0), ("Sharpness", 0.5), ("Contrast", -0.2)] * 4
    no_stats = [("Rotate", 30.0), ("Posterize", 3.0), ("Color", 0.5), ("Identity", 0.0)] * 4
    C, H, W = 3, 29, 45
    n = C * H * W
    for chosen, launches in ((ops, 2), (no_stats, 1)):
        buf = torch.full(((len(imgs) + 2) * n,), 0xA5, dtype=torch.uint8, device="cuda")
        out = buf[n:-n].view(len(imgs), C, H, W)
        lib.hb_launch_count_reset()
        _autoaugment.apply_ops(imgs, chosen, BILINEAR, None, out=out)
        assert lib.hb_launch_count() == launches
        assert bool((buf[:n] == 0xA5).all()) and bool((buf[-n:] == 0xA5).all())
        again = _autoaugment.apply_ops(imgs, chosen, BILINEAR, None)
        assert torch.equal(out, again)
    tf = T.TrivialAugmentWide(interpolation=BILINEAR, fill=5)
    tf(list(imgs))  # warm-up: first launches load modules
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(8):
            lib.hb_launch_count_reset()
            tf(list(imgs))
            assert lib.hb_launch_count() <= 2
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


def test_ambiguous_band_is_narrow():
    """The affine sweeps above leave only a thin band of pixels to the tolerance (runs after them, in file order)."""
    img = _image("random", 3, 176, 176, seed=1)
    for interp in (NEAREST, BILINEAR):
        _sweep(img, interp, [128.0], [o for o in _every_op() if o[0] in GEOMETRIC])
    assert STATS["geometric"] > 0
    print(f"ambiguous share {STATS['ambiguous'] / STATS['geometric']:.5f}, "
          f"mismatched share {STATS['mismatched'] / STATS['geometric']:.6f}")
    assert STATS["ambiguous"] <= 0.05 * STATS["geometric"]
    assert STATS["mismatched"] <= STATS["ambiguous"]
