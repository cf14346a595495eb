"""The classification Compose and Normalize of holocron_b200.transforms on the GPU, against torchvision's per-image
``T.Compose`` on the same CUDA tensors under the same seed: the recipe's four chains, erasing before and after
Normalize and on uint8 before the conversion, scalar, per-channel and random fills, widths off the 16- and 4-element
vectors, sources off a 16-byte boundary and ``unbind`` views, a single tensor, and the standalone Normalize. Runs and
tails must be bit-identical; pixels of TrivialAugmentWide's affine ops may differ only where the oracle of
``_autoaugment_oracle.py`` marks them ambiguous. Every chain runs under ``torch.cuda.set_sync_debug_mode("error")``,
and the launches are counted."""
import pytest
import torch
from torchvision.transforms import InterpolationMode, autoaugment as TVA, transforms as TV

from _autoaugment_oracle import apply_op as oracle_op
from holocron_b200 import _lib
from holocron_b200 import transforms as HT
from holocron_b200.transforms import _autoaugment, classification as C

pytestmark = pytest.mark.gpu

BILINEAR = InterpolationMode.BILINEAR
MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
GEOMETRIC = ("ShearX", "ShearY", "TranslateX", "TranslateY", "Rotate")


def imagenette_train(p):
    return [TV.RandomResizedCrop(176, scale=(0.3, 1.0), interpolation=BILINEAR), TV.RandomHorizontalFlip(),
            TVA.TrivialAugmentWide(interpolation=BILINEAR), TV.PILToTensor(), TV.ConvertImageDtype(torch.float32),
            TV.Normalize(MEAN, STD), TV.RandomErasing(p=p, scale=(0.02, 0.2), value="random")]


def imagenette_val():
    return [TV.Resize(232, interpolation=BILINEAR), TV.CenterCrop(224), TV.PILToTensor(),
            TV.ConvertImageDtype(torch.float32), TV.Normalize(MEAN, STD)]


def cifar_train(p):
    return [TV.RandomHorizontalFlip(), TVA.TrivialAugmentWide(interpolation=BILINEAR), TV.PILToTensor(),
            TV.ConvertImageDtype(torch.float32), TV.Normalize(MEAN, STD), TV.RandomErasing(p=p, value="random")]


def cifar_val():
    return [TV.PILToTensor(), TV.ConvertImageDtype(torch.float32), TV.Normalize(MEAN, STD)]


def _images(sizes, seed, dtype=torch.uint8):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, 256, (3, h, w), generator=g, dtype=torch.uint8).to(dtype).cuda() for h, w in sizes]


def _random_sizes(n, seed, lo=300, hi=500):
    g = torch.Generator().manual_seed(seed)
    return [tuple(int(v) for v in torch.randint(lo, hi + 1, (2,), generator=g)) for _ in range(n)]


def _reference(chain, images, seed, monkeypatch):
    """torchvision's Compose applied image by image, and the input and op of each TrivialAugmentWide call."""
    ops = []
    real = TVA._apply_op

    def op(img, name, magnitude, interpolation, fill):
        ops.append((img.clone(), name, magnitude))
        return real(img, name, magnitude, interpolation, fill)

    tf = TV.Compose([t for t in chain if not isinstance(t, TV.PILToTensor)])  # PIL images only
    torch.manual_seed(seed)
    with monkeypatch.context() as m:
        m.setattr(TVA, "_apply_op", op)
        outs = [tf(x) for x in images]
    return outs, ops, torch.random.get_rng_state()


def _ours(chain, images, seed):
    """Our Compose under the sync debug mode "error": (output, launches, generator state after)."""
    lib = _lib.lib()
    torch.cuda.synchronize()
    torch.manual_seed(seed)
    lib.hb_launch_count_reset()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = C.Compose(chain)(images)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    launches = lib.hb_launch_count()
    return out, launches, torch.random.get_rng_state()


def _check(chain, images, seed, monkeypatch, launches=None):
    """Our Compose against torchvision's image by image; ``images`` a list, or one tensor."""
    single = isinstance(images, torch.Tensor)
    got, n, state = _ours(chain, images, seed)
    want, ops, want_state = _reference(chain, [images] if single else images, seed, monkeypatch)
    assert torch.equal(state, want_state)
    if single:
        got = got[None]
    assert got.dtype == want[0].dtype and got.shape == (len(want), *want[0].shape)
    for k, w in enumerate(want):
        if ops and ops[k][1] in GEOMETRIC:
            img, name, magnitude = ops[k]
            _, amb = oracle_op(img.cpu().numpy(), name, magnitude, True, None)
            bad = (got[k] != w).any(0).cpu().numpy() & ~amb
            assert not bad.any(), (k, name, magnitude, int(bad.sum()))
        else:
            assert torch.equal(got[k], w), (k, ops[k][1:] if ops else None, int((got[k] != w).sum()))
    if launches is not None:
        stat = any(o[1] in _autoaugment.STAT_OPS for o in ops)
        assert n == launches + stat, (n, launches, stat)


@pytest.mark.parametrize("seed", [0, 1])
@pytest.mark.parametrize("p", [0.0, 0.5, 1.0])
def test_imagenette_train(monkeypatch, seed, p):
    _check(imagenette_train(p), _images(_random_sizes(12, seed), seed), seed, monkeypatch, launches=3)


@pytest.mark.parametrize("seed", [0, 3])
def test_imagenette_val(monkeypatch, seed):
    _check(imagenette_val(), _images(_random_sizes(12, seed, 200, 500), seed), seed, monkeypatch, launches=2)


@pytest.mark.parametrize("seed", [0, 1])
@pytest.mark.parametrize("p", [0.0, 0.5, 1.0])
def test_cifar_train(monkeypatch, seed, p):
    _check(cifar_train(p), _images([(32, 32)] * 64, seed), seed, monkeypatch, launches=3)


def test_cifar_val(monkeypatch):
    _check(cifar_val(), _images([(32, 32)] * 64, 5), 5, monkeypatch, launches=1)


FILLS = [0.7, (0.1, -2.5, 3.25), "random", 300.7, (-3.5, 255.9, 1000.2)]


@pytest.mark.parametrize("value", FILLS)
@pytest.mark.parametrize("where", ["after_normalize", "before_normalize", "uint8_before_convert"])
@pytest.mark.parametrize("H, W", [(37, 50), (20, 13), (9, 3), (64, 64)])
def test_erasing_in_the_tail(monkeypatch, value, where, H, W):
    erase = TV.RandomErasing(p=0.8, scale=(0.05, 0.5), value=value)
    convert, normalize = TV.ConvertImageDtype(torch.float32), TV.Normalize(MEAN, STD)
    chain = {"after_normalize": [convert, normalize, erase], "before_normalize": [convert, erase, normalize],
             "uint8_before_convert": [erase, convert, normalize]}[where]
    _check(chain, _images([(H, W)] * 16, H * W), W, monkeypatch, launches=1)


@pytest.mark.parametrize("dtype", [torch.uint8, torch.float32])
@pytest.mark.parametrize("H, W", [(33, 61), (16, 16), (5, 7), (31, 4)])
def test_strided_and_misaligned_sources(monkeypatch, dtype, H, W):
    """Sources 1-3 elements off a 16-byte boundary, unbind views of a batch, and a channels-last batch."""
    g = torch.Generator().manual_seed(H + W)
    base = torch.randint(0, 256, (4 * 3 * H * W + 3,), generator=g, dtype=torch.uint8).to(dtype).cuda()
    off = [base[o:o + 3 * H * W].view(3, H, W) for o in (1, 2, 3)]
    batch = torch.randint(0, 256, (4, 3, H, W), generator=g, dtype=torch.uint8).to(dtype).cuda()
    chl = batch.contiguous(memory_format=torch.channels_last)
    chain = [TV.ConvertImageDtype(torch.float32), TV.RandomErasing(p=1.0, value="random"), TV.Normalize(MEAN, STD)]
    for images in (off, batch.unbind(0), chl.unbind(0)):
        _check(chain, list(images), 7, monkeypatch, launches=1)
    _check([TV.RandomResizedCrop(24), TV.RandomHorizontalFlip()] + chain, off, 7, monkeypatch, launches=2)


def test_single_tensor(monkeypatch):
    _check(imagenette_train(1.0), _images([(300, 400)], 1)[0], 4, monkeypatch, launches=3)
    _check(imagenette_val(), _images([(300, 400)], 1)[0], 4, monkeypatch, launches=2)
    _check(cifar_val(), _images([(32, 32)], 2)[0], 4, monkeypatch, launches=1)


def test_standalone_normalize():
    g = torch.Generator().manual_seed(0)
    batch = torch.rand(6, 3, 45, 61, generator=g).cuda() * 2 - 0.5
    tv = TV.Normalize(MEAN, STD)
    for mean, std in ((MEAN, STD), (0.5, 0.25), ([0.1], (3.0, 0.7, 1e-3))):
        ours, theirs = HT.Normalize(mean, std), TV.Normalize(mean, std)
        lib = _lib.lib()
        torch.cuda.synchronize()
        lib.hb_launch_count_reset()
        torch.cuda.set_sync_debug_mode("error")
        try:
            a, b, c = ours(batch.unbind(0)), ours(batch), ours(batch[0])
        finally:
            torch.cuda.set_sync_debug_mode(0)
        assert lib.hb_launch_count() == 3
        assert torch.equal(a, theirs(batch)) and torch.equal(b, theirs(batch)) and torch.equal(c, theirs(batch[0]))
    x = batch.clone()
    out = HT.Normalize(MEAN, STD, inplace=True)(x)
    assert torch.equal(x, batch) and torch.equal(out, tv(batch))
