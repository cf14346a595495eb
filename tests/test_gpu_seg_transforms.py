"""holocron_b200.transforms.segmentation on the GPU. Each fused run against this package's own ``Resize`` followed by
pad / crop / flip done by indexing, bit for bit, for every dtype; images against torchvision's tensor chain within the
bounds tests/test_gpu_transforms.py holds the resampler to; masks bit for bit against torchvision's tensor chain; the
whole training recipe (ColorJitter included) and the validation chain against a per-image torchvision oracle
(tests/_seg_transforms_oracle.py) under the same seed. Then the batching properties: one launch per run for the
images and one for the masks, strided sources, nothing written outside the outputs, identical bits on a second run, no
host synchronisation."""
import numpy as np
import pytest
import torch
from torchvision.transforms import transforms as TT
from torchvision.transforms.functional import InterpolationMode

import _seg_transforms_oracle as SO
import _transforms_oracle as O
from holocron_b200 import _lib
from holocron_b200 import transforms as T
from holocron_b200.transforms import _resample
from holocron_b200.transforms import segmentation as S
from test_gpu_transforms import DEV, DTYPES, _image, check_oracle

pytestmark = pytest.mark.gpu

INTERPS = {"bilinear": InterpolationMode.BILINEAR, "bicubic": InterpolationMode.BICUBIC}
# (source sizes, RandomResize range, crop): down- and upscales, odd sides, 1-pixel sides, sides below, equal to and
# above the crop
CASES = [([(37, 53), (61, 20), (33, 33)], (12, 30), 24),
         ([(9, 13), (1, 7), (7, 1), (1, 1)], (5, 40), 16),
         ([(50, 23), (23, 50)], (23, 24), 23)]
NORMALIZE = TT.Normalize(mean=[0.485, 0.456, 0.406], std=[0.229, 0.224, 0.225])


def _mask(h, w, seed):
    """21 classes with a 255 border, as VOC's masks."""
    g = torch.Generator().manual_seed(seed)
    m = torch.randint(0, 21, (h, w), generator=g, dtype=torch.uint8)
    m[:, :1] = 255
    m[-1:, :] = 255
    return m.to(DEV)


def _pairs(sizes, dtype, seed):
    return ([_image((3, h, w), dtype, seed + k) for k, (h, w) in enumerate(sizes)],
            [_mask(h, w, 100 + seed + k) for k, (h, w) in enumerate(sizes)])


def _render(inner, fold, fill):
    """A folded run applied by indexing on an already resized box."""
    Hc, Wc = fold.canvas
    ys = torch.arange(Hc, device=inner.device)[:, None] - fold.top
    us = torch.arange(Wc, device=inner.device)
    xs = ((Wc - 1 - us) if fold.mirror else us)[None, :] - fold.left
    h, w = inner.shape[-2:]
    live = (ys >= 0) & (ys < h) & (xs >= 0) & (xs < w)
    out = inner[..., ys.clamp(0, h - 1), xs.clamp(0, w - 1)]
    return torch.where(live, out, torch.full_like(out, fill))


def _folds(steps, sizes, seed):
    torch.manual_seed(seed)
    return [S.fold_run(steps, s) for s in sizes]


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
@pytest.mark.parametrize("interp", INTERPS)
@pytest.mark.parametrize("case", range(len(CASES)))
def test_fused_run_is_exact(dtype, interp, case):
    """The fused run equals Resize to (h_r, w_r), then pad / crop / flip by indexing, bit for bit: the taps of a canvas
    pixel do not depend on the tile it falls in."""
    sizes, (lo, hi), crop = CASES[case]
    images, masks = _pairs(sizes, dtype, 10 * case)
    resize = S.RandomResize(lo, hi, INTERPS[interp])
    for steps in ([resize, S.RandomCrop(crop), S.RandomHorizontalFlip(0.5)],
                  [resize, S.RandomHorizontalFlip(0.5), S.RandomCrop(crop), S.RandomHorizontalFlip(0.5)]):
        for seed in range(3):
            torch.manual_seed(seed)
            x, y = S.Compose(steps)(images, masks)
            assert x.shape == (len(sizes), 3, crop, crop) and y.shape == (len(sizes), crop, crop)
            for k, (fold, img, m) in enumerate(zip(_folds(steps, sizes, seed), images, masks)):
                resized = T.Resize(fold.inner, interpolation=INTERPS[interp], antialias=True)([img])[0]
                assert torch.equal(x[k], _render(resized, fold, 0)), (k, fold)
                mr = T.Resize(fold.inner, interpolation=InterpolationMode.NEAREST)([m[None]])[0, 0]
                assert torch.equal(y[k], _render(mr, fold, 255)), (k, fold)


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
@pytest.mark.parametrize("interp", INTERPS)
def test_images_and_masks_against_torchvision(dtype, interp):
    """Images within the resampler's bounds of the fp64 oracle, as torchvision's chain is; masks bit for bit."""
    sizes = [(37, 53), (61, 20), (9, 13), (1, 7)]
    images, masks = _pairs(sizes, dtype, 3)
    steps = [S.RandomResize(8, 40, INTERPS[interp]), S.RandomCrop(24), S.RandomHorizontalFlip(0.5)]
    for seed in range(3):
        torch.manual_seed(seed)
        x, y = S.Compose(steps)(images, masks)
        torch.manual_seed(seed)
        tv = SO.apply_batch(steps, images, masks)
        for k, (fold, img) in enumerate(zip(_folds(steps, sizes, seed), images)):
            value, mag = O.resize_pad(img, fold.inner, fold.inner, interp, True)
            value = _render(torch.from_numpy(value), fold, 0).numpy()
            mag = _render(torch.from_numpy(mag), fold, 0).numpy()
            check_oracle(x[k], value, mag, interp, img)
            check_oracle(tv[k][0], value, mag, interp, img)
            assert torch.equal(y[k], tv[k][1])


def _recipe():
    return S.Compose([S.RandomResize(160, 640), S.RandomCrop(256), S.RandomHorizontalFlip(0.5),
                      S.ImageTransform(TT.ColorJitter(brightness=0.3, contrast=0.3, saturation=0.1, hue=0.02)),
                      S.ToTensor(), S.ImageTransform(NORMALIZE)])


def _voc_batch(n=32, seed=0):
    g = np.random.default_rng(seed)
    sizes = [(int(a), int(b)) for a, b in g.integers(300, 501, (n, 2))]
    return _pairs(sizes, torch.uint8, 1000 + seed)


def test_train_recipe_against_per_image_oracle(monkeypatch):
    """32 images of VOC-like sizes through the recipe: masks and int64 targets bit for bit; images before ColorJitter
    within a rounding of torchvision's; after it, bit for bit given the same jittered input."""
    images, masks = _voc_batch()
    seen = {}
    real_jitter = S.jitter

    def recording_jitter(sources, draws):
        seen["pre"] = torch.stack(list(sources)).clone()
        return real_jitter(sources, draws)
    monkeypatch.setattr(S, "jitter", recording_jitter)
    torch.manual_seed(0)
    x, y = _recipe()(images, masks)
    state = torch.get_rng_state()
    assert x.shape == (32, 3, 256, 256) and x.dtype == torch.float32
    assert y.shape == (32, 256, 256) and y.dtype == torch.int64
    torch.manual_seed(0)
    ref = SO.apply_batch(_recipe().transforms, images, masks, pre_jitter=seen["pre"])
    assert torch.equal(torch.get_rng_state(), state)
    assert torch.equal(y, torch.stack([r[1] for r in ref]))
    before = torch.stack([r[2] for r in ref])
    diff = (seen["pre"].int() - before.int()).abs()
    assert diff.max() <= 1 and (diff != 0).float().mean() < 1e-3
    assert torch.equal(x, torch.stack([r[0] for r in ref]))


def test_val_chain_against_per_image_oracle():
    images, masks = _voc_batch(8, seed=1)
    val = S.Compose([S.Resize((256, 256)), S.ToTensor(), S.ImageTransform(NORMALIZE)])
    x, y = val(images, masks)
    ref = SO.apply_batch(val.transforms, images, masks)
    assert torch.equal(y, torch.stack([r[1] for r in ref]))
    diff = (x - torch.stack([r[0] for r in ref])).abs() * torch.tensor([0.229, 0.224, 0.225], device=DEV)[:, None, None]
    assert diff.max() <= 1.0001 / 255


def test_launches_per_run():
    images, masks = _voc_batch(8, seed=2)
    lib = _lib.lib()
    recipe = _recipe()
    recipe(images, masks)  # warm up
    for tf, launches in ((S.Compose(recipe.transforms[:3]), 2), (recipe, 4),
                         (S.Compose([S.RandomResize(300, 400), S.RandomCrop(320), S.RandomHorizontalFlip(0.5),
                                     S.RandomCrop(256), S.RandomHorizontalFlip(0.5)]), 4),
                         (S.RandomResize(160, 640), 2), (S.RandomHorizontalFlip(0.5), 2)):
        torch.cuda.synchronize()
        lib.hb_launch_count_reset()
        tf(images, masks)
        assert lib.hb_launch_count() == launches, tf  # the recipe: 2 resample + the jitter's statistics and apply


def test_ragged_results_and_single_pairs():
    images, masks = _pairs([(37, 53), (61, 20)], torch.uint8, 7)
    torch.manual_seed(0)
    x, y = S.RandomResize(10, 30)(images, masks)
    torch.manual_seed(0)
    ref = SO.apply_batch([S.RandomResize(10, 30)], images, masks)
    assert isinstance(x, list) and isinstance(y, list)
    assert x[0].untyped_storage().data_ptr() == x[1].untyped_storage().data_ptr()
    for a, b, (ra, rb) in zip(x, y, ref):
        assert a.shape[-2:] == b.shape and torch.equal(b, rb)
    torch.manual_seed(1)
    xs, ys = S.RandomHorizontalFlip(0.5)(images[1], masks[1])
    torch.manual_seed(1)
    rx, ry = SO.apply([S.RandomHorizontalFlip(0.5)], images[1], masks[1])
    assert torch.equal(xs, rx) and torch.equal(ys, ry)


def test_strided_sources():
    """unbind of a stacked batch (channels_last) and (1, H, W) masks give what contiguous sources give."""
    batch = _image((6, 3, 45, 70), torch.uint8, 40).to(memory_format=torch.channels_last)
    mbatch = torch.stack([_mask(45, 70, 50 + k) for k in range(6)])[:, None]
    views = list(batch.unbind(0))
    assert not views[0].is_contiguous()
    steps = [S.RandomResize(30, 60), S.RandomCrop(40), S.RandomHorizontalFlip(0.5)]
    torch.manual_seed(3)
    a, am = S.Compose(steps)(views, list(mbatch.unbind(0)))
    torch.manual_seed(3)
    b, bm = S.Compose(steps)([v.contiguous() for v in views], [m[0].contiguous() for m in mbatch])
    assert am.shape == (6, 1, 40, 40) and bm.shape == (6, 40, 40)
    assert torch.equal(a, b) and torch.equal(am[:, 0], bm)
    torch.manual_seed(3)
    ref = SO.apply_batch(steps, views, list(mbatch.unbind(0)))
    assert torch.equal(am, torch.stack([r[1] for r in ref]))


def test_sentinels_fill_and_two_runs():
    """Placed, mirrored and filled canvases of every dtype: stacked into a fenced output, nothing is written outside it;
    ragged, each view holds exactly its canvas. A second run of the recipe gives the same bits."""
    inner, offsets, mirrors = [(20, 30), (10, 20)], [(-3, 2), (1, -4)], [True, False]
    for dtype in DTYPES:
        imgs = [_image((3, 33, 47), dtype, 60), _image((3, 10, 20), dtype, 61)]
        n = 2 * 3 * 24 * 30
        buf = torch.full((n + 2048,), 7, dtype=dtype, device=DEV)
        out = buf[1024:1024 + n].view(2, 3, 24, 30)
        _resample.resample(imgs, inner, (24, 30), InterpolationMode.BILINEAR, True, out=out, offsets=offsets,
                           mirrors=mirrors, fill=255.0)
        ragged = _resample.resample(imgs, inner, None, InterpolationMode.BILINEAR, True, offsets=offsets,
                                    canvases=[(24, 24), (12, 30)], mirrors=mirrors, fill=255.0)
        assert (buf[:1024] == 7).all() and (buf[1024 + n:] == 7).all()
        assert ragged[1].data_ptr() - ragged[0].data_ptr() == 3 * 24 * 24 * ragged[0].element_size()
        for k, img in enumerate(imgs):
            resized = T.Resize(inner[k], antialias=True)([img])[0]
            for o in (out[k], ragged[k]):
                fold = S._Fold(inner[k], tuple(o.shape[-2:]), *offsets[k], mirrors[k])
                assert torch.equal(o, _render(resized, fold, 255)), (dtype, k)
    images, masks = _voc_batch(8, seed=3)
    runs = []
    for _ in range(2):
        torch.manual_seed(5)
        runs.append(_recipe()(images, masks))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
    imgs, masks = _pairs([(10, 12), (5, 30)], torch.uint8, 70)
    x, y = S.RandomCrop(32)(imgs, masks)
    assert (y[0, 10:] == 255).all() and (y[0, :, 12:] == 255).all() and (x[1, :, 5:] == 0).all()


def test_no_host_synchronisation():
    images, masks = _voc_batch(8, seed=4)
    recipe = S.Compose(_recipe().transforms[:5])  # torchvision's Normalize checks its std on the device
    val = S.Compose([S.Resize((256, 256)), S.ToTensor()])
    recipe(images, masks)
    val(images, masks)
    S.RandomResize(160, 640)(images, masks)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        recipe(images, masks)
        val(images, masks)
        S.RandomResize(160, 640)(images, masks)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
