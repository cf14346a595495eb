"""RandomResizedCrop, RandomHorizontalFlip and RandomErasing of holocron_b200.transforms on the GPU. Crops: per element
against the fp64 oracle (tests/_transforms_oracle.py) within the bounds tests/test_gpu_transforms.py holds the
resampler to, and torchvision's ``resized_crop`` on the same CUDA images within the same bounds. Flips and erasing: bit
for bit against torchvision run image by image on the same CUDA images under the same seed. Then the batching
properties: one launch per call, identical bits on a second run, nothing written outside the output, no host
synchronisation."""
import pytest
import torch
import torchvision.transforms.functional as TF
from torchvision.transforms import transforms as TV
from torchvision.transforms.functional import InterpolationMode

import _transforms_oracle as O
from holocron_b200 import _lib
from holocron_b200 import transforms as T
from holocron_b200.transforms import _erase, _resample
from test_gpu_transforms import DEV, DTYPES, INTERP, _image, check_pair

pytestmark = pytest.mark.gpu

ERASE_VALUES = [0, 0.75, (0.5, -1.5, 300.25), "random"]


def _crop_check(imgs, boxes, size, interp, antialias, out):
    """Each canvas against the oracle of its crop and torchvision's resized_crop of the same CUDA image. uint8 outputs
    may differ from the oracle only at rounding ties; small crops upscaled by simple ratios put many values on exact .5
    ties, so their number is not bounded here."""
    for x, (i, j, h, w), y in zip(imgs, boxes, out):
        crop = x[:, i:i + h, j:j + w]
        value, mag = O.resize_pad(crop, size, size, interp, antialias)
        tv = TF.resized_crop(x, i, j, h, w, list(size), INTERP[interp], antialias=antialias)
        check_pair(y, tv, value, mag, interp, crop)


def _channels_last_views(n, shape, dtype, seed):
    batch = _image((n, *shape), dtype, seed).to(memory_format=torch.channels_last)
    views = list(batch.unbind(0))
    assert not views[0].is_contiguous()
    return batch, views


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=str)
@pytest.mark.parametrize("interp", O.FILTERS)
@pytest.mark.parametrize("antialias", [True, False])
def test_random_resized_crop_every_dtype_filter(dtype, interp, antialias):
    imgs = [_image(s, dtype, 60 + k) for k, s in enumerate([(3, 57, 83), (3, 90, 41), (3, 33, 33), (3, 120, 17)])]
    tf = T.RandomResizedCrop((24, 31), scale=(0.05, 1.0), interpolation=INTERP[interp], antialias=antialias)
    torch.manual_seed(5)
    out = tf(imgs)
    torch.manual_seed(5)
    boxes = [tf.get_params(x, tf.scale, tf.ratio) for x in imgs]
    assert out.shape == (4, 3, 24, 31) and out.dtype == dtype
    _crop_check(imgs, boxes, (24, 31), interp, antialias, out)


@pytest.mark.parametrize("interp", O.FILTERS)
@pytest.mark.parametrize("antialias", [True, False])
def test_crop_one_pixel_sides_and_heavy_downscales(interp, antialias):
    """Crop boxes of 1-pixel sides (upscaled) and of whole large images (downscaled 1/8 and more), fp32 and uint8."""
    for dtype in (torch.float32, torch.uint8):
        imgs = [_image((3, 300, 256), dtype, 70), _image((3, 41, 37), dtype, 71), _image((3, 9, 260), dtype, 72)]
        for boxes, size in [([(0, 0, 300, 256), (3, 5, 1, 30), (4, 100, 1, 1)], (30, 32)),
                            ([(17, 200, 1, 1), (0, 36, 41, 1), (0, 0, 9, 260)], (7, 5))]:
            out = _resample.resample(imgs, [size] * 3, size, INTERP[interp], antialias, boxes=boxes)
            _crop_check(imgs, boxes, size, interp, antialias, out)


def test_crop_strided_sources_and_single_tensor():
    batch, views = _channels_last_views(5, (3, 64, 48), torch.float32, 73)
    tf = T.RandomResizedCrop(32, scale=(0.3, 1.0), interpolation=InterpolationMode.BICUBIC)
    torch.manual_seed(9)
    a = tf(views)
    torch.manual_seed(9)
    assert torch.equal(a, tf([v.contiguous() for v in views]))
    # a 2-D tensor: torchvision's resize fails in torch's interpolate
    for cls in (T.RandomResizedCrop, TV.RandomResizedCrop):
        torch.manual_seed(10)
        with pytest.raises(ValueError):
            cls(32, scale=(0.3, 1.0))(batch[0, 0])
    # one tensor: one draw, leading dimensions carried along, and torchvision's output on it
    for x in (batch, batch[0]):
        torch.manual_seed(10)
        ours = tf(x)
        torch.manual_seed(10)
        i, j, h, w = tf.get_params(x, tf.scale, tf.ratio)
        torch.manual_seed(10)
        theirs = TV.RandomResizedCrop(32, scale=(0.3, 1.0), interpolation=InterpolationMode.BICUBIC)(x)
        assert ours.shape == theirs.shape == (*x.shape[:-2], 32, 32)
        planes = x.reshape(-1, 1, *x.shape[-2:])
        for y, z, plane in zip(ours.reshape(-1, 1, 32, 32), theirs.reshape(-1, 1, 32, 32), planes):
            crop = plane[:, i:i + h, j:j + w]
            value, mag = O.resize_pad(crop, (32, 32), (32, 32), "bicubic", True)
            check_pair(y, z, value, mag, "bicubic", crop)


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_flip_bit_identical_to_torchvision(dtype):
    batch, views = _channels_last_views(12, (3, 21, 34), dtype, 80)
    contiguous = [_image((3, 21, 34), dtype, 81 + k) for k in range(12)]
    for imgs in (views, contiguous):
        for p in (0.0, 0.5, 1.0):
            torch.manual_seed(4)
            ours = T.RandomHorizontalFlip(p)(imgs)
            torch.manual_seed(4)
            theirs = torch.stack([TV.RandomHorizontalFlip(p)(x) for x in imgs])
            assert torch.equal(ours, theirs)
    for x in (batch, batch[3], batch[3, 1]):  # one tensor, leading dimensions included
        for seed in range(4):
            torch.manual_seed(seed)
            ours = T.RandomHorizontalFlip()(x)
            torch.manual_seed(seed)
            assert torch.equal(ours, TV.RandomHorizontalFlip()(x))


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
@pytest.mark.parametrize("value", ERASE_VALUES, ids=str)
@pytest.mark.parametrize("inplace", [False, True])
def test_erase_bit_identical_to_torchvision(dtype, value, inplace):
    """Every dtype (the fp32 values cast as torch's copy casts them, uint8 included), scalar, per-channel and random
    values, on contiguous images and on the strided images of a channels_last batch."""
    kwargs = {"p": 0.7, "scale": (0.02, 0.33), "value": value, "inplace": inplace}
    for layout in ("contiguous", "channels_last"):
        if layout == "contiguous":
            base = [_image((3, 37, 45), dtype, 90 + k) for k in range(10)]
        else:
            base = _channels_last_views(10, (3, 37, 45), dtype, 90)[1]
        ours_in = [x.clone(memory_format=torch.preserve_format) for x in base] if inplace else base
        theirs_in = [x.clone(memory_format=torch.preserve_format) for x in base]
        torch.manual_seed(21)
        ours = T.RandomErasing(**kwargs)(ours_in)
        after_ours = torch.random.get_rng_state()
        torch.manual_seed(21)
        theirs = [TV.RandomErasing(**kwargs)(x) for x in theirs_in]
        assert torch.equal(torch.random.get_rng_state(), after_ours)
        if inplace:
            assert ours is ours_in
            ours = torch.stack(ours_in)
        else:  # the sources are read, not written
            assert all(torch.equal(a, b) for a, b in zip(base, theirs_in))
        assert torch.equal(ours, torch.stack(theirs)), layout
        assert not torch.equal(ours, torch.stack(base))


@pytest.mark.parametrize("value", ERASE_VALUES, ids=str)
def test_erase_single_tensor(value):
    for dtype in (torch.uint8, torch.bfloat16, torch.float32):
        batch = _image((2, 3, 30, 26), dtype, 95)
        for x in (batch, batch[1]):
            for inplace in (False, True):
                for seed in range(5):
                    a, b = x.clone(), x.clone()
                    torch.manual_seed(seed)
                    ours = T.RandomErasing(p=0.6, value=value, inplace=inplace)(a)
                    torch.manual_seed(seed)
                    theirs = TV.RandomErasing(p=0.6, value=value, inplace=inplace)(b)
                    assert torch.equal(ours, theirs) and torch.equal(a, b)
                    assert (ours is a) == (theirs is b)


def test_one_launch_per_call_and_two_runs_identical():
    imgs = [_image((3, 300 + 7 * k, 500 - 11 * k), torch.uint8, 100 + k) for k in range(8)]
    crop = T.RandomResizedCrop(176, scale=(0.3, 1.0))
    flip = T.RandomHorizontalFlip()
    erase = T.RandomErasing(p=1.0, scale=(0.02, 0.2), value="random")
    erase_inplace = T.RandomErasing(p=1.0, scale=(0.02, 0.2), value="random", inplace=True)
    runs = []
    for _ in range(2):
        torch.manual_seed(33)
        lib = _lib.lib()
        outs = []
        for tf, arg in ((crop, lambda: imgs), (flip, lambda: outs[0].unbind(0)), (erase, lambda: outs[1].unbind(0)),
                        (erase_inplace, lambda: outs[2].clone().unbind(0))):
            x = arg()
            lib.hb_launch_count_reset()
            y = tf(x)
            assert lib.hb_launch_count() == 1
            outs.append(torch.stack(list(y)) if isinstance(y, tuple) else y)
        runs.append(outs)
    for a, b in zip(*runs):
        assert torch.equal(a, b)


def test_sentinels_around_the_output_stay_untouched():
    imgs = [_image((3, 33, 47), torch.uint8, 110), _image((3, 60, 20), torch.uint8, 111)]
    n = 2 * 3 * 24 * 24
    buf = torch.full((n + 2048,), 0xA5, dtype=torch.uint8, device=DEV)
    out = buf[1024:1024 + n].view(2, 3, 24, 24)
    _resample.resample(imgs, [(24, 24)] * 2, (24, 24), InterpolationMode.BILINEAR, True, out=out,
                       boxes=[(5, 3, 28, 44), (0, 0, 60, 20)], flips=[True, False])
    torch.cuda.synchronize()
    assert (buf[:1024] == 0xA5).all() and (buf[1024 + n:] == 0xA5).all()
    _crop_check([imgs[0].flip(-1), imgs[1]], [(5, 47 - 3 - 44, 28, 44), (0, 0, 60, 20)], (24, 24), "bilinear", True,
                out)
    # erasing: a copy into a fenced output, and rectangles written in place into images fenced by their own margins
    for dtype in (torch.uint8, torch.float16, torch.float64):
        src = [_image((3, 29, 31), dtype, 112 + k) for k in range(3)]
        rects = [(0, 0, 29, 31, torch.randn(3, 29, 31)), (28, 30, 1, 1, torch.tensor([2.0])[:, None, None]),
                 (3, 1, 20, 29, torch.randn(3, 20, 29))]
        m = 3 * 29 * 31
        fenced = torch.full((3 * m + 64,), 7, dtype=dtype, device=DEV)
        out = fenced[32:32 + 3 * m].view(3, 3, 29, 31)
        _erase.erase(src, rects, False, out=out)
        assert (fenced[:32] == 7).all() and (fenced[32 + 3 * m:] == 7).all()
        for x, (i, j, h, w, v), y in zip(src, rects, out):
            assert torch.equal(y, TF.erase(x, i, j, h, w, v.to(DEV)))
        frame = torch.full((3, 3, 31, 35), 7, dtype=dtype, device=DEV)
        inner = [f[:, 1:30, 2:33] for f in frame]
        for f, x in zip(inner, src):
            f.copy_(x)
        assert _erase.erase(inner, rects, True) is None
        border = frame.clone()
        border[:, :, 1:30, 2:33] = 7
        assert (border == 7).all()
        for x, (i, j, h, w, v), y in zip(src, rects, inner):
            assert torch.equal(y, TF.erase(x, i, j, h, w, v.to(DEV)))


def test_no_host_synchronisation():
    imgs = [_image((3, 300 + 7 * k, 500 - 11 * k), torch.uint8, 120 + k) for k in range(4)]
    tfs = (T.RandomResizedCrop(176, scale=(0.3, 1.0)), T.RandomHorizontalFlip(),
           T.RandomErasing(p=1.0, value="random"), T.RandomErasing(p=1.0, value=(1, 2, 3), inplace=True))
    for tf in tfs:  # warm up: module loads and pinned-buffer allocations
        tf(imgs if isinstance(tf, T.RandomResizedCrop) else [x[:, :300, :400] for x in imgs])
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        x = tfs[0](imgs)
        x = tfs[1](x.unbind(0))
        x = tfs[2](x.unbind(0))
        tfs[3](x.unbind(0))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
