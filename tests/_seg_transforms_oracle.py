"""The reference's segmentation transforms (references/segmentation/transforms.py) restated on tensors, one image at a
time, with torchvision's tensor ops: ``resize`` (antialiased) for the image and ``resize`` nearest for the mask,
``pad`` with 0 / 255 on the bottom and right, ``crop``, ``hflip``, torchvision's ``ColorJitter`` and ``Normalize``, and
``ToTensor`` as ``x.to(float32).div(255)`` / int64. Draws are the reference's, in its order, on the default CPU
generator, one image after the other as its ``Compose`` applied sample by sample makes them."""
import torch
import torchvision.transforms.functional as TF
from torchvision.transforms import transforms as TT
from torchvision.transforms.functional import InterpolationMode

from holocron_b200.transforms import segmentation as S


def _pad_if_smaller(x, size, fill):
    h, w = x.shape[-2:]
    if min(h, w) < size:
        x = TF.pad(x, [0, 0, size - w if w < size else 0, size - h if h < size else 0], fill=fill)
    return x


def apply(steps, image, mask, pre_jitter=None):
    """(image, mask) after ``steps`` (this package's segmentation classes, read for their parameters). With
    ``pre_jitter``, a ColorJitter takes that image instead of the one the oracle computed (its draws are unchanged), and
    the image it was given is returned third."""
    before = None
    for t in steps:
        if isinstance(t, (S.Resize, S.RandomResize)):
            if isinstance(t, S.Resize):
                size = t.output_size
            else:
                size = t.min_size if t.min_size == t.max_size else torch.randint(t.min_size, t.max_size, (1,)).item()
            image = TF.resize(image, size, interpolation=t.interpolation, antialias=True)
            # torch's interpolate takes no (H, W) tensor: resize an (H, W) mask as one channel
            flat = mask.ndim == 2
            mask = TF.resize(mask[None] if flat else mask, size, interpolation=InterpolationMode.NEAREST)
            mask = mask[0] if flat else mask
        elif isinstance(t, S.RandomCrop):
            image = _pad_if_smaller(image, t.size, 0)
            mask = _pad_if_smaller(mask, t.size, 255)
            params = TT.RandomCrop.get_params(image, (t.size, t.size))
            image, mask = TF.crop(image, *params), TF.crop(mask, *params)
        elif isinstance(t, S.RandomHorizontalFlip):
            if torch.rand(1).item() < t.prob:
                image, mask = TF.hflip(image), TF.hflip(mask)
        elif isinstance(t, S.ToTensor):
            image, mask = image.to(torch.float32).div(255), mask.to(torch.int64)
        elif isinstance(t.transform, TT.ColorJitter):
            before = image
            j = t.transform
            fn_idx, b, c, s, h = j.get_params(j.brightness, j.contrast, j.saturation, j.hue)
            image = pre_jitter if pre_jitter is not None else image
            for k in fn_idx:
                if k == 0 and b is not None:
                    image = TF.adjust_brightness(image, b)
                elif k == 1 and c is not None:
                    image = TF.adjust_contrast(image, c)
                elif k == 2 and s is not None:
                    image = TF.adjust_saturation(image, s)
                elif k == 3 and h is not None:
                    image = TF.adjust_hue(image, h)
        else:
            image = t.transform(image)
    return (image, mask) if pre_jitter is None else (image, mask, before)


def apply_batch(steps, images, masks, pre_jitter=None):
    """``apply`` image by image, in list order."""
    return [apply(steps, x, m, None if pre_jitter is None else pre_jitter[k])
            for k, (x, m) in enumerate(zip(images, masks))]
