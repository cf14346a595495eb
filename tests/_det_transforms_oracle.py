"""The reference's detection transforms (references/detection/transforms.py) restated one image at a time: torchvision's
tensor ops for the image (``resize`` with antialias, ``resized_crop``, ``center_crop``, ``hflip``, the wrapped
transforms) and separate torch fp32 ops for the boxes, each rounding as the reference's do. Draws are the reference's,
in its order, on the default CPU generator, one image after the other.

Divisions by an image side divide by a 0-dim tensor on the boxes' device: torch's CUDA division by a Python scalar
multiplies by its reciprocal, which rounds differently from the reference's CPU division."""
import torch
import torchvision.transforms.functional as TF
from torchvision.transforms import transforms as TT

from holocron_b200.transforms import detection as D


def _scale(boxes, sx, sy):
    boxes[:, [0, 2]] *= sx
    boxes[:, [1, 3]] *= sy


def _clamp_shift(boxes, x_lo, x_hi, y_lo, y_hi):
    boxes[:, [0, 2]] = boxes[:, [0, 2]].clamp(x_lo, x_hi)
    boxes[:, [1, 3]] = boxes[:, [1, 3]].clamp(y_lo, y_hi)
    boxes[:, [0, 2]] -= x_lo
    boxes[:, [1, 3]] -= y_lo


def apply(steps, image, target, pre_jitter=None):
    """(image, target) after ``steps`` (this package's detection classes, read for their parameters). ``target`` holds
    ``boxes`` and ``labels`` (it is not modified), or is a VOC annotation dict when ``steps`` start with a
    ``VOCTargetTransform``. With ``pre_jitter``, a ColorJitter takes that image instead of the one the oracle computed
    (its draws are unchanged), and the image it was given is returned third."""
    if steps and isinstance(steps[0], D.VOCTargetTransform):
        boxes, labels = steps[0].parse(target)
        target = {"boxes": torch.tensor(boxes, dtype=torch.float32).reshape(-1, 4).to(image.device),
                  "labels": torch.tensor(labels, dtype=torch.int64).to(image.device)}
        steps = steps[1:]
    boxes, labels = target["boxes"].clone(), target["labels"].clone()
    before = None
    for t in steps:
        H, W = image.shape[-2:]
        if isinstance(t, D.Resize):
            if isinstance(t.size, int):
                boxes *= t.size / (H if H < W else W)
            elif isinstance(t.size, tuple):
                _scale(boxes, t.size[0] / W, t.size[1] / H)
            image = TF.resize(image, t.size, t.interpolation, t.max_size, t.antialias)
        elif isinstance(t, D.RandomResizedCrop):
            i, j, h, w = t.get_params(image, t.scale, t.ratio)
            image = TF.resized_crop(image, i, j, h, w, t.size, t.interpolation, antialias=t.antialias)
            _clamp_shift(boxes, j, j + w, i, i + h)
            keep = (boxes[:, 0] != boxes[:, 2]) & (boxes[:, 1] != boxes[:, 3])
            boxes, labels = boxes[keep], labels[keep]
            _scale(boxes, t.size[0] / w, t.size[1] / h)
        elif isinstance(t, D.CenterCrop):
            image = TF.center_crop(image, t.size)
            h, w = image.shape[-2:]
            x, y = int(w / 2 - t.size[0] / 2), int(h / 2 - t.size[1] / 2)
            _clamp_shift(boxes, x, x + t.size[0], y, y + t.size[1])
        elif isinstance(t, D.RandomHorizontalFlip):
            if torch.rand(1).item() < t.p:
                image = TF.hflip(image)
                boxes[:, [0, 2]] = H - boxes[:, [0, 2]]
                boxes = boxes[:, [2, 1, 0, 3]]
        elif t is D.convert_to_relative:
            boxes[:, [0, 2]] /= torch.tensor(float(W), device=boxes.device)
            boxes[:, [1, 3]] /= torch.tensor(float(H), device=boxes.device)
            boxes[:, [0, 2]] = boxes[:, [0, 2]].clamp(0, 1)
            boxes[:, [1, 3]] = boxes[:, [1, 3]].clamp(0, 1)
        elif isinstance(t.transform, TT.ColorJitter):
            before = image
            j = t.transform
            fn_idx, b, c, s, hue = j.get_params(j.brightness, j.contrast, j.saturation, j.hue)
            image = pre_jitter if pre_jitter is not None else image
            for k in fn_idx:
                if k == 0 and b is not None:
                    image = TF.adjust_brightness(image, b)
                elif k == 1 and c is not None:
                    image = TF.adjust_contrast(image, c)
                elif k == 2 and s is not None:
                    image = TF.adjust_saturation(image, s)
                elif k == 3 and hue is not None:
                    image = TF.adjust_hue(image, hue)
        elif isinstance(t.transform, TT.PILToTensor):
            pass
        else:
            image = t.transform(image)
    out = {"boxes": boxes, "labels": labels}
    return (image, out) if pre_jitter is None else (image, out, before)


def apply_batch(steps, images, targets, pre_jitter=None):
    """``apply`` image by image, in list order."""
    return [apply(steps, x, t, None if pre_jitter is None else pre_jitter[k])
            for k, (x, t) in enumerate(zip(images, targets))]
