"""Generates tests/golden/det_transforms.pt by running the UNMODIFIED reference's detection transforms
(references/detection/transforms.py of frgfm/Holocron, a checkout named by the HOLOCRON_REFERENCE environment variable)
on seeded PIL images and targets:

    HOLOCRON_REFERENCE=/path/to/Holocron python tests/golden/make_golden_det_transforms.py

It records each class's constructor signature and ``repr``, and for each chain and seed, applied sample by sample as
the recipe's dataset applies it: every ``torch.randint`` / ``torch.rand`` call and every ``RandomResizedCrop.get_params``
result made while the reference runs (arguments and value), the (H, W) of the image after each step, the output boxes
(fp32) and labels (int64), and the default generator's state afterwards. Box outputs depend on the sizes and draws
only, not on the pixels. Chains are given as data ``[(name, args)]`` so the tests can build the same chain from this
package; targets are given as data too (VOC annotation dicts, or boxes and labels).
"""
import importlib.util
import sys
from pathlib import Path

import numpy as np
import torch
from PIL import Image
from torchvision.transforms import transforms as T

sys.path.insert(0, str(Path(__file__).resolve().parent))
from make_golden import OUT, describe_signature  # noqa: E402  (loads the reference)
from oracle.reference_loader import REFERENCE_ROOT  # noqa: E402

_spec = importlib.util.spec_from_file_location("ref_det_transforms",
                                               REFERENCE_ROOT / "references" / "detection" / "transforms.py")
REF = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(REF)

VOC_CLASSES = ["aeroplane", "bicycle", "bird", "boat", "bottle", "bus", "car", "cat", "chair", "cow", "diningtable",
               "dog", "horse", "motorbike", "person", "pottedplant", "sheep", "sofa", "train", "tvmonitor"]
JITTER = ("ColorJitter", (0.3, 0.3, 0.1, 0.02))
NORMALIZE = ("Normalize", ([0.485, 0.456, 0.406], [0.229, 0.224, 0.225]))
TENSOR = [("ImageTransform", ("PILToTensor", ())), ("ImageTransform", ("ConvertImageDtype", (torch.float32,))),
          ("ImageTransform", NORMALIZE)]
CHAINS = {
    # references/detection/train.py:116-125 (--source holocron) and its validation chain
    "recipe": [("VOCTargetTransform", (VOC_CLASSES,)), ("Resize", ((416, 416),)), ("RandomHorizontalFlip", ()),
               ("convert_to_relative", ()), ("ImageTransform", JITTER)] + TENSOR,
    "val": [("VOCTargetTransform", (VOC_CLASSES,)), ("Resize", ((416, 416),)), ("convert_to_relative", ())] + TENSOR,
    "rrc": [("RandomResizedCrop", (416,)), ("RandomHorizontalFlip", (0.5,)), ("convert_to_relative", ())],
    "rrc_small": [("RandomResizedCrop", ((96, 64), (0.02, 0.2))), ("convert_to_relative", ())],
    "center_crop": [("CenterCrop", (200,)), ("RandomHorizontalFlip", (0.5,))],
    "center_crop_large": [("CenterCrop", (600,)), ("convert_to_relative", ())],
    "center_crop_rect": [("CenterCrop", ((150, 250),)), ("RandomHorizontalFlip", (0.5,)), ("convert_to_relative", ())],
    "resize_int": [("Resize", (200,)), ("RandomHorizontalFlip", (0.5,))],
    "resize_tuple": [("Resize", ((100, 200),)), ("convert_to_relative", ())],
    "resize_list": [("Resize", ([100, 200],)), ("convert_to_relative", ())],
    "resize_list1": [("Resize", ([150],))],
    "flips_two_runs": [("RandomHorizontalFlip", (0.5,)), ("CenterCrop", (120,)), ("RandomHorizontalFlip", (0.5,)),
                       ("Resize", (90,)), ("CenterCrop", ((60, 80),)), ("RandomHorizontalFlip", (0.7,)),
                       ("RandomResizedCrop", ((40, 50), (0.5, 1.0))), ("RandomHorizontalFlip", (0.5,)),
                       ("convert_to_relative", ())],
    "flip": [("RandomHorizontalFlip", (1.0,))],
}
# (H, W) per sample; square and non-square, so every quirk shows
SIZES = {
    "recipe": [(375, 500), (500, 375), (333, 500), (300, 300), (281, 500), (500, 486)],
    "val": [(375, 500), (500, 375), (416, 416)],
}
DEFAULT_SIZES = [(300, 400), (400, 300), (256, 256), (123, 457), (500, 331), (64, 64)]
SEEDS = (0, 1, 7)
# box counts per sample, cycled: zero, one, a few, many
COUNTS = (3, 0, 1, 17, 40, 5)
REPRS = [("Resize", ((416, 416),)), ("Resize", (200,)), ("RandomResizedCrop", (416,)), ("CenterCrop", (200,)),
         ("RandomHorizontalFlip", ()), ("RandomHorizontalFlip", (0.7,)), ("ImageTransform", JITTER),
         ("ImageTransform", NORMALIZE)]


def build(name, args):
    if name == "ImageTransform":
        inner, inner_args = args
        return REF.ImageTransform(getattr(T, inner)(*inner_args))
    if name == "convert_to_relative":
        return REF.convert_to_relative
    return getattr(REF, name)(*args)


def voc_objects(h, w, n, g):
    """n VOC objects inside an h x w image (integer pixel boxes, xmin < xmax, ymin < ymax)."""
    objs = []
    for _ in range(n):
        x0, x1 = sorted(g.choice(w + 1, 2, replace=False).tolist())
        y0, y1 = sorted(g.choice(h + 1, 2, replace=False).tolist())
        objs.append({"name": VOC_CLASSES[int(g.integers(0, 20))],
                     "bndbox": {"xmin": str(x0), "ymin": str(y0), "xmax": str(x1), "ymax": str(y1)}})
    return objs


def boxes_for(h, w, n, g):
    """n fp32 boxes around an h x w image: integer and fractional boxes inside, straddling its edges, fully outside,
    touching its sides, and degenerate (x1 == x2 or y1 == y2)."""
    out = []
    for k in range(n):
        kind = k % 6
        if kind == 0:  # integer, inside
            x0, x1 = sorted(g.choice(w + 1, 2, replace=False).tolist())
            y0, y1 = sorted(g.choice(h + 1, 2, replace=False).tolist())
        elif kind == 1:  # fractional, inside
            x0, x1 = sorted(g.uniform(0, w, 2).tolist())
            y0, y1 = sorted(g.uniform(0, h, 2).tolist())
        elif kind == 2:  # straddling the image's edges
            x0, x1 = sorted(g.uniform(-0.3 * w, 1.3 * w, 2).tolist())
            y0, y1 = sorted(g.uniform(-0.3 * h, 1.3 * h, 2).tolist())
        elif kind == 3:  # outside
            x0, x1 = sorted(g.uniform(1.05 * w, 1.5 * w, 2).tolist())
            y0, y1 = sorted(g.uniform(0, h, 2).tolist())
        elif kind == 4:  # touching the sides
            x0, x1, y0, y1 = 0.0, float(w), float(g.integers(0, h)), float(h)
        else:  # degenerate
            x0 = x1 = float(g.integers(0, w + 1))
            y0, y1 = sorted(g.uniform(0, h, 2).tolist())
        out.append([x0, y0, x1, y1])
    return torch.tensor(out, dtype=torch.float32).reshape(-1, 4)


def make_samples(name, seed):
    """The chain's inputs: (H, W) and a target (VOC annotation dict or boxes / labels) per sample."""
    g = np.random.default_rng(10_000 + seed)
    samples = []
    for k, (h, w) in enumerate(SIZES.get(name, DEFAULT_SIZES)):
        n = COUNTS[k % len(COUNTS)]
        if CHAINS[name][0][0] == "VOCTargetTransform":
            target = {"annotation": {"object": voc_objects(h, w, max(n, 1), g)}}
        else:
            target = {"boxes": boxes_for(h, w, n, g), "labels": torch.from_numpy(g.integers(0, 20, n))}
        samples.append(((h, w), target))
    return samples


class DrawLog:
    """Records torch.randint / torch.rand calls and RandomResizedCrop.get_params results while active."""

    def __init__(self):
        self.calls = []

    def __enter__(self):
        self._randint, self._rand = torch.randint, torch.rand
        self._get_params = T.RandomResizedCrop.get_params

        def randint(*args, **kwargs):
            out = self._randint(*args, **kwargs)
            self.calls.append(("randint", tuple(int(a) if isinstance(a, int) else tuple(a) for a in args),
                               out.tolist()))
            return out

        def rand(*args, **kwargs):
            out = self._rand(*args, **kwargs)
            self.calls.append(("rand", tuple(tuple(a) if isinstance(a, (tuple, list)) else a for a in args),
                               out.tolist()))
            return out

        def get_params(img, scale, ratio):
            out = self._get_params(img, scale, ratio)
            self.calls.append(("get_params", (tuple(scale), tuple(ratio)), tuple(int(v) for v in out)))
            return out
        torch.randint, torch.rand = randint, rand
        T.RandomResizedCrop.get_params = staticmethod(get_params)
        return self

    def __exit__(self, *exc):
        torch.randint, torch.rand = self._randint, self._rand
        T.RandomResizedCrop.get_params = staticmethod(self._get_params)


def _image(h, w, seed):
    g = np.random.default_rng(seed)
    return Image.fromarray(g.integers(0, 256, (h, w, 3), dtype=np.uint8), "RGB")


def run_chain(steps, samples, seed):
    """Applies the chain sample by sample; per sample the draws, the (H, W) after each step and the output target."""
    torch.manual_seed(seed)
    out = []
    for k, ((h, w), target) in enumerate(samples):
        img = _image(h, w, 1000 * seed + k)
        if "boxes" in target:
            target = {"boxes": target["boxes"].clone(), "labels": target["labels"].clone()}
        after = []
        with DrawLog() as log:
            for t in steps:
                img, target = t(img, target)
                after.append((img.size[1], img.size[0]) if isinstance(img, Image.Image) else tuple(img.shape[-2:]))
        out.append({"draws": log.calls, "after": after, "boxes": target["boxes"].clone(),
                    "labels": target["labels"].clone()})
    return out, torch.get_rng_state()


def main():
    names = ("Compose", "ImageTransform", "CenterCrop", "Resize", "RandomResizedCrop", "RandomHorizontalFlip",
             "VOCTargetTransform", "convert_to_relative")
    rec = {"signatures": {n: describe_signature(getattr(REF, n)) for n in names},
           "reprs": [(n, a, repr(build(n, a))) for n, a in REPRS], "chains": {}}
    for name, spec in CHAINS.items():
        compose = REF.Compose([build(n, a) for n, a in spec])
        for seed in SEEDS:
            samples = make_samples(name, seed)
            outs, state = run_chain(compose.transforms, samples, seed)
            rec["chains"].setdefault(name, []).append({"spec": spec, "seed": seed, "inputs": samples,
                                                        "outputs": outs, "state": state})
    torch.save(rec, OUT / "det_transforms.pt")
    print(f"wrote {OUT / 'det_transforms.pt'}: {sum(len(v) for v in rec['chains'].values())} chain records")


if __name__ == "__main__":
    main()
