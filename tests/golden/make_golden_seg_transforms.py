"""Generates tests/golden/seg_transforms.pt by running the UNMODIFIED reference's segmentation transforms
(references/segmentation/transforms.py of frgfm/Holocron, a checkout named by the HOLOCRON_REFERENCE environment
variable) on seeded PIL images and masks:

    HOLOCRON_REFERENCE=/path/to/Holocron python tests/golden/make_golden_seg_transforms.py

It records each class's constructor signature and ``repr``, and for each chain, seed and list of input sizes, applied
sample by sample as the recipe's dataset applies it: every ``torch.randint`` / ``torch.rand`` call made while the
reference runs (arguments and value), the (H, W) of image and mask after each step, and the default generator's state
afterwards. Chains are given as data ``[(class name, args)]`` so the tests can build the same chain from this package.
"""
import importlib.util
import sys
from pathlib import Path

import numpy as np
import torch
from PIL import Image

sys.path.insert(0, str(Path(__file__).resolve().parent))
from make_golden import OUT, describe_signature  # noqa: E402  (loads the reference)
from oracle.reference_loader import REFERENCE_ROOT  # noqa: E402

_spec = importlib.util.spec_from_file_location("ref_seg_transforms",
                                               REFERENCE_ROOT / "references" / "segmentation" / "transforms.py")
REF = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(REF)

JITTER = ("ColorJitter", (0.3, 0.3, 0.1, 0.02))
NORMALIZE = ("Normalize", ([0.485, 0.456, 0.406], [0.229, 0.224, 0.225]))
CHAINS = {
    # references/segmentation/train.py:133-140 and :174-178
    "recipe": [("RandomResize", (160, 640)), ("RandomCrop", (256,)), ("RandomHorizontalFlip", (0.5,)),
               ("ImageTransform", JITTER), ("ToTensor", ()), ("ImageTransform", NORMALIZE)],
    "val": [("Resize", ((256, 256),)), ("ToTensor", ()), ("ImageTransform", NORMALIZE)],
    "fixed_size": [("RandomResize", (256,)), ("RandomCrop", (256,)), ("RandomHorizontalFlip", (0.5,))],
    # resized sides below, equal to and above the crop
    "small": [("RandomResize", (24, 40)), ("RandomCrop", (32,)), ("RandomHorizontalFlip", (0.5,))],
    "flips_around_crop": [("RandomHorizontalFlip", (0.5,)), ("RandomCrop", (8,)), ("RandomHorizontalFlip", (0.5,))],
    "two_runs": [("Resize", (12,)), ("RandomCrop", (10,)), ("RandomHorizontalFlip", (0.7,)), ("RandomCrop", (6,)),
                 ("RandomResize", (5, 9)), ("RandomHorizontalFlip", (0.3,))],
}
SIZES = {
    "recipe": [(375, 500), (500, 375), (333, 500), (281, 500), (500, 486), (366, 500), (112, 500), (500, 353)],
    "val": [(375, 500), (500, 375), (256, 256), (1, 7)],
    "fixed_size": [(375, 500), (256, 300), (400, 256), (200, 190)],
    "small": [(30, 40), (32, 50), (50, 32), (32, 32), (20, 70), (1, 7), (7, 1)],
    "flips_around_crop": [(5, 7), (8, 8), (8, 11), (1, 1), (13, 3)],
    "two_runs": [(9, 14), (20, 11), (1, 5), (6, 6)],
}
SEEDS = (0, 1, 7)
# standalone transforms: (class name, args)
STANDALONE = [("RandomResize", (160, 640)), ("RandomResize", (256,)), ("Resize", (256,)), ("Resize", ((256, 256),)),
              ("RandomCrop", (256,)), ("RandomCrop", (32,)), ("RandomHorizontalFlip", (0.5,))]
REPRS = [("Resize", ((256, 256),)), ("Resize", (256,)), ("RandomResize", (160, 640)), ("RandomResize", (256,)),
         ("RandomCrop", (256,)), ("RandomHorizontalFlip", (0.5,)), ("ToTensor", ()), ("ImageTransform", JITTER),
         ("ImageTransform", NORMALIZE)]


def build(name, args):
    from torchvision.transforms import transforms as T
    if name == "ImageTransform":
        inner, inner_args = args
        return REF.ImageTransform(getattr(T, inner)(*inner_args))
    return getattr(REF, name)(*args)


def _sample(h, w, seed):
    g = np.random.default_rng(seed)
    img = Image.fromarray(g.integers(0, 256, (h, w, 3), dtype=np.uint8), "RGB")
    mask = Image.fromarray(g.integers(0, 21, (h, w), dtype=np.uint8), "L")
    return img, mask


class DrawLog:
    """Records torch.randint / torch.rand calls and their values while active."""

    def __init__(self):
        self.calls = []

    def __enter__(self):
        self._randint, self._rand = torch.randint, torch.rand

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
        torch.randint, torch.rand = randint, rand
        return self

    def __exit__(self, *exc):
        torch.randint, torch.rand = self._randint, self._rand


def run_chain(steps, sizes, seed):
    """Applies the chain sample by sample; per sample the draws and the (H, W) after each step."""
    torch.manual_seed(seed)
    per_sample = []
    for k, (h, w) in enumerate(sizes):
        img, mask = _sample(h, w, 1000 * seed + k)
        after = []
        with DrawLog() as log:
            for t in steps:
                img, mask = t(img, mask)
                hw = lambda x: (x.size[1], x.size[0]) if isinstance(x, Image.Image) else tuple(x.shape[-2:])  # noqa
                after.append((hw(img), hw(mask)))
        per_sample.append({"draws": log.calls, "after": after})
    return per_sample, torch.get_rng_state()


def main():
    rec = {"signatures": {n: describe_signature(getattr(REF, n)) for n in
                          ("Compose", "Resize", "RandomResize", "RandomCrop", "RandomHorizontalFlip", "ToTensor",
                           "ImageTransform")},
           "reprs": [(n, a, repr(build(n, a))) for n, a in REPRS],
           "chains": {}, "standalone": []}
    for name, spec in CHAINS.items():
        compose = REF.Compose([build(n, a) for n, a in spec])
        rec["compose_repr_" + name] = repr(compose)
        for seed in SEEDS:
            samples, state = run_chain(compose.transforms, SIZES[name], seed)
            rec["chains"].setdefault(name, []).append({"spec": spec, "sizes": SIZES[name], "seed": seed,
                                                        "samples": samples, "state": state})
    for n, a in STANDALONE:
        for seed in SEEDS:
            sizes = [(375, 500), (30, 40), (256, 256), (1, 7), (500, 256)]
            samples, state = run_chain([build(n, a)], sizes, seed)
            rec["standalone"].append({"spec": [(n, a)], "sizes": sizes, "seed": seed, "samples": samples,
                                      "state": state})
    torch.save(rec, OUT / "seg_transforms.pt")
    print(f"wrote {OUT / 'seg_transforms.pt'}: {sum(len(v) for v in rec['chains'].values())} chain records, "
          f"{len(rec['standalone'])} standalone records")


if __name__ == "__main__":
    main()
