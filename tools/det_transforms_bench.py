"""Times the detection recipe's image-and-box transforms (holocron_b200.transforms.detection) on a batch of images and
VOC annotations, against the per-image oracle run image by image on the same CUDA tensors.

Workload: 32 seeded uint8 3xHxW images with sides drawn in [300, 500] (VOC-like), each with 1-40 VOC objects, through
the train recipe (references/detection/train.py:116-125: VOCTargetTransform, Resize((416, 416)),
RandomHorizontalFlip(), convert_to_relative, ColorJitter(0.3, 0.3, 0.1, 0.02), PILToTensor, ConvertImageDtype(float32),
Normalize), the val chain (the same without flip and jitter) and a RandomResizedCrop(416) chain (VOCTargetTransform,
RandomResizedCrop(416), RandomHorizontalFlip(), convert_to_relative). The baseline is tests/_det_transforms_oracle.py:
the same steps with torchvision's tensor ops for the images and separate torch ops for the boxes, image by image,
drawing the same values under the same seed.

Before timing, both paths run under one seed and their boxes and labels are compared (they must be equal). Reported
per chain: the time per batch on a host clock around the call and a device synchronise (median of several windows);
the host time of the draws alone; launches of this package's kernels and device-to-host synchronisations per batch
(torch's sync debug mode); with ``--profile`` (a run of its own), the device time of each kernel of one batch from a
torch.profiler trace; and the card name and power limit, read in the same run.

Usage: ``python tools/det_transforms_bench.py [--images 32] [--iters 10] [--windows 5] [--json out] [--profile]``.
"""
import argparse
import json
import re
import statistics
import subprocess
import sys
import time
import warnings
from pathlib import Path

import numpy as np
import torch
from torchvision.transforms import transforms as TVT

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

from holocron_b200 import _lib  # noqa: E402
from holocron_b200.transforms import _fold  # noqa: E402
from holocron_b200.transforms import detection as D  # noqa: E402
import _det_transforms_oracle as DO  # noqa: E402

SEED = 2024
NORMALIZE = TVT.Normalize(mean=[0.485, 0.456, 0.406], std=[0.229, 0.224, 0.225])
VOC = ["aeroplane", "bicycle", "bird", "boat", "bottle", "bus", "car", "cat", "chair", "cow", "diningtable", "dog",
       "horse", "motorbike", "person", "pottedplant", "sheep", "sofa", "train", "tvmonitor"]
TENSOR = [D.ImageTransform(TVT.PILToTensor()), D.ImageTransform(TVT.ConvertImageDtype(torch.float32)),
          D.ImageTransform(NORMALIZE)]


def _chains():
    jitter = D.ImageTransform(TVT.ColorJitter(brightness=0.3, contrast=0.3, saturation=0.1, hue=0.02))
    return {"train": D.Compose([D.VOCTargetTransform(VOC), D.Resize((416, 416)), D.RandomHorizontalFlip(),
                                D.convert_to_relative, jitter] + TENSOR),
            "val": D.Compose([D.VOCTargetTransform(VOC), D.Resize((416, 416)), D.convert_to_relative] + TENSOR),
            "random_resized_crop": D.Compose([D.VOCTargetTransform(VOC), D.RandomResizedCrop(416),
                                              D.RandomHorizontalFlip(), D.convert_to_relative])}


def _kernel_name(key):
    key = re.sub(r"^void ", "", key.replace("(anonymous namespace)::", ""))
    return key.split("(")[0][:80]


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                              "-i", "0"], capture_output=True, text=True, timeout=30).stdout
    except (OSError, subprocess.SubprocessError):
        out = "unknown"
    return out.strip()


def _batch(n):
    g = np.random.default_rng(SEED)
    tg = torch.Generator().manual_seed(SEED)
    images, targets = [], []
    for h, w in g.integers(300, 501, (n, 2)).tolist():
        images.append(torch.randint(0, 256, (3, h, w), generator=tg, dtype=torch.uint8).cuda())
        objs = []
        for _ in range(int(g.integers(1, 41))):
            x0, x1 = sorted(g.choice(w + 1, 2, replace=False).tolist())
            y0, y1 = sorted(g.choice(h + 1, 2, replace=False).tolist())
            objs.append({"name": VOC[int(g.integers(0, 20))], "bndbox": {"xmin": str(x0), "ymin": str(y0),
                                                                        "xmax": str(x1), "ymax": str(y1)}})
        targets.append({"annotation": {"object": objs}})
    return images, targets


def _time(fn, iters, windows):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(windows):
        t0 = time.perf_counter()
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1e3 / iters)
    return round(statistics.median(times), 3)


def _syncs(fn):
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    return sum("called a synchronizing CUDA operation" in str(w.message) for w in caught)


def _draws_ms(tf, images, iters):
    """Host time of the draws and folds of one batch alone (no parsing, no table, no launch)."""
    segments = _fold.group(tf.transforms[1:], D._kind, D._starts_run, "detection")
    jitters = _fold.jitters_of(segments, D.ImageTransform)
    sizes = _fold.sizes_of(images)
    t0 = time.perf_counter()
    for _ in range(iters):
        for size in sizes:
            D._draw(segments, jitters, size)
    return round((time.perf_counter() - t0) * 1e3 / iters, 3)


def _same_targets(a, b):
    return len(a) == len(b) and all(torch.equal(x["boxes"], y["boxes"]) and torch.equal(x["labels"], y["labels"])
                                    for x, y in zip(a, b))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=32)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--json", type=str, default="")
    ap.add_argument("--profile", action="store_true", help="only trace one batch per chain and report kernel times")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("det_transforms_bench needs a CUDA device")
    images, targets = _batch(args.images)
    lib = _lib.lib()
    res = {"card": _card(), "workload": f"{args.images} x uint8 3xHxW (H, W in [300, 500]) + 1-40 VOC objects each",
           "boxes_per_batch": sum(len(t["annotation"]["object"]) for t in targets)}
    for name, tf in _chains().items():
        ours = lambda: tf(images, targets)  # noqa: E731
        theirs = lambda: DO.apply_batch(tf.transforms, images, targets)  # noqa: E731
        if args.profile:
            from torch.profiler import ProfilerActivity, profile
            ours()
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                ours()
                torch.cuda.synchronize()
            res[name] = {"kernels_count_us": {_kernel_name(e.key): [e.count, round(e.device_time_total, 2)]
                                              for e in prof.key_averages() if e.device_type.name == "CUDA"}}
            continue
        torch.manual_seed(SEED)
        _, y = ours()
        torch.manual_seed(SEED)
        ref = theirs()
        if not _same_targets(y, [r[1] for r in ref]):
            raise SystemExit(f"{name}: boxes or labels differ from the oracle's")
        r = {"boxes_equal": True, "ms_per_batch": _time(ours, args.iters, args.windows),
             "draws_host_ms": _draws_ms(tf, images, args.iters)}
        r["draws_share"] = round(r["draws_host_ms"] / r["ms_per_batch"], 3)
        lib.hb_launch_count_reset()
        ours()
        r["launches"] = lib.hb_launch_count()
        r["syncs"] = _syncs(ours)
        r["oracle_ms_per_batch"] = _time(theirs, max(1, args.iters // 2), args.windows)
        r["oracle_syncs"] = _syncs(theirs)
        res[name] = r
    line = json.dumps(res)
    print(line)
    if args.json:
        Path(args.json).write_text(line + "\n")


if __name__ == "__main__":
    main()
