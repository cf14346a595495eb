"""Times the segmentation recipe's paired transforms (holocron_b200.transforms.segmentation) on a batch of images and
masks, against torchvision's tensor ops run image by image on the same CUDA tensors.

Workload: 32 seeded uint8 3xHxW images with sides drawn in [300, 500] (VOC-like) and uint8 masks of 21 classes, as
lists of CUDA tensors, through the train recipe (references/segmentation/train.py:133-140: RandomResize(160, 640),
RandomCrop(256), RandomHorizontalFlip(0.5), ColorJitter(0.3, 0.3, 0.1, 0.02), ToTensor, Normalize) and the val chain
(:174-178: Resize((256, 256)), ToTensor, Normalize). The baseline is tests/_seg_transforms_oracle.py: the same steps
with torchvision's tensor ops, image by image, drawing the same values under the same seed.

Before timing, both paths run under one seed and their masks are compared (they must be equal). Reported per chain:
the time per batch on a host clock around the call and a device synchronise (so the host draws and table building
are in it; median of several windows); the host time of the draws alone; launches of this package's kernels and
device-to-host synchronisations per batch (torch's sync debug mode); with ``--profile`` (a run of its own), the device
time of each kernel of one batch from a torch.profiler trace; and the card name and power limit, read in the same run.

Usage: ``python tools/seg_transforms_bench.py [--images 32] [--iters 10] [--windows 5] [--json out] [--profile]``.
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
from holocron_b200.transforms import segmentation as S  # noqa: E402
import _seg_transforms_oracle as SO  # noqa: E402

SEED = 2024
NORMALIZE = TVT.Normalize(mean=[0.485, 0.456, 0.406], std=[0.229, 0.224, 0.225])


def _chains():
    return {"train": S.Compose([S.RandomResize(160, 640), S.RandomCrop(256), S.RandomHorizontalFlip(0.5),
                                S.ImageTransform(TVT.ColorJitter(0.3, 0.3, 0.1, 0.02)), S.ToTensor(),
                                S.ImageTransform(NORMALIZE)]),
            "val": S.Compose([S.Resize((256, 256)), S.ToTensor(), S.ImageTransform(NORMALIZE)])}


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
    images, masks = [], []
    for h, w in g.integers(300, 501, (n, 2)):
        images.append(torch.randint(0, 256, (3, int(h), int(w)), generator=tg, dtype=torch.uint8).cuda())
        masks.append(torch.randint(0, 21, (int(h), int(w)), generator=tg, dtype=torch.uint8).cuda())
    return images, masks


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
    """Host time of the draws and folds of one batch alone (no table, no launch)."""
    segments = S._segments(tf.transforms)
    jitters = [s for s in segments if isinstance(s, S.ImageTransform) and isinstance(s.transform, TVT.ColorJitter)]
    sizes = [(int(x.shape[-2]), int(x.shape[-1])) for x in images]
    t0 = time.perf_counter()
    for _ in range(iters):
        for size in sizes:
            S._draw(segments, jitters, size)
    return round((time.perf_counter() - t0) * 1e3 / iters, 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=32)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--json", type=str, default="")
    ap.add_argument("--profile", action="store_true", help="only trace one batch per chain and report kernel times")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("seg_transforms_bench needs a CUDA device")
    images, masks = _batch(args.images)
    lib = _lib.lib()
    res = {"card": _card(), "workload": f"{args.images} x uint8 3xHxW (H, W in [300, 500]) + uint8 masks"}
    for name, tf in _chains().items():
        ours = lambda: tf(images, masks)  # noqa: E731
        theirs = lambda: SO.apply_batch(tf.transforms, images, masks)  # noqa: E731
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
        if not torch.equal(y, torch.stack([r[1] for r in ref])):
            raise SystemExit(f"{name}: masks differ from torchvision's")
        r = {"masks_equal": True, "ms_per_batch": _time(ours, args.iters, args.windows),
             "draws_host_ms": _draws_ms(tf, images, args.iters)}
        r["draws_share"] = round(r["draws_host_ms"] / r["ms_per_batch"], 3)
        lib.hb_launch_count_reset()
        ours()
        r["launches"] = lib.hb_launch_count()
        r["syncs"] = _syncs(ours)
        r["torchvision_ms_per_batch"] = _time(theirs, max(1, args.iters // 2), args.windows)
        r["torchvision_syncs"] = _syncs(theirs)
        res[name] = r
    line = json.dumps(res)
    print(line)
    if args.json:
        Path(args.json).write_text(line + "\n")


if __name__ == "__main__":
    main()
