"""Times the classification recipe's transform chains (holocron_b200.transforms.classification.Compose) on a batch of
images, against torchvision's ``T.Compose`` applied image by image on the same CUDA tensors under the same seed.

Workload: 256 seeded uint8 3xHxW CUDA images with H and W drawn in [300, 500], through the ImageNette train chain
(references/classification/train.py:100-107: RandomResizedCrop(176, scale=(0.3, 1.0)), RandomHorizontalFlip(),
TrivialAugmentWide, PILToTensor, ConvertImageDtype(float32), Normalize, RandomErasing(scale=(0.02, 0.2),
value="random"), bilinear) with erasing at p = 0 (the recipe's default) and p = 0.5, and the validation chain (:162-168:
Resize(232), CenterCrop(224), PILToTensor, ConvertImageDtype(float32), Normalize). The normalisation is the
reference's IMAGENETTE preset.

Before timing, both paths run under one seed and their outputs are compared: the validation chain must be
bit-identical; the train chains report the share of elements that differ (TrivialAugmentWide's affine ops may differ
where a sampling coordinate is within fp32 rounding of a decision, its docstring says where). Reported per chain: the
time per batch on a host clock around the call and a device synchronise (median of several windows); the host time of
the draws alone; launches of this package's kernels and host synchronisations per batch (torch's sync debug mode); with
``--profile`` (a run of its own), the device time of each kernel of one batch from a torch.profiler trace and the
tail's algorithmic rate (1 B read and 4 B written per element of a uint8 batch); and the card name and power limit,
read in the same run.

Usage: ``python tools/cls_transforms_bench.py [--images 256] [--iters 5] [--windows 5] [--json out] [--profile]``;
with ``--profile`` and ``--json``, the kernel times are added to that file's record under "profile".
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
from torchvision.transforms import InterpolationMode, autoaugment as TVA, transforms as TV

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from holocron_b200 import _lib  # noqa: E402
from holocron_b200.transforms import _fold, classification as C  # noqa: E402

SEED = 2024
# the reference's IMAGENETTE normalisation preset
MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


def _chains():
    bilinear = InterpolationMode.BILINEAR

    def train(p):
        return [TV.RandomResizedCrop(176, scale=(0.3, 1.0), interpolation=bilinear), TV.RandomHorizontalFlip(),
                TVA.TrivialAugmentWide(interpolation=bilinear), TV.PILToTensor(), TV.ConvertImageDtype(torch.float32),
                TV.Normalize(MEAN, STD), TV.RandomErasing(p=p, scale=(0.02, 0.2), value="random")]

    return {"train_erase_p0": train(0.0), "train_erase_p0.5": train(0.5),
            "val": [TV.Resize(232, interpolation=bilinear), TV.CenterCrop(224), TV.PILToTensor(),
                    TV.ConvertImageDtype(torch.float32), TV.Normalize(MEAN, STD)]}


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
    return [torch.randint(0, 256, (3, h, w), generator=tg, dtype=torch.uint8).cuda()
            for h, w in g.integers(300, 501, (n, 2)).tolist()]


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


def _draws_ms(chain, images, iters):
    """Host time of the draws and folds of one batch alone (no table, no launch)."""
    segments = C._segments(chain)
    spaces = {id(s): s._augmentation_space(s.num_magnitude_bins) for s in segments
              if isinstance(s, TVA.TrivialAugmentWide)}

    def other(s, size):
        if isinstance(s, TVA.TrivialAugmentWide):
            return C.trivial_draw(spaces[id(s)])
        erasing = s.step(TV.RandomErasing)
        return C.erase_draw(erasing, torch.empty(3, *size, device="meta")) if erasing is not None else None

    sizes = _fold.sizes_of(images)
    t0 = time.perf_counter()
    for _ in range(iters):
        for size in sizes:
            _fold.draw(segments, [], size, C.fold_run, other)
    return round((time.perf_counter() - t0) * 1e3 / iters, 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=256)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--json", type=str, default="")
    ap.add_argument("--profile", action="store_true", help="only trace one batch per chain and report kernel times")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("cls_transforms_bench needs a CUDA device")
    images = _batch(args.images)
    elements = args.images * 3 * 176 * 176, args.images * 3 * 224 * 224
    lib = _lib.lib()
    res = {"card": _card(), "workload": f"{args.images} x uint8 3xHxW (H, W in [300, 500])"}
    for name, chain in _chains().items():
        tf = C.Compose(chain)
        tv = TV.Compose([t for t in chain if not isinstance(t, TV.PILToTensor)])  # PIL images only
        ours = lambda: tf(images)  # noqa: E731
        theirs = lambda: [tv(x) for x in images]  # noqa: E731
        if args.profile:
            from torch.profiler import ProfilerActivity, profile
            ours()
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                ours()
                torch.cuda.synchronize()
            kernels = {_kernel_name(e.key): [e.count, round(e.device_time_total, 2)]
                       for e in prof.key_averages() if e.device_type.name == "CUDA"}
            tail_us = sum(us for k, (_, us) in kernels.items() if "tail_kernel" in k)
            n = elements[1] if name == "val" else elements[0]
            res[name] = {"kernels_count_us": kernels, "tail_us": tail_us,
                         "tail_algorithmic_GBps": round(5 * n / (tail_us * 1e3), 1) if tail_us else None}
            continue
        torch.manual_seed(SEED)
        got = ours()
        torch.manual_seed(SEED)
        want = torch.stack(theirs())
        differ = int((got != want).sum())
        if name == "val" and differ:
            raise SystemExit(f"{name}: {differ} elements differ from torchvision's")
        r = {"elements_differing": differ, "share_differing": differ / want.numel(),
             "ms_per_batch": _time(ours, args.iters, args.windows), "draws_host_ms": _draws_ms(chain, images, 3)}
        lib.hb_launch_count_reset()
        ours()
        r["launches"] = lib.hb_launch_count()
        r["syncs"] = _syncs(ours)
        r["torchvision_ms_per_batch"] = _time(theirs, 1, max(3, args.windows // 2))
        r["torchvision_syncs"] = _syncs(theirs)
        res[name] = r
    if args.profile and args.json and Path(args.json).exists():
        record = json.loads(Path(args.json).read_text())
        record["profile"] = res
        res = record
    line = json.dumps(res)
    print(line)
    if args.json:
        Path(args.json).write_text(line + "\n")


if __name__ == "__main__":
    main()
