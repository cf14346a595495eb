"""Times ColorJitter of the reference's segmentation and detection recipes on a batch of images, batched here against
torchvision run image by image.

Workload: 256 uint8 3x256x256 images with seeded content (the segmentation recipe's crop,
references/segmentation/train.py:133-140), as ``batch.unbind(0)`` of one CUDA tensor, through
``ColorJitter(brightness=0.3, contrast=0.3, saturation=0.1, hue=0.02)``, the factors of both recipes. Baselines:
torchvision's ``ColorJitter`` applied image by image, once on the same CUDA tensors and once on CPU copies with the
host's torch thread count stated. Both paths draw under the same seed, so their outputs are compared as well as timed.

Reported: the CUDA-event time per batch after warm-up (median of several windows; the CPU baseline uses a host clock),
which includes the host work of each call; the host time of the draws alone; launches and device-to-host
synchronisations per batch of each path (synchronisations counted with torch's sync debug mode); with ``--profile`` (a
run of its own), the kernel time of each launch from a profiler trace and the algorithmic bytes (C*H*W read twice and
written once per image when contrast is drawn, read and written once otherwise) over kernel time; the output
comparison under the bars of tests/test_gpu_color_jitter.py (bit-identical for uint8 images of this size); and the card
name and power limit, read in the same run.

Usage: ``python tools/color_jitter_bench.py [--images 256] [--iters 20] [--windows 5] [--cpu-iters 1] [--json out]
[--profile]``.
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

import torch
from torchvision.transforms import transforms as TVT

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from holocron_b200 import _lib  # noqa: E402
from holocron_b200 import transforms as T  # noqa: E402
from holocron_b200.transforms import augmentation  # noqa: E402

HBM_PEAK = 3.35e12
SIDE = 256
SEED = 2024
RECIPE = {"brightness": 0.3, "contrast": 0.3, "saturation": 0.1, "hue": 0.02}


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                              "-i", "0"], capture_output=True, text=True, timeout=30).stdout
    except (OSError, subprocess.SubprocessError):
        out = "unknown"
    return out.strip()


def _time_gpu(fn, iters, windows):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(windows):
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        for _ in range(iters):
            fn()
        end.record()
        end.synchronize()
        times.append(start.elapsed_time(end) / iters)
    return statistics.median(times)


def _syncs(fn):
    """Device-to-host synchronisations one call makes, as torch's sync debug mode reports them."""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--cpu-iters", type=int, default=1)
    ap.add_argument("--json", type=str, default="")
    ap.add_argument("--profile", action="store_true", help="only trace one batch and report kernel times")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("color_jitter_bench needs a CUDA device")
    g = torch.Generator().manual_seed(SEED)
    batch = torch.randint(0, 256, (args.images, 3, SIDE, SIDE), generator=g, dtype=torch.uint8).cuda()
    images = list(batch.unbind(0))
    ours = T.ColorJitter(**RECIPE)
    theirs = TVT.ColorJitter(**RECIPE)
    lib = _lib.lib()
    res = {"card": _card(), "workload": f"{args.images} x uint8 3x{SIDE}x{SIDE}, ColorJitter(0.3, 0.3, 0.1, 0.02)"}

    if args.profile:
        from torch.profiler import ProfilerActivity, profile

        ours(images)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            ours(images)
            torch.cuda.synchronize()
        us = {re.search(r"(\w+_kernel)\(", e.key).group(1): round(e.device_time_total, 2)
              for e in prof.key_averages() if e.device_type.name == "CUDA" and "_kernel(" in e.key}
        total = sum(us.values())
        nbytes = 3 * 3 * SIDE * SIDE * len(images)  # every image has a contrast factor with these ranges
        res.update({"kernels_us": us, "bytes": nbytes, "GB_per_s": round(nbytes / total / 1e3, 1),
                    "share_of_hbm_peak": round(nbytes / (total * 1e-6) / HBM_PEAK, 3)})
        line = json.dumps(res)
        print(line)
        if args.json:
            Path(args.json).write_text(line + "\n")
        return

    # batched: time per batch, launches, syncs, host draw time
    res["batched_ms"] = round(_time_gpu(lambda: ours(images), args.iters, args.windows), 4)
    lib.hb_launch_count_reset()
    ours(images)
    res["batched_launches"] = lib.hb_launch_count()
    res["batched_syncs"] = _syncs(lambda: ours(images))
    real = augmentation.jitter
    augmentation.jitter = lambda s, draws: None
    try:
        t0 = time.perf_counter()
        for _ in range(args.iters):
            ours(images)
        res["draws_host_ms"] = round((time.perf_counter() - t0) * 1e3 / args.iters, 4)
    finally:
        augmentation.jitter = real

    # torchvision image by image, on CUDA and on CPU copies
    per_image = lambda xs: [theirs(x) for x in xs]  # noqa: E731
    res["torchvision_cuda_ms"] = round(_time_gpu(lambda: per_image(images), max(1, args.iters // 4),
                                                 args.windows), 4)
    res["torchvision_cuda_syncs"] = _syncs(lambda: per_image(images))
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        per_image(images)
        torch.cuda.synchronize()
    res["torchvision_cuda_launches"] = sum(e.count for e in prof.key_averages() if e.device_type.name == "CUDA"
                                           and "Memcpy" not in e.key and "Memset" not in e.key)
    cpu = [x.cpu() for x in images]
    per_image(cpu)
    t0 = time.perf_counter()
    for _ in range(args.cpu_iters):
        per_image(cpu)
    res["torchvision_cpu_ms"] = round((time.perf_counter() - t0) * 1e3 / args.cpu_iters, 2)
    res["cpu_threads"] = torch.get_num_threads()

    # outputs: same seed for both paths; uint8 images of 256^2 pixels are under the bit-identical bar
    torch.manual_seed(SEED)
    out = ours(images)
    torch.manual_seed(SEED)
    ref = torch.stack(per_image(images))
    res["comparison"] = {"pixels_differing": int((out != ref).sum()), "pixels": out.numel()}
    line = json.dumps(res)
    print(line)
    if args.json:
        Path(args.json).write_text(line + "\n")


if __name__ == "__main__":
    main()
