"""Times TrivialAugmentWide of the reference's classification recipe on a batch of images, batched here against
torchvision run image by image.

Workload: 256 uint8 3x176x176 images with seeded content (the size RandomResizedCrop(176) gives in
references/classification/train.py:100-107), as ``batch.unbind(0)`` of one CUDA tensor, through
``TrivialAugmentWide(interpolation=BILINEAR)``. Baselines: torchvision's ``TrivialAugmentWide`` applied image by image,
once on the same CUDA tensors and once on CPU copies with the host's torch thread count stated. Both paths draw under
the same seed, so their outputs are compared as well as timed.

Reported: the CUDA-event time per batch after warm-up (median of several windows; the CPU baseline uses a host clock),
which includes the host work of each call; the host time of the draws alone; launches and device-to-host
synchronisations per batch of each path (synchronisations counted with torch's sync debug mode); per-op batches forced
through ``apply_ops`` (every image one op), their call time with CUDA events and, with ``--profile`` (a run of its
own), their kernel times from a profiler trace with the algorithmic bytes (C*H*W read and written per image, plus one
more read of it for the histogram ops) over kernel time; the output comparison under the bars of
tests/test_gpu_autoaugment.py; and the card name and power limit, read in the same run.

Usage: ``python tools/autoaugment_bench.py [--images 256] [--iters 20] [--windows 5] [--cpu-iters 1] [--json out]
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
from torchvision.transforms import InterpolationMode
from torchvision.transforms import autoaugment as TVA

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

from holocron_b200 import _lib  # noqa: E402
from holocron_b200 import transforms as T  # noqa: E402
from holocron_b200.transforms import _autoaugment, augmentation  # noqa: E402

HBM_PEAK = 3.35e12
SIDE = 176
SEED = 2024
BILINEAR = InterpolationMode.BILINEAR
GEOMETRIC = ("ShearX", "ShearY", "TranslateX", "TranslateY", "Rotate")
FORCED = {"Identity": 0.0, "ShearX": 0.3, "Rotate": 30.0, "TranslateX": 12.0, "Brightness": 0.4, "Color": 0.4,
          "Contrast": 0.4, "Sharpness": 0.4, "Posterize": 4.0, "Solarize": 128.0, "AutoContrast": 0.0,
          "Equalize": 0.0}


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


def _compare(images, ops, out, ref):
    """Pixels outside the tolerated band, and the share of affine pixels the band holds."""
    from _autoaugment_oracle import apply_op as oracle_op
    bad = amb = geo = 0
    for x, (op, m), got, want in zip(images, ops, out, ref):
        mism = (got != want).cpu().numpy()
        if op in GEOMETRIC:
            _, a = oracle_op(x.cpu().numpy(), op, m, True, None)
            bad += int((mism & ~a[None]).sum())
            amb += int(a.sum())
            geo += a.size
        else:
            bad += int(mism.sum())
    return {"pixels_outside_bars": bad, "affine_ambiguous_share": amb / max(geo, 1)}


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
        raise SystemExit("autoaugment_bench needs a CUDA device")
    g = torch.Generator().manual_seed(SEED)
    batch = torch.randint(0, 256, (args.images, 3, SIDE, SIDE), generator=g, dtype=torch.uint8).cuda()
    images = list(batch.unbind(0))
    ours = T.TrivialAugmentWide(interpolation=BILINEAR)
    theirs = TVA.TrivialAugmentWide(interpolation=BILINEAR)
    lib = _lib.lib()
    res = {"card": _card(), "workload": f"{args.images} x uint8 3x{SIDE}x{SIDE}, TrivialAugmentWide(BILINEAR)"}

    if args.profile:
        from torch.profiler import ProfilerActivity, profile

        def kernel_us(fn):
            fn()
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                fn()
                torch.cuda.synchronize()
            return {re.search(r"(\w+_kernel)\(", e.key).group(1): round(e.device_time_total, 2)
                    for e in prof.key_averages() if e.device_type.name == "CUDA" and "_kernel(" in e.key}

        res["kernels_us_one_mixed_batch"] = kernel_us(lambda: ours(images))
        plane = 3 * SIDE * SIDE * len(images)
        per_op = {}
        for op, m in FORCED.items():
            us = kernel_us(lambda: _autoaugment.apply_ops(images, [(op, m)] * len(images), BILINEAR, None))
            nbytes = plane * (3 if op in _autoaugment.STAT_OPS else 2)
            total = sum(us.values())
            per_op[op] = {"kernels_us": us, "bytes": nbytes, "GB_per_s": round(nbytes / total / 1e3, 1),
                          "share_of_hbm_peak": round(nbytes / (total * 1e-6) / HBM_PEAK, 3)}
        res["forced_ops_kernel_time"] = per_op
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
    real = augmentation.apply_ops
    augmentation.apply_ops = lambda s, ops, *a: None
    try:
        t0 = time.perf_counter()
        for _ in range(args.iters):
            ours(images)
        res["draws_host_ms"] = round((time.perf_counter() - t0) * 1e3 / args.iters, 4)
    finally:
        augmentation.apply_ops = real

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

    # per-op forced batches (every image the same op): call time, host work included
    res["forced_ops_call_ms"] = {
        op: round(_time_gpu(lambda: _autoaugment.apply_ops(images, [(op, m)] * len(images), BILINEAR, None),
                            args.iters, args.windows), 4) for op, m in FORCED.items()}

    # outputs under the test bars, same seed for both paths
    recorded = []
    augmentation.apply_ops = lambda s, ops, *a: recorded.extend(ops) or real(s, ops, *a)
    try:
        torch.manual_seed(SEED)
        out = ours(images)
    finally:
        augmentation.apply_ops = real
    torch.manual_seed(SEED)
    ref = per_image(images)
    res["comparison"] = _compare(images, recorded, out, ref)
    line = json.dumps(res)
    print(line)
    if args.json:
        Path(args.json).write_text(line + "\n")


if __name__ == "__main__":
    main()
