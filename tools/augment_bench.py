"""Times the random augmentations of the reference's classification recipe on a batch of images, batched here against
torchvision run image by image.

Workload: the training transforms of references/classification/train.py on 256 uint8 3-channel images with seeded
random sides of 300-500 pixels, as a list of CUDA tensors:

  RandomResizedCrop(176, scale=(0.3, 1.0)) -> RandomHorizontalFlip() -> ConvertImageDtype(float32) -> Normalize
      -> RandomErasing(p=1, scale=(0.02, 0.2), value="random")

Batched: the crop takes the list, the flip and the erasing take ``batch.unbind(0)`` (one launch each); the dtype
conversion and ``Normalize`` run once on the stacked batch. Baselines: torchvision's classes applied image by image,
once on the same CUDA tensors and once on CPU copies with the host's torch thread count stated. They run stage by stage
(every image's crop, then every image's flip, ...), which makes the draws of the batched chain, so the outputs are
compared as well as timed.

Reported: the CUDA-event time per batch after warm-up (median of several windows; the CPU baseline uses a host clock),
which includes the host work of each call (torchvision's get_params, the descriptor rows); the kernel time per batch and
per kernel from a profiler trace of one batch taken in a run of its own; the launches per batch; the algorithmic bytes
of the two transform kernels (each crop source pixel read once and each canvas pixel written once; each flipped and each
erased pixel read and written once, plus the fp32 random fill) over their kernel time; and, separately, the host time of
drawing the random fill, which matching torchvision's draws requires (``torch.empty([C, h, w]).normal_()`` per image).
The card name and power limit are read in the same run.

Usage: ``python tools/augment_bench.py [--images 256] [--iters 10] [--windows 5] [--cpu-iters 1] [--json out.json]``.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time
from pathlib import Path

import torch
import torchvision.transforms.functional as TF
from torchvision.transforms import transforms as TV

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

import holocron_b200 as hb  # noqa: E402

HBM_PEAK = 3.35e12
DEV = torch.device("cuda", 0)
CROP = 176
MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


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
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) / iters)
    return statistics.median(times)


def _time_cpu(fn, iters):
    fn()
    t0 = time.perf_counter()
    for _ in range(iters):
        fn()
    return (time.perf_counter() - t0) * 1e3 / iters


def _trace(fn):
    """Kernels and memcpys one call enqueues, and the kernel time per kernel name, from a profiler trace of it alone."""
    fn()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {"kernel": 0, "memcpy": 0, "kernel_ms": 0.0, "by_kernel_ms": {}}
    for evt in prof.events():
        if evt.device_type != torch.autograd.DeviceType.CUDA:
            continue
        if "memcpy" in evt.name.lower():
            out["memcpy"] += 1
            continue
        ms = evt.time_range.elapsed_us() / 1e3
        out["kernel"] += 1
        out["kernel_ms"] += ms
        name = "erase_kernel" if "erase_kernel" in evt.name else (
            "resample_kernel" if "resample_kernel" in evt.name else "other")
        out["by_kernel_ms"][name] = out["by_kernel_ms"].get(name, 0.0) + ms
    out["kernel_ms"] = round(out["kernel_ms"], 4)
    out["by_kernel_ms"] = {k: round(v, 4) for k, v in out["by_kernel_ms"].items()}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=256)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--cpu-iters", type=int, default=1)
    ap.add_argument("--json", type=str, default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("augment_bench needs a CUDA device")

    g = torch.Generator().manual_seed(0)
    sides = torch.randint(300, 501, (args.images, 2), generator=g).tolist()
    cpu_imgs = [torch.randint(0, 256, (3, h, w), generator=g, dtype=torch.uint8) for h, w in sides]
    gpu_imgs = [x.to(DEV) for x in cpu_imgs]

    kw_crop, kw_erase = {"scale": (0.3, 1.0)}, {"p": 1.0, "scale": (0.02, 0.2), "value": "random"}
    crop, flip, erase = (hb.transforms.RandomResizedCrop(CROP, **kw_crop), hb.transforms.RandomHorizontalFlip(),
                         hb.transforms.RandomErasing(**kw_erase))
    tv_crop, tv_flip, tv_erase = (TV.RandomResizedCrop(CROP, **kw_crop), TV.RandomHorizontalFlip(),
                                  TV.RandomErasing(**kw_erase))

    def ours():
        x = flip(crop(gpu_imgs).unbind(0))
        x = TF.normalize(TF.convert_image_dtype(x, torch.float32), MEAN, STD)
        return erase(x.unbind(0))

    def reference(imgs):
        xs = [tv_crop(x) for x in imgs]
        xs = [tv_flip(x) for x in xs]
        xs = [TF.normalize(TF.convert_image_dtype(x, torch.float32), MEAN, STD) for x in xs]
        return [tv_erase(x) for x in xs]

    # the same seed makes the same draws in both: compare what they compute (the crops round uint8 ties by one step)
    torch.manual_seed(0)
    a = ours()
    torch.manual_seed(0)
    b = torch.stack(reference(gpu_imgs))
    diff = (a - b).abs()
    check = {"max_abs_diff": float(diff.max()), "differing": float((diff != 0).float().mean()),
             "one_uint8_step": round(1 / 255 / min(STD), 5)}

    # algorithmic bytes of the transform kernels, from the draws of the seeded batch above: crop boxes, the flip draws
    # (which only advance the generator here), then the erase rectangles, timed as the host's share of the erasing
    torch.manual_seed(0)
    boxes = [crop.get_params(x, crop.scale, crop.ratio) for x in gpu_imgs]
    for _ in gpu_imgs:
        torch.rand(1)
    canvas = args.images * 3 * CROP * CROP
    t0 = time.perf_counter()
    rects = [erase._draw(torch.empty(3, CROP, CROP, device="meta"))[1] for _ in gpu_imgs]
    draw_ms = (time.perf_counter() - t0) * 1e3
    fill = sum(r[4].numel() for r in rects if r is not None)
    resample_bytes = sum(3 * h * w for _, _, h, w in boxes) + canvas + 2 * canvas  # uint8: crop, then flip
    erase_bytes = 2 * 4 * canvas + 4 * fill

    card = _card()
    torch.manual_seed(0)
    t_ours = _time_gpu(ours, args.iters, args.windows)
    hb.lib().hb_launch_count_reset()
    ours()
    launches = hb.lib().hb_launch_count()
    t_ref = _time_gpu(lambda: reference(gpu_imgs), max(1, args.iters // 5), args.windows)
    t_cpu = _time_cpu(lambda: reference(cpu_imgs), args.cpu_iters)
    trace = _trace(ours)
    ref_trace = _trace(lambda: reference(gpu_imgs))
    k = trace["by_kernel_ms"]
    ours_kernel_bytes = resample_bytes + erase_bytes
    ours_kernel_ms = k.get("resample_kernel", 0.0) + k.get("erase_kernel", 0.0)
    row = {
        "workload": f"{args.images} uint8 images of 300-500 px: RandomResizedCrop({CROP}, scale=(0.3, 1.0)), "
                    "RandomHorizontalFlip, ConvertImageDtype + Normalize, RandomErasing(p=1, scale=(0.02, 0.2), "
                    "value='random')",
        "card": card, "ms_per_batch": round(t_ours, 4), "hb_launches_per_batch": launches, "trace": trace,
        "transform_kernel_bytes": ours_kernel_bytes, "transform_kernel_ms": round(ours_kernel_ms, 4),
        "transform_kernel_GB_per_s": round(ours_kernel_bytes / (ours_kernel_ms * 1e-3) / 1e9, 1),
        "transform_kernel_fraction_of_hbm_peak": round(ours_kernel_bytes / (ours_kernel_ms * 1e-3) / HBM_PEAK, 3),
        "resample_GB_per_s": round(resample_bytes / (k.get("resample_kernel", float("nan")) * 1e-3) / 1e9, 1),
        "erase_GB_per_s": round(erase_bytes / (k.get("erase_kernel", float("nan")) * 1e-3) / 1e9, 1),
        "host_random_fill_draw_ms": round(draw_ms, 3),
        "reference_cuda_ms": round(t_ref, 3), "reference_cuda_trace": ref_trace,
        "reference_cpu_ms": round(t_cpu, 1), "cpu_threads": torch.get_num_threads(), "cpu_cores": os.cpu_count(),
        "speedup_vs_reference_cuda": round(t_ref / t_ours, 1), "speedup_vs_reference_cpu": round(t_cpu / t_ours, 1),
        "vs_reference_output": check,
    }
    print(json.dumps(row))
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(row, indent=1))


if __name__ == "__main__":
    main()
