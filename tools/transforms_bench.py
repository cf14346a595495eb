"""Times holocron_b200.transforms on a batch of images against the reference's execution of the same calls.

Workload: 256 uint8 3-channel images with seeded random sides of 300-500 pixels, as a list of CUDA tensors (the shape of
a detection / segmentation input pipeline feeding a 224x224 model). Timed calls:

  - Resize((224, 224), mode=ResizeMethod.PAD)   (antialiased bilinear resize to the aspect-preserving box, zero pad);
  - Resize((224, 224))                           (squish, antialiased bilinear);
  - RandomZoomOut((224, 224))                    (scale (0.5, 1), antialiased bilinear, zero pad).

Baselines restate what holocron.transforms runs per image: torchvision's ``resize`` then ``pad`` (``resize`` alone for
squish), once on the same CUDA tensors and once on CPU copies with the host's torch thread count stated. For each call
it reports the CUDA-event time per batch after warm-up (median of several windows; the CPU baseline uses a host clock),
the kernel launches per batch, the algorithmic bytes (each source pixel read once, each output pixel written once) and
the rate over them against the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s), both for the event time (which includes
the host work of each call: get_params, the descriptor table) and for the kernel time alone (from a profiler trace of
one call, taken outside the timed windows). The card name and power limit are read in the same run.

Usage: ``python tools/transforms_bench.py [--images 256] [--iters 10] [--windows 5] [--cpu-iters 1] [--json out.json]``.
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

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

import holocron_b200 as hb  # noqa: E402
from holocron_b200.transforms.interpolation import ResizeMethod  # noqa: E402

HBM_PEAK = 3.35e12
DEV = torch.device("cuda", 0)
SIZE = (224, 224)


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


def _kernels_per_call(fn):
    """CUDA kernels (and memcpys) one call enqueues, from a profiler trace of that call alone."""
    fn()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    kinds = {"kernel": 0, "memcpy": 0, "kernel_ms": 0.0}
    for evt in prof.events():
        if evt.device_type == torch.autograd.DeviceType.CUDA:
            kind = "memcpy" if "memcpy" in evt.name.lower() else "kernel"
            kinds[kind] += 1
            if kind == "kernel":
                kinds["kernel_ms"] += evt.time_range.elapsed_us() / 1e3
    kinds["kernel_ms"] = round(kinds["kernel_ms"], 4)
    return kinds


def _reference_chain(img, inner, pad=True):
    """One image as holocron.transforms runs it: torchvision resize (antialiased bilinear), then zero pad."""
    y = TF.resize(img, list(inner), TF.InterpolationMode.BILINEAR)
    if not pad:
        return y
    dh, dw = SIZE[0] - inner[0], SIZE[1] - inner[1]
    return TF.pad(y, [dw // 2, dh // 2, dw - dw // 2, dh - dh // 2])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=256)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--cpu-iters", type=int, default=1)
    ap.add_argument("--json", type=str, default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("transforms_bench needs a CUDA device")

    g = torch.Generator().manual_seed(0)
    sides = torch.randint(300, 501, (args.images, 2), generator=g).tolist()
    cpu_imgs = [torch.randint(0, 256, (3, h, w), generator=g, dtype=torch.uint8) for h, w in sides]
    gpu_imgs = [x.to(DEV) for x in cpu_imgs]
    src_bytes = sum(x.numel() for x in cpu_imgs)
    out_bytes = args.images * 3 * SIZE[0] * SIZE[1]

    pad_tf = hb.transforms.Resize(SIZE, mode=ResizeMethod.PAD)
    squish_tf = hb.transforms.Resize(SIZE)
    zoom_tf = hb.transforms.RandomZoomOut(SIZE)

    def zoom_inner(imgs):
        return [zoom_tf.get_params(x) for x in imgs]

    calls = {
        "Resize(pad)": (lambda: pad_tf(gpu_imgs),
                        lambda imgs: [_reference_chain(x, pad_tf.get_params(x)) for x in imgs]),
        "Resize(squish)": (lambda: squish_tf(gpu_imgs),
                           lambda imgs: [_reference_chain(x, SIZE, pad=False) for x in imgs]),
        "RandomZoomOut": (lambda: zoom_tf(gpu_imgs),
                          lambda imgs: [_reference_chain(x, hw) for x, hw in zip(imgs, zoom_inner(imgs))]),
    }
    # the batched call computes what the per-image chain computes (uint8: at most one step, at rounding ties)
    torch.manual_seed(0)
    ours = pad_tf(gpu_imgs)
    theirs = torch.stack(calls["Resize(pad)"][1](gpu_imgs))
    max_step = int((ours.int() - theirs.int()).abs().max())
    differing = float((ours != theirs).float().mean())

    card = _card()
    rows = []
    for name, (fn, ref) in calls.items():
        torch.manual_seed(0)
        t_ours = _time_gpu(fn, args.iters, args.windows)
        hb.lib().hb_launch_count_reset()
        fn()
        launches = hb.lib().hb_launch_count()
        t_ref = _time_gpu(lambda: ref(gpu_imgs), max(1, args.iters // 5), args.windows)
        t_cpu = _time_cpu(lambda: ref(cpu_imgs), args.cpu_iters)
        trace = _kernels_per_call(fn)
        rate = (src_bytes + out_bytes) / (t_ours * 1e-3)
        kernel_rate = (src_bytes + out_bytes) / (trace["kernel_ms"] * 1e-3)
        rows.append({
            "call": name, "images": args.images, "ms_per_batch": round(t_ours, 4), "launches_per_batch": launches,
            "trace": trace, "kernel_GB_per_s": round(kernel_rate / 1e9, 1),
            "kernel_fraction_of_hbm_peak": round(kernel_rate / HBM_PEAK, 3), "reference_cuda_ms": round(t_ref, 3),
            "reference_cuda_launches": _kernels_per_call(lambda: ref(gpu_imgs)),
            "reference_cpu_ms": round(t_cpu, 1), "cpu_threads": torch.get_num_threads(),
            "cpu_cores": os.cpu_count(), "algorithmic_bytes": src_bytes + out_bytes,
            "GB_per_s": round(rate / 1e9, 1), "fraction_of_hbm_peak": round(rate / HBM_PEAK, 3),
            "speedup_vs_reference_cuda": round(t_ref / t_ours, 1), "speedup_vs_reference_cpu": round(t_cpu / t_ours, 1),
        })
    result = {"card": card, "pad_vs_reference_max_step": max_step, "pad_vs_reference_differing": differing,
              "rows": rows}
    for r in rows:
        print(json.dumps(r))
    print(json.dumps({"card": card, "pad_vs_reference_max_step": max_step,
                      "pad_vs_reference_differing": differing}))
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
