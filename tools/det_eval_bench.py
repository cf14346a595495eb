"""Times the ground-truth matching of DetectionTrainer.evaluate: the per-image loop (assign_iou image by image, as
evaluate runs it on CPU batches) against one hb_assign_iou_batch launch per batch (what it runs on CUDA batches).

Workload: 32 images per batch, each with a seeded 0-40 VOC-like targets (20 classes) and 0-300 detections (jittered
copies of its targets and spurious boxes, on a 1/64 grid so that IoU ties occur), all on the GPU. Before timing, both
paths' (assigned, correct) counts are compared (they must be equal). Reported per path: the time per batch from CUDA
events and from a host clock after a device synchronise (median of several windows, the two paths alternating window
by window); the synchronising calls per batch (torch's sync debug mode, "warn"); with ``--profile`` (a run of its own),
the kernels launched per batch and their device time from a torch.profiler trace. ``--e2e`` adds DetectionTrainer.evaluate
on a randomly initialised yolov2 at 416x416 over a few batches with each path. The card name and power limit are read in
the same run.

Usage: ``python tools/det_eval_bench.py [--images 32] [--iters 20] [--windows 7] [--e2e] [--profile] [--json out]``
(``--json`` updates the file: the timing, end-to-end and profile runs each write their own key).
"""
import argparse
import json
import statistics
import subprocess
import sys
import time
import warnings
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from holocron_b200 import _lib  # noqa: E402
from holocron_b200.trainer import DetectionTrainer, assign_iou, trainers  # noqa: E402

SEED = 2024
THR = 0.5


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                              "-i", "0"], capture_output=True, text=True, timeout=30).stdout
    except (OSError, subprocess.SubprocessError):
        out = "unknown"
    return out.strip()


def _voc_boxes(n, g):
    xy = torch.rand(n, 2, generator=g) * 0.8
    wh = 0.02 + torch.rand(n, 2, generator=g) * 0.5
    return torch.cat([xy, (xy + wh).clamp(max=1.0)], 1)


def _batch(n_img, g):
    gts, preds, gl, pl = [], [], [], []
    for _ in range(n_img):
        n = int(torch.randint(0, 41, (1,), generator=g))
        m = int(torch.randint(0, 301, (1,), generator=g))
        gt = _voc_boxes(n, g)
        lab = torch.randint(0, 20, (n,), generator=g)
        k = min(m, 4 * n)
        src = torch.randint(0, max(n, 1), (k,), generator=g)
        near = gt[src] + 0.03 * torch.randn(k, 4, generator=g) if n else torch.zeros(0, 4)
        pred = torch.round(torch.cat([near, _voc_boxes(m - k, g)]) * 64) / 64
        plab = torch.randint(0, 20, (m,), generator=g)
        if n:
            hit = torch.rand(k, generator=g) < 0.7
            plab[:k] = torch.where(hit, lab[src], plab[:k])
        for lst, t in ((gts, gt), (preds, pred), (gl, lab), (pl, plab)):
            lst.append(t.cuda())
    return gts, preds, gl, pl


def _loop(gts, preds, gl, pl):
    """DetectionTrainer.evaluate's per-image loop: (assigned, correct)."""
    assigned = correct = 0
    for g, p, a, b in zip(gts, preds, gl, pl):
        if g.shape[0] > 0 and p.shape[0] > 0:
            gi, pi = assign_iou(g, p, THR)
            assigned += len(gi)
            correct += (a[gi] == b[pi]).sum().item()
    return assigned, correct


def _kernel(gts, preds, gl, pl, counts):
    trainers._assign_batch(gts, preds, THR, gl, pl, counts)


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


def _window(fn, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / iters, start.elapsed_time(end) / iters


def _timing(args):
    g = torch.Generator().manual_seed(SEED)
    batch = _batch(args.images, g)
    counts = torch.zeros(2, dtype=torch.int64, device="cuda")
    _kernel(*batch, counts)
    want = _loop(*batch)
    assert tuple(counts.tolist()) == want, (counts.tolist(), want)
    paths = {"loop": lambda: _loop(*batch), "kernel": lambda: _kernel(*batch, counts)}
    for fn in paths.values():
        fn(), fn()
    runs = {k: [] for k in paths}
    for _ in range(args.windows):
        for k, fn in paths.items():
            runs[k].append(_window(fn, args.iters))
    out = {"card": _card(), "workload": f"{args.images} images, 0-40 targets and 0-300 detections each",
           "targets_per_batch": sum(int(t.shape[0]) for t in batch[0]),
           "detections_per_batch": sum(int(t.shape[0]) for t in batch[1]),
           "assigned_per_batch": want[0], "correct_per_batch": want[1], "counts_equal": True}
    for k, fn in paths.items():
        n = _lib.lib().hb_launch_count()
        syncs = _syncs(fn)
        out[k] = {"host_ms_per_batch": round(statistics.median(h for h, _ in runs[k]), 4),
                  "event_ms_per_batch": round(statistics.median(e for _, e in runs[k]), 4),
                  "host_ms_windows": [round(h, 4) for h, _ in runs[k]],
                  "syncs_per_batch": syncs, "holocron_launches_per_batch": _lib.lib().hb_launch_count() - n}
    out["kernel"]["note"] = "no read-back per batch: evaluate reads the accumulator once per call"
    out["speedup_host"] = round(out["loop"]["host_ms_per_batch"] / out["kernel"]["host_ms_per_batch"], 1)
    return out


def _profile(args):
    g = torch.Generator().manual_seed(SEED)
    batch = _batch(args.images, g)
    counts = torch.zeros(2, dtype=torch.int64, device="cuda")
    paths = {"loop": lambda: _loop(*batch), "kernel": lambda: _kernel(*batch, counts)}
    out = {"card": _card()}
    for k, fn in paths.items():
        fn(), fn()
        torch.cuda.synchronize()
        acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
        with torch.profiler.profile(activities=acts) as prof:
            fn()
            torch.cuda.synchronize()
        kernels, copies, names = 0, 0, {}
        device_us = 0.0
        for e in prof.events():
            if e.device_type != torch.autograd.DeviceType.CUDA:
                continue
            us = e.time_range.elapsed_us()
            if e.name.startswith(("Memcpy", "Memset")):
                copies += 1
                continue
            kernels += 1
            device_us += us
            key = e.name.replace("(anonymous namespace)::", "").split("(")[0][:60]
            names[key] = names.get(key, 0) + 1
        out[k] = {"kernels_per_batch": kernels, "kernel_device_us_per_batch": round(device_us, 2),
                  "copies_per_batch": copies, "kernels": dict(sorted(names.items(), key=lambda kv: -kv[1])[:8])}
    return out


def _e2e(args):
    from holocron_b200.models.detection import yolov2
    torch.manual_seed(SEED)
    model = yolov2(num_classes=20, box_score_thresh=0.0).cuda().eval()
    g = torch.Generator().manual_seed(SEED + 1)
    loader = []
    for _ in range(args.e2e_batches):
        gts, _, gl, _ = _batch(args.e2e_batch_size, g)
        xs = [torch.randn(3, 416, 416, generator=g).cuda() for _ in gts]
        loader.append((xs, [{"boxes": b, "labels": lab} for b, lab in zip(gts, gl)]))
    tr = DetectionTrainer(model, loader, loader, None, torch.optim.SGD(model.parameters(), lr=1e-3), gpu=None)
    matchable = trainers._matchable

    def run(path):
        trainers._matchable = matchable if path == "kernel" else (lambda *a: False)
        try:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            res = tr.evaluate()
            torch.cuda.synchronize()
            return res, (time.perf_counter() - t0) * 1e3
        finally:
            trainers._matchable = matchable

    with torch.no_grad():
        dets = [model(xs) for xs, _ in loader]
    per_image = [int(d["boxes"].shape[0]) for batch in dets for d in batch]
    results, times = {}, {"loop": [], "kernel": []}
    for path in ("loop", "kernel"):
        results[path], _ = run(path)
    for _ in range(args.e2e_repeats):
        for path in ("loop", "kernel"):
            times[path].append(run(path)[1])
    syncs = {}
    for path in ("loop", "kernel"):
        trainers._matchable = matchable if path == "kernel" else (lambda *a: False)
        try:
            syncs[path] = _syncs(tr.evaluate)
        finally:
            trainers._matchable = matchable
    return {"card": _card(), "model": "yolov2(num_classes=20, box_score_thresh=0.0), random init, 416x416",
            "batches": args.e2e_batches, "batch_size": args.e2e_batch_size,
            "detections_per_image_mean": round(statistics.mean(per_image), 1),
            "detections_per_image_max": max(per_image),
            "metrics_equal": results["loop"] == results["kernel"], "metrics": results["kernel"],
            **{f"{p}_ms_per_evaluate": round(statistics.median(times[p]), 2) for p in times},
            **{f"{p}_ms_windows": [round(t, 2) for t in times[p]] for p in times},
            **{f"{p}_syncs_per_evaluate": syncs[p] for p in syncs}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=32)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--e2e", action="store_true", help="also time DetectionTrainer.evaluate on yolov2")
    ap.add_argument("--e2e-batches", type=int, default=4)
    ap.add_argument("--e2e-batch-size", type=int, default=16)
    ap.add_argument("--e2e-repeats", type=int, default=3)
    ap.add_argument("--profile", action="store_true", help="only trace one batch per path and report its kernels")
    ap.add_argument("--json", type=str, default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("det_eval_bench needs a CUDA device")
    rec = {}
    if args.profile:
        rec["profile_run"] = _profile(args)
    else:
        rec["timing_run"] = _timing(args)
        if args.e2e:
            rec["e2e_run"] = _e2e(args)
    print(json.dumps(rec, indent=1))
    if args.json:
        path = Path(args.json)
        old = json.loads(path.read_text()) if path.exists() else {}
        old.update(rec)
        path.write_text(json.dumps(old, indent=1) + "\n")


if __name__ == "__main__":
    main()
