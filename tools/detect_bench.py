"""Times the YOLOv4 eval forward with the per-image post-processing loop and with the batched kernels, alternated.

Usage: ``python tools/detect_bench.py [--batch 16] [--size 512] [--iters 10] [--out results.json]``. Both variants run
the same backbone, neck and heads. "per-image" then post-processes each scale with the reference's Python loop (one
torchvision nms per image and scale) and concatenates per image; "batched" is ``model(x)`` (three scales in one launch
chain, one read-back). Wall time is taken from a host clock after a device synchronise, per batch. The synchronisation
count comes from torch's CUDA sync debug mode, the launch count from torch.profiler, both for the post-processing
alone. Two head settings: the zero-initialised output convolutions of a fresh model (every candidate passes, all scores
tie) and random output convolutions."""
import argparse
import json
import statistics
import subprocess
import sys
import time
import warnings
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from holocron_b200.models.detection import yolov4  # noqa: E402
from holocron_b200.models.detection.yolov4 import YoloLayer  # noqa: E402


def _per_image(head, outs):
    layers = (head.yolo1, head.yolo2, head.yolo3)
    ys = [YoloLayer._post_process_per_image(*layer._format_outputs(o), layer.rpn_nms_thresh, layer.box_score_thresh)
          for layer, o in zip(layers, outs)]
    return [{k: torch.cat((d1[k], d2[k], d3[k]), dim=0) for k in ("boxes", "scores", "labels")} for d1, d2, d3 in zip(*ys)]


def _batched(head, outs):
    from holocron_b200.models.detection._postprocess import to_detections
    return to_detections(*head._detect(outs))


def _syncs(fn, *args):
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn(*args)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    return sum("synchroniz" in str(w.message) for w in rec)


def _launches(fn, *args):
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn(*args)
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)


def _power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", type=str, default=None)
    args = ap.parse_args()
    dev = torch.device("cuda")
    torch.manual_seed(0)
    model = yolov4(num_classes=80).to(dev).eval()
    x = torch.rand(args.batch, 3, args.size, args.size, device=dev)
    result = {"device": torch.cuda.get_device_name(0), "power_limit": _power_limit(), "batch": args.batch,
              "size": args.size, "iters": args.iters, "heads": {}}
    for setting in ("zero-init", "random"):
        if setting == "random":
            for head in (model.head.head1, model.head.head2_2, model.head.head3):
                torch.nn.init.normal_(head[-1].weight, std=0.05)
                torch.nn.init.normal_(head[-1].bias, std=1.0)
        with torch.no_grad():
            outs = model.head._heads(list(model.neck(model.backbone(x))))
            a, b = _per_image(model.head, outs), _batched(model.head, outs)
            same = all(torch.equal(p[k], q[k]) for p, q in zip(a, b) for k in p)
            times = {"per-image": [], "batched": []}
            for _ in range(args.iters + 1):          # the first round is a warm-up
                for name in times:
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    if name == "batched":
                        model(x)
                    else:
                        _per_image(model.head, model.head._heads(list(model.neck(model.backbone(x)))))
                    torch.cuda.synchronize()
                    times[name].append(time.perf_counter() - t0)
            rec = {"equal": same, "detections": sum(len(d["scores"]) for d in b)}
            for name, fn in (("per-image", _per_image), ("batched", _batched)):
                rec[name] = {"forward_ms_median": 1e3 * statistics.median(times[name][1:]),
                             "post_process_syncs": _syncs(fn, model.head, outs),
                             "post_process_launches": _launches(fn, model.head, outs)}
        result["heads"][setting] = rec
    line = json.dumps(result)
    print(line)
    if args.out:
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
