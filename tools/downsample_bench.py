"""Times BlurPool2d, GlobalMaxPool2d and z_pool against the reference's eager formulations on the same GPU:

  - BlurPool2d: ReflectionPad2d then a depth-wise F.conv2d with the binomial filter (bf16 channels_last, cuDNN);
  - GlobalMaxPool2d: x.view(N, C, -1).max(-1) (the reference's view needs a contiguous NCHW input);
  - z_pool: cat([x.max(dim, keepdim=True).values, x.mean(dim, keepdim=True)], dim) (bf16 channels_last).

For each op it reports forward and forward+backward time (CUDA events after warm-up, the median of several windows),
the algorithmic bytes (each tensor read or written once: forward x + y, backward dy + dx), the rate over those bytes
and its share of the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s), and the relative L2 distance between the two
formulations' outputs. The card name, power limit and SM clock are read in the same run.

Usage: ``python tools/downsample_bench.py [--iters 20] [--windows 5] [--json out.json]``.
"""
import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch
import torch.nn.functional as F

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

import holocron_b200 as hb  # noqa: E402
from holocron_b200.nn import _pooling as P  # noqa: E402

HBM_PEAK = 3.35e12
DEV = torch.device("cuda", 0)

# (op, argument, N, C, H): BlurPool2d (kernel_size, stride), GlobalMaxPool2d, z_pool dim
SHAPES = [("blur", (3, 2), 256, 64, 112), ("blur", (5, 2), 256, 256, 56), ("gmp", None, 256, 2048, 7),
          ("gmp", None, 256, 512, 28), ("zpool", 1, 64, 64, 56), ("zpool", 2, 64, 64, 56), ("zpool", 3, 64, 64, 56)]


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                              "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30).stdout
    except (OSError, subprocess.SubprocessError):
        out = "unknown"
    return out.strip()


def _time(fn, iters, windows):
    for _ in range(5):
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


def _eager(op, arg, c):
    if op == "blur":
        k, s = arg
        mod = hb.nn.BlurPool2d(c, k, s)
        filt = (mod._coeffs[:, None] * mod._coeffs[None, :]).to(torch.bfloat16)[None, None].repeat(c, 1, 1, 1).to(DEV)
        pad = P.blur_padding(k, s)
        return lambda x: F.conv2d(F.pad(x, [pad] * 4, mode="reflect"), filt, stride=s, groups=c)
    if op == "gmp":
        return lambda x: x.view(x.size(0), x.size(1), -1).max(-1).values.view(x.size(0), x.size(1), 1, 1)
    return lambda x: torch.cat([x.max(arg, keepdim=True).values, x.mean(arg, keepdim=True)], dim=arg)


def _ours(op, arg, c):
    if op == "blur":
        return hb.nn.BlurPool2d(c, *arg)
    if op == "gmp":
        return hb.nn.GlobalMaxPool2d()
    return hb.nn.ZPool(arg)


def _measure(fn, x, iters, windows):
    with torch.no_grad():
        y = fn(x)
    fwd = _time(lambda: fn(x), iters, windows)
    xg = x.detach().requires_grad_(True)
    dy = torch.randn_like(fn(xg))

    def step():
        torch.autograd.grad(fn(xg), xg, dy)
    both = _time(step, iters, windows)
    return y, fwd, both


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--json", type=str, default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("downsample_bench.py needs a CUDA device")
    card = _card()
    print(f"card (name, power limit, SM clock, max SM clock): {card}")
    rows = []
    for op, arg, n, c, h in SHAPES:
        torch.manual_seed(0)
        x_cl = torch.randn(n, c, h, h, device=DEV).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        # the reference's GlobalMaxPool2d views its input as (N, C, H*W): it needs a contiguous NCHW tensor
        x_eager = x_cl.contiguous() if op == "gmp" else x_cl
        y_ours, f_ours, b_ours = _measure(_ours(op, arg, c), x_cl, args.iters, args.windows)
        y_eager, f_eager, b_eager = _measure(_eager(op, arg, c), x_eager, args.iters, args.windows)
        diff = float((y_ours.double() - y_eager.double()).norm() / y_eager.double().norm())
        x_bytes, y_bytes = x_cl.numel() * 2, y_ours.numel() * 2
        fwd_bytes, both_bytes = x_bytes + y_bytes, 2 * (x_bytes + y_bytes)
        row = {"op": op, "arg": arg, "shape": [n, c, h, h], "dtype": "bf16", "fwd_bytes": fwd_bytes,
               "fwd_bwd_bytes": both_bytes, "rel_l2_vs_eager": diff}
        for tag, f, b in (("ours", f_ours, b_ours), ("eager", f_eager, b_eager)):
            row[tag] = {"fwd_ms": round(f, 4), "fwd_bwd_ms": round(b, 4),
                        "fwd_GBps": round(fwd_bytes / f / 1e6, 1), "fwd_bwd_GBps": round(both_bytes / b / 1e6, 1),
                        "fwd_peak_frac": round(fwd_bytes / f / 1e-3 / HBM_PEAK, 3),
                        "fwd_bwd_peak_frac": round(both_bytes / b / 1e-3 / HBM_PEAK, 3)}
        rows.append(row)
        print(json.dumps(row))
        del x_cl, x_eager, y_ours, y_eager
        torch.cuda.empty_cache()
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps({"card": card, "rows": rows}, indent=1))


if __name__ == "__main__":
    main()
