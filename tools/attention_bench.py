"""Times SAM and TripletAttention against the reference's formulation on stock torch, on the same GPU, in bf16
channels_last:

  - SAM: x * torch.sigmoid(F.conv2d(x, w, b)) (holocron/nn/modules/attention.py:29-30);
  - TripletAttention: three DimAttention branches, each transpose(dim, 1).contiguous(), z_pool, a 7x7 F.conv2d,
    F.batch_norm with batch statistics, sigmoid, the product and the transpose back, then (x_c + x_h + x_w) / 3
    (:50-77), in training mode.

For each layer and shape it reports forward and forward+backward time (CUDA events after warm-up, the median of several
windows), the algorithmic bytes of the fused passes (SAM: forward x + y, backward x + dy + dx; TripletAttention:
forward x (pool) + x + y (apply), backward x + dy (pool) + dy + dx (dx pass)), the rate over those bytes and its share of
the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s), and the relative L2 distance between the fused and the stock-torch
outputs. The card name, power limit and SM clock are read in the same run.

Usage: ``python tools/attention_bench.py [--iters 20] [--windows 5] [--json out.json]``.
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

HBM_PEAK = 3.35e12
DEV = torch.device("cuda", 0)

# ResNet-50 stage outputs at batch 64 (SAM: up to its 1024-channel limit in bf16)
SHAPES = [("sam", 64, 256, 56), ("sam", 64, 512, 28), ("sam", 64, 1024, 14),
          ("triplet", 64, 256, 56), ("triplet", 64, 512, 28), ("triplet", 64, 1024, 14), ("triplet", 64, 2048, 7)]
# tensor passes of the fused kernels: (forward, forward + backward)
PASSES = {"sam": (2, 5), "triplet": (3, 7)}


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


def _stock_sam(mod):
    w, b = mod.conv.weight.to(torch.bfloat16), mod.conv.bias.to(torch.bfloat16)
    return lambda x: x * torch.sigmoid(F.conv2d(x, w, b))


def _stock_triplet(mod):
    params = []
    for br in (mod.c_branch, mod.h_branch, mod.w_branch):
        conv, bn = br.compress[1], br.compress[2]
        params.append((br.dim, conv.weight.to(torch.bfloat16), bn.weight.to(torch.bfloat16),
                       bn.bias.to(torch.bfloat16), bn.running_mean.clone(), bn.running_var.clone()))

    def branch(x, dim, w, g, b, rm, rv):
        if dim != 1:
            x = x.transpose(dim, 1).contiguous()
        zp = torch.cat([x.max(1, keepdim=True).values, x.mean(1, keepdim=True)], dim=1)
        out = x * torch.sigmoid(F.batch_norm(F.conv2d(zp, w, padding=3), rm, rv, g, b, True, 0.01, 1e-5))
        return out.transpose(dim, 1).contiguous() if dim != 1 else out

    def fn(x):
        xc, xh, xw = (branch(x, *p) for p in params)
        return (xc + xh + xw) / 3
    return fn


def _measure(fn, x, iters, windows):
    with torch.no_grad():
        y = fn(x)
    fwd = _time(lambda: fn(x), iters, windows)
    xg = x.detach().requires_grad_(True)
    dy = torch.randn_like(y)

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
        raise SystemExit("attention_bench.py needs a CUDA device")
    card = _card()
    print(f"card (name, power limit, SM clock, max SM clock): {card}")
    rows = []
    for layer, n, c, h in SHAPES:
        torch.manual_seed(0)
        x = torch.randn(n, c, h, h, device=DEV).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        mod = (hb.nn.SAM(c) if layer == "sam" else hb.nn.TripletAttention()).to(DEV).train()
        stock = _stock_sam(mod) if layer == "sam" else _stock_triplet(mod)
        # the comparison output comes from the first call of each (same running statistics, same input)
        y_ours, f_ours, b_ours = _measure(mod, x, args.iters, args.windows)
        y_stock, f_stock, b_stock = _measure(stock, x, args.iters, args.windows)
        diff = float((y_ours.double() - y_stock.double()).norm() / y_stock.double().norm())
        tensor = x.numel() * 2
        fwd_bytes, both_bytes = PASSES[layer][0] * tensor, PASSES[layer][1] * tensor
        row = {"layer": layer, "shape": [n, c, h, h], "dtype": "bf16", "tensor_bytes": tensor, "fwd_bytes": fwd_bytes,
               "fwd_bwd_bytes": both_bytes, "rel_l2_vs_stock": diff}
        for tag, f, b in (("fused", f_ours, b_ours), ("stock", f_stock, b_stock)):
            row[tag] = {"fwd_ms": round(f, 4), "fwd_bwd_ms": round(b, 4),
                        "fwd_GBps": round(fwd_bytes / f / 1e6, 1), "fwd_bwd_GBps": round(both_bytes / b / 1e6, 1),
                        "fwd_peak_frac": round(fwd_bytes / f / 1e-3 / HBM_PEAK, 3),
                        "fwd_bwd_peak_frac": round(both_bytes / b / 1e-3 / HBM_PEAK, 3)}
        rows.append(row)
        print(json.dumps(row))
        del x, y_ours, y_stock
        torch.cuda.empty_cache()
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps({"card": card, "rows": rows}, indent=1))


if __name__ == "__main__":
    main()
