"""Times Involution2d on RedNet-50-style layers (batch 64, bf16, K = 7, G = C/16, reduction 4): the four stage widths at
their resolutions and the stride-2 layers at the stage transitions. For each shape it reports

  - forward and forward+backward time of the module, and the time of each involution kernel;
  - the rate of each kernel over its algorithmic bytes (each tensor read or written once), and the share of the forward
    bytes that is the generated kernel tensor;
  - the peak memory of a forward+backward step (torch.cuda.max_memory_allocated above the live tensors);
  - the same module figures for the reference's formulation (unfold, broadcast product, sum over the taps) run in eager
    bf16 on the same GPU, with cuDNN for the pooling and the two 1x1 convolutions;

and prints the card name and power limit of the run. Usage: ``python tools/involution_bench.py [--iters 20] [--json out]``.
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch
import torch.nn.functional as F

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

# (C, H, stride): stride-1 layers of the four stages, then the stride-2 layers entering stages 2-4
SHAPES = [(64, 56, 1), (128, 28, 1), (256, 14, 1), (512, 7, 1), (128, 56, 2), (256, 28, 2), (512, 14, 2)]
BATCH, KSIZE = 64, 7


def _card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = "unknown"
    return name, out


def _time(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def _peak(fn):
    fn()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def _eager_forward(mod, x):
    import _involution_oracle as O
    u = mod.unfold
    kernel = F.avg_pool2d(x, u.stride, u.stride) if u.stride > 1 else x
    kernel = F.conv2d(kernel, mod.reduce.weight.bfloat16(), mod.reduce.bias.bfloat16())
    kernel = F.conv2d(kernel, mod.span.weight.bfloat16(), mod.span.bias.bfloat16())
    return O.involution2d_unfold(x, kernel, mod.k_size, u.stride, u.padding, u.dilation, mod.groups)


def bench_shape(c, h, s, iters):
    import holocron_b200 as hb
    from holocron_b200._lib import lib, ptr, stream_ptr
    from holocron_b200.nn import _fused as K
    dev = torch.device("cuda", 0)
    g, k = c // 16, KSIZE
    torch.manual_seed(0)
    mod = hb.nn.Involution2d(c, k, padding=k // 2, stride=s, groups=g, reduction_ratio=4).to(dev)
    x = torch.randn(BATCH, c, h, h, device=dev).bfloat16().contiguous(memory_format=torch.channels_last)
    xg = x.clone().requires_grad_(True)
    ho = h // s
    dy = torch.randn(BATCH, c, ho, ho, device=dev).bfloat16().contiguous(memory_format=torch.channels_last)

    def fwd():
        with torch.no_grad():
            mod(x)

    def fwd_bwd(f=mod):
        xg.grad = None
        f(xg).backward(dy)

    row = {"C": c, "H": h, "stride": s, "K": k, "G": g, "N": BATCH}
    row["module_fwd_ms"] = _time(fwd, iters)
    row["module_fwd_bwd_ms"] = _time(fwd_bwd, iters)
    row["module_peak_mb"] = _peak(fwd_bwd) / 2**20

    # the three involution kernels on their own, through the C ABI
    kp = K.round_up(g * k * k, 16)
    ker = torch.randn(BATCH, kp, ho, ho, device=dev).bfloat16().contiguous(memory_format=torch.channels_last)
    y = torch.empty_like(dy)
    dx = torch.empty_like(x)
    dker = torch.empty_like(ker)
    L = lib()
    args = (BATCH, h, h, c, c, kp, k, g, s, k // 2, 1)
    calls = {"fwd": lambda: L.hb_involution_fwd_bf16(ptr(x), ptr(ker), ptr(y), *args, stream_ptr()),
             "bwd_data": lambda: L.hb_involution_bwd_data_bf16(ptr(dy), ptr(ker), ptr(dx), *args, stream_ptr()),
             "bwd_kernel": lambda: L.hb_involution_bwd_kernel_bf16(ptr(x), ptr(dy), ptr(dker), *args, stream_ptr())}
    xb, yb, kb = x.numel() * 2, dy.numel() * 2, BATCH * ho * ho * g * k * k * 2
    nbytes = {"fwd": xb + kb + yb, "bwd_data": yb + kb + xb, "bwd_kernel": xb + yb + kb}
    for name, call in calls.items():
        assert call() == 0, name
        ms = _time(call, iters)
        row[f"{name}_ms"] = ms
        row[f"{name}_GBps"] = nbytes[name] / ms / 1e6
    row["fwd_kernel_tensor_share"] = kb / nbytes["fwd"]

    def eager_fwd():
        with torch.no_grad():
            _eager_forward(mod, x)

    row["eager_fwd_ms"] = _time(eager_fwd, iters)
    row["eager_fwd_bwd_ms"] = _time(lambda: fwd_bwd(lambda t: _eager_forward(mod, t)), iters)
    row["eager_peak_mb"] = _peak(lambda: fwd_bwd(lambda t: _eager_forward(mod, t))) / 2**20
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--json", type=str, default=None, help="also write the rows to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "involution_bench.py needs a CUDA device"
    name, power = _card()
    print(f"card: {name}, power limit: {power}")
    rows = []
    hdr = ("C", "HxW", "s", "fwd ms", "fwd+bwd ms", "peak MB", "k.fwd ms (GB/s)", "k.dgrad ms (GB/s)",
           "k.kgrad ms (GB/s)", "ker share", "eager fwd", "eager fwd+bwd", "eager peak MB")
    print(" | ".join(hdr))
    for c, h, s in SHAPES:
        r = bench_shape(c, h, s, args.iters)
        rows.append(r)
        print(" | ".join([str(c), f"{h}x{h}", str(s), f"{r['module_fwd_ms']:.3f}", f"{r['module_fwd_bwd_ms']:.3f}",
                          f"{r['module_peak_mb']:.0f}", f"{r['fwd_ms']:.3f} ({r['fwd_GBps']:.0f})",
                          f"{r['bwd_data_ms']:.3f} ({r['bwd_data_GBps']:.0f})",
                          f"{r['bwd_kernel_ms']:.3f} ({r['bwd_kernel_GBps']:.0f})", f"{r['fwd_kernel_tensor_share']:.0%}",
                          f"{r['eager_fwd_ms']:.3f}", f"{r['eager_fwd_bwd_ms']:.3f}", f"{r['eager_peak_mb']:.0f}"]),
              flush=True)
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps({"card": name, "power_limit": power, "rows": rows}, indent=1))


if __name__ == "__main__":
    main()
