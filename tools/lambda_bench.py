"""Times LambdaLayer at batch 64 in bf16 channels_last: 128 channels at 28² and 256 channels at 14² (dim_u 1 and 4) with
r = 23, the global variant at 14², and the reference test's layer. For each shape it reports

  - forward and forward+backward time of the module, and the peak memory of a forward+backward step
    (torch.cuda.max_memory_allocated above the live tensors);
  - the time of each lambda kernel (torch.profiler over one forward+backward, summed by kernel name), with the algorithmic
    FLOPs and bytes of that kernel computed from the shapes and the achieved rates;
  - the same module figures for the eager formulation (the conv3d position lambda of the reference, restated in
    tests/_lambda_oracle.py) run in bf16 on the same GPU with cuDNN for the convolutions;

and prints the card name and power limit of the run. Usage: ``python tools/lambda_bench.py [--iters 10] [--json out]``.
"""
import argparse
import json
import subprocess
import sys
from collections import defaultdict
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

BATCH = 64
# (name, in_channels, out_channels, dim_k, n, r, heads, dim_u, H, W, batch)
SHAPES = [
    ("128@28² r23", 128, 128, 16, None, 23, 4, 1, 28, 28, BATCH),
    ("256@14² r23 u1", 256, 256, 16, None, 23, 4, 1, 14, 14, BATCH),
    ("256@14² r23 u4", 256, 256, 16, None, 23, 4, 4, 14, 14, BATCH),
    ("256@14² global", 256, 256, 16, 196, None, 4, 1, 14, 14, BATCH),
    ("reference test", 8, 32, 16, None, 13, 4, 1, 32, 32, 2),
]


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
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def kernel_work(b, hw, dk, u, heads, dv, r):
    """Algorithmic (FLOPs, bytes) per lambda kernel: 2 FLOPs per multiply-add, bf16 activations and fp32 lambdas, each
    tensor read or written once. The local position terms count the Qr form the kernels run."""
    n = b * hw
    taps = r * r if r else 0
    cq, ck, cv, co = heads * dk, dk * u, dv * u, heads * dv
    w = {
        "lam_content_kernel": (2.0 * n * dk * u * dv + 3.0 * n * ck, 2.0 * n * (ck + cv) + 4.0 * b * dk * dv),
        "lam_out_kernel": (2.0 * n * heads * (dk * dv + (u * taps * (dk + dv) if r else dk * dv)),
                           2.0 * n * (cq + cv + co) + (4.0 * n * dk * dv if not r else 0.0)),
        "lam_bwd_content_kernel": (2.0 * n * dk * (heads * dv + 2 * u * dv), 2.0 * n * (cq + co + 2 * cv + 2 * ck)),
        "lam_dlp_kernel": (2.0 * n * heads * dk * dv, 2.0 * n * (cq + co + dk * dv)),
        "lam_dq_kernel": (2.0 * n * heads * (dk * dv + (u * taps * (dk + dv) if r else dk * dv)),
                          2.0 * n * (co + cv + cq) + (4.0 * n * dk * dv if not r else 0.0)),
        "lam_dv_kernel": (2.0 * n * dk * u * dv * (1 + taps), 2.0 * n * (ck + dk * dv + cv)),
        "lam_dr_partial_kernel": (2.0 * n * dk * u * taps * dv, 2.0 * n * (dk * dv + cv)),
    }
    return w


def _kernel_times(step):
    from torch.profiler import ProfilerActivity, profile
    step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    out = defaultdict(float)
    for ev in prof.events():
        if ev.device_type.name == "CUDA" and "lam_" in ev.name:
            key = ev.name.split("lam_", 1)[1].split("<", 1)[0].split("(", 1)[0]
            out["lam_" + key] += ev.device_time / 1000.0
    return dict(out)


def run(iters):
    import holocron_b200 as hb
    import _lambda_oracle as O

    name, power = _card()
    print(f"# {name}, power limit {power}")
    rows = []
    for label, cin, cout, dk, n, r, heads, u, h, w, b in SHAPES:
        torch.manual_seed(0)
        mod = hb.nn.LambdaLayer(cin, cout, dk, n=n, r=r, num_heads=heads, dim_u=u).cuda()
        x = torch.randn(b, cin, h, w, device="cuda").bfloat16().contiguous(memory_format=torch.channels_last)
        x.requires_grad_(True)

        def fwd():
            with torch.no_grad():
                mod(x)

        def step():
            mod(x).float().sum().backward()

        def eager_fwd():
            with torch.no_grad():
                O.lambda_module(x, mod, training=True, dtype=torch.bfloat16, core=O.lambda_core_conv3d)

        def eager_step():
            O.lambda_module(x, mod, training=True, dtype=torch.bfloat16, core=O.lambda_core_conv3d).float().sum().backward()

        row = {"shape": label, "batch": b, "fwd_ms": _time(fwd, iters), "step_ms": _time(step, iters),
               "peak_mb": _peak(step), "eager_fwd_ms": _time(eager_fwd, iters), "eager_step_ms": _time(eager_step, iters),
               "eager_peak_mb": _peak(eager_step)}
        work = kernel_work(b, h * w, dk, u, heads, cout // heads, r or 0)
        kt = _kernel_times(step)
        row["kernels"] = {k: {"ms": t, "gflops": work[k][0] / t / 1e6 if k in work else None,
                              "gbps": work[k][1] / t / 1e6 if k in work else None} for k, t in sorted(kt.items())}
        rows.append(row)
        print(json.dumps(row))
    return {"card": name, "power_limit": power, "rows": rows}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--json", type=str, default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lambda_bench needs a CUDA device")
    res = run(args.iters)
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
