"""Times the focal loss forward + backward (the register-resident hard-target kernels) on a segmentation-sized input:
16 x 21 x 512 x 512 bf16 logits, int64 targets, reduction 'mean'. Prints one JSON line with the GPU's name and power
limit, the median and spread of per-iteration times over several windows of CUDA-event timing, and the bytes the two
passes must move (logits read twice, dlogits written once, targets read twice) over the median."""
import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import holocron_b200 as hb  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shape", type=int, nargs=4, default=[16, 21, 512, 512])
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--windows", type=int, default=7)
    a = ap.parse_args()
    n, k, h, w = a.shape
    torch.manual_seed(0)
    x = (torch.randn(n, k, h, w, device="cuda") * 2).to(torch.bfloat16).requires_grad_(True)
    t = torch.randint(0, k, (n, h, w), device="cuda")

    def step():
        loss = hb.nn.functional.focal_loss(x, t, gamma=2.0)
        (g,) = torch.autograd.grad(loss, x)
        return g

    for _ in range(10):
        step()
    torch.cuda.synchronize()
    times = []
    for _ in range(a.windows):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.iters):
            step()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) / a.iters)
    med = statistics.median(times)
    nbytes = 3 * x.numel() * 2 + 2 * t.numel() * 8
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    print(json.dumps({"workload": f"focal_loss fwd+bwd bf16 {n}x{k}x{h}x{w}", "gpu": gpu, "ms_median": round(med, 4),
                      "ms_min": round(min(times), 4), "ms_max": round(max(times), 4),
                      "GB/s": round(nbytes / med / 1e6, 1)}))


if __name__ == "__main__":
    main()
