"""Times the RepVGG-A0 (batch 256, 224x224) weight-gradient shapes that run on the generic wgrad kernel (conv_wgrad.cu):
the 1280->1280 3x3 and 1x1 filters at 7x7, the 3x3 and 1x1 filters of the four stride-2 blocks, and the stem's 1x1
GEMM over its 32 im2col columns. The 48-192-channel stride-1 blocks run on the row-window kernel and are not here.

Usage: ``python tools/wgrad_bench.py [--lib PATH] [--iters 50] [--out FILE]``. ``--lib`` loads another build of
libholocron_b200.so (e.g. one of an earlier commit), so two builds can be compared shape by shape from the same tree, one
process per build; ``HB_WGRAD_TAPS_PER_UNIT`` in the environment caps the taps a CTA runs together. Each shape is
warmed up, then timed with CUDA events around ``--iters`` back-to-back calls (the reduction pass over the per-range
partials included), and reported as algorithmic TFLOP/s next to a bf16 ``torch.matmul`` of the same M x N x K
(M = Cout, N = Cin x taps, K = output pixels). ``--out`` also writes the SHA-1 digest of each dW, so that two builds or
two executions can be checked for identical results on the same seeded inputs."""
import argparse
import hashlib
import json
import os
import sys
import zlib
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

BATCH = 256


def shapes():
    """(name, (H, Cin, Cout, k, stride)) with padding k // 2."""
    out = [("3x3 s1 1280->1280 @7", (7, 1280, 1280, 3, 1)), ("1x1 s1 1280->1280 @7", (7, 1280, 1280, 1, 1))]
    for h, ci, co in ((112, 48, 48), (56, 48, 96), (28, 96, 192), (14, 192, 1280)):
        out.append((f"3x3 s2 {ci}->{co} @{h}", (h, ci, co, 3, 2)))
        out.append((f"1x1 s2 {ci}->{co} @{h}", (h, ci, co, 1, 2)))
    out.append(("stem 1x1 32->48 @112", (112, 32, 48, 1, 1)))
    return out


def build_case(K, args, dev):
    """Returns (call, flops, (M, N, K) of the equivalent GEMM); inputs are seeded on the CPU."""
    h, ci, co, k, stride = args
    g = torch.Generator().manual_seed(zlib.crc32(repr(args).encode()))
    pad = k // 2
    ho = K.conv_out_size(h, k, stride, pad, 1)
    x = torch.randn(BATCH, ci, h, h, generator=g).to(torch.bfloat16).to(dev).contiguous(memory_format=torch.channels_last)
    dy = torch.randn(BATCH, co, ho, ho, generator=g).to(torch.bfloat16).to(dev).contiguous(memory_format=torch.channels_last)
    m = BATCH * ho * ho

    def call():
        return K.wgrad_raw(x, dy, co, k, stride, pad)
    return call, 2.0 * m * co * ci * k * k, (co, ci * k * k, m)


def time_it(fn, iters):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None, help="path of the libholocron_b200.so to load (default: the in-tree build)")
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--no-matmul", action="store_true", help="skip the torch.matmul yardstick")
    ap.add_argument("--out", default=None, help="write timings and dW digests as JSON")
    args = ap.parse_args()
    if args.iters < 50:
        ap.error("--iters must be at least 50")
    if not torch.cuda.is_available():
        raise SystemExit("wgrad_bench.py needs a CUDA device")
    from holocron_b200 import _lib
    if args.lib:
        _lib._LIB_PATH = Path(args.lib).resolve()
    from holocron_b200.nn import _fused as K
    dev = torch.device("cuda", 0)
    res = {"lib": str(_lib.lib_path()), "device": torch.cuda.get_device_name(dev),
           "taps_per_unit": os.environ.get("HB_WGRAD_TAPS_PER_UNIT"), "rows": []}
    total_ms = 0.0
    for name, a in shapes():
        call, flops, (m, n, kk) = build_case(K, a, dev)
        dw = call()
        torch.cuda.synchronize()
        row = {"shape": name, "gemm_mnk": [m, n, kk], "sha1": hashlib.sha1(dw.cpu().numpy().tobytes()).hexdigest()}
        del dw
        ms = time_it(call, args.iters)
        total_ms += ms
        row.update(ms=round(ms, 4), tflops=round(flops / ms / 1e9, 1))
        if not args.no_matmul:
            am = torch.randn(m, kk, device=dev, dtype=torch.bfloat16)
            bm = torch.randn(kk, n, device=dev, dtype=torch.bfloat16)
            mm = time_it(lambda: torch.matmul(am, bm), args.iters)
            row.update(matmul_ms=round(mm, 4), matmul_tflops=round(2.0 * m * n * kk / mm / 1e9, 1))
            del am, bm
        res["rows"].append(row)
        print(f"{name:26s} {ms:8.3f} ms {row['tflops']:7.1f} TFLOP/s"
              + ("" if args.no_matmul else f"   matmul {row['matmul_ms']:7.3f} ms {row['matmul_tflops']:7.1f} TFLOP/s"),
              flush=True)
    res["total_ms"] = round(total_ms, 4)
    print(f"{'all shapes':26s} {total_ms:8.3f} ms", flush=True)
    if args.out:
        Path(args.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
