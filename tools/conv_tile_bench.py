"""Times the RepVGG-A0 (batch 256, 224x224) convolution shapes that run on the generic implicit-GEMM kernel
(conv_fprop.cu): forward 3x3 and 1x1 (stride 1 and 2), the stride-1 data gradient with the 1x1 branch as K extension and
the identity gradient as epilogue residual, and the parity-class data gradient of the stride-2 blocks.

Usage: ``python tools/conv_tile_bench.py [--lib PATH] [--iters 50] [--out FILE]``. ``--lib`` loads another build of
libholocron_b200.so (e.g. one of an earlier commit), so two builds can be compared shape by shape from the same tree, one
process per build. Each shape is warmed up, then timed with CUDA events around ``--iters`` back-to-back launches, and
reported as algorithmic TFLOP/s next to a bf16 ``torch.matmul`` of the same M x N x K. ``--out`` also writes the
outputs' SHA-1 digests and the per-channel sums of the statistics partials, so that two builds can be checked for
identical results on the same seeded inputs."""
import argparse
import hashlib
import json
import sys
import zlib
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

BATCH = 256


def shapes():
    """(name, kind, args): kind 'fwd' = (H, Cin, Cout, k, stride, stats); 'kext' = (H, C, Cd); 's2' = (H, C, Cd)."""
    out = []
    for h, c in ((14, 192), (7, 1280)):
        out.append((f"fwd 3x3 s1 {c}->{c} @{h}", "fwd", (h, c, c, 3, 1, True)))
        out.append((f"fwd 1x1 s1 {c}->{c} @{h}", "fwd", (h, c, c, 1, 1, c >= 1024)))
        out.append((f"dgrad kext {c}->{c} @{h}", "kext", (h, c, c)))
    for h, ci, co in ((28, 96, 192), (14, 192, 1280)):
        out.append((f"fwd 3x3 s2 {ci}->{co} @{h}", "fwd", (h, ci, co, 3, 2, 9 * ci >= 1024)))
        out.append((f"fwd 1x1 s2 {ci}->{co} @{h}", "fwd", (h, ci, co, 1, 2, False)))
        out.append((f"dgrad s2 {co}->{ci} @{h}", "s2", (h, co, ci)))
    return out


def _cl(t):
    return t.contiguous(memory_format=torch.channels_last)


def build_case(K, kind, args, dev):
    """Returns (launch, flops, (M, N, K) of the equivalent GEMM); inputs are seeded on the CPU."""
    g = torch.Generator().manual_seed(zlib.crc32(repr((kind, args)).encode()))

    def rnd(*shape, scale=1.0):
        return (torch.randn(*shape, generator=g) * scale).to(torch.bfloat16).to(dev)

    if kind == "fwd":
        h, ci, co, k, stride, stats = args
        x = _cl(rnd(BATCH, ci, h, h))
        wf = rnd(co, k, k, ci, scale=(k * k * ci) ** -0.5).contiguous()
        pad = k // 2
        ho = K.conv_out_size(h, k, stride, pad, 1)
        m, kk = BATCH * ho * ho, k * k * ci

        def launch():
            return K.conv2d_forward_raw(x, wf, co, k, k, stride, pad, 1, want_stats=stats)
        return launch, 2.0 * m * co * kk, (m, co, kk)
    if kind == "kext":
        h, c, cd = args
        dy3, dy1, dxid = (_cl(rnd(BATCH, c, h, h)) for _ in range(3))
        wd3 = rnd(cd, 3, 3, c, scale=(9 * c) ** -0.5).contiguous()
        wd1 = rnd(cd, 1, 1, c, scale=c ** -0.5).contiguous()
        m, kk = BATCH * h * h, 10 * c

        def launch():
            return K.conv2d_forward_raw(dy3, wd3, cd, 3, 3, 1, 1, 1, None, dxid, K.ACT_NONE, xe=dy1, we=wd1, kind="dgrad")
        return launch, 2.0 * m * cd * kk, (m, cd, kk)
    h, c, cd = args
    ho = (h - 1) // 2 + 1
    dy3, dy1 = _cl(rnd(BATCH, c, ho, ho)), _cl(rnd(BATCH, c, ho, ho))
    w3 = torch.nn.Parameter((torch.randn(c, cd, 3, 3, generator=g) * (9 * cd) ** -0.5).to(dev))
    wd1 = rnd(cd, 1, 1, c, scale=c ** -0.5).contiguous()
    taps = sum((1 + a) * (1 + b) * ((h - a + 1) // 2) * ((h - b + 1) // 2) for a in (0, 1) for b in (0, 1))
    flops = 2.0 * BATCH * cd * c * (taps + ho * ho)
    m, kk = BATCH * h * h, (taps + ho * ho) * c // (h * h)

    def launch():
        return K.dgrad_s2_raw(dy3, w3, cd, h, h, dy1, wd1)
    return launch, flops, (m, cd, kk)


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
    ap.add_argument("--out", default=None, help="write timings, output digests and statistics sums as JSON")
    args = ap.parse_args()
    if args.iters < 50:
        ap.error("--iters must be at least 50")
    if not torch.cuda.is_available():
        raise SystemExit("conv_tile_bench.py needs a CUDA device")
    from holocron_b200 import _lib
    if args.lib:
        _lib._LIB_PATH = Path(args.lib).resolve()
    from holocron_b200.nn import _fused as K
    dev = torch.device("cuda", 0)
    res = {"lib": str(_lib.lib_path()), "device": torch.cuda.get_device_name(dev), "rows": []}
    for name, kind, a in shapes():
        launch, flops, (m, n, kk) = build_case(K, kind, a, dev)
        out = launch()
        torch.cuda.synchronize()
        row = {"shape": name, "gemm_mnk": [m, n, kk], "sha1": hashlib.sha1(out.cpu().view(torch.int16).numpy().tobytes()).hexdigest()}
        st = K.get_stats(out)
        if st is not None:
            parts, slots = st
            row["stats_sum"] = parts[:slots].double().sum(0).cpu().flatten().tolist()
        del out
        ms = time_it(launch, args.iters)
        row.update(ms=round(ms, 4), tflops=round(flops / ms / 1e9, 1))
        if not args.no_matmul:
            am = torch.randn(m, kk, device=dev, dtype=torch.bfloat16)
            bm = torch.randn(kk, n, device=dev, dtype=torch.bfloat16)
            mm = time_it(lambda: torch.matmul(am, bm), args.iters)
            row.update(matmul_ms=round(mm, 4), matmul_tflops=round(2.0 * m * n * kk / mm / 1e9, 1))
            del am, bm
        res["rows"].append(row)
        print(f"{name:28s} {ms:8.3f} ms {row['tflops']:7.1f} TFLOP/s"
              + ("" if args.no_matmul else f"   matmul {row['matmul_ms']:7.3f} ms {row['matmul_tflops']:7.1f} TFLOP/s"),
              flush=True)
    if args.out:
        Path(args.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
