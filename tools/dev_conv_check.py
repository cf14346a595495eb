"""Dev harness (GPU): checks the wgmma conv kernels against torch's conv2d on the same bf16 inputs."""
import ctypes
import sys
import time

import torch
import torch.nn.functional as F

sys.path.insert(0, ".")
from holocron_b200._lib import lib, ptr, stream_ptr


def run_fprop(N, H, W, Cin, Cout, k, stride, pad, bias=False, act=0, residual=False, seed=0, ctas=0):
    torch.manual_seed(seed)
    dev = "cuda"
    x = torch.randn(N, Cin, H, W, device=dev).to(torch.bfloat16)
    w = (torch.randn(Cout, Cin, k, k, device=dev) / (Cin * k * k) ** 0.5).to(torch.bfloat16)
    b = torch.randn(Cout, device=dev) if bias else None
    x_nhwc = x.permute(0, 2, 3, 1).contiguous()
    w_krsc = w.permute(0, 2, 3, 1).contiguous()
    Ho = (H + 2 * pad - (k - 1) - 1) // stride + 1
    Wo = (W + 2 * pad - (k - 1) - 1) // stride + 1
    res = torch.randn(N, Ho, Wo, Cout, device=dev).to(torch.bfloat16) if residual else None
    y = torch.full((N, Ho, Wo, Cout), float("nan"), device=dev, dtype=torch.bfloat16)
    rc = lib().hb_conv2d_fprop_bf16(ptr(x_nhwc), ptr(w_krsc), ptr(y), ptr(b), ptr(res), N, H, W, Cin, Cout, k, k,
                                    stride, pad, 1, act, ctas, stream_ptr())
    torch.cuda.synchronize()
    ref = F.conv2d(x.float(), w.float(), b, stride=stride, padding=pad)
    ref = ref.permute(0, 2, 3, 1)
    if residual:
        ref = ref + res.float()
    if act == 1:
        ref = ref.relu()
    err = (y.float() - ref).abs()
    denom = ref.abs().max().item() + 1e-6
    nan = torch.isnan(y.float()).sum().item()
    rel = err.max().item() / denom
    tag = "OK " if (rc == 0 and nan == 0 and rel < 1e-2) else "BAD"
    print(f"{tag} fprop N{N} {H}x{W} C{Cin}->{Cout} k{k} s{stride} p{pad} bias={bias} act={act} res={residual}: rc={rc} "
          f"nan={nan} max_abs_err={err.max().item():.4g} rel_to_max={rel:.3g}", flush=True)
    if tag == "BAD" and nan == 0:
        # locate the error pattern
        bad = (err > 1e-2 * denom).nonzero()
        print("   first bad idx:", bad[:5].tolist(), "count", bad.shape[0], "of", err.numel())
    return tag == "OK "


def main():
    print(torch.cuda.get_device_name(0))
    ok = True
    # plain GEMM mode (1x1 s1 p0)
    ok &= run_fprop(1, 16, 8, 64, 64, 1, 1, 0)
    ok &= run_fprop(2, 16, 16, 64, 128, 1, 1, 0)
    ok &= run_fprop(2, 16, 16, 128, 64, 1, 1, 0)
    ok &= run_fprop(2, 14, 14, 192, 192, 1, 1, 0)
    ok &= run_fprop(2, 14, 14, 48, 48, 1, 1, 0)
    ok &= run_fprop(2, 7, 7, 256, 1280, 1, 1, 0)
    # im2col mode
    ok &= run_fprop(1, 16, 8, 64, 64, 3, 1, 1)
    ok &= run_fprop(2, 16, 16, 64, 64, 3, 1, 1)
    ok &= run_fprop(2, 14, 14, 48, 48, 3, 1, 1)
    ok &= run_fprop(3, 14, 14, 192, 192, 3, 1, 1)
    ok &= run_fprop(2, 28, 28, 96, 96, 3, 1, 1, bias=True, act=1)
    ok &= run_fprop(2, 28, 28, 96, 96, 3, 1, 1, residual=True, act=1)
    ok &= run_fprop(2, 28, 28, 48, 96, 3, 2, 1)
    ok &= run_fprop(2, 28, 28, 48, 96, 1, 2, 0)
    ok &= run_fprop(2, 7, 7, 192, 1280, 3, 1, 1)
    ok &= run_fprop(2, 56, 56, 8, 48, 3, 2, 1)
    ok &= run_fprop(4, 112, 112, 48, 48, 3, 1, 1)
    ok &= run_fprop(64, 14, 14, 1280, 1280, 3, 1, 1, ctas=0)
    print("ALL OK" if ok else "SOME BAD")
    # quick timing of a mid layer
    N, H, W, C = 256, 14, 14, 192
    x = torch.randn(N, H, W, C, device="cuda").to(torch.bfloat16)
    w = torch.randn(C, 3, 3, C, device="cuda").to(torch.bfloat16)
    y = torch.empty(N, H, W, C, device="cuda", dtype=torch.bfloat16)
    for shape in [(256, 14, 14, 192, 192), (256, 28, 28, 96, 96), (256, 56, 56, 48, 48), (256, 112, 112, 48, 48),
                  (256, 7, 7, 1280, 1280)]:
        N, H, W, Ci, Co = shape
        x = torch.randn(N, H, W, Ci, device="cuda").to(torch.bfloat16)
        w = torch.randn(Co, 3, 3, Ci, device="cuda").to(torch.bfloat16)
        y = torch.empty(N, H, W, Co, device="cuda", dtype=torch.bfloat16)
        args = (ptr(x), ptr(w), ptr(y), ptr(None), ptr(None), N, H, W, Ci, Co, 3, 3, 1, 1, 1, 0, 0, stream_ptr())
        for _ in range(3):
            lib().hb_conv2d_fprop_bf16(*args)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(10):
            lib().hb_conv2d_fprop_bf16(*args)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 10
        flops = 2 * N * H * W * Co * Ci * 9
        byts = (N * H * W * (Ci + Co) + Co * Ci * 9) * 2
        xc = x.permute(0, 3, 1, 2)  # channels_last view
        wc = w.permute(0, 3, 1, 2)
        for _ in range(3):
            F.conv2d(xc, wc, padding=1)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(10):
            F.conv2d(xc, wc, padding=1)
        e1.record()
        torch.cuda.synchronize()
        ms_t = e0.elapsed_time(e1) / 10
        print(f"time {shape}: ours {ms:.3f} ms  {flops/ms/1e9:.1f} TFLOP/s  {byts/ms/1e6:.1f} GB/s | cudnn {ms_t:.3f} ms")


if __name__ == "__main__":
    main()
