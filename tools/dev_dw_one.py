"""Dev tool (GPU): the depth-wise kernels on the two largest ReXNet-1.0x shapes (for ncu captures / timing)."""
import sys

import torch

sys.path.insert(0, ".")
from holocron_b200._lib import lib, ptr, stream_ptr

L = lib()
for (N, H, W, C, stride) in [(256, 112, 112, 96, 2), (256, 56, 56, 176, 1)]:
    Ho, Wo = (H + 2 - 3) // stride + 1, (W + 2 - 3) // stride + 1
    x = torch.randn(N, H, W, C, device="cuda").bfloat16()
    dy = torch.randn(N, Ho, Wo, C, device="cuda").bfloat16()
    w = torch.randn(C, 3, 3, device="cuda")
    y = torch.empty(N, Ho, Wo, C, device="cuda", dtype=torch.bfloat16)
    dx = torch.empty_like(x)
    dw = torch.empty(C, 3, 3, device="cuda")
    sums = torch.empty(L.hb_dwconv_wgrad_scratch_doubles(C, 3), device="cuda", dtype=torch.float64)
    for _ in range(2):
        L.hb_dwconv_fwd_bf16(ptr(x), ptr(w), ptr(None), ptr(y), N, H, W, C, 3, stride, 1, stream_ptr())
        L.hb_dwconv_bwd_data_bf16(ptr(dy), ptr(w), ptr(dx), N, H, W, C, 3, stride, 1, stream_ptr())
        L.hb_dwconv_bwd_weight_bf16(ptr(x), ptr(dy), ptr(dw), ptr(None), ptr(sums), N, H, W, C, 3, stride, 1, stream_ptr())
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    ev[0].record()
    L.hb_dwconv_fwd_bf16(ptr(x), ptr(w), ptr(None), ptr(y), N, H, W, C, 3, stride, 1, stream_ptr())
    ev[1].record()
    L.hb_dwconv_bwd_data_bf16(ptr(dy), ptr(w), ptr(dx), N, H, W, C, 3, stride, 1, stream_ptr())
    ev[2].record()
    L.hb_dwconv_bwd_weight_bf16(ptr(x), ptr(dy), ptr(dw), ptr(None), ptr(sums), N, H, W, C, 3, stride, 1, stream_ptr())
    ev[3].record()
    torch.cuda.synchronize()
    gb = (x.numel() + y.numel()) * 2 / 1e9
    print(f"N{N} {H}x{W} C{C} s{stride}: fwd {ev[0].elapsed_time(ev[1]):.3f} ms, bwd_data {ev[1].elapsed_time(ev[2]):.3f} ms, "
          f"bwd_weight {ev[2].elapsed_time(ev[3]):.3f} ms  (x + y = {gb:.2f} GB)", flush=True)
