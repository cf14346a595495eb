"""The 144..256-column Cout tiles of the generic implicit-GEMM kernel (conv_fprop.cu) against the CPU oracle.

A Cout tile wider than 128 columns is only chosen for filters with more than one tap and while the layer still has at
least one tile per SM, so these shapes are sized for it (2 x 92 x 92 output pixels = 133 pixel tiles; 28 pixel tiles x
5 Cout tiles for Cout = 1280), next to 1x1 and small shapes that must keep the narrow tiles (Cout 192 / 256 split in
two). Covered: 1x1, 3x3 and stride-2 forward, the stride-1 data gradient with a K extension and an epilogue residual,
and the parity-class stride-2 data gradient. A launch with output-column statistics keeps the narrow tiles (so the
partial sums are grouped as before); its output must equal, bit for bit, the same convolution on the wide tiles, and
its partials must match sums over that output and repeat bit for bit. Besides the relative L2 bar, every element must lie
within the per-element bound of tests/_bounds.py."""
import pytest
import torch
import torch.nn.functional as TF

from holocron_b200.nn import _fused as K

from _bounds import assert_within, conv_ref, dgrad_ref, epilogue_ref, ulp

pytestmark = pytest.mark.gpu


def rel_l2(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-20)).item()


def bf16(*shape, scale=1.0):
    return (torch.randn(*shape) * scale).bfloat16()


def cl(t):
    return t.cuda().contiguous(memory_format=torch.channels_last)


FWD = {
    # name: (N, H, Cin, Cout, k, stride)
    "1x1_192": (2, 92, 192, 192, 1, 1),
    "1x1_256": (2, 92, 64, 256, 1, 1),
    "3x3_192": (2, 92, 192, 192, 3, 1),
    "3x3_160": (2, 92, 48, 160, 3, 1),
    "3x3_s2_192": (2, 184, 96, 192, 3, 2),
    "3x3_s2_256": (2, 184, 64, 256, 3, 2),
    "3x3_1280": (2, 42, 64, 1280, 3, 1),      # 5 Cout tiles of 256
    "3x3_1152": (2, 42, 64, 1152, 3, 1),      # 6 Cout tiles of 192
    "1x1_192_one_tile": (1, 8, 192, 192, 1, 1),   # a single pixel tile: keeps the narrow tiles
    "3x3_256_small": (2, 7, 64, 256, 3, 1),
}


@pytest.mark.parametrize("name", list(FWD))
def test_fprop_wide_tiles_vs_oracle(name):
    n, h, cin, cout, k, stride = FWD[name]
    torch.manual_seed(cout + h)
    x = bf16(n, cin, h, h)
    w = bf16(cout, cin, k, k, scale=(cin * k * k) ** -0.5)
    bias = torch.randn(cout)
    ref = TF.conv2d(x.float(), w.float(), bias, stride=stride, padding=k // 2)
    wf = w.permute(0, 2, 3, 1).contiguous().cuda()
    y = K.conv2d_forward_raw(cl(x), wf, cout, k, k, stride, k // 2, 1, bias.cuda())
    assert rel_l2(y, ref) < 4e-3
    assert_within(y, *conv_ref(x, w, bias, stride, k // 2), name)


@pytest.mark.parametrize("cd", [192, 256])
def test_dgrad_kext_residual_wide_tiles(cd):
    # dX = dgrad3x3(dY3) + dgrad1x1(dY1) + dXid in one launch, as the stride-1 RepVGG block's backward issues it
    torch.manual_seed(cd)
    n, h, c = 2, 92, 64
    dy3, dy1, dxid = bf16(n, c, h, h), bf16(n, c, h, h), bf16(n, cd, h, h)
    wd3 = bf16(cd, c, 3, 3, scale=(9 * c) ** -0.5)
    wd1 = bf16(cd, c, 1, 1, scale=c ** -0.5)
    ref = TF.conv2d(dy3.float(), wd3.float(), padding=1) + TF.conv2d(dy1.float(), wd1.float()) + dxid.float()
    y = K.conv2d_forward_raw(cl(dy3), wd3.permute(0, 2, 3, 1).contiguous().cuda(), cd, 3, 3, 1, 1, 1, None, cl(dxid),
                             K.ACT_NONE, xe=cl(dy1), we=wd1.permute(0, 2, 3, 1).contiguous().cuda(), kind="dgrad")
    assert rel_l2(y, ref) < 4e-3
    r3, a3 = conv_ref(dy3, wd3, None, 1, 1)
    r1, a1 = conv_ref(dy1, wd1)
    ref, a, slack = epilogue_ref(r3 + r1, a3 + a1, dxid)             # residual added to the bf16-rounded sum
    assert_within(y, ref, a, "dX", slack=slack)


@pytest.mark.parametrize("h", [184, 183, 12])
def test_dgrad_s2_parity_classes_cd192(h):
    # parity-class data gradient of a stride-2 3x3 conv (+ its 1x1 stride-2 branch), Cd = 192: the two-tap classes
    # (0, 1) and (1, 0) of the 184 grid have 133 pixel tiles (wide tile); the 183 and 12 grids keep the narrow tiles
    torch.manual_seed(h)
    n, c, cd = 2, 64, 192
    ho = (h - 1) // 2 + 1
    w3 = (torch.randn(c, cd, 3, 3) * (9 * cd) ** -0.5)
    w3 = w3.bfloat16().float()
    w1 = bf16(c, cd, 1, 1, scale=cd ** -0.5)
    dy3, dy1 = bf16(n, c, ho, ho), bf16(n, c, ho, ho)
    op = h - ((ho - 1) * 2 - 2 + 3)
    ref = TF.conv_transpose2d(dy3.float(), w3, stride=2, padding=1, output_padding=op)
    ref = ref + TF.conv_transpose2d(dy1.float(), w1.float(), stride=2, output_padding=h - ((ho - 1) * 2 + 1))
    wd1 = w1.permute(1, 2, 3, 0).contiguous().cuda()   # [Cd, 1, 1, C]
    dx = K.dgrad_s2_raw(cl(dy3), torch.nn.Parameter(w3.cuda()), cd, h, h, cl(dy1), wd1)
    assert rel_l2(dx, ref) < 4e-3
    # the 1x1 branch is stored (bf16) first; class (0, 0) of the 3x3 part is rounded to bf16 and added onto it
    r3, a3 = dgrad_ref((n, cd, h, h), w3, dy3, 2, 1)
    r1, a1 = dgrad_ref((n, cd, h, h), w1, dy1, 2, 0)
    slack = torch.zeros_like(r3)
    slack[:, :, ::2, ::2] = 0.5 * (ulp(r3) + ulp(r1))[:, :, ::2, ::2]
    assert_within(dx, r3 + r1, a3 + a1, "dX", slack=slack)


@pytest.mark.parametrize("shape", [(2, 92, 192, 192), (2, 42, 128, 1280), (1, 8, 128, 256)])
def test_stats_launch_matches_wide_tiles(shape):
    n, h, cin, cout = shape
    torch.manual_seed(cout)
    x = cl(bf16(n, cin, h, h))
    wf = bf16(cout, 3, 3, cin, scale=(9 * cin) ** -0.5).cuda()
    y1 = K.conv2d_forward_raw(x, wf, cout, 3, 3, 1, 1, 1, want_stats=True)
    parts1, slots1 = K.get_stats(y1)
    p1 = parts1[:slots1].clone()
    y2 = K.conv2d_forward_raw(x, wf, cout, 3, 3, 1, 1, 1, want_stats=True)
    parts2, slots2 = K.get_stats(y2)
    assert slots1 == slots2
    assert torch.equal(y1, y2)
    assert torch.equal(p1, parts2[:slots2])
    # same accumulation order per output element whatever the Cout tile: the plain launch (wide tiles where the layer
    # allows them) gives the statistics launch's output bit for bit
    assert torch.equal(K.conv2d_forward_raw(x, wf, cout, 3, 3, 1, 1, 1), y1)
    assert_within(y1, *conv_ref(x, wf.permute(0, 3, 1, 2), None, 1, 1), "y")
    yf = y1.double().permute(0, 2, 3, 1).reshape(-1, cout)
    tot = p1.double().sum(0)
    torch.testing.assert_close(tot[:, 0], yf.sum(0), rtol=1e-4, atol=1e-2)
    torch.testing.assert_close(tot[:, 1], (yf * yf).sum(0), rtol=1e-4, atol=1e-2)
