"""GPU parity tests for the tensor-core convolution kernels (fprop / dgrad / wgrad) and the fused BatchNorm/branch-sum/
activation kernels, through the C ABI, against the CPU oracle (torch fp32 on the same bf16-rounded inputs).

Tolerances: outputs stored in bf16 -> relative L2 error < 4e-3 (bf16 rounding, 2^-9 rms) and max-abs < 2 bf16 ulp of the
largest value; fp32 outputs (weight gradients, BN statistics, dgamma/dbeta) -> rel L2 < 1e-3 (north_star). The convolution
cases also check every element against the per-element bound of tests/_bounds.py."""
import pytest
import torch
import torch.nn.functional as TF

from holocron_b200.nn import _fused as K

from _bounds import FP32_BITS, assert_within, conv_ref, dgrad_ref, wgrad_ref

pytestmark = pytest.mark.gpu


def rel_l2(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-20)).item()


CONV_CASES = [
    # N, H, W, Cin, Cout, k, stride, pad
    (2, 16, 16, 64, 64, 1, 1, 0),
    (2, 14, 14, 48, 48, 3, 1, 1),       # RepVGG-A0 widths: channel count not a multiple of the 64-wide K block
    (3, 14, 14, 192, 192, 3, 1, 1),
    (2, 28, 28, 48, 96, 3, 2, 1),       # stride-2 stage entry
    (2, 28, 28, 48, 96, 1, 2, 0),
    (1, 7, 7, 192, 1280, 3, 2, 1),      # ragged M tile (16 pixels) + 5 N tiles
    (2, 9, 11, 16, 32, 3, 1, 1),        # odd spatial sizes, M tail
    (2, 1, 9, 32, 48, 3, 2, 1),         # stride 2 on a one-pixel side: data gradient by zero insertion, no parity classes
    (2, 32, 32, 3, 48, 3, 2, 1),        # stem: 3 input channels (padded to 8 internally)
    (1, 1, 1, 1280, 1008, 1, 1, 0),     # GEMV-like
]


@pytest.mark.parametrize("case", CONV_CASES)
def test_conv2d_forward_backward_vs_oracle(case):
    n, h, w, cin, cout, k, stride, pad = case
    torch.manual_seed(0)
    x = torch.randn(n, cin, h, w).bfloat16()
    wt = (torch.randn(cout, cin, k, k) / (cin * k * k) ** 0.5).bfloat16().float()  # bf16-representable master weights
    xo = x.float().requires_grad_(True)
    wo = wt.clone().requires_grad_(True)
    yo = TF.conv2d(xo, wo, stride=stride, padding=pad)
    up = torch.randn_like(yo).bfloat16()
    yo.backward(up.float())
    xd = x.cuda().requires_grad_(cin >= 8)
    wd = wt.cuda().requires_grad_(True)
    y = K.conv2d(xd, wd, None, stride, pad)
    assert y.dtype == torch.bfloat16 and y.shape == yo.shape and y.is_contiguous(memory_format=torch.channels_last)
    y.backward(up.cuda())
    assert rel_l2(y, yo) < 4e-3
    assert rel_l2(wd.grad, wo.grad) < 1e-3           # fp32 weight gradient
    if cin >= 8:
        assert rel_l2(xd.grad, xo.grad) < 4e-3
    # per element: fp64 on the same bf16 operands, one ulp of the output type + 1e-5 * sum|terms|
    assert_within(y, *conv_ref(x, wt, None, stride, pad), "y")
    assert_within(wd.grad, *wgrad_ref(x, up, k, stride, pad), "dw", bits=FP32_BITS)
    if cin >= 8:
        assert_within(xd.grad, *dgrad_ref(x.shape, wt, up, stride, pad), "dx")


def test_conv_bias_relu_residual_epilogue():
    torch.manual_seed(1)
    x = torch.randn(2, 32, 12, 12).bfloat16()
    wt = (torch.randn(64, 32, 3, 3) * 0.1).bfloat16().float()
    b = torch.randn(64)
    ref = torch.relu(TF.conv2d(x.float(), wt, b, padding=1))
    with torch.no_grad():
        y = K.conv2d_bias_act(x.cuda(), wt.cuda(), b.cuda(), 1, 1, K.ACT_RELU)
    assert rel_l2(y, ref) < 4e-3
    # with autograd the same function goes conv -> fused activation pass
    xw = wt.cuda().requires_grad_(True)
    y2 = K.conv2d_bias_act(x.cuda(), xw, b.cuda().requires_grad_(True), 1, 1, K.ACT_RELU)
    assert rel_l2(y2, ref) < 6e-3
    y2.float().sum().backward()
    wo = wt.clone().requires_grad_(True)
    torch.relu(TF.conv2d(x.float(), wo, b, padding=1)).sum().backward()
    assert rel_l2(xw.grad, wo.grad) < 1e-2


def test_conv_linearity_at_full_size():
    """Size-independent property at a BASELINE-sized layer (256 x 48 x 112 x 112, RepVGG-A0 stage 0):
    conv(x, a*w1 + b*w2) == a*conv(x, w1) + b*conv(x, w2) up to bf16 rounding, and a sampled comparison with the oracle."""
    torch.manual_seed(2)
    x = torch.randn(256, 48, 112, 112, device="cuda").bfloat16().contiguous(memory_format=torch.channels_last)
    w1 = (torch.randn(48, 48, 3, 3, device="cuda") * 0.05)
    w2 = (torch.randn(48, 48, 3, 3, device="cuda") * 0.05)
    with torch.no_grad():
        y1 = K.conv2d(x, w1, None, 1, 1).float()
        y2 = K.conv2d(x, w2, None, 1, 1).float()
        y12 = K.conv2d(x, 0.5 * w1 + 2 * w2, None, 1, 1).float()
    assert rel_l2(y12, 0.5 * y1 + 2 * y2) < 1e-2
    idx = [0, 100, 255]
    ref = TF.conv2d(x[idx].float().cpu(), w1.bfloat16().float().cpu(), padding=1)
    assert rel_l2(y1[idx], ref) < 4e-3


ACTS = {0: lambda t: t, 1: torch.relu, 2: TF.relu6, 3: TF.silu, 4: lambda t: TF.leaky_relu(t, 0.1), 5: TF.mish,
        6: lambda t: 0.5 * t * (t + 2).clamp(0, 2)}


@pytest.mark.parametrize("cfg", [(1000, 48, 3, 1, False), (777, 1280, 2, 1, False), (2048, 96, 3, 0, True),
                                 (2048, 320, 1, 3, False), (512, 8, 2, 6, False), (3000, 192, 1, 2, True),
                                 (640, 64, 1, 5, False), (640, 32, 1, 4, True)])
def test_bn_act_fused_vs_oracle(cfg):
    m, c, nb, act, has_res = cfg
    torch.manual_seed(3)
    n, h, w = 1, m // 8, 8
    m = n * h * w
    us = [(torch.randn(n, c, h, w) * (1 + b) + 0.5 * b).bfloat16() for b in range(nb)]
    bns = [torch.nn.BatchNorm2d(c) for _ in range(nb)]
    for bn in bns:
        bn.weight.data.uniform_(0.5, 1.5); bn.bias.data.normal_(0, 0.2)
    res = torch.randn(n, c, h, w).bfloat16() if has_res else None
    up = torch.randn(n, c, h, w).bfloat16()
    # oracle
    import copy
    obns = [copy.deepcopy(b) for b in bns]
    uo = [u.float().requires_grad_(True) for u in us]
    ro = res.float().requires_grad_(True) if has_res else None
    z = sum(bn(u) for bn, u in zip(obns, uo))
    if has_res:
        z = z + ro
    yo = ACTS[act](z)
    yo.backward(up.float())
    # cuda
    dbns = [b.cuda() for b in bns]
    ud = [u.cuda().requires_grad_(True) for u in us]
    rd = res.cuda().requires_grad_(True) if has_res else None
    y = K.bn_act(ud, dbns, act, 0.1, rd, training=True)
    y.backward(up.cuda())
    assert rel_l2(y, yo) < 5e-3
    for i in range(nb):
        assert rel_l2(dbns[i].running_mean, obns[i].running_mean) < 1e-3
        assert rel_l2(dbns[i].running_var, obns[i].running_var) < 1e-3
        assert int(dbns[i].num_batches_tracked) == 1
        assert rel_l2(ud[i].grad, uo[i].grad) < 8e-3
        assert rel_l2(dbns[i].weight.grad, obns[i].weight.grad) < 2e-3
        assert rel_l2(dbns[i].bias.grad, obns[i].bias.grad) < 2e-3
    if has_res:
        assert rel_l2(rd.grad, ro.grad) < 5e-3
    # eval mode uses the running statistics
    for b in dbns + obns:
        b.eval()
    with torch.no_grad():
        ye = K.bn_act([u.cuda() for u in us], dbns, act, 0.1, None if res is None else res.cuda())
        zo = sum(bn(u.float()) for bn, u in zip(obns, us))
        if has_res:
            zo = zo + res.float()
        assert rel_l2(ye, ACTS[act](zo)) < 5e-3


def test_global_avg_pool():
    x = torch.randn(4, 1280, 7, 7).bfloat16()
    xd = x.cuda().contiguous(memory_format=torch.channels_last).requires_grad_(True)
    y = K.global_avg_pool_flat(xd)
    ref = x.float().mean((2, 3))
    assert rel_l2(y, ref) < 4e-3
    y.float().sum().backward()
    assert torch.allclose(xd.grad.float().cpu(), torch.full_like(x.float(), 1 / 49), rtol=1e-2)


@pytest.mark.parametrize("stride,cout,bias", [(2, 32, False), (1, 32, True), (2, 64, False)])
def test_stem_convolution_im2col_path_vs_torch_and_generic_path(stride, cout, bias, monkeypatch):
    """3-channel 3x3 / pad-1 stems (ReXNet, Darknet, YOLOv4, UNet3+) run as one im2col pass + a dense 1x1 GEMM: output, weight and
    bias gradients against torch's fp32 convolution on the bf16-rounded operands, and against the implicit-GEMM path."""
    from holocron_b200.nn import _fused as K
    torch.manual_seed(0)
    x = torch.randn(4, 3, 33, 29, device="cuda")
    w = (torch.randn(cout, 3, 3, 3, device="cuda") / 27 ** 0.5).requires_grad_(True)
    b = torch.randn(cout, device="cuda").requires_grad_(True) if bias else None
    up = torch.randn(4, cout, (33 + 2 - 3) // stride + 1, (29 + 2 - 3) // stride + 1, device="cuda")

    def run():
        for t in (w, b):
            if t is not None:
                t.grad = None
        y = K.conv2d(x, w, b, stride, 1)
        (y.float() * up).sum().backward()
        return y.detach().float(), w.grad.clone(), None if b is None else b.grad.clone()

    y1, gw1, gb1 = run()
    monkeypatch.setenv("HB_DISABLE_STEM_IM2COL", "1")
    y0, gw0, gb0 = run()
    xr, wr = x.bfloat16().float(), w.detach().bfloat16().float().requires_grad_(True)
    br = None if b is None else b.detach().clone().requires_grad_(True)
    ref = TF.conv2d(xr, wr, br, stride, 1)
    (ref * up.bfloat16().float()).sum().backward()
    assert rel_l2(y1, ref) < 4e-3 and rel_l2(y0, ref) < 4e-3
    assert rel_l2(gw1, wr.grad) < 4e-3 and rel_l2(gw0, wr.grad) < 4e-3
    if bias:
        assert rel_l2(gb1, br.grad) < 4e-3
