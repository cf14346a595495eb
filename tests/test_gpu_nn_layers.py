"""GPU parity tests for the remaining holocron.nn hot-path layers: FReLU (depth-wise conv + BN + max), NormConv2d,
Add2d, SlimConv2d, DropBlock2d — CUDA path vs golden fixtures from the unmodified reference and vs the oracle.
fp32 layers (NormConv2d/Add2d/DropBlock): rtol 1e-4; bf16 activations (FReLU, SlimConv fast path): rel L2 < 1e-2."""
import pytest
import torch
import torch.nn.functional as TF

import holocron_b200 as hb
from holocron_b200.nn import functional as F
from oracle import functional as OF

from conftest import load_golden

pytestmark = pytest.mark.gpu


def close(a, b, rtol=1e-4, atol=1e-5):
    torch.testing.assert_close(a.detach().cpu().float(), b.detach().cpu().float(), rtol=rtol, atol=atol)


def rel_l2(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-20)).item()


CFGS = (("p1", dict(padding=1)), ("s2p1", dict(stride=2, padding=1)), ("d2p2", dict(dilation=2, padding=2)), ("p0", dict()))


def test_norm_conv2d_and_add2d_vs_golden(monkeypatch):
    g = load_golden("convs")
    x, w, b = g["x"].cuda(), g["w"], g["b"]
    for tag, kw in CFGS:
        # default path: wgmma implicit GEMM with the patch standardisation in the epilogue. Operands are rounded to bf16
        # (2^-9 relative each) and so is the stored output: the bar against the fp32 reference is 1e-2 rel-L2;
        # the weight gradient comes from the fp32 kernel fed with the bf16-path statistics.
        monkeypatch.delenv("HB_NORMCONV_FP32", raising=False)
        wd = w.cuda().requires_grad_(True); bd = b.cuda().requires_grad_(True)
        y = F.norm_conv2d(x, wd, bd, **kw)
        y.sum().backward()
        assert y.dtype == torch.float32 and y.is_contiguous() and y.shape == g[f"normconv_{tag}"].shape
        assert rel_l2(y, g[f"normconv_{tag}"]) < 1e-2, (tag, rel_l2(y, g[f"normconv_{tag}"]))
        assert rel_l2(wd.grad, g[f"normconv_{tag}_gw"]) < 1e-2
        close(bd.grad, g[f"normconv_{tag}_gb"], 1e-4, 1e-4)
        # fp32 CUDA-core kernel behind the switch: fp32-level agreement with the reference
        monkeypatch.setenv("HB_NORMCONV_FP32", "1")
        wd = w.cuda().requires_grad_(True); bd = b.cuda().requires_grad_(True)
        y = F.norm_conv2d(x, wd, bd, **kw)
        y.sum().backward()
        close(y, g[f"normconv_{tag}"], 1e-4, 1e-5)
        close(wd.grad, g[f"normconv_{tag}_gw"], 1e-3, 1e-4)
        close(bd.grad, g[f"normconv_{tag}_gb"], 1e-4, 1e-4)
        monkeypatch.delenv("HB_NORMCONV_FP32", raising=False)
        for ns in (False, True):
            xd = x.clone().requires_grad_(not ns)
            wd = w.cuda().requires_grad_(True); bd = b.cuda().requires_grad_(True)
            y = F.add2d(xd, wd, bd, normalize_slices=ns, **kw)
            y.sum().backward()
            close(y, g[f"add2d_{tag}_n{int(ns)}"], 1e-4, 1e-4)
            close(wd.grad, g[f"add2d_{tag}_n{int(ns)}_gw"], 1e-3, 1e-3)
            close(bd.grad, g[f"add2d_{tag}_n{int(ns)}_gb"], 1e-4, 1e-4)
            if not ns:
                close(xd.grad, g[f"add2d_{tag}_n0_gx"], 1e-4, 1e-4)


@pytest.mark.parametrize("shape", [(4, 64, 56, 56, 64, 3, 1, 1), (2, 24, 33, 29, 40, 3, 2, 1), (2, 16, 20, 20, 32, 5, 1, 2),
                                   (3, 128, 14, 14, 256, 1, 1, 0)])
def test_norm_conv2d_tensor_core_path_vs_fp32_formula(shape):
    """Config-size check of the tensor-core path against the reference formula in fp32 (unfold -> standardise -> matmul),
    with a positive-mean input (image-like): the mean-times-filter-sum term is large, the epilogue algebra must cancel it."""
    n, cin, h, w, cout, k, stride, pad = shape
    torch.manual_seed(0)
    x = torch.rand(n, cin, h, w, device="cuda") + 0.5
    wt = torch.randn(cout, cin, k, k, device="cuda") / (cin * k * k) ** 0.5
    b = torch.randn(cout, device="cuda")
    ref = OF.norm_conv2d(x.cpu(), wt.cpu(), b.cpu(), stride, pad, 1)
    y = F.norm_conv2d(x, wt, b, stride, pad)
    assert rel_l2(y, ref) < 1e-2, rel_l2(y, ref)


def test_conv_modules_like_reference_tests():
    # reference tests/test_nn_conv.py: output shapes + backward, zeros and reflect padding; groups are ignored
    for mod in (hb.nn.NormConv2d(8, 16, 3, padding=1), hb.nn.NormConv2d(8, 16, 3, padding=1, padding_mode="reflect"),
                hb.nn.Add2d(8, 16, 3, padding=1), hb.nn.Add2d(8, 16, 3, padding=1, padding_mode="reflect")):
        mod = mod.cuda()
        out = mod(torch.rand(2, 8, 16, 16, device="cuda"))
        assert out.shape == (2, 16, 16, 16)
        out.sum().backward()
        assert mod.weight.grad is not None and torch.isfinite(mod.weight.grad).all()
    slim = hb.nn.SlimConv2d(8, 3, padding=1, r=32, L=2).cuda()
    out = slim(torch.rand(2, 8, 16, 16, device="cuda"))
    assert out.shape == (2, 6, 16, 16)
    out.sum().backward()
    with pytest.raises(RuntimeError):   # grouped weight: shape error, like the reference's matmul failure (SURVEY §9.3)
        hb.nn.NormConv2d(8, 16, 3, padding=1, groups=2).cuda()(torch.rand(2, 8, 16, 16, device="cuda"))
    with pytest.raises(RuntimeError):   # input gradient through the slice normalisation: undefined in the reference too
        xx = torch.rand(2, 8, 9, 9, device="cuda", requires_grad=True)
        F.norm_conv2d(xx, torch.rand(4, 8, 3, 3, device="cuda")).sum().backward()


def test_norm_conv2d_larger_vs_oracle():
    torch.manual_seed(0)
    x = torch.randn(3, 24, 37, 29)
    w = torch.randn(40, 24, 3, 3) * 0.1
    b = torch.randn(40)
    ref = OF.norm_conv2d(x, w, b, stride=2, padding=1)
    assert rel_l2(F.norm_conv2d(x.cuda(), w.cuda(), b.cuda(), stride=2, padding=1), ref) < 1e-2      # tensor-core path (bf16 operands)
    import os
    os.environ["HB_NORMCONV_FP32"] = "1"
    try:
        close(F.norm_conv2d(x.cuda(), w.cuda(), b.cuda(), stride=2, padding=1), ref, 1e-4, 1e-4)     # fp32 CUDA-core kernel
    finally:
        del os.environ["HB_NORMCONV_FP32"]
    close(F.add2d(x.cuda(), w.cuda(), b.cuda(), padding=1), OF.add2d(x, w, b, padding=1), 1e-4, 1e-3)


def test_slimconv_vs_golden_and_fast_path():
    g = load_golden("convs")
    slim = hb.nn.SlimConv2d(8, 3, padding=1, r=4, L=2)
    slim.load_state_dict(g["slim_state"])
    slim = slim.cuda().eval()
    x = g["x"].cuda().requires_grad_(True)
    y = slim(x)
    y.sum().backward()
    close(y, g["slim_eval"], 1e-3, 1e-4)
    close(x.grad, g["slim_eval_gx"], 1e-3, 1e-4)
    # realistic width: all three convolutions on the tensor-core kernel; compare with the same module run by torch
    torch.manual_seed(1)
    big = hb.nn.SlimConv2d(64, 3, padding=1, r=32, L=2).cuda().eval()
    xb = torch.randn(2, 64, 20, 20, device="cuda")
    y = big(xb)
    assert y.shape == (2, 48, 20, 20)
    half = 32
    z = xb.mean((2, 3), keepdim=True)
    wgt = torch.sigmoid(big.fc2(torch.relu(big.bn(big.fc1(z)))))
    xw = xb * wgt
    top = big.conv_top(xw[:, :half] + xw[:, half:])
    xw = xb * wgt.flip(dims=(1,))
    bot = big.conv_bot2(big.conv_bot1(xw[:, :half] + xw[:, half:]))
    assert rel_l2(y, torch.cat((top, bot), 1)) < 1e-2


def test_frelu_vs_golden():
    g = load_golden("convs")
    fr = hb.nn.FReLU(8)
    fr.load_state_dict(g["frelu_state"])
    fr = fr.cuda().eval()
    x = g["x"].cuda().requires_grad_(True)
    y = fr(x)
    y.float().sum().backward()
    assert rel_l2(y, g["frelu_eval"]) < 6e-3
    assert rel_l2(x.grad, g["frelu_eval_gx"]) < 8e-2
    fr.train()
    x2 = g["x"].cuda().requires_grad_(True)
    y = fr(x2)
    y.float().sum().backward()
    assert rel_l2(y, g["frelu_train"]) < 6e-3
    # the max() gate flips wherever |x - BN(t)| is below the bf16 rounding of t: a handful of the 1440 elements
    assert rel_l2(x2.grad, g["frelu_train_gx"]) < 8e-2
    assert rel_l2(fr.bn.running_mean, g["frelu_train_running_mean"]) < 5e-3
    assert rel_l2(fr.bn.running_var, g["frelu_train_running_var"]) < 5e-3
    assert fr.conv.weight.grad is not None and fr.conv.bias.grad is not None and fr.bn.weight.grad is not None
    assert len(repr(fr).split("\n")) == 4   # reference tests/test_nn_activation.py:44


@pytest.mark.parametrize("stride,c", [(1, 96), (2, 96), (1, 328), (2, 16)])
def test_depthwise_conv_vs_oracle(stride, c):
    from holocron_b200.nn._dwconv import dwconv2d
    torch.manual_seed(2)
    x = torch.randn(2, c, 15, 17).bfloat16()
    w = torch.randn(c, 1, 3, 3) * 0.3
    b = torch.randn(c) * 0.1
    xo = x.float().requires_grad_(True); wo = w.clone().requires_grad_(True); bo = b.clone().requires_grad_(True)
    yo = TF.conv2d(xo, wo, bo, stride=stride, padding=1, groups=c)
    up = torch.randn_like(yo).bfloat16()
    yo.backward(up.float())
    xd = x.cuda().requires_grad_(True); wd = w.cuda().requires_grad_(True); bd = b.cuda().requires_grad_(True)
    y = dwconv2d(xd, wd, bd, stride, 1)
    y.backward(up.cuda())
    assert rel_l2(y, yo) < 4e-3 and rel_l2(xd.grad, xo.grad) < 4e-3
    assert rel_l2(wd.grad, wo.grad) < 1e-3 and rel_l2(bd.grad, bo.grad) < 1e-3


@pytest.mark.parametrize("shape", [(2, 96, 37, 29, 1, 1, False), (2, 40, 16, 16, 2, 1, True), (3, 176, 14, 14, 1, 1, False),
                                   (2, 24, 9, 7, 2, 1, False), (1, 8, 5, 4, 1, 1, True), (2, 32, 8, 8, 1, 0, False),
                                   (2, 16, 6, 3, 1, 1, False)])
def test_depthwise_quad_kernel_edges(shape):
    """Four-outputs-per-thread depth-wise kernel (forward stride 1 / 2, data gradient stride 1 as a flipped correlation): ragged
    widths (W % 4 != 0), padding 0 and 1, widths below one quad (falls back to the one-output kernel), bias."""
    from holocron_b200.nn._dwconv import dwconv2d
    n, c, h, w, stride, pad, bias = shape
    torch.manual_seed(3)
    x = torch.randn(n, c, h, w, device="cuda").bfloat16().contiguous(memory_format=torch.channels_last).requires_grad_(True)
    wt = torch.randn(c, 1, 3, 3, device="cuda", requires_grad=True)
    b = torch.randn(c, device="cuda", requires_grad=True) if bias else None
    y = dwconv2d(x, wt, b, stride, pad)
    xr = x.detach().float().requires_grad_(True)
    wr = wt.detach().clone().requires_grad_(True)
    br = b.detach().clone().requires_grad_(True) if bias else None
    ref = TF.conv2d(xr, wr, br, stride, pad, 1, c)
    g = torch.randn_like(ref).bfloat16()
    y.backward(g)
    ref.backward(g.float())
    assert rel_l2(y, ref) < 4e-3 and rel_l2(x.grad, xr.grad) < 4e-3
    # weight / bias gradients (one filter row x four outputs per thread; per-block partials folded in a fixed order)
    assert rel_l2(wt.grad, wr.grad) < 1e-3
    if bias:
        assert rel_l2(b.grad, br.grad) < 1e-3
    first = wt.grad.clone()
    wt.grad = None
    dwconv2d(x, wt, b, stride, pad).backward(g)
    assert torch.equal(first, wt.grad)          # deterministic: no atomics


@pytest.mark.parametrize("k", [1, 5, 7])
def test_depthwise_other_filter_sizes_weight_gradient(k):
    """k != 3 takes the one-output-per-thread kernels; their weight gradient uses the same per-block partials + ordered fold."""
    from holocron_b200.nn._dwconv import dwconv2d
    torch.manual_seed(k)
    c = 40
    x = torch.randn(3, c, 13, 11, device="cuda").bfloat16().contiguous(memory_format=torch.channels_last).requires_grad_(True)
    wt = torch.randn(c, 1, k, k, device="cuda", requires_grad=True)
    b = torch.randn(c, device="cuda", requires_grad=True)
    y = dwconv2d(x, wt, b, 1, k // 2)
    xr = x.detach().float().requires_grad_(True)
    wr, br = wt.detach().clone().requires_grad_(True), b.detach().clone().requires_grad_(True)
    ref = TF.conv2d(xr, wr, br, 1, k // 2, 1, c)
    g = torch.randn_like(ref).bfloat16()
    y.backward(g)
    ref.backward(g.float())
    assert rel_l2(y, ref) < 4e-3 and rel_l2(x.grad, xr.grad) < 4e-3
    assert rel_l2(wt.grad, wr.grad) < 1e-3 and rel_l2(b.grad, br.grad) < 1e-3


def test_dropblock_vs_golden_and_edge_cases():
    g = load_golden("convs")
    x = g["dropblock_x"].cuda()
    out = F.dropblock2d(x, 0.3, 3, noise=g["dropblock_noise"].cuda())
    close(out, g["dropblock_out"], 1e-5, 1e-6)
    close(out, OF.dropblock2d_with_noise(g["dropblock_x"], g["dropblock_noise"], 0.3, 3), 1e-5, 1e-6)
    # channels_last bf16 input, gradient = mask * scale
    xc = x.bfloat16().contiguous(memory_format=torch.channels_last).requires_grad_(True)
    oc = F.dropblock2d(xc, 0.3, 3, noise=g["dropblock_noise"].cuda())
    assert rel_l2(oc, g["dropblock_out"]) < 6e-3
    oc.float().sum().backward()
    ratio = (g["dropblock_out"] / g["dropblock_x"]).nan_to_num(0.0)
    assert rel_l2(xc.grad, ratio) < 6e-3
    # reference tests/test_nn.py:6-36
    xx = torch.rand(2, 4, 16, 16, device="cuda")
    mod = hb.nn.DropBlock2d(0.0, 1).train()
    assert mod(xx) is xx                                     # p = 0 -> same tensor object
    mod = hb.nn.DropBlock2d(1.0, 1).train()
    assert torch.equal(mod(xx), torch.zeros_like(xx))        # p = 1, block 1 -> everything dropped
    mod = hb.nn.DropBlock2d(0.5, 3, inplace=True).train()
    xi = xx.clone()
    assert mod(xi).data_ptr() == xi.data_ptr()
    assert hb.nn.DropBlock2d(0.5, 3).eval()(xx) is xx
    assert repr(hb.nn.DropBlock2d()) == "DropBlock2d(p=0.1, block_size=7, inplace=False)"


@pytest.mark.parametrize("c,hw,act", [(96, (14, 14), 2), (304, (7, 9), 3), (16, (56, 56), 0), (1280, (7, 7), 1)])
def test_se_gate_activation_and_pooling(c, hw, act):
    """hb_gate_act_{fwd,bwd}_bf16 / hb_gap_fwd_bf16 (SEBlock `x * y` + the block's activation, rexnet.py:63-66, 125-131)
    against torch fp32 on the same bf16-rounded inputs."""
    from holocron_b200.nn import _fused as K
    torch.manual_seed(3)
    n = 3
    x = (torch.randn(n, c, *hw) * 2).bfloat16()
    g = torch.rand(n, c, 1, 1)
    acts = {0: lambda t: t, 1: torch.relu, 2: TF.relu6, 3: TF.silu}
    xo, go = x.float().requires_grad_(True), g.clone().requires_grad_(True)
    yo = acts[act](xo * go)
    up = torch.randn_like(yo).bfloat16()
    yo.backward(up.float())
    xd = x.cuda().contiguous(memory_format=torch.channels_last).requires_grad_(True)
    gd = g.cuda().requires_grad_(True)
    y = K.gate_act(xd, gd, act)
    assert y.dtype == torch.bfloat16 and y.shape == yo.shape
    y.backward(up.cuda())
    assert rel_l2(y, yo) < 4e-3
    assert rel_l2(xd.grad, xo.grad) < 6e-3
    assert rel_l2(gd.grad, go.grad) < 2e-3 and gd.grad.shape == gd.shape
    pooled = K.global_avg_pool_flat(xd.detach())
    assert rel_l2(pooled, x.float().mean((2, 3))) < 4e-3
