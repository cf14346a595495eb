"""Every MMA width of the convolution kernels against the CPU oracle. The Cout tile (fprop, row-window kernel) and the
Cin tile (weight gradient) are template parameters, one kernel instantiation per multiple of 16 up to 128, so each
width is its own code: run all of them through forward, data gradient and weight gradient, for the generic
implicit-GEMM kernels (1x1, 3x3 on a grid narrower than 8 pixels, stride 2) and the row-window kernels (3x3 stride 1).
Tolerances as in test_gpu_conv_bn.py: bf16 outputs rel L2 < 4e-3, fp32 weight gradients rel L2 < 1e-3, and every element
within the per-element bound of tests/_bounds.py."""
import pytest
import torch
import torch.nn.functional as TF

from holocron_b200.nn import _fused as K

from _bounds import FP32_BITS, assert_within, conv_ref, dgrad_ref, wgrad_ref

pytestmark = pytest.mark.gpu

WIDTHS = list(range(16, 129, 16))
KINDS = {
    # name: (H = W, k, stride, pad)
    "1x1": (10, 1, 1, 0),
    "3x3_generic": (7, 3, 1, 1),
    "3x3_rows": (12, 3, 1, 1),
    "3x3_s2": (12, 3, 2, 1),
}


def rel_l2(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-20)).item()


@pytest.mark.parametrize("kind", list(KINDS))
@pytest.mark.parametrize("width", WIDTHS)
def test_conv_every_width_vs_oracle(width, kind):
    hw, k, stride, pad = KINDS[kind]
    torch.manual_seed(width)
    x = torch.randn(2, width, hw, hw).bfloat16()
    wt = (torch.randn(width, width, k, k) / (width * k * k) ** 0.5).bfloat16().float()
    xo = x.float().requires_grad_(True)
    wo = wt.clone().requires_grad_(True)
    yo = TF.conv2d(xo, wo, stride=stride, padding=pad)
    up = torch.randn_like(yo).bfloat16()
    yo.backward(up.float())
    xd = x.cuda().requires_grad_(True)
    wd = wt.cuda().requires_grad_(True)
    y = K.conv2d(xd, wd, None, stride, pad)
    y.backward(up.cuda())
    assert rel_l2(y, yo) < 4e-3
    assert rel_l2(xd.grad, xo.grad) < 4e-3
    assert rel_l2(wd.grad, wo.grad) < 1e-3
    assert_within(y, *conv_ref(x, wt, None, stride, pad), "y")
    assert_within(xd.grad, *dgrad_ref(x.shape, wt, up, stride, pad), "dx")
    assert_within(wd.grad, *wgrad_ref(x, up, k, stride, pad), "dw", bits=FP32_BITS)
