"""The per-element bound of tests/_bounds.py is not vacuous, and the whole-tensor relative L2 bar the convolution tests
used alone is blind to local faults.

An emulation of the convolution kernels - fp32 accumulation of the bf16 operands, bias added, rounded to bf16, then the
residual added and rounded again - must pass the bound. Each fault below is one a persistent tile walk or an epilogue can
plausibly make; injected into that emulation, each keeps the relative L2 error under 4e-3 and must break the bound.
The layer is a 7x7 convolution with 64 input channels (K = 3136) over 12 x 97 x 97 output pixels: M = 112908 = 882 tiles
of 128 pixels and a tail of 12, 16 output channels (one Cout tile)."""
import pytest
import torch
import torch.nn.functional as TF

from _bounds import conv_ref, epilogue_ref, excess

N, CIN, HW, COUT, KS = 12, 64, 97, 16, 7
PAD = KS // 2
M = N * HW * HW
TILE = 128


def _nhwc(t):          # NCHW -> [M, C]
    return t.permute(0, 2, 3, 1).reshape(-1, t.shape[1])


@pytest.fixture(scope="module")
def layer():
    torch.manual_seed(0)
    x = torch.randn(N, CIN, HW, HW).bfloat16()
    w = (torch.randn(COUT, CIN, KS, KS) / (CIN * KS * KS) ** 0.5).bfloat16()
    bias = torch.randn(COUT) * 0.1
    res = (torch.randn(N, COUT, HW, HW) * 0.05).bfloat16()
    acc, abs_sum = conv_ref(x, w, bias, 1, PAD)
    acc32 = TF.conv2d(x.float(), w.float(), bias, 1, PAD)           # fp32 accumulation of the bf16 operands
    y = acc32.bfloat16()
    y_res = (y.float() + res.float()).bfloat16()                      # bf16(acc + bias) + residual, rounded again
    ref_res, abs_res, slack = epilogue_ref(acc, abs_sum, res)
    return dict(x=x, w=w, res=res, acc=_nhwc(acc), abs=_nhwc(abs_sum), acc32=_nhwc(acc32), y=_nhwc(y), y_res=_nhwc(y_res),
                ref_res=_nhwc(ref_res), abs_res=_nhwc(abs_res), slack=_nhwc(slack), res_m=_nhwc(res))


def _rel_l2(got, ref):
    return float((got.double() - ref).norm() / ref.norm())


def _tap_contrib(L, ms, r, s, c0, c1):
    """fp32 contribution of filter tap (r, s), input channels [c0, c1), to output pixels ``ms`` ([len(ms), Cout])."""
    xp = TF.pad(L["x"].float(), (PAD, PAD, PAD, PAD)).permute(0, 2, 3, 1)
    n, i, j = ms // (HW * HW), (ms // HW) % HW, ms % HW
    return xp[n, i + r, j + s, c0:c1] @ L["w"].float()[:, c0:c1, r, s].t()


def test_emulation_meets_the_bound(layer):
    L = layer
    assert float(excess(L["y"], L["acc"], L["abs"]).max()) <= 0
    assert float(excess(L["y_res"], L["ref_res"], L["abs_res"], slack=L["slack"]).max()) <= 0


def _check_fault(got, ref, abs_sum, slack=None):
    assert _rel_l2(got, ref) < 4e-3, "the fault should pass the relative L2 bar"
    assert float(excess(got, ref, abs_sum, slack=slack).max()) > 0, "the per-element bound should catch the fault"


def test_wrong_16_byte_chunk(layer):
    L = layer
    y = L["y"].clone()
    m = 40000
    y[m, 8:16] = y[m + 4000, 8:16]              # one 16-byte store of 8 channels taken from another pixel
    _check_fault(y, L["acc"], L["abs"])


def test_tap_dropped_on_one_pixel(layer):
    L = layer
    y = L["y"].clone()
    m = torch.tensor([3 * HW * HW + 50 * HW + 50])
    y[m] = (L["acc32"][m] - _tap_contrib(L, m, PAD, PAD, 0, CIN)).bfloat16()
    _check_fault(y, L["acc"], L["abs"])


def test_k_step_dropped_for_one_tile(layer):
    L = layer
    y = L["y"].clone()
    ms = torch.arange(300 * TILE, 301 * TILE)
    y[ms] = (L["acc32"][ms] - _tap_contrib(L, ms, 2, 4, 16, 32)).bfloat16()   # one 16-channel wgmma k-step skipped
    _check_fault(y, L["acc"], L["abs"])


def test_residual_added_twice_on_one_tile(layer):
    L = layer
    y = L["y_res"].clone()
    ms = torch.arange(100 * TILE, 101 * TILE)
    y[ms] = (y[ms].float() + L["res_m"][ms].float()).bfloat16()
    _check_fault(y, L["ref_res"], L["abs_res"], L["slack"])


def test_m_tail_pixel_from_wrong_row(layer):
    L = layer
    assert M % TILE == 12
    y = L["y"].clone()
    y[M - 1] = y[M - 2]                         # last pixel of the partial tile written from its neighbour's row
    _check_fault(y, L["acc"], L["abs"])
