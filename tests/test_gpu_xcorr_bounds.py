"""The NormConv2d / Add2d kernels (csrc/xcorr.cu, csrc/patch_stats.cu, the norm epilogue of csrc/conv_fprop.cu) per
element against fp64, on every path of tests/_xcorr_cases.py.

Every kernel runs through its C entry point with its outputs (out, mean / rstd, dw, dx, y) pre-filled with NaN, so an
element left unwritten fails; dw is zeroed by its launcher, so that check covers the launcher's memset. Each bound is the
sum of the error sources of the kernel it checks (see ``tests/_bounds.py`` for the idiom); the fp64 oracles run on the
device. u = 2^-24 is the fp32 unit roundoff.

* fp32 patch statistics (warp-strided sums, chain length d = ceil(K / 32) + 5): |dmean| <= (d + 1) u mean|p|;
  rstd relative <= ((d + 3) u var + dmean^2) / (2 (var + eps)) + 3 u (two-pass, so no cancellation beyond dmean^2).
* bf16 patch statistics (per-pixel fp32 sums over Cp padded channels, then fp64): |dmean| <= (Cp + 2) u mean|p|;
  rstd relative <= 1.5 (Cp + 1) u E[p^2] / (var + eps) + 2 u: E[x^2] - mean^2 cancels by the factor E[p^2] / var.
* fp32 forward: one fp32 ulp + (K + 3) u sum|p^||w| (norm_conv; |p - w| for add2d, where nothing cancels) + the
  statistics error carried through: drstd |ref - bias| + rstd dmean sum|w| (norm_conv), drstd sum|p^| + K rstd dmean
  (normalised add2d).
* tensor-core NormConv2d (bf16 operands, bf16 output): one bf16 ulp + 1e-5 rstd (sum|p||w| + |mean| sum|w|) +
  (drstd + u) |ref - bias| + rstd dmean sum|w|. The |mean| sum|w| term is the cancellation the epilogue fold
  rstd (acc - mean wsum) has to survive; the inputs have a positive mean so that it is large.
* weight gradient, fed the statistics its forward saved: (chain + 2) u sum|g h|, chain = one thread's rows plus one
  atomicAdd per split (tests/_xcorr_cases.py); the normalised adder adds 2 |g| for every term whose fp64 |p^ - w| lies
  within the fp32 rounding of p^ (2.5 u |p^|): the sign of such a term may flip.
* Add2d data gradient: (KH KW Cout + 1) u sum|g|; pixels no window reads are exactly 0.

The weight gradient is summed with atomics, so it is not bit-reproducible and nothing here asserts that it is."""
import ctypes

import pytest
import torch
import torch.nn.functional as TF

import holocron_b200 as hb
from holocron_b200._lib import ConvArgs, lib, ptr, stream_ptr
from holocron_b200.nn import functional as F
from oracle import functional as OF

import _xcorr_cases as D
from _bounds import BF16_BITS, FP32_BITS, assert_within

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24
EPS = 1e-14
NAN = float("nan")


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _gen(name):
    g = torch.Generator(device=DEV)
    g.manual_seed(sum(map(ord, name)))
    return g


def nan(*shape, dtype=torch.float32):
    return torch.full(shape, NAN, device=DEV, dtype=dtype)


def patches(x, cs):
    """fp64 [N, L, K] windows of x (channel-major inside a window, zero padding included: the order of F.unfold)."""
    return TF.unfold(x.double(), (cs.kh, cs.kw), dilation=cs.dil, padding=cs.pad, stride=cs.stride).transpose(1, 2)


def stats_ref(p):
    """fp64 two-pass (mean, var, rstd) of each window, [N, L]."""
    mu = p.mean(-1)
    var = ((p - mu[..., None]) ** 2).mean(-1)
    return mu, var, 1.0 / torch.sqrt(var + EPS)


def fp32_stats_bounds(p, cs):
    """(dmean, relative drstd) of patch_stats_kernel in xcorr.cu, per window."""
    mu, var, _ = stats_ref(p)
    d = -(-cs.k // 32) + 5
    dmu = (d + 1) * U * p.abs().mean(-1)
    return dmu, ((d + 3) * U * var + dmu ** 2) / (2 * (var + EPS)) + 3 * U


def bf16_stats_bounds(p, cin_p):
    """(dmean, relative drstd) of hb_patch_stats_bf16 on the bf16-rounded input, per window."""
    mu, var, _ = stats_ref(p)
    return (cin_p + 2) * U * p.abs().mean(-1), 1.5 * (cin_p + 1) * U * (p * p).mean(-1) / (var + EPS) + 2 * U


def check_stats(mean, rstd, p, dmu, drel, what):
    mu, _, r = stats_ref(p)
    assert_within(mean.view_as(mu), mu, torch.zeros_like(mu), f"{what} mean", rel=0, bits=FP32_BITS, slack=dmu)
    assert_within(rstd.view_as(r), r, torch.zeros_like(r), f"{what} rstd", rel=0, bits=FP32_BITS, slack=drel * r)


def sign_sum(gm, a, b, absolute=False, tie=None):
    """sum_m gm[m, co] * sign(a[m, k] - b[co, k]) -> [Cout, K] (or, ``absolute``, the same with |gm| and |sign|; ``tie``:
    the sum of |gm| over the terms with |a - b| <= tie[m, k]), in row chunks that keep [rows, Cout, K] small."""
    m, co, k = gm.shape[0], b.shape[0], b.shape[1]
    out = torch.zeros(co, k, device=a.device, dtype=torch.float64)
    step = max(1, (1 << 24) // (co * k))
    for i in range(0, m, step):
        diff = a[i:i + step, None, :] - b[None]
        g = gm[i:i + step, :, None]
        if tie is not None:
            out += (g.abs() * (diff.abs() <= tie[i:i + step, None, :])).sum(0)
        elif absolute:
            out += (g.abs() * diff.sign().abs()).sum(0)
        else:
            out += (g * diff.sign()).sum(0)
    return out


def dgrad_terms(gm, a, b):
    """-sum_co gm[m, co] * sign(a[m, k] - b[co, k]) and sum_co |gm[m, co] sign| -> two [M, K]."""
    m, k = a.shape
    val = torch.empty(m, k, device=a.device, dtype=torch.float64)
    mag = torch.empty_like(val)
    step = max(1, (1 << 24) // (b.shape[0] * k))
    for i in range(0, m, step):
        s = (a[i:i + step, None, :] - b[None]).sign()
        g = gm[i:i + step, :, None]
        val[i:i + step] = -(g * s).sum(1)
        mag[i:i + step] = (g.abs() * s.abs()).sum(1)
    return val, mag


# ---------------------------------------------------------------------------------------------------------------------
# raw launches of the fp32 kernels
# ---------------------------------------------------------------------------------------------------------------------
def xc_fwd(x, w, b, cs, mode, normalize):
    out = nan(cs.n, cs.cout, cs.ho, cs.wo)
    mean, rstd = (nan(cs.m), nan(cs.m)) if normalize else (None, None)
    rc = lib().hb_xcorr2d_fwd(ptr(x), ptr(w), ptr(b), ptr(out), ptr(mean), ptr(rstd), cs.n, cs.cin, cs.h, cs.w, cs.cout,
                              cs.kh, cs.kw, cs.stride, cs.pad, cs.dil, mode, int(normalize), ctypes.c_float(EPS),
                              stream_ptr())
    assert rc == 0, f"hb_xcorr2d_fwd returned {rc}"
    torch.cuda.synchronize()
    return out, mean, rstd


def xc_wgrad(x, w, g, mean, rstd, cs, mode, normalize):
    dw = nan(cs.cout, cs.cin, cs.kh, cs.kw)
    rc = lib().hb_xcorr2d_wgrad(ptr(x), ptr(w), ptr(g), ptr(mean), ptr(rstd), ptr(dw), cs.n, cs.cin, cs.h, cs.w, cs.cout,
                                cs.kh, cs.kw, cs.stride, cs.pad, cs.dil, mode, int(normalize), ctypes.c_float(EPS),
                                stream_ptr())
    assert rc == 0, f"hb_xcorr2d_wgrad returned {rc}"
    torch.cuda.synchronize()
    return dw


def add_dgrad(x, w, g, cs):
    dx = nan(cs.n, cs.cin, cs.h, cs.w)
    rc = lib().hb_add2d_dgrad(ptr(x), ptr(w), ptr(g), ptr(dx), cs.n, cs.cin, cs.h, cs.w, cs.cout, cs.kh, cs.kw, cs.stride,
                              cs.pad, cs.dil, stream_ptr())
    assert rc == 0, f"hb_add2d_dgrad returned {rc}"
    torch.cuda.synchronize()
    return dx


# ---------------------------------------------------------------------------------------------------------------------
# fp64 forward references with their bounds: (ref [N, Cout, L], bound without the ulp [N, Cout, L])
# ---------------------------------------------------------------------------------------------------------------------
def _ncl(t):
    return t.transpose(1, 2)


def fwd_ref(p, w, b, cs, mode, normalize, stat_bounds=None):
    w64 = w.double().reshape(cs.cout, -1)
    b64 = torch.zeros(cs.cout, device=DEV, dtype=torch.float64) if b is None else b.double()
    rel = (cs.k + 3) * U
    if not normalize:
        ph = p
    else:
        mu, _, r = stats_ref(p)
        ph = (p - mu[..., None]) * r[..., None]
        dmu, drel = stat_bounds(p)
    if mode == 0:
        core = ph @ w64.t()
        bound = rel * (ph.abs() @ w64.abs().t())
        if normalize:
            bound = bound + drel[..., None] * core.abs() + (r * dmu)[..., None] * w64.abs().sum(1)
    else:
        dist = torch.cdist(ph, w64.expand(cs.n, -1, -1), p=1)
        core = -dist
        bound = rel * dist
        if normalize:
            s = ph.abs().sum(-1)
            bound = bound + ((drel + 2 * U) * s + cs.k * r * dmu)[..., None]
    return _ncl(core + b64), _ncl(bound)


def assert_fwd(out, ref, bound, what, bits=FP32_BITS):
    assert_within(out.reshape(ref.shape), ref, torch.zeros_like(ref), what, rel=0, bits=bits, slack=bound)


# ---------------------------------------------------------------------------------------------------------------------
# 1. the fp32 kernels, every case, both modes, with and without normalisation
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(D.CASES))
def test_fp32_kernels_per_element(name):
    cs = D.CASES[name]
    sms = _sms()
    what = D.describe(name, sms)
    print(what)
    gen = _gen(name)
    x = torch.randn(cs.n, cs.cin, cs.h, cs.w, device=DEV, generator=gen) + 0.5
    w = torch.randn(cs.cout, cs.cin, cs.kh, cs.kw, device=DEV, generator=gen) * cs.k ** -0.5
    b = torch.randn(cs.cout, device=DEV, generator=gen)
    g = torch.randn(cs.n, cs.cout, cs.ho, cs.wo, device=DEV, generator=gen)
    p = patches(x, cs)
    w64 = w.double().reshape(cs.cout, -1)
    gm = g.double().reshape(cs.n, cs.cout, -1).transpose(1, 2).reshape(-1, cs.cout)       # [M, Cout]
    chain = D.wgrad_geo(cs, sms).chain
    for mode in (0, 1):
        for normalize in (False, True):
            tag = f"{name} mode={mode} normalize={normalize}"
            for bias in (b, None):
                out, mean, rstd = xc_fwd(x, w, bias, cs, mode, normalize)
                ref, bound = fwd_ref(p, w, bias, cs, mode, normalize, lambda q: fp32_stats_bounds(q, cs))
                assert_fwd(out, ref, bound, f"{tag} bias={bias is not None} out [{what}]")
            if normalize:
                check_stats(mean, rstd, p, *fp32_stats_bounds(p, cs), f"{tag} patch_stats_kernel")
                h = (p - mean.double().view(cs.n, -1, 1)) * rstd.double().view(cs.n, -1, 1)
            else:
                h = p
            h = h.reshape(-1, cs.k)                                                          # [M, K]
            dw = xc_wgrad(x, w, g, mean, rstd, cs, mode, normalize)
            rel = (chain + 2) * U
            if mode == 0:
                ref, abs_sum, slack = gm.t() @ h, gm.abs().t() @ h.abs(), None
            else:
                ref, abs_sum = sign_sum(gm, h, w64), sign_sum(gm, h, w64, absolute=True)
                slack = None
                if normalize:
                    ties = sign_sum(gm, h, w64, tie=2.5 * U * h.abs())
                    abs_sum, slack = abs_sum + ties, 2 * ties
            assert_within(dw.reshape(ref.shape), ref, abs_sum, f"{tag} dw [{what}]", rel=rel, bits=FP32_BITS,
                          slack=slack)
    # Add2d data gradient: -sum g sign(x - w) over the windows that read each pixel
    dx = add_dgrad(x, w, g, cs)
    val, mag = dgrad_terms(gm, p.reshape(-1, cs.k), w64)
    fold = dict(output_size=(cs.h, cs.w), kernel_size=(cs.kh, cs.kw), dilation=cs.dil, padding=cs.pad, stride=cs.stride)
    ref = TF.fold(val.view(cs.n, -1, cs.k).transpose(1, 2), **fold)
    abs_sum = TF.fold(mag.view(cs.n, -1, cs.k).transpose(1, 2), **fold)
    assert_within(dx, ref, abs_sum, f"{name} dx [{what}]", rel=(cs.kh * cs.kw * cs.cout + 1) * U, bits=FP32_BITS)
    rows, cols = D.dgrad_uncovered(cs)
    assert bool((dx[:, :, rows, :] == 0).all()) and bool((dx[:, :, :, cols] == 0).all()), \
        f"{name}: an input pixel no window reads has a non-zero gradient"


# ---------------------------------------------------------------------------------------------------------------------
# 2. tensor-core NormConv2d: hb_patch_stats_bf16 + hb_conv2d_fused_bf16 with the norm epilogue
# ---------------------------------------------------------------------------------------------------------------------
def tc_inputs(name, cs):
    gen = _gen(name)
    x = torch.rand(cs.n, cs.cin, cs.h, cs.w, device=DEV, generator=gen) + 0.5      # image-like: positive patch means
    w = torch.randn(cs.cout, cs.cin, cs.kh, cs.kw, device=DEV, generator=gen) * cs.k ** -0.5
    b = torch.randn(cs.cout, device=DEV, generator=gen)
    return x, w, b


def tc_pack(x, w, b, t):
    """(x NHWC bf16 with Cin_p channels, w [Cout_p, kh, kw, Cin_p] bf16, bias [Cout_p] fp32), zero-padded."""
    n, cin, h, wd = x.shape
    cout = w.shape[0]
    xb = torch.zeros(n, h, wd, t.cin_p, device=DEV, dtype=torch.bfloat16)
    xb[..., :cin] = x.permute(0, 2, 3, 1).bfloat16()
    wf = torch.zeros(t.cout_p, w.shape[2], w.shape[3], t.cin_p, device=DEV, dtype=torch.bfloat16)
    wf[:cout, ..., :cin] = w.permute(0, 2, 3, 1).bfloat16()
    bp = torch.zeros(t.cout_p, device=DEV)
    bp[:cout] = b
    return xb, wf, bp


def tc_stats(xb, cs):
    mean, rstd = nan(cs.m), nan(cs.m)
    scratch = nan(2 * cs.n * cs.h * cs.w)
    rc = lib().hb_patch_stats_bf16(ptr(xb), ptr(mean), ptr(rstd), ptr(scratch), cs.n, cs.h, cs.w, xb.shape[-1], cs.kh,
                                   cs.kw, cs.stride, cs.pad, cs.dil, cs.k, ctypes.c_float(EPS), stream_ptr())
    assert rc == 0, f"hb_patch_stats_bf16 returned {rc}"
    torch.cuda.synchronize()
    return mean, rstd


def tc_conv(xb, wf, bp, mean, rstd, wsum, cs, num_ctas=0):
    cout_p = wf.shape[0]
    y = nan(cs.n, cs.ho, cs.wo, cout_p, dtype=torch.bfloat16)
    a = ConvArgs()
    a.x, a.w, a.y, a.bias = xb.data_ptr(), wf.data_ptr(), y.data_ptr(), bp.data_ptr()
    a.N, a.H, a.W, a.Cin, a.Cout, a.R, a.S = cs.n, cs.h, cs.w, xb.shape[-1], cout_p, cs.kh, cs.kw
    a.stride, a.pad, a.dil, a.act, a.num_ctas = cs.stride, cs.pad, cs.dil, 0, num_ctas
    a.norm_mean, a.norm_rstd, a.norm_wsum = mean.data_ptr(), rstd.data_ptr(), wsum.data_ptr()
    slots = ctypes.c_int(-1)
    rc = lib().hb_conv2d_fused_bf16(ctypes.byref(a), ctypes.byref(slots), stream_ptr())
    assert rc == 0, f"hb_conv2d_fused_bf16 returned {rc}"
    torch.cuda.synchronize()
    return y


def tc_ref(x, w, b, cs, cin_p):
    """fp64 NormConv2d of the bf16-rounded x and w, and its bound without the ulp; both [N, Cout, L]."""
    p = patches(x.bfloat16(), cs)
    w64 = w.bfloat16().double().reshape(cs.cout, -1)
    mu, _, r = stats_ref(p)
    core = ((p - mu[..., None]) * r[..., None]) @ w64.t()
    dmu, drel = bf16_stats_bounds(p, cin_p)
    wabs = w64.abs().sum(1)
    bound = (1e-5 * r[..., None] * (p.abs() @ w64.abs().t() + mu.abs()[..., None] * wabs)
             + (drel + U)[..., None] * core.abs() + (r * dmu)[..., None] * wabs)
    return _ncl(core + b.double()), _ncl(bound), p


FORCED_GRID_CASES = ["tc_rgb_stem", "tc_masked144", "tc_wide192"]


@pytest.mark.parametrize("name", list(D.TC_CASES))
def test_tensor_core_norm_conv_per_element(name):
    cs = D.TC_CASES[name]
    sms = _sms()
    t = D.tc_launch(cs, sms)
    what = D.describe(name, sms)
    print(what)
    x, w, b = tc_inputs(name, cs)
    xb, wf, bp = tc_pack(x, w, b, t)
    ref, bound, p = tc_ref(x, w, b, cs, t.cin_p)
    mean, rstd = tc_stats(xb, cs)
    check_stats(mean, rstd, p, *bf16_stats_bounds(p, t.cin_p), f"{name} hb_patch_stats_bf16")
    wsum = wf.float().sum((1, 2, 3))
    y = tc_conv(xb, wf, bp, mean, rstd, wsum, cs)
    yl = y.float().reshape(cs.n, -1, t.cout_p)
    assert_fwd(_ncl(yl[..., :cs.cout]), ref, bound, f"{name} y [{what}]", bits=BF16_BITS)
    assert bool((yl[..., cs.cout:] == 0).all()), f"{name}: a padded output column is not 0"
    if name in FORCED_GRID_CASES:
        # one CTA walks several pixel tiles and reloads the mean / rstd rows of each; the K order of an element does
        # not depend on the grid (nor on the Cout tile the small grids switch to), so the bits do not either
        for g in (1, 2, 3):
            bn = D.tc_launch(cs, sms, g).bn
            assert torch.equal(tc_conv(xb, wf, bp, mean, rstd, wsum, cs, g), y), f"{name} num_ctas={g} (BN={bn})"
    # the module path: its statistics must be those of the Cin kh kw logical window (not of the padded channels)
    got = F.norm_conv2d(x, w, b, cs.stride, cs.pad, cs.dil)
    assert_fwd(got, ref, bound, f"{name} F.norm_conv2d [{what}]", bits=BF16_BITS)


@pytest.mark.parametrize("name", ["tc_rgb_stem", "tc_dil2", "tc_masked144"])
def test_tensor_core_norm_conv_weight_gradient(name):
    """The statistics saved by the tensor-core forward come from the bf16 input; the weight gradient reads the fp32
    input: dw = sum g (x - mean_bf16) rstd_bf16 over the fp32 windows."""
    cs = D.TC_CASES[name]
    t = D.tc_launch(cs, _sms())
    x, w, b = tc_inputs(name, cs)
    x = x + 1e-3 * torch.randn(x.shape, device=DEV, generator=_gen(name + "x"))        # not bf16 values
    g = torch.randn(cs.n, cs.cout, cs.ho, cs.wo, device=DEV, generator=_gen(name + "g"))
    wd = w.clone().requires_grad_(True)
    F.norm_conv2d(x, wd, b, cs.stride, cs.pad, cs.dil).backward(g)
    xb, _, _ = tc_pack(x, w, b, t)
    mean, rstd = tc_stats(xb, cs)
    h = ((patches(x, cs) - mean.double().view(cs.n, -1, 1)) * rstd.double().view(cs.n, -1, 1)).reshape(-1, cs.k)
    gm = g.double().reshape(cs.n, cs.cout, -1).transpose(1, 2).reshape(-1, cs.cout)
    rel = (D.wgrad_geo(cs, _sms()).chain + 2) * U
    assert_within(wd.grad.reshape(cs.cout, -1), gm.t() @ h, gm.abs().t() @ h.abs(), f"{name} dw", rel=rel,
                  bits=FP32_BITS)


# ---------------------------------------------------------------------------------------------------------------------
# 3. exact edges
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("stride", [1, 2])
def test_add2d_ties_contribute_zero(stride):
    """Integer-valued x, w and g: every sum is exact in fp32, so both Add2d gradients must equal torch's fp64 autograd
    of the oracle to the bit, whose abs backward gives 0 at p == w. Many windows tie, zero padding against w = 0
    included."""
    cs = D.Case(2, 4, 9, 8, 12, 3, 3, stride, 1)
    gen = _gen(f"ties{stride}")
    x = torch.randint(-2, 3, (cs.n, cs.cin, cs.h, cs.w), device=DEV, generator=gen).float()
    w = torch.randint(-2, 3, (cs.cout, cs.cin, 3, 3), device=DEV, generator=gen).float()
    g = torch.randint(-3, 4, (cs.n, cs.cout, cs.ho, cs.wo), device=DEV, generator=gen).float()
    p = patches(x, cs)
    pad_zero = (patches(torch.ones_like(x), cs) == 0)[..., None, :] & (w.reshape(1, 1, cs.cout, -1) == 0)
    assert bool(pad_zero.any()) and bool((p[..., None, :] == w.double().reshape(1, 1, cs.cout, -1)).sum() > 1000)
    x64, w64 = x.double().cpu().requires_grad_(True), w.double().cpu().requires_grad_(True)
    ref = OF.add2d(x64, w64, None, stride, 1)
    ref.backward(g.double().cpu())
    out, _, _ = xc_fwd(x, w, None, cs, 1, False)
    assert torch.equal(out.double().cpu(), ref.detach())
    assert torch.equal(xc_wgrad(x, w, g, None, None, cs, 1, False).double().cpu(), w64.grad)
    assert torch.equal(add_dgrad(x, w, g, cs).double().cpu(), x64.grad)


def test_zero_regions_give_the_bias():
    """Windows that see only zeros (a black border, a ReLU output) have mean 0 and rstd 1 / sqrt(eps): the normalised
    window is exactly 0 and NormConv2d returns exactly the bias, fp32 on the fp32 kernel, bf16-rounded on the tensor
    cores."""
    gen = _gen("zeros")
    x = torch.relu(torch.randn(2, 8, 16, 14, device=DEV, generator=gen))
    x[:, :, :7] = 0
    b = torch.randn(24, device=DEV, generator=gen)
    for kh, kw in ((3, 3), (3, 1)):
        cs = D.Case(2, 8, 16, 14, 24, kh, kw, 1, 1)
        w = torch.randn(24, 8, kh, kw, device=DEV, generator=gen)
        dark = (patches(x, cs).abs().sum(-1) == 0).view(cs.n, 1, cs.ho, cs.wo).expand(-1, 24, -1, -1)
        assert bool(dark.any())
        want = b.view(1, -1, 1, 1).expand_as(dark)
        out, _, _ = xc_fwd(x, w, b, cs, 0, True)
        assert torch.equal(out[dark], want[dark]), f"{kh}x{kw} fp32 kernel"
        got = F.norm_conv2d(x, w, b, 1, 1)                    # 3x3: tensor cores; 3x1: fp32 kernel
        want = want if kh != kw else b.bfloat16().float().view(1, -1, 1, 1).expand_as(dark)
        assert torch.equal(got[dark], want[dark]), f"{kh}x{kw} F.norm_conv2d"


def test_constant_patches_stay_finite():
    """A saturated region: constant non-zero windows have variance 0 in exact arithmetic, and rounding leaves a tiny
    variance of either sign. With eps = 1e-14 the reference itself is ill-conditioned there (rstd up to 1e7), so only
    finiteness is asserted."""
    x = torch.rand(2, 8, 16, 16, device=DEV, generator=_gen("const")) + 0.5
    x[:, :, 4:12, 4:12] = 0.7
    w = torch.randn(16, 8, 3, 3, device=DEV, generator=_gen("constw"))
    for kh, kw in ((3, 3), (3, 1)):
        wk = w[..., :kw].contiguous()
        assert bool(torch.isfinite(F.norm_conv2d(x, wk, None, 1, 1)).all()), f"{kh}x{kw} norm_conv2d"
        assert bool(torch.isfinite(F.add2d(x, wk, None, 1, 1, normalize_slices=True)).all()), f"{kh}x{kw} add2d"


# ---------------------------------------------------------------------------------------------------------------------
# 4. modules: reflect padding, bf16 input, no bias, a 3 x 1 filter
# ---------------------------------------------------------------------------------------------------------------------
def test_norm_conv2d_module_reflect_bf16_rect():
    gen = _gen("mod_nc")
    mod = hb.nn.NormConv2d(8, 16, (3, 1), padding=(1, 0), padding_mode="reflect", bias=False).to(DEV)
    x = (torch.rand(2, 8, 11, 10, device=DEV, generator=gen) + 0.5).bfloat16()
    y = mod(x)
    assert y.dtype == torch.bfloat16 and y.shape == (2, 16, 11, 10)
    xp = TF.pad(x.double(), (0, 0, 1, 1), mode="reflect")
    cs = D.Case(2, 8, 13, 10, 16, 3, 1)                      # the reflect-padded input, padding 0
    ref, bound = fwd_ref(patches(xp, cs), mod.weight.detach(), None, cs, 0, True, lambda q: fp32_stats_bounds(q, cs))
    assert_fwd(y, ref, bound, "NormConv2d 3x1 reflect bf16", bits=BF16_BITS)
    assert torch.allclose(ref.reshape(y.shape), OF.norm_conv2d(xp, mod.weight.double(), None), rtol=1e-12, atol=1e-12)
    g = torch.randn(y.shape, device=DEV, generator=gen)
    y.backward(g.bfloat16())
    xpf = TF.pad(x.float(), (0, 0, 1, 1), mode="reflect")
    _, mean, rstd = xc_fwd(xpf, mod.weight.detach(), None, cs, 0, True)
    h = ((patches(xpf, cs) - mean.double().view(2, -1, 1)) * rstd.double().view(2, -1, 1)).reshape(-1, cs.k)
    gm = g.bfloat16().double().reshape(2, 16, -1).transpose(1, 2).reshape(-1, 16)
    rel = (D.wgrad_geo(cs, _sms()).chain + 2) * U
    assert_within(mod.weight.grad.reshape(16, -1), gm.t() @ h, gm.abs().t() @ h.abs(), "NormConv2d 3x1 dw", rel=rel,
                  bits=FP32_BITS)


@pytest.mark.parametrize("normalize", [False, True])
def test_add2d_module_reflect_bf16_rect(normalize):
    gen = _gen(f"mod_add{normalize}")
    mod = hb.nn.Add2d(8, 8, (3, 1), padding=(1, 0), padding_mode="reflect", bias=False,
                      normalize_slices=normalize).to(DEV)
    x = torch.randn(2, 8, 11, 10, device=DEV, generator=gen).bfloat16().requires_grad_(not normalize)
    y = mod(x)
    assert y.dtype == torch.bfloat16 and y.shape == (2, 8, 11, 10)
    cs = D.Case(2, 8, 13, 10, 8, 3, 1)
    xp = TF.pad(x.detach().double(), (0, 0, 1, 1), mode="reflect")
    ref, bound = fwd_ref(patches(xp, cs), mod.weight.detach(), None, cs, 1, normalize,
                         lambda q: fp32_stats_bounds(q, cs))
    assert_fwd(y, ref, bound, f"Add2d 3x1 reflect bf16 normalize={normalize}", bits=BF16_BITS)
    # g in {-1, 0, 1}: without normalisation both gradients are sums of integers (dx: 24 terms per padded pixel, a
    # border pixel gets two of those through the reflection: exact in fp32 and in the bf16 of dx), so they must equal
    # fp64 autograd of the oracle to the bit
    g = torch.randint(-1, 2, y.shape, device=DEV, generator=gen).bfloat16()
    y.backward(g)
    x64 = x.detach().double().requires_grad_(True)
    w64 = mod.weight.detach().double().requires_grad_(True)
    OF.add2d(TF.pad(x64, (0, 0, 1, 1), mode="reflect"), w64, None, normalize_slices=normalize).backward(g.double())
    if not normalize:
        assert torch.equal(mod.weight.grad.double(), w64.grad), "Add2d dw"
        assert torch.equal(x.grad.double(), x64.grad), "Add2d dx"
    else:
        # the sums are still exact, but the kernel normalises in fp32: a term within the fp32 rounding of a tie may
        # take the other sign than in fp64, which moves dw by 2 |g| = 2 (random operands leave at most a few such)
        diff = (mod.weight.grad.double() - w64.grad).abs()
        assert bool((diff % 2 == 0).all()) and float(diff.sum()) <= 8, f"Add2d normalised dw: off by {diff.sum()}"


# ---------------------------------------------------------------------------------------------------------------------
# 5. empty batch
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("op", ["norm_conv2d", "add2d"])
def test_empty_batch(op):
    x = torch.rand(0, 3, 9, 9, device=DEV, requires_grad=op == "add2d")
    w = torch.rand(4, 3, 3, 3, device=DEV, requires_grad=True)
    b = torch.rand(4, device=DEV, requires_grad=True)
    y = getattr(F, op)(x, w, b, 2, 1)
    ref = getattr(OF, op)(x.detach().cpu(), w.detach().cpu(), b.detach().cpu(), 2, 1)
    assert y.shape == ref.shape == (0, 4, 5, 5) and y.dtype == ref.dtype
    y.sum().backward()
    assert torch.equal(w.grad, torch.zeros_like(w)) and torch.equal(b.grad, torch.zeros_like(b))
    if op == "add2d":
        assert x.grad.shape == x.shape
