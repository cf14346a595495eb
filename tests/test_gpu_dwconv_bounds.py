"""The depth-wise convolution kernels (csrc/dwconv.cu) per element, on every path their dispatch takes.

Each case of tests/_dwconv_cases.py runs the three C entry points directly, so a failure names the kernel the routing
mirror says the case takes. Outputs (y, dx, dw, db and the weight-gradient scratch, sized exactly as
``hb_dwconv_wgrad_scratch_doubles`` asks) are pre-filled with NaN so an unwritten element shows, and sit in front of a
guard band that must come back unchanged. Every element is checked against an fp64 reference fed the same operands
(tests/_bounds.py). Each launch runs twice and must give the same bits; each case also runs without a bias and with
db = NULL. The rows of the scratch the weight-gradient kernel writes must be exactly the first gx of the mirror, which
ties the mirror's grid (and the dw bound derived from it) to the launcher.

``HB_DISABLE_DW_QUAD`` is read once per process, so the one-output 3x3 kernels and ``dw_bwd_weight_kernel<3>`` on the
same wide shapes run in a child process with the variable set."""
import ctypes
import os
import subprocess
import sys
from pathlib import Path

import pytest
import torch

from holocron_b200._lib import lib, ptr, stream_ptr
from holocron_b200.nn._dwconv import dwconv2d
from torch.nn.grad import conv2d_input

import _dwconv_cases as D
from _bounds import FP32_BITS, assert_within, conv_ref, dgrad_ref, wgrad_ref

pytestmark = pytest.mark.gpu
DEV = "cuda"
GUARD = 64
SENTINEL = 12288.0          # exact in bf16, fp32 and fp64
QUAD_ON = os.environ.get("HB_DISABLE_DW_QUAD") is None
ROOT = Path(__file__).resolve().parents[1]


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def guarded(n, dtype):
    """(view of n elements pre-filled with NaN, whole buffer): the view is followed by GUARD sentinels."""
    buf = torch.full((n + GUARD,), SENTINEL, device=DEV, dtype=dtype)
    buf[:n] = float("nan")
    return buf[:n], buf


def assert_guard(buf, n, what):
    assert bool((buf[n:] == SENTINEL).all()), f"{what}: guard band overwritten"


def _nchw(t):
    return t.permute(0, 3, 1, 2)


# ---------------------------------------------------------------------------------------------------------------------
# raw launches: NHWC bf16 activations, fp32 filter [C, K, K]
# ---------------------------------------------------------------------------------------------------------------------
def fwd(x, w, bias, cs):
    y, buf = guarded(cs.n * cs.ho * cs.wo * cs.c, torch.bfloat16)
    rc = lib().hb_dwconv_fwd_bf16(ptr(x), ptr(w), ptr(bias), ptr(y), cs.n, cs.h, cs.w, cs.c, cs.k, cs.stride, cs.pad,
                                  stream_ptr())
    assert rc == 0, f"hb_dwconv_fwd_bf16 returned {rc}"
    torch.cuda.synchronize()
    assert_guard(buf, y.numel(), "y")
    return y.view(cs.n, cs.ho, cs.wo, cs.c)


def dgrad(dy, w, cs):
    dx, buf = guarded(cs.n * cs.h * cs.w * cs.c, torch.bfloat16)
    rc = lib().hb_dwconv_bwd_data_bf16(ptr(dy), ptr(w), ptr(dx), cs.n, cs.h, cs.w, cs.c, cs.k, cs.stride, cs.pad,
                                       stream_ptr())
    assert rc == 0, f"hb_dwconv_bwd_data_bf16 returned {rc}"
    torch.cuda.synchronize()
    assert_guard(buf, dx.numel(), "dx")
    return dx.view(cs.n, cs.h, cs.w, cs.c)


def wgrad(x, dy, cs, with_db=True):
    """(dw [C, K, K], db [C] or None, scratch): every buffer guarded; the scratch is exactly what the library asks for."""
    kk = cs.k * cs.k
    dw, dwbuf = guarded(cs.c * kk, torch.float32)
    db, dbbuf = guarded(cs.c, torch.float32)
    ns = lib().hb_dwconv_wgrad_scratch_doubles(cs.c, cs.k)
    scratch, sbuf = guarded(ns, torch.float64)
    rc = lib().hb_dwconv_bwd_weight_bf16(ptr(x), ptr(dy), ptr(dw), ptr(db) if with_db else None, ptr(scratch), cs.n,
                                         cs.h, cs.w, cs.c, cs.k, cs.stride, cs.pad, stream_ptr())
    assert rc == 0, f"hb_dwconv_bwd_weight_bf16 returned {rc}"
    torch.cuda.synchronize()
    assert_guard(dwbuf, dw.numel(), "dw")
    assert_guard(dbbuf, cs.c, "db")
    assert_guard(sbuf, ns, "wgrad scratch")
    return dw.view(cs.c, cs.k, cs.k), (db if with_db else None), scratch


# ---------------------------------------------------------------------------------------------------------------------
# 1. every kernel, per element, through the C ABI
# ---------------------------------------------------------------------------------------------------------------------
def untouched(cs):
    """[H, W] mask of the input pixels no output pixel reads (their dx must be exactly 0)."""
    ones = conv2d_input((1, 1, cs.h, cs.w), torch.ones(1, 1, cs.k, cs.k, dtype=torch.float64),
                        torch.ones(1, 1, cs.ho, cs.wo, dtype=torch.float64), cs.stride, cs.pad)
    return ones[0, 0] == 0


def check_case(name, quad=QUAD_ON):
    cs = D.CASES[name]
    sms = _sms()
    r = D.route(cs, sms, quad)
    what = D.describe(name, sms, quad)
    print(what)
    if cs.wrap:
        for d, v in r.items():
            assert v.min_iters >= 2, f"{what}: {d} does not wrap its grid"
    assert lib().hb_dwconv_wgrad_scratch_doubles(cs.c, cs.k) == D.scratch_doubles(cs.c, cs.k, sms), what
    g = torch.Generator(device=DEV)
    g.manual_seed(sum(map(ord, name)))
    c, k = cs.c, cs.k
    x = torch.randn(cs.n, cs.h, cs.w, c, device=DEV, generator=g).bfloat16()
    dy = torch.randn(cs.n, cs.ho, cs.wo, c, device=DEV, generator=g).bfloat16()
    # fp32 filter and bias that are not bf16 values: the products of the forward and data gradient are not exact in fp32
    w = torch.randn(c, k, k, device=DEV, generator=g) / k
    bias = torch.randn(c, device=DEV, generator=g)
    big = x.numel() > 1 << 20
    rdev = DEV if big else "cpu"
    xr, dyr, wr = _nchw(x), _nchw(dy), w.view(c, 1, k, k)
    # y and dx are bf16: (K^2 + 1) fp32 roundings of the non-exact products and the bias, <= 50 * 2^-24 < 1e-5 of
    # sum|terms| for K <= 7, and the final rounding (one bf16 ulp)
    for b in (bias, None):
        tag = f"{r['fwd'].kernel} bias={b is not None}"
        y = fwd(x, w, b, cs)
        ref, abs_sum = conv_ref(xr, wr, b, cs.stride, cs.pad, groups=c, device=rdev)
        assert_within(_nchw(y), ref, abs_sum, f"{name} y [{tag}]")
        assert torch.equal(fwd(x, w, b, cs), y), f"{name} y [{tag}]: not bit-reproducible"
    tag = r["dgrad"].kernel
    dx = dgrad(dy, w, cs)
    ref, abs_sum = dgrad_ref((cs.n, c, cs.h, cs.w), wr, dyr, cs.stride, cs.pad, groups=c, device=rdev)
    assert_within(_nchw(dx), ref, abs_sum, f"{name} dx [{tag}]")
    assert torch.equal(dgrad(dy, w, cs), dx), f"{name} dx [{tag}]: not bit-reproducible"
    hole = untouched(cs)
    if hole.any():
        assert bool((dx[:, hole.to(DEV)] == 0).all()), f"{name} dx [{tag}]: a pixel no output reads is not 0"
    # dw / db are fp32: the products of bf16 x and dy are exact, the error is one thread's fp32 chain (the fp64 folds of
    # the partials add < 2^-40 relative) and the final rounding (one fp32 ulp)
    wl = r["wgrad"]
    tag = f"{wl.kernel} gx={wl.gx} chain={wl.chain}" + (" finalize unrolled" if D.finalize_unrolled(wl.gx) else "")
    dw, db, scratch = wgrad(x, dy, cs)
    e = c * (k * k + 1)
    assert not bool(scratch[:wl.gx * e].isnan().any()), f"{name} [{tag}]: a partial-sum row below gx is unwritten"
    assert bool(scratch[wl.gx * e:].isnan().all()), f"{name} [{tag}]: more partial-sum rows written than gx"
    rel = wl.chain * 2.0 ** -24
    ref, abs_sum = wgrad_ref(xr, dyr, k, cs.stride, cs.pad, groups=c, device=rdev)
    assert_within(dw.view(c, 1, k, k), ref, abs_sum, f"{name} dw [{tag}]", rel=rel, bits=FP32_BITS)
    d64 = dyr.to(rdev, torch.float64)
    assert_within(db, d64.sum((0, 2, 3)), d64.abs().sum((0, 2, 3)), f"{name} db [{tag}]", rel=rel, bits=FP32_BITS)
    dw2, db2, _ = wgrad(x, dy, cs)
    assert torch.equal(dw2, dw) and torch.equal(db2, db), f"{name} dw/db [{tag}]: not bit-reproducible"
    dw3, _, _ = wgrad(x, dy, cs, with_db=False)
    assert torch.equal(dw3, dw), f"{name} dw [{tag}]: differs with db = NULL"


@pytest.mark.parametrize("name", list(D.CASES))
def test_kernels_per_element(name):
    check_case(name)


def test_quad_kernels_disabled():
    """The K = 3, stride 1 / 2 cases again with HB_DISABLE_DW_QUAD set, in a child process that runs to completion."""
    env = dict(os.environ, HB_DISABLE_DW_QUAD="1")
    code = ("import sys; sys.path[:0] = [sys.argv[1], sys.argv[2]]\n"
            "import test_gpu_dwconv_bounds as T\n"
            "assert not T.QUAD_ON\n"
            "for name in sys.argv[3:]:\n"
            "    T.check_case(name)\n")
    proc = subprocess.run([sys.executable, "-c", code, str(ROOT / "tests"), str(ROOT), *D.QUAD_CASES], env=env,
                          capture_output=True, text=True, timeout=900)
    print(proc.stdout)
    assert proc.returncode == 0, proc.stdout[-2000:] + proc.stderr[-4000:]


# ---------------------------------------------------------------------------------------------------------------------
# 2. the autograd binding end to end: the same bits as the C ABI
# ---------------------------------------------------------------------------------------------------------------------
def _bf16_valued(*shape, gen):
    return torch.randn(*shape, device=DEV, generator=gen).bfloat16().float()


@pytest.mark.parametrize("name", ["rexnet_s2_odd", "k5_s2", "slab_tail_c328"])
def test_binding_nchw_fp32_matches_abi(name):
    cs = D.CASES[name]
    g = torch.Generator(device=DEV)
    g.manual_seed(7)
    x = _bf16_valued(cs.n, cs.c, cs.h, cs.w, gen=g).requires_grad_(True)        # NCHW fp32
    dy = _bf16_valued(cs.n, cs.c, cs.ho, cs.wo, gen=g)
    w = (torch.randn(cs.c, 1, cs.k, cs.k, device=DEV, generator=g) / cs.k).requires_grad_(True)
    b = torch.randn(cs.c, device=DEV, generator=g).requires_grad_(True)
    y = dwconv2d(x, w, b, cs.stride, cs.pad)
    y.backward(dy)
    xh = x.detach().permute(0, 2, 3, 1).bfloat16().contiguous()
    dyh = dy.permute(0, 2, 3, 1).bfloat16().contiguous()
    w3 = w.detach().view(cs.c, cs.k, cs.k)
    assert torch.equal(y.detach().permute(0, 2, 3, 1), fwd(xh, w3, b.detach(), cs)), "y"
    assert torch.equal(x.grad.permute(0, 2, 3, 1).float(), dgrad(dyh, w3, cs).float()), "dx"
    dw, db, _ = wgrad(xh, dyh, cs)
    assert torch.equal(w.grad.view(cs.c, cs.k, cs.k), dw) and torch.equal(b.grad, db), "dw / db"


def test_binding_bias_grad_only():
    cs = D.CASES["stride3"]
    g = torch.Generator(device=DEV)
    g.manual_seed(8)
    x = _bf16_valued(cs.n, cs.c, cs.h, cs.w, gen=g)
    w = torch.randn(cs.c, 1, 3, 3, device=DEV, generator=g)
    b = torch.randn(cs.c, device=DEV, generator=g).requires_grad_(True)
    dy = _bf16_valued(cs.n, cs.c, cs.ho, cs.wo, gen=g)
    dwconv2d(x, w, b, cs.stride, cs.pad).backward(dy)
    assert w.grad is None and x.grad is None
    _, db, _ = wgrad(x.permute(0, 2, 3, 1).bfloat16().contiguous(), dy.permute(0, 2, 3, 1).bfloat16().contiguous(), cs)
    assert torch.equal(b.grad, db)


def test_binding_unsupported_wgrad_filter_raises():
    c = 16
    g = torch.Generator(device=DEV)
    g.manual_seed(9)
    x = _bf16_valued(2, c, 12, 12, gen=g).requires_grad_(True)
    w = torch.randn(c, 1, 9, 9, device=DEV, generator=g).requires_grad_(True)
    y = dwconv2d(x, w, None, 1, 4)          # the generic forward takes any K
    assert_within(y, *conv_ref(x, w, None, 1, 4, groups=c), "y K=9")
    with pytest.raises(RuntimeError, match="hb_dwconv_bwd_weight_bf16"):
        y.backward(torch.ones_like(y))


def test_binding_empty_batch():
    x = torch.zeros(0, 16, 9, 9, device=DEV, requires_grad=True)
    w = torch.randn(16, 1, 3, 3, device=DEV, requires_grad=True)
    b = torch.randn(16, device=DEV, requires_grad=True)
    y = dwconv2d(x, w, b, 2, 1)
    assert y.shape == (0, 16, 5, 5)
    y.sum().backward()
    assert x.grad.shape == x.shape
    assert torch.equal(w.grad, torch.zeros_like(w)) and torch.equal(b.grad, torch.zeros_like(b))
