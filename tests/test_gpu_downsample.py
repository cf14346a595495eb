"""BlurPool2d, GlobalMaxPool2d and z_pool on the H100: the pooling kernels against fp64 on the same values and against
the torch restatement (tests/_downsample_oracle.py), the padding channels of the raw entry points, the modules against
the reference's fixture (tests/golden/downsample.pt), the reference's own test cases, realistic sizes, determinism and
CUDA-graph replay."""
import ctypes

import pytest
import torch
from torch import nn

import holocron_b200 as hb
from holocron_b200._lib import lib, ptr, stream_ptr
from holocron_b200.nn import _pooling as P

import _downsample_oracle as O
from _bounds import BF16_BITS, FP32_BITS, assert_within
from conftest import load_golden

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
DS = hb.nn.modules.downsample
BITS = {torch.bfloat16: BF16_BITS, torch.float32: FP32_BITS}
DTYPES = [torch.bfloat16, torch.float32]


def _cl(t: torch.Tensor) -> torch.Tensor:
    return t.contiguous(memory_format=torch.channels_last)


def _same_bits(a, b):
    """torch.equal with NaN equal to NaN and -0.0 different from +0.0."""
    a, b = a.cpu(), b.cpu()
    return (torch.equal(a.isnan(), b.isnan()) and torch.equal(a.nan_to_num(), b.nan_to_num())
            and torch.equal(torch.signbit(a), torch.signbit(b)))


def _rel_l2(a, b):
    a, b = a.detach().cpu().double(), b.detach().cpu().double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


# ---------------------------------------------------------------------------------------------------------------------
# blur pooling against fp64


def _check_blur(n, c, h, w, k, s, dtype, seed=0, device="cpu"):
    torch.manual_seed(seed)
    x = _cl(torch.randn(n, c, h, w, device=DEV).to(dtype)).requires_grad_(True)
    mod = DS.BlurPool2d(c, k, s)
    y = mod(x)
    dy = _cl(torch.randn(y.shape, device=DEV).to(dtype))
    y.backward(dy)
    # channels_last; a view of the channel-padded buffer when C is not a whole number of 16-byte vectors
    assert y.dtype == dtype and (y.is_contiguous(memory_format=torch.channels_last)
                                 or (y.stride(1) == 1 and c != P._pitch(c, dtype)))
    f = O.blur_filter(k, dtype).double()
    x64, dy64 = x.detach().to(device).double(), dy.to(device).double()
    ref = O.blur_pool2d(x64, k, s, f)
    ref_abs = O.blur_pool2d(x64.abs(), k, s, f)
    dref = O.blur_pool2d_backward(dy64, x.shape, k, s, f)
    dref_abs = O.blur_pool2d_backward(dy64.abs(), x.shape, k, s, f)
    assert_within(y.detach(), ref, ref_abs, "y", bits=BITS[dtype])
    assert_within(x.grad, dref, dref_abs, "dx", bits=BITS[dtype])


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp32"])
@pytest.mark.parametrize("c", [8, 12, 64, 256])
@pytest.mark.parametrize("s", [1, 2, 3])
@pytest.mark.parametrize("k", [2, 3, 4, 5, 6, 7])
def test_blur_kernels_vs_fp64(k, s, c, dtype):
    p = P.blur_padding(k, s)
    side = max(p + 1, k - 2 * p)
    _check_blur(2, c, 11, 9, k, s, dtype, seed=k * 10 + s)
    # the smallest legal sides: every pixel is within p of a border, mirrors on both sides included
    _check_blur(1, c, side, side + 1, k, s, dtype, seed=k * 10 + s + 1)
    _check_blur(1, c, side + 2, side, k, s, dtype, seed=k * 10 + s + 2)


def test_blur_realistic_size():
    """BlurPool2d(64, 3, 2) on a 32 x 64 x 112^2 bf16 activation (the reference computed in fp64 on the GPU)."""
    _check_blur(32, 64, 112, 112, 3, 2, torch.bfloat16, device=DEV)


# ---------------------------------------------------------------------------------------------------------------------
# max / mean reductions against the restatement

OPS = ["gmp", 1, 2, 3, -1, -2, -3]


def _planted(shape, seed):
    """Small integers (ties along every dim), NaNs, and +-0.0 ties in rows that only zeros decide."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(-4, 4, shape, generator=g).float()
    n, c, h, w = shape
    x[0, 1, 2, 3] = x[0, 1, 4, 1] = float("nan")
    x[1, 2] = -torch.rand(h, w, generator=g) - 1.0
    x[1, 2, 0, 2], x[1, 2, 3, 4] = 0.0, -0.0
    x[1, 3] = -torch.rand(h, w, generator=g) - 1.0
    x[1, 3, 1, 1], x[1, 3, 2, 5] = -0.0, 0.0
    x[0, :, 5, 6] = 0.0
    x[0, 0, 5, 6] = -0.0
    x[1, :, 0, 0] = float("nan")
    return x


def _run_op(op, x):
    if op == "gmp":
        return DS.GlobalMaxPool2d()(x)
    return hb.nn.functional.z_pool(x, op)


def _restated(op, x, w):
    """(y, dx) of the restatement on the CPU; dx in fp32 for a bf16 x (the kernel rounds dmax + dmean / L once)."""
    if op == "gmp":
        y, idx = O.global_max_pool2d(x)
        return y, O.global_max_pool2d_backward(w.float(), idx, x.shape)
    y, idx = O.z_pool(x, op)
    return y, O.z_pool_backward(w.float(), idx, x.shape, op)


def _check_reduction(op, x_cpu, w_seed=0):
    x = x_cpu.to(DEV).requires_grad_(True)
    y = _run_op(op, x)
    g = torch.Generator().manual_seed(w_seed)
    w = torch.randn(y.shape, generator=g).to(x.dtype)
    (y * w.to(DEV)).sum().backward()
    ry, rdx = _restated(op, x_cpu, w)
    assert y.shape == ry.shape and y.dtype == x.dtype
    if op == "gmp":
        assert _same_bits(y, ry)
    else:
        dim = op % 4
        mx, mean = y.detach().cpu().split(1, dim)
        rmx, _ = ry.split(1, dim)
        assert _same_bits(mx, rmx), "max values"
        xd = x_cpu.double()
        ref_mean = xd.sum(dim, keepdim=True) / x.shape[dim]
        abs_mean = xd.abs().sum(dim, keepdim=True) / x.shape[dim]
        finite = torch.isfinite(ref_mean)
        assert torch.equal(mean.isnan(), ref_mean.isnan())
        assert_within(mean[finite], ref_mean[finite], abs_mean[finite], "mean", bits=BITS[x.dtype])
    # the gradient, routing included, is the restatement's (rounded once to bf16 for a bf16 x)
    assert _same_bits(x.grad, rdx.to(x.dtype)), "dx"


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp32"])
@pytest.mark.parametrize("op", OPS, ids=[str(o) for o in OPS])
@pytest.mark.parametrize("c", [5, 8, 64])
def test_reductions_vs_restatement(op, c, dtype):
    _check_reduction(op, _planted((2, c, 6, 7), c).to(dtype), w_seed=c)
    _check_reduction(op, torch.randn(3, c, 9, 5, generator=torch.Generator().manual_seed(c)).to(dtype), w_seed=c + 1)


def test_reductions_realistic_sizes():
    g = torch.Generator().manual_seed(0)
    # GlobalMaxPool2d on a 256 x 2048 x 7^2 bf16 head; small integers make ties in every row
    _check_reduction("gmp", torch.randint(-50, 50, (256, 2048, 7, 7), generator=g).to(torch.bfloat16))
    # H*W > 65 536 splits a row across the threads of a CTA
    _check_reduction("gmp", torch.randn(2, 8, 300, 300, generator=g))
    _check_reduction(-1, torch.randint(-3, 3, (2, 4, 300, 300), generator=g).float())
    # z_pool over H with W*C > 2^16 (grid.y slabs)
    _check_reduction(2, torch.randn(2, 256, 8, 300, generator=g).to(torch.bfloat16))
    _check_reduction(1, torch.randn(4, 200, 30, 31, generator=g).to(torch.bfloat16))


# ---------------------------------------------------------------------------------------------------------------------
# padding channels of the raw entry points


@pytest.mark.parametrize("dtype,c", [(torch.bfloat16, 12), (torch.float32, 6), (torch.bfloat16, 3)])
def test_padded_channels_are_zero(dtype, c):
    """Channels C..Cp-1 of every output and input gradient are written as zeros, whatever the padded inputs hold."""
    torch.manual_seed(2)
    n, h, w, k, s = 2, 9, 7, 3, 2
    cp = P._pitch(c, dtype)
    code = 1 if dtype == torch.bfloat16 else 0
    x = _cl(torch.randn(n, cp, h, w, device=DEV).to(dtype))
    x[:, c:] = float("nan")
    taps = ctypes.cast(P.blur_taps(DS.BlurPool2d(c, k, s)._coeffs, dtype), ctypes.c_void_p)
    pad = P.blur_padding(k, s)
    ho, wo = (h + 2 * pad - k) // s + 1, (w + 2 * pad - k) // s + 1
    y = _cl(torch.full((n, cp, ho, wo), float("nan"), device=DEV, dtype=dtype))
    dx = torch.full_like(x, float("nan"))
    assert lib().hb_blurpool_fwd(ptr(x), ptr(y), taps, n, h, w, c, cp, k, s, code, stream_ptr()) == 0
    dy = y.clone()
    dy[:, c:] = float("nan")
    assert lib().hb_blurpool_bwd(ptr(dy), ptr(dx), taps, n, h, w, c, cp, k, s, code, stream_ptr()) == 0
    torch.cuda.synchronize()
    for t in (y, dx):
        assert torch.equal(t[:, c:], torch.zeros_like(t[:, c:])) and torch.isfinite(t[:, :c]).all()
    # middle-axis reductions: GlobalMaxPool2d (A=N, L=HW, M=Cp) and z_pool over H (A=N, L=H, M=W*Cp)
    for a, l_, m, with_mean, shape in ((n, h * w, cp, 0, (n, cp, 1, 1)), (n, h, w * cp, 1, (n, cp, 2, w))):
        out = _cl(torch.full(shape, float("nan"), device=DEV, dtype=dtype))
        idx = torch.full((a * m,), -7, dtype=torch.int32, device=DEV)
        assert lib().hb_pool_mid_fwd(ptr(x), ptr(out), ptr(idx), a, l_, m, c, cp, with_mean, code, stream_ptr()) == 0
        dout = out.clone()
        dout[:, c:] = float("nan")
        dxr = torch.full_like(x, float("nan"))
        assert lib().hb_pool_mid_bwd(ptr(dout), ptr(idx), ptr(dxr), a, l_, m, c, cp, with_mean, code,
                                     stream_ptr()) == 0
        torch.cuda.synchronize()
        for t in (out, dxr):
            assert torch.equal(t[:, c:], torch.zeros_like(t[:, c:])) and torch.isfinite(t[:, :c]).all()
        assert (idx.view(-1, cp)[:, c:] == 0).all()
    # channel-axis reduction (z_pool over C): the padding lanes are not part of the reduction
    out = _cl(torch.empty(n, 2, h, w, device=DEV, dtype=dtype))
    idx = torch.empty(n * h * w, dtype=torch.int32, device=DEV)
    assert lib().hb_pool_last_fwd(ptr(x), ptr(out), ptr(idx), n * h * w, c, cp, code, stream_ptr()) == 0
    dxr = torch.full_like(x, float("nan"))
    assert lib().hb_pool_last_bwd(ptr(out), ptr(idx), ptr(dxr), n * h * w, c, cp, code, stream_ptr()) == 0
    torch.cuda.synchronize()
    assert torch.isfinite(out).all() and bool((idx < c).all())
    assert torch.equal(dxr[:, c:], torch.zeros_like(dxr[:, c:])) and torch.isfinite(dxr[:, :c]).all()


# ---------------------------------------------------------------------------------------------------------------------
# modules against the reference's fixture


def _bar(dtype):
    return 1e-2 if dtype == torch.bfloat16 else 1e-5


def test_modules_vs_fixture():
    gold = load_golden("downsample")
    for case in gold["blur"]:
        x = case["x"].to(DEV).requires_grad_(True)
        y = DS.BlurPool2d(x.shape[1], case["k"], case["s"])(x)
        (y * case["w"].to(DEV)).sum().backward()
        assert y.dtype == x.dtype and y.shape == case["y"].shape
        assert _rel_l2(y, case["y"]) <= _bar(x.dtype), (case["k"], case["s"])
        assert _rel_l2(x.grad, case["dx"]) <= _bar(x.dtype), (case["k"], case["s"])
    for key in ("gmp", "zpool"):
        for case in gold[key]:
            x = case["x"].to(DEV).requires_grad_(True)
            if key == "gmp":
                y = DS.GlobalMaxPool2d(case["flatten"])(x)
                mx, mean, rmx, rmean = y, None, case["y"], None
            else:
                dim = case["dim"]
                y = DS.ZPool(dim)(x)
                (mx, mean), (rmx, rmean) = y.split(1, dim), case["y"].split(1, dim)
            assert y.shape == case["y"].shape and y.dtype == x.dtype
            (y * case["w"].to(DEV)).sum().backward()
            if x.dtype == torch.float32:
                assert _same_bits(mx, rmx), (key, case["tag"])
            else:
                assert _rel_l2(mx.nan_to_num(), rmx.nan_to_num()) <= _bar(x.dtype)
            if mean is not None:
                assert torch.equal(mean.isnan().cpu(), rmean.isnan())
                assert _rel_l2(mean.nan_to_num(), rmean.nan_to_num()) <= _bar(x.dtype)
            assert _rel_l2(x.grad, case["dx"]) <= _bar(x.dtype), (key, case["tag"])
            if key == "gmp":
                assert torch.equal((x.grad != 0).cpu(), case["dx"] != 0), f"{case['tag']}: gradient routing"


# ---------------------------------------------------------------------------------------------------------------------
# the reference's own tests/test_nn_downsample.py cases, on the GPU


def test_reference_globalmaxpool2d():
    x = torch.rand(2, 4, 16, 16, device=DEV)
    ref = nn.AdaptiveMaxPool2d(1)
    out = DS.GlobalMaxPool2d(flatten=False)(x)
    assert torch.equal(out, ref(x))
    x = torch.rand(2, 4, 16, 16, device=DEV)
    assert torch.equal(DS.GlobalMaxPool2d(flatten=True)(x), ref(x).view(*x.shape[:2]))


def test_reference_blurpool2d():
    x = torch.rand((2, 8, 5, 5), device=DEV)
    mod = DS.BlurPool2d(8, stride=2)
    with torch.no_grad():
        out = mod(x)
    assert out.shape == (2, 8, 3, 3)
    k = torch.tensor([[0.0625, 0.125, 0.0625], [0.125, 0.25, 0.125], [0.0625, 0.125, 0.0625]], device=DEV)
    assert torch.allclose(out[..., 1, 1], (x[..., 1:-1, 1:-1] * k[None, None, ...]).sum(dim=(2, 3)), atol=1e-7)


def test_reference_zpool():
    x = torch.rand((2, 4, 32, 32), device=DEV)
    out = hb.nn.functional.z_pool(x, 1)
    assert out.shape == (2, 2, 32, 32)
    assert out[0, 0, 0, 0].item() == x[0, :, 0, 0].max().item()
    # the mean is a sum of four fp32 values in another order than torch's: within one fp32 ulp
    mean = x[0, :, 0, 0].mean().item()
    assert abs(out[0, 1, 0, 0].item() - mean) <= 2.0 ** -23 * abs(mean)
    assert torch.equal(DS.ZPool(1)(x), out)


def test_other_dtypes_and_layouts():
    """fp16 / fp64 compute in fp32 and come back in their dtype; a bf16 channels_last input with C % 8 == 0 is read in
    place; 4-D outputs are channels_last."""
    torch.manual_seed(0)
    x = torch.randn(2, 16, 10, 12, device=DEV)
    for dt in (torch.float16, torch.float64):
        xd = x.to(dt)
        y = DS.BlurPool2d(16, 5, 2)(xd)
        assert y.dtype == dt
        assert _rel_l2(y, O.blur_pool2d(xd.double().cpu(), 5, 2)) <= 1e-3
        z = hb.nn.functional.z_pool(xd, 2)
        assert z.dtype == dt and torch.equal(z.split(1, 2)[0].cpu(), xd.amax(2, keepdim=True).cpu())
    xb = _cl(x.bfloat16())
    before = torch.cuda.memory_allocated()
    y = DS.BlurPool2d(16, 3, 2)(xb)
    assert torch.cuda.memory_allocated() - before < xb.numel() * xb.element_size(), "no layout copy of the input"
    for out in (y, DS.GlobalMaxPool2d()(xb), DS.ZPool(1)(xb), DS.ZPool(2)(xb), DS.ZPool(3)(xb)):
        assert out.is_contiguous(memory_format=torch.channels_last)


# ---------------------------------------------------------------------------------------------------------------------
# determinism and CUDA-graph replay


class _Chain(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.blur = DS.BlurPool2d(c, 5, 2)
        self.gmp = DS.GlobalMaxPool2d()
        self.z = nn.ModuleList([DS.ZPool(d) for d in (1, 2, 3)])

    def forward(self, x):
        b = self.blur(x)
        return [b, self.gmp(b)] + [z(b) for z in self.z]


def _run(mod, x, ws):
    x.grad = None
    outs = mod(x)
    sum((o * w).sum() for o, w in zip(outs, ws)).backward()
    return [o.detach().clone() for o in outs] + [x.grad.clone()]


@pytest.mark.parametrize("dtype,c", [(torch.bfloat16, 64), (torch.float32, 12)])
def test_deterministic_and_graph_replay(dtype, c):
    torch.manual_seed(0)
    mod = _Chain(c)
    # a long spatial extent so the max / mean rows are split across threads
    x = _cl(torch.randint(-8, 8, (2, c, 300, 260), device=DEV).to(dtype)).requires_grad_(True)
    ws = [torch.randn(o.shape, device=DEV).to(dtype) for o in mod(x)]
    first, second = _run(mod, x, ws), _run(mod, x, ws)
    for a, b in zip(first, second):
        assert _same_bits(a, b)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        _run(mod, x, ws)
    torch.cuda.current_stream().wait_stream(side)
    x.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = mod(x)
        sum((o * w).sum() for o, w in zip(outs, ws)).backward()
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(first, list(outs) + [x.grad]):
        assert _same_bits(a, b)
