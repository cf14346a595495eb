"""DropBlock (csrc/dropblock.cu), global average pooling (csrc/se_gate.cu, csrc/conv_aux.cu), HardMish / NLReLU
(csrc/pointwise.cu) and the pairwise box backward (csrc/boxes.cu) per element, against the fp64 oracles and bounds of
tests/_small_kernels_oracle.py, on every path of the case tables there.

Kernels are launched through the C ABI where the Python wrapper would hide a path (an unaligned base, in-place
aliasing, a NULL gradient). Outputs are NaN-filled and followed by a guard band that must come back unchanged."""
import ctypes

import pytest
import torch

import _small_kernels_oracle as O
from holocron_b200._lib import dtype_code, lib, ptr, stream_ptr
from holocron_b200 import ops
from holocron_b200.nn import functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"
GUARD = 64
SENTINEL = 12345.0
DTYPES = [torch.float32, torch.bfloat16, torch.float16]
BITS = {torch.float32: 24, torch.bfloat16: 8, torch.float16: 11}


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def guarded(n, dtype=torch.float32, fill=float("nan"), offset=0):
    """(view of n elements starting `offset` elements into the buffer, whole buffer): the view is pre-filled with
    ``fill`` and followed by GUARD sentinels."""
    buf = torch.full((offset + n + GUARD,), SENTINEL, device=DEV, dtype=dtype)
    buf[offset:offset + n] = fill
    return buf[offset:offset + n], buf


def assert_guard(buf, n, what, offset=0):
    assert bool((buf[offset + n:] == SENTINEL).all()), f"{what}: guard band overwritten"
    assert bool((buf[:offset] == SENTINEL).all()), f"{what}: bytes before the base overwritten"


def ulp(ref, bits):
    """One ulp at |ref| for a format of `bits` significant bits (subnormal spacing of fp16 / bf16 / fp32 below)."""
    emin = {24: -126, 8: -126, 11: -14}[bits]
    a = ref.abs().clamp_min(2.0 ** emin)
    return torch.exp2(torch.floor(torch.log2(a)) - (bits - 1))


def assert_bound(got, ref, bound, what):
    """|got - ref| <= bound per element; NaN in ref must be NaN in got, +-inf must match exactly."""
    got = got.detach().to(torch.float64)
    ref = ref.to(got.device)
    special = ~torch.isfinite(ref)
    nan_ok = torch.isnan(got[special]) == torch.isnan(ref[special])
    inf_ok = torch.where(torch.isnan(ref[special]), True, got[special] == ref[special])
    assert bool(nan_ok.all() and inf_ok.all()), f"{what}: NaN / inf pattern differs"
    fin = torch.isfinite(ref)
    err = (got[fin] - ref[fin]).abs()
    bad = ~(err <= bound.to(got.device)[fin])
    if bad.any():
        i = int(bad.nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {int(fin.sum())} elements off; first: got "
                             f"{float(got[fin][i]):.9g}, ref {float(ref[fin][i]):.9g}, bound {float(bound[fin][i]):.3g}")


# ---------------------------------------------------------------------------------------------------------------------
# activations
# ---------------------------------------------------------------------------------------------------------------------
def _act_inputs(n, dtype, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = (torch.randn(n, device=DEV, generator=g, dtype=torch.float64) * 3).to(dtype)
    plant = torch.tensor([-2.0, 0.0, float("nan"), float("inf"), -float("inf"), -1.0, 2.0 ** -30, -0.0], device=DEV)
    k = min(n, plant.numel())
    x[:k] = plant[:k].to(dtype)
    x[-k:] = plant[:k].to(dtype)
    dy = (torch.randn(n, device=DEV, generator=g, dtype=torch.float64) + 0.5).to(dtype)
    return x, dy


def _launch_unary(fn, x, n, dtype, offset, *extra):
    y, buf = guarded(n, dtype, offset=offset)
    assert fn(ptr(x), ptr(y), n, *extra, dtype_code(x), stream_ptr()) == 0
    torch.cuda.synchronize()
    assert_guard(buf, n, "forward output", offset)
    return y


def _launch_binary(fn, a, b, n, dtype, offset, *extra):
    y, buf = guarded(n, dtype, offset=offset)
    assert fn(ptr(a), ptr(b), ptr(y), n, *extra, dtype_code(a), stream_ptr()) == 0
    torch.cuda.synchronize()
    assert_guard(buf, n, "backward output", offset)
    return y


def _in_place_of(src, offset):
    """A copy of src at `offset` elements into a fresh buffer (for unaligned bases)."""
    buf = torch.full((offset + src.numel(),), 0, device=DEV, dtype=src.dtype)
    buf[offset:] = src
    return buf[offset:]


def _one_plus_beta_x(x64, beta):
    """fp32 1 + beta * relu(x) both ways the compiler may evaluate it: fused (one rounding) or not (two)."""
    r = torch.where(x64 < 0, torch.zeros_like(x64), x64)       # relu_nan keeps NaN
    b32 = torch.tensor(beta, dtype=torch.float32).item()
    fused = (1 + b32 * r).float().double()
    split = (1 + (b32 * r).float().double()).float().double()
    return fused, split


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
@pytest.mark.parametrize("case", O.ACT_CASES, ids=lambda c: c[0])
def test_activations(case, dtype):
    name, nvec, tail, aligned, route = case
    n = nvec * O.vec_width(dtype) + tail
    for binary in (False, True):
        assert O.route_act(n, dtype, binary, aligned, _sms()) == frozenset(route)
    off = 0 if aligned else 1
    x, dy = _act_inputs(n, dtype, 7 + n)
    x, dy = _in_place_of(x, off), _in_place_of(dy, off)
    x64, dy64 = x.double(), dy.double()
    L = lib()
    bits, fp32 = BITS[dtype], dtype == torch.float32
    u = O.U32
    store = 0.0 if fp32 else 0.5          # one rounding to the storage type, in its ulps

    # HardMish forward: (0.5 x) * clamp(fl32(x + 2)); fp32 intermediates as the kernel rounds them
    t32 = (x64 + 2).float().double()
    ref = 0.5 * x64 * t32.clamp(0, 2)
    ref = torch.where(torch.isnan(x64), x64, ref)
    y = _launch_unary(L.hb_hard_mish_fwd, x, n, dtype, off)
    assert_bound(y, ref, (0.5 if fp32 else store) * ulp(ref, bits) + u * ref.abs(), f"{name} hard_mish fwd")
    # and the plain fp64 value on the planted clamp ends and specials
    assert_bound(y, O.hard_mish_ref(x64), ulp(O.hard_mish_ref(x64), bits) + 4 * u * x64.abs().nan_to_num(0, 0, 0),
                 f"{name} hard_mish fwd vs fp64")

    # HardMish backward: dy * (0.5 c + [0 <= t <= 2] 0.5 x), t = fl32(x + 2)
    inner = torch.where((t32 >= 0) & (t32 <= 2), 0.5 * x64, torch.zeros_like(x64))
    c = torch.where(torch.isnan(t32), t32, t32.clamp(0, 2))
    ref = dy64 * (0.5 * c + inner)
    ref = torch.where(torch.isinf(x64), O.hard_mish_grad_ref(x64, dy64), ref)
    mag = dy64.abs() * (0.5 * c.abs() + inner.abs())
    dx = _launch_binary(L.hb_hard_mish_bwd, x, dy, n, dtype, off)
    assert_bound(dx, ref, store * ulp(ref, bits) + 2 * u * mag.nan_to_num(0, 0, 0), f"{name} hard_mish bwd")
    assert_bound(dx, O.hard_mish_grad_ref(x64, dy64), ulp(O.hard_mish_grad_ref(x64, dy64), bits) +
                 4 * u * (dy64 * (x64.abs() + 2)).abs().nan_to_num(0, 0, 0), f"{name} hard_mish bwd vs autograd")

    for beta in (1.0, 0.5):
        fused, split = _one_plus_beta_x(x64, beta)
        # forward: logf (fp32: 1 ulp) or __logf (16-bit: 2^-21.4 absolute) of the fp32 argument, then the storage rounding
        y = _launch_unary(L.hb_nl_relu_fwd, x, n, dtype, off, ctypes.c_float(beta))
        errs = []
        for a in (fused, split):
            ref = torch.log(a)
            if fp32:
                bound = ulp(ref, 24) + 2.0 ** -149
            else:
                bound = store * ulp(ref.abs() + O.LOG_FAST_ABS, bits) + O.LOG_FAST_ABS
            errs.append(((y.double() - ref).abs() - bound).nan_to_num(0, 0, 0))
        worst = torch.minimum(*errs)
        assert bool((worst <= 0).all()), f"{name} nl_relu fwd beta={beta}: max excess {float(worst.max()):.3g}"
        assert_bound(y, O.nl_relu_ref(x64, beta), torch.full_like(x64, float("inf")), f"{name} nl_relu fwd specials")

        # backward from the input: dy * beta / a (IEEE division in fp32, __fdividef in 16-bit: 2 ulps)
        dx = _launch_binary(L.hb_nl_relu_bwd, x, dy, n, dtype, off, ctypes.c_float(beta))
        errs = []
        for a in (fused, split):
            ref = torch.where(x64 <= 0, torch.zeros_like(x64), dy64 * beta / a)
            bound = store * ulp(ref, bits) + (2 if fp32 else 6) * u * ref.abs()
            errs.append(((dx.double() - ref).abs() - bound).nan_to_num(0, 0, 0))
        worst = torch.minimum(*errs)
        assert bool((worst <= 0).all()), f"{name} nl_relu bwd beta={beta}: max excess {float(worst.max()):.3g}"
        ref = O.nl_relu_grad_ref(x64, dy64, beta)
        assert_bound(dx, ref, torch.full_like(ref, float("inf")), f"{name} nl_relu bwd specials")

        # backward from the output (the in-place path): dy * beta * expf(-y) on the stored y (expf: 2 ulps, 2 products)
        y64 = y.double()
        dx = _launch_binary(L.hb_nl_relu_bwd_from_out, y, dy, n, dtype, off, ctypes.c_float(beta))
        ref = O.nl_relu_grad_from_out_ref(y64, dy64, beta)
        assert_bound(dx, ref, store * ulp(ref, bits) + 6 * u * ref.abs(), f"{name} nl_relu bwd_from_out beta={beta}")


def test_nl_relu_in_place_gradient_pinned():
    """The in-place backward sees y, not x. Where 0 < beta x < 2^-24, y rounds to 0 and the gradient is 0 (the
    out-of-place one is beta dy); in 16-bit, the rounding of y moves the gradient by up to y * 2^-8 (bf16) relative."""
    L = lib()
    beta = 1.0
    x = torch.tensor([2.0 ** -30, 2.0 ** -26, 1e-3, 1.0, 3.0, 8.0] * 64, device=DEV)
    dy = torch.ones_like(x)
    n = x.numel()
    y = _launch_unary(L.hb_nl_relu_fwd, x, n, torch.float32, 0, ctypes.c_float(beta))
    from_out = _launch_binary(L.hb_nl_relu_bwd_from_out, y, dy, n, torch.float32, 0, ctypes.c_float(beta))
    from_in = _launch_binary(L.hb_nl_relu_bwd, x, dy, n, torch.float32, 0, ctypes.c_float(beta))
    tiny = x < 2.0 ** -24
    assert bool((y[tiny] == 0).all()) and bool((from_out[tiny] == 0).all())
    assert bool((from_in[tiny] == beta).all())
    for dtype, bits in ((torch.bfloat16, 8), (torch.float16, 11)):
        xs = torch.linspace(0.01, 20, 4096, device=DEV).to(dtype)
        n = xs.numel()
        ones = torch.ones_like(xs)
        ys = _launch_unary(L.hb_nl_relu_fwd, xs, n, dtype, 0, ctypes.c_float(beta))
        g = _launch_binary(L.hb_nl_relu_bwd_from_out, ys, ones, n, dtype, 0, ctypes.c_float(beta)).double()
        exact = O.nl_relu_grad_ref(xs.double(), ones.double(), beta)
        yv = torch.log1p(beta * xs.double())
        rel = (g - exact).abs() / exact
        allowed = yv * 2.0 ** -bits + 2.0 ** -21 + 2.0 ** -bits    # y's rounding + __logf + the storage rounding of dx
        assert bool((rel <= allowed).all()), f"{dtype}: from-output gradient error {float((rel - allowed).max()):.3g}"
        assert float(rel.max()) > 2.0 ** -bits, f"{dtype}: the rounding of y no longer shows"


# ---------------------------------------------------------------------------------------------------------------------
# DropBlock
# ---------------------------------------------------------------------------------------------------------------------
def _mask(noise, gamma, bs):
    n, h, w = noise.shape
    mask, mbuf = guarded(n * h * w)
    kept = torch.full((1,), -1, device=DEV, dtype=torch.int64)
    assert lib().hb_dropblock_mask(ptr(noise), ptr(mask), ptr(kept), n, h, w, bs, ctypes.c_float(gamma),
                                   stream_ptr()) == 0
    torch.cuda.synchronize()
    assert_guard(mbuf, n * h * w, "mask")
    return mask.view(n, h, w), kept


def _apply(x, mask, kept, n, c, h, w, cl, dtype, offset, inplace):
    """Runs hb_dropblock_apply on a copy of x (physical NCHW or NHWC) placed `offset` elements into a guarded buffer;
    returns the output in logical NCHW."""
    phys = x.permute(0, 2, 3, 1).contiguous() if cl else x.contiguous()
    total = phys.numel()
    src, sbuf = guarded(total, dtype, offset=offset)
    src.copy_(phys.reshape(-1))
    if inplace:
        out, obuf = src, sbuf
    else:
        out, obuf = guarded(total, dtype, offset=offset)
    assert lib().hb_dropblock_apply(ptr(src), ptr(out), ptr(mask), ptr(kept), n, c, h, w, int(cl), dtype_code(src),
                                    stream_ptr()) == 0
    torch.cuda.synchronize()
    assert_guard(obuf, total, "dropblock output", offset)
    out = out.view(n, h, w, c).permute(0, 3, 1, 2) if cl else out.view(n, c, h, w)
    return out


def _noise(n, h, w, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.rand((n, h, w), device=DEV, generator=g)


@pytest.mark.parametrize("bs,h,w", [(1, 9, 11), (3, 9, 11), (7, 9, 11), (13, 9, 11), (3, 1, 17), (5, 17, 1), (3, 1, 1)])
def test_dropblock_mask_exact(bs, h, w):
    gamma = 0.3 / bs ** 2
    noise = _noise(3, h, w, 11 * bs + h)
    g32 = torch.tensor(gamma, dtype=torch.float32)
    # plant noise at exactly fp32(gamma) and one ulp on either side
    flat = noise.view(-1)
    k = flat.numel()
    flat[0] = g32
    flat[k // 2] = torch.nextafter(g32, torch.tensor(1.0)).item()
    flat[k - 1] = torch.nextafter(g32, torch.tensor(0.0)).item()
    mask, kept = _mask(noise, gamma, bs)
    ref, count = O.dropblock_mask_ref(noise.cpu(), gamma, bs)
    assert torch.equal(mask.cpu().double(), ref)
    assert int(kept.item()) == count


def test_dropblock_all_or_none_dropped():
    n, c, h, w = 2, 8, 9, 11
    x = torch.randn(n, c, h, w, device=DEV)
    # every cell a seed: everything dropped, kept 0, scale 1, output 0
    mask, kept = _mask(torch.zeros(n, h, w, device=DEV), 0.5, 3)
    assert int(kept.item()) == 0 and bool((mask == 0).all())
    out = _apply(x, mask, kept, n, c, h, w, False, torch.float32, 0, False)
    assert bool((out == 0).all())
    # no seed: nothing dropped, scale numel / numel = 1, output x
    mask, kept = _mask(torch.ones(n, h, w, device=DEV), 0.5, 3)
    assert int(kept.item()) == n * h * w
    out = _apply(x, mask, kept, n, c, h, w, True, torch.float32, 0, False)
    assert torch.equal(out, x)


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
@pytest.mark.parametrize("case", O.DB_APPLY_CASES, ids=lambda c: c[0])
def test_dropblock_apply(case, dtype):
    """Forward and backward (the same kernel on the upstream gradient) on each path. fp32 is bit-identical to the
    reference's op sequence; 16-bit lies within one ulp of x * numel / kept with the exact count."""
    name, n, c, h, w, cl, offset, inplace, route = case
    assert O.route_dropblock(n, c, h, w, dtype, cl, offset == 0, _sms()) == frozenset(route)
    gamma = 0.3 / 9
    noise = _noise(n, h, w, 5 + c)
    mask, kept = _mask(noise, gamma, 3)
    ref_mask, count = O.dropblock_mask_ref(noise.cpu(), gamma, 3)
    for seed in (1, 2):      # forward on x, backward on dy
        x = torch.randn(n, c, h, w, device=DEV, generator=torch.Generator(device=DEV).manual_seed(seed)).to(dtype)
        out = _apply(x, mask, kept, n, c, h, w, cl, dtype, offset, inplace)
        if dtype == torch.float32:
            ref = O.dropblock_reference_ops(x.cpu(), noise.cpu(), gamma, 3)
            assert torch.equal(out.cpu(), ref), (f"{name}: {int((out.cpu() != ref).sum())} of {ref.numel()} elements "
                                                 f"differ from the reference's op sequence")
        else:
            ref = O.dropblock_out_ref(x.cpu(), ref_mask, count)
            assert_bound(out.cpu(), ref, ulp(ref, BITS[dtype]), f"{name} {dtype}")


def test_dropblock_scale_bit_exact_over_counts():
    """fp32 output equals the reference's ops for many kept counts of one 2 x 56 x 56 mask: the scale numel / kept is
    rounded twice there (fl(fl(1 / kept) * numel)), which a single division misses for about a quarter of the counts."""
    n, c, h, w = 2, 8, 56, 56
    x = torch.randn(n, c, h, w, device=DEV, generator=torch.Generator(device=DEV).manual_seed(3))
    gen = torch.Generator(device=DEV).manual_seed(4)
    mismatched = []
    for trial in range(48):
        noise = torch.rand((n, h, w), device=DEV, generator=gen)
        drop = 0.02 + 0.9 * trial / 48
        mask, kept = _mask(noise, drop / 9, 3)
        out = _apply(x, mask, kept, n, c, h, w, trial % 2 == 1, torch.float32, 0, False)
        ref = O.dropblock_reference_ops(x.cpu(), noise.cpu(), drop / 9, 3)
        if not torch.equal(out.cpu(), ref):
            mismatched.append(int(kept.item()))
    assert not mismatched, f"kept counts whose output differs from the reference's: {mismatched}"


def test_dropblock_count_above_2_24_exact_and_deterministic():
    """4100 x 4100 cells (> 2^24): the kept count is exact and two runs give identical bits."""
    n, c, h, w, route = O.DB_BIG
    assert O.route_dropblock(n, c, h, w, torch.float32, False, True, _sms()) == frozenset(route)
    noise = torch.ones((n, h, w), device=DEV)
    noise.view(-1)[::4098] = 0.0          # isolated seeds (block 1): each drops one cell
    mask, kept = _mask(noise, 0.5, 1)
    count = n * h * w - (n * h * w + 4097) // 4098
    assert count % 2 == 1 and count > 2 ** 24
    assert int(kept.item()) == count, f"kept {int(kept.item())}, exact {count}"
    _, kept2 = _mask(noise, 0.5, 1)
    assert torch.equal(kept, kept2)
    x = torch.randn(n, 2, h, w, device=DEV)
    out = _apply(x, mask, kept, n, 2, h, w, False, torch.float32, 0, False)
    scale = (torch.ones(1) / torch.tensor([float(count)])) * (n * h * w)
    assert torch.equal(out, (x * mask[:, None]) * scale.to(DEV))


def test_dropblock2d_wrapper_bf16_uses_exact_count():
    """Through dropblock2d: the bf16 output is x * numel / kept with the exact count, not the reference's bf16-rounded
    count (6000 kept cells become 6016 there)."""
    n, c, h, w = 2, 16, 56, 56
    x = torch.randn(n, c, h, w, device=DEV).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    noise = _noise(n, h, w, 9)
    out = F.dropblock2d(x, 0.1, 3, noise=noise)
    mask, count = O.dropblock_mask_ref(noise.cpu(), 0.1 / 9, 3)
    ref = O.dropblock_out_ref(x.cpu(), mask, count)
    assert_bound(out.cpu(), ref, ulp(ref, 8), "dropblock2d bf16")


# ---------------------------------------------------------------------------------------------------------------------
# global average pooling
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", O.GAP_CASES, ids=lambda c: f"n{c[0]}_hw{c[1]}_c{c[2]}")
def test_gap(case):
    n, hw, c, route = case
    assert O.route_gap(n, hw, c, _sms()) == frozenset(route)
    g = torch.Generator(device=DEV).manual_seed(hw + c)
    x = (torch.randn(n, hw, c, device=DEV, generator=g, dtype=torch.float64) + 0.3).to(torch.bfloat16)
    y, ybuf = guarded(n * c, torch.bfloat16)
    assert lib().hb_gap_fwd_bf16(ptr(x), ptr(y), n, hw, c, stream_ptr()) == 0
    torch.cuda.synchronize()
    assert_guard(ybuf, n * c, "gap forward")
    x64 = x.double()
    mean = x64.mean(1)
    L = O.gap_chain(hw, c)
    bound = ulp(mean, 8) + L * O.U32 * x64.abs().sum(1) / hw
    assert_bound(y.view(n, c), mean, bound, f"gap fwd L={L}")

    dy = torch.randn(n, c, device=DEV, generator=g).to(torch.bfloat16)
    dx, dbuf = guarded(n * hw * c, torch.bfloat16)
    assert lib().hb_gap_bwd_bf16(ptr(dy), ptr(dx), n, hw, c, stream_ptr()) == 0
    torch.cuda.synchronize()
    assert_guard(dbuf, n * hw * c, "gap backward")
    ref = (dy.double() / hw)[:, None, :].expand(n, hw, c)
    bound = 0.5 * ulp(ref, 8) + 2 * O.U32 * ref.abs()
    assert_bound(dx.view(n, hw, c), ref, bound, "gap bwd")


# ---------------------------------------------------------------------------------------------------------------------
# pairwise box backward
# ---------------------------------------------------------------------------------------------------------------------
def _box_sets(m, n, gen):
    """Integer boxes (ties, touching, identical, contained), some clipped to a border, and a few real-valued ones."""
    b1 = O.integer_boxes(m, gen, span=8, border=6 if m % 2 else 0)
    b2 = O.integer_boxes(n, gen, span=8)
    k = min(m, n, 3)
    b2[:k] = b1[:k]                                       # identical pairs
    if n > k:
        b2[k] = torch.tensor([-50.0, -50.0, 50.0, 50.0])  # contains every other box
    if m > 4:                                             # two real-valued boxes: x1 <= y1 <= x2 <= y2 from sorted draws
        b1[-2:] = torch.rand(2, 4, generator=gen, dtype=torch.float64).sort(1).values * 9
    return b1.float(), b2.float()


@pytest.mark.parametrize("mode", [O.IOU, O.GIOU, O.PENALTY, O.DIOU], ids=["iou", "giou", "penalty", "diou"])
@pytest.mark.parametrize("case", O.BOX_SIZES, ids=lambda c: c[0])
def test_box_backward(case, mode):
    name, m, n, (want1, want2), route = case
    assert O.route_box(m, n, want1, want2) == frozenset(route)
    gen = torch.Generator().manual_seed(m * 1000 + n + mode)
    b1, b2 = _box_sets(m, n, gen)
    # keep union and enclosure away from zero here; the degenerate pairs have their own test
    if m:
        b1[:, 2:] = torch.maximum(b1[:, 2:], b1[:, :2] + 1)
    if n:
        b2[:, 2:] = torch.maximum(b2[:, 2:], b2[:, :2] + 1)
    gout = torch.randn(m, n, generator=gen)
    d1, d2 = b1.to(DEV), b2.to(DEV)
    g1, buf1 = guarded(4 * m)
    g2, buf2 = guarded(4 * n)
    rc = lib().hb_box_pairwise_bwd(ptr(d1), ptr(d2), ptr(gout.to(DEV)), ptr(g1) if want1 else None,
                                   ptr(g2) if want2 else None, m, n, mode, stream_ptr())
    assert rc == 0
    torch.cuda.synchronize()
    assert_guard(buf1, 4 * m, "g1")
    assert_guard(buf2, 4 * n, "g2")
    r1, r2, bound1, bound2 = O.box_grads_ref(mode, b1, b2, gout)
    if want1:
        assert_bound(g1.view(m, 4).cpu(), r1, bound1 + 2.0 ** -140, f"{name} g1")
    else:
        assert bool(torch.isnan(g1).all()), "g1 written although not requested"
    if want2:
        assert_bound(g2.view(n, 4).cpu(), r2, bound2 + 2.0 ** -140, f"{name} g2")
    else:
        assert bool(torch.isnan(g2).all()), "g2 written although not requested"


@pytest.mark.parametrize("mode", [O.IOU, O.GIOU, O.PENALTY, O.DIOU], ids=["iou", "giou", "penalty", "diou"])
def test_box_backward_degenerate_pairs_match_autograd(mode):
    """Zero-area boxes give zero-union pairs, a point repeated gives a zero enclosure: the kernel's NaN / inf pattern is
    that of torch autograd of the reference's operators in fp32, and its finite values agree."""
    b1 = torch.tensor([[1, 1, 1, 1], [2, 2, 2, 5], [0, 0, 4, 4], [3, 3, 3, 3], [1, 2, 3, 2]], dtype=torch.float32)
    b2 = torch.tensor([[1, 1, 1, 1], [2, 3, 2, 4], [0, 0, 4, 4], [5, 5, 6, 6]], dtype=torch.float32)
    gout = torch.linspace(0.5, 1.5, 20).view(5, 4)
    g1, buf1 = guarded(20)
    g2, buf2 = guarded(16)
    assert lib().hb_box_pairwise_bwd(ptr(b1.to(DEV)), ptr(b2.to(DEV)), ptr(gout.to(DEV)), ptr(g1), ptr(g2), 5, 4, mode,
                                     stream_ptr()) == 0
    torch.cuda.synchronize()
    a1, a2 = O.box_autograd(mode, b1, b2, gout)
    r1, r2, bound1, bound2 = O.box_grads_ref(mode, b1, b2, gout)
    for got, auto, ref, bound, what in ((g1.view(5, 4).cpu(), a1, r1, bound1, "g1"), (g2.view(4, 4).cpu(), a2, r2, bound2, "g2")):
        assert torch.equal(torch.isnan(got), torch.isnan(auto)), f"{what}: NaN pattern differs from autograd"
        assert torch.equal(torch.isinf(got), torch.isinf(auto)), f"{what}: inf pattern differs from autograd"
        assert_bound(got, ref, bound.nan_to_num(0, 0, 0) + 2.0 ** -140, what)


@pytest.mark.parametrize("fn", ["box_giou", "diou_loss", "ciou_loss"])
def test_box_backward_bf16_through_wrapper(fn):
    """bf16 boxes: the kernel runs in fp32 on the widened values and the gradients come back rounded to bf16; only the
    boxes1 side asks for a gradient (the ground-truth side of the YOLOv4 loss needs none)."""
    gen = torch.Generator().manual_seed(21)
    b1, b2 = _box_sets(40, 30, gen)
    b1[:, 2:] = torch.maximum(b1[:, 2:], b1[:, :2] + 1)
    b2[:, 2:] = torch.maximum(b2[:, 2:], b2[:, :2] + 1)
    a = b1.to(torch.bfloat16).to(DEV).requires_grad_(True)
    b = b2.to(torch.bfloat16).to(DEV)
    gout = torch.randn(40, 30, generator=gen)
    (getattr(ops, fn)(a, b) * gout.to(DEV)).sum().backward()
    assert a.grad.dtype == torch.bfloat16
    mode = O.GIOU if fn == "box_giou" else O.DIOU
    r1, _, bound1, _ = O.box_grads_ref(mode, a.detach().float().cpu(), b.float().cpu(), gout)
    assert_bound(a.grad.cpu(), r1, 0.5 * ulp(r1 + bound1, 8) + bound1 + 2.0 ** -130, f"{fn} bf16 g1")
