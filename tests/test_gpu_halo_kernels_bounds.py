"""The involution (csrc/involution.cu) and lambda (csrc/lambda_layer.cu) kernels per element, through the C ABI, on every
path of the case tables in tests/_halo_kernels_oracle.py.

Each entry point is checked on its own against the fp64 oracle of that file, fed exactly the operands the kernel gets
(the upstream intermediates are the oracle's, rounded to the type the kernel reads), with the per-element bound of
tests/_bounds.py: one ulp of the output type plus 1e-5 of the sum of |terms|. Outputs, and the dR scratch, start
NaN-filled between guard words that must come back unchanged; padding channels of every output must come out exactly
zero; the padding the kernels' headers say is never read holds NaN. Every launch runs twice and must give the same
bits. Refused calls must change no byte and launch nothing. Keys of -inf must follow torch.softmax."""
import pytest
import torch

import _halo_kernels_oracle as O
from _bounds import assert_within
from _lambda_oracle import lambda_core
from holocron_b200._lib import lib, ptr, stream_ptr

pytestmark = pytest.mark.gpu
DEV = "cuda"
GUARD = 64          # elements on each side of an output; keeps the view 16-byte aligned
NAN = float("nan")
BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


class Out:
    """A NaN-filled output of ``shape`` between GUARD elements of random bits on each side (``.t`` is the view)."""

    def __init__(self, shape, dtype):
        n = 1
        for s in shape:
            n *= s
        self.n = n
        self.buf = torch.empty(n + 2 * GUARD, dtype=dtype, device=DEV)
        ib = torch.int16 if dtype == BF16 else torch.int32
        self.buf.view(ib).random_(-2 ** 15, 2 ** 15)
        self.guard = self.buf.clone()
        self.t = self.buf[GUARD:GUARD + n].view(shape)
        self.refill()

    def refill(self):
        self.t.fill_(NAN)

    def bits(self):
        return self.t.view(torch.int16 if self.t.dtype == BF16 else torch.int32).clone()

    def check_guard(self, what):
        ib = torch.int16 if self.buf.dtype == BF16 else torch.int32
        a, b = self.buf.view(ib), self.guard.view(ib)
        assert torch.equal(a[:GUARD], b[:GUARD]), f"{what}: guard words before the output overwritten"
        assert torch.equal(a[GUARD + self.n:], b[GUARD + self.n:]), f"{what}: guard words after the output overwritten"


def _launch(call, outs, what):
    """Runs ``call`` twice into NaN-refilled outputs: both runs return 0, leave the guards alone and give the same bits."""
    assert call() == 0, f"{what}: launch failed"
    torch.cuda.synchronize()
    first = [o.bits() for o in outs]
    for o in outs:
        o.check_guard(what)
        o.refill()
    assert call() == 0, f"{what}: second launch failed"
    torch.cuda.synchronize()
    for o, f in zip(outs, first):
        o.check_guard(what)
        same = o.bits() == f
        if not bool(same.all()):
            i = tuple(int(j) for j in (~same).nonzero()[0])
            raise AssertionError(f"{what}: two runs differ in {int((~same).sum())} elements, first at {i}")


def _assert_zero(t, c0, what):
    """The padding channels c0.. of t (the last dimension) hold exactly zero."""
    pad = t[..., c0:]
    bad = pad.float() != 0
    if bool(bad.any()):
        i = tuple(int(j) for j in bad.nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} padding elements not zero, first at {i[:-1] + (c0 + i[-1],)}: "
                             f"{float(pad[i])}")


def _assert_equal(got, ref, what):
    bad = got.to(F64) != ref
    if bool(bad.any()):
        i = tuple(int(j) for j in bad.nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} elements differ, first at {i}: got {float(got[i])}, "
                             f"ref {float(ref[i])}")


def _operand(gen, shape, c, scale=1.0, pad=NAN):
    """bf16 [..., Cp] with c random logical channels and the padding channels set to ``pad``."""
    t = torch.full(shape, pad, device=DEV, dtype=BF16)
    t[..., :c] = (torch.randn(*shape[:-1], c, generator=gen, device=DEV, dtype=F32) * scale).to(BF16)
    return t


# ---------------------------------------------------------------------------------------------------------------------
# involution
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", O.INV_CASES, ids=lambda c: c[0])
def test_involution(case):
    N, H, W, C, Cp, Kp, K, G, s, p, d = geom = O.inv_case_geom(case)
    assert case[-1] <= O.route_involution(*geom, _sms())
    Ho, Wo = O.window_out(H, K, s, p, d), O.window_out(W, K, s, p, d)
    gk = G * K * K
    gen = torch.Generator(device=DEV).manual_seed(len(case[0]) * 1000 + N * H * W)
    x = _operand(gen, (N, H, W, Cp), C)
    ker = _operand(gen, (N, Ho, Wo, Kp), gk)
    dy = _operand(gen, (N, Ho, Wo, Cp), C)
    y, dx, dker = Out((N, Ho, Wo, Cp), BF16), Out((N, H, W, Cp), BF16), Out((N, Ho, Wo, Kp), BF16)
    L = lib()
    args = (N, H, W, C, Cp, Kp, K, G, s, p, d)
    _launch(lambda: L.hb_involution_fwd_bf16(ptr(x), ptr(ker), ptr(y.t), *args, stream_ptr()), [y], "fwd")
    _launch(lambda: L.hb_involution_bwd_data_bf16(ptr(dy), ptr(ker), ptr(dx.t), *args, stream_ptr()), [dx], "bwd_data")
    _launch(lambda: L.hb_involution_bwd_kernel_bf16(ptr(x), ptr(dy), ptr(dker.t), *args, stream_ptr()), [dker],
            "bwd_kernel")
    (y_ref, dx_ref, dk_ref), (y_abs, dx_abs, dk_abs) = O.inv_oracle(
        x[..., :C].to(F64), ker[..., :gk].to(F64), dy[..., :C].to(F64), K, G, s, p, d)
    assert_within(y.t[..., :C], y_ref, y_abs, "y")
    assert_within(dx.t[..., :C], dx_ref, dx_abs, "dx")
    assert_within(dker.t[..., :gk], dk_ref, dk_abs, "dker")
    _assert_zero(y.t, C, "y")
    _assert_zero(dx.t, C, "dx")
    _assert_zero(dker.t, gk, "dker")


def _snapshot(ts):
    return [t.view(torch.uint8).clone() for t in ts]


def _assert_untouched(ts, before, what):
    for i, (t, b) in enumerate(zip(ts, before)):
        assert torch.equal(t.view(torch.uint8), b), f"{what}: buffer {i} changed"


def _refused(call, bufs, what):
    torch.cuda.synchronize()
    before = _snapshot(bufs)
    L = lib()
    L.hb_launch_count_reset()
    rc = call()
    launches = L.hb_launch_count()
    torch.cuda.synchronize()
    assert rc == 1, f"{what}: returned {rc}, expected cudaErrorInvalidValue"
    assert launches == 0, f"{what}: {launches} kernels launched"
    _assert_untouched(bufs, before, what)


SPACE = 1 << 20     # elements of every buffer of the refusal tests: more than any refused geometry could reach


def _space(dtype, gen):
    t = torch.empty(SPACE, device=DEV, dtype=dtype)
    t.view(torch.int16 if dtype == BF16 else torch.int32).random_(-2 ** 15, 2 ** 15, generator=gen)
    return t


def test_involution_refusals_touch_nothing():
    gen = torch.Generator(device=DEV).manual_seed(5)
    bufs = [_space(BF16, gen) for _ in range(3)]
    L = lib()
    n = 0
    for name, changes, want in O.INV_ROWS:
        g = {**O.INV_BASE, **changes}
        if g["N"] * max(g["H"], 1) * max(g["W"], 1) * max(g["Cp"], g["Kp"], 1) > 1 << 16:
            continue        # the 2^31 rows: a launch could reach past these buffers, so they are checked without a GPU
        geom = [g[k] for k in O.INV_KEYS]
        assert O.inv_refused(*geom) == want
        if not want:
            continue
        for entry in ("fwd", "bwd_data", "bwd_kernel"):
            fn = getattr(L, f"hb_involution_{entry}_bf16")
            _refused(lambda: fn(ptr(bufs[0]), ptr(bufs[1]), ptr(bufs[2]), *geom, stream_ptr()), bufs, f"{name} {entry}")
            n += 1
    assert n >= 30


# ---------------------------------------------------------------------------------------------------------------------
# lambda
# ---------------------------------------------------------------------------------------------------------------------
def _lam_inputs(geom, seed):
    B, H, W, dk, u, heads, dv, r, Cqp, Ckp, Cvp, Cop = geom
    hw = H * W
    gen = torch.Generator(device=DEV).manual_seed(seed)
    q = _operand(gen, (B, hw, Cqp), heads * dk)
    k = _operand(gen, (B, hw, Ckp), dk * u, 2.0)
    v = _operand(gen, (B, hw, Cvp), dv * u, pad=0.0)      # v's padding is read (weighted by zero): it holds zeros
    dy = _operand(gen, (B, hw, Cop), heads * dv)
    R = Rt = lp = dvpos = None
    if r:
        R = torch.randn(dk, u, r, r, generator=gen, device=DEV).to(BF16).float()
        Rt = R.reshape(dk, u, r * r).permute(2, 1, 0).contiguous()
    else:
        lp = torch.randn(B, hw, dk, dv, generator=gen, device=DEV) * 0.5
        dvpos = torch.randn(B, hw, dv * u, generator=gen, device=DEV) * 0.5
    return q, k, v, dy, R, Rt, lp, dvpos


def _f64(t, c=None):
    return None if t is None else (t if c is None else t[..., :c]).to(F64)


@pytest.mark.parametrize("case", O.LAM_CASES, ids=lambda c: c[0])
def test_lambda(case):
    geom = O.lam_case_geom(case)
    B, H, W, dk, u, heads, dv, r, Cqp, Ckp, Cvp, Cop = geom
    assert case[-1] <= O.route_lambda(*geom[:8], _sms())
    hw, dvp, rr = H * W, O.round_up(dv, 8), r * r
    q, k, v, dy, R, Rt, lp, dvpos = _lam_inputs(geom, sum(geom))
    q64, k64, v64, dy64 = _f64(q, heads * dk), _f64(k, dk * u), _f64(v, dv * u), _f64(dy, heads * dv)
    R64, lp64, dvpos64 = _f64(R), _f64(lp), _f64(dvpos)
    L = lib()
    st = stream_ptr

    # key softmax statistics and the content lambda
    stats, lc = Out((B, dk * u, 2), F32), Out((B, dk, dv), F32)
    _launch(lambda: L.hb_lambda_content_fwd_bf16(ptr(k), ptr(v), ptr(stats.t), ptr(lc.t), *geom, st()), [stats, lc],
            "content_fwd")
    mx, sm = O.lam_stats(k64, dk, u)
    _assert_equal(stats.t[..., 0], mx, "stats max")
    assert_within(stats.t[..., 1], sm, sm, "stats sum", bits=24)
    sig = O.lam_sigma(k64, mx, sm, dk, u)
    lc_ref, lc_abs = O.lam_lc(sig, v64, dv, u)
    assert_within(lc.t, lc_ref, lc_abs, "lc", bits=24)
    # what the later kernels are fed: the oracle's intermediates in the kernels' types
    stats_in = torch.stack([mx, sm], -1).float()
    mx_in, sm_in = stats_in[..., 0].to(F64), stats_in[..., 1].to(F64)
    lc_in = lc_ref.float()

    y = Out((B, hw, Cop), BF16)
    _launch(lambda: L.hb_lambda_out_fwd_bf16(ptr(q), ptr(v), ptr(Rt), ptr(lc_in), ptr(lp), ptr(y.t), *geom, st()), [y],
            "out_fwd")
    y_ref, y_abs = O.lam_y(q64, v64, R64, lc_in.to(F64), lp64, H, W, dk, u, heads, dv, r)
    assert_within(y.t[..., :heads * dv], y_ref, y_abs, "y")
    _assert_zero(y.t, heads * dv, "y")

    dlc, dkt = Out((B, dk, dv), F32), Out((B, hw, Ckp), BF16)
    _launch(lambda: L.hb_lambda_bwd_content_bf16(ptr(q), ptr(k), ptr(v), ptr(dy), ptr(stats_in), ptr(dlc.t),
                                                  ptr(dkt.t), *geom, st()), [dlc, dkt], "bwd_content")
    dlc_ref, dlc_abs = O.lam_dlc(q64, dy64, dk, heads, dv)
    assert_within(dlc.t, dlc_ref, dlc_abs, "dlc", bits=24)
    dk_ref, dk_abs = O.lam_dk(k64, v64, mx_in, sm_in, dlc_ref, dlc_abs, dk, u, dv)
    assert_within(dkt.t[..., :dk * u], dk_ref, dk_abs, "dk")
    _assert_zero(dkt.t, dk * u, "dk")
    dlc_in = dlc_ref.float()

    dlp = Out((B, hw, dk, dvp), BF16)
    _launch(lambda: L.hb_lambda_dlp_bf16(ptr(q), ptr(dy), ptr(dlp.t), *geom, st()), [dlp], "dlp")
    dlp_ref, dlp_abs = O.lam_dlp(q64, dy64, dk, heads, dv)
    assert_within(dlp.t[..., :dv], dlp_ref, dlp_abs, "dlp")
    _assert_zero(dlp.t, dv, "dlp")
    dlp_in = torch.zeros(B, hw, dk, dvp, device=DEV, dtype=BF16)
    dlp_in[..., :dv] = dlp_ref.to(BF16)

    dq = Out((B, hw, Cqp), BF16)
    _launch(lambda: L.hb_lambda_bwd_q_bf16(ptr(dy), ptr(v), ptr(Rt), ptr(lc_in), ptr(lp), ptr(dq.t), *geom, st()), [dq],
            "bwd_q")
    dq_ref, dq_abs = O.lam_dq(dy64, v64, R64, lc_in.to(F64), lp64, H, W, dk, u, heads, dv, r)
    assert_within(dq.t[..., :heads * dk], dq_ref, dq_abs, "dq")
    _assert_zero(dq.t, heads * dk, "dq")

    dvo = Out((B, hw, Cvp), BF16)
    _launch(lambda: L.hb_lambda_bwd_v_bf16(ptr(k), ptr(stats_in), ptr(dlc_in), ptr(dlp_in), ptr(Rt), ptr(dvpos),
                                           ptr(dvo.t), *geom, st()), [dvo], "bwd_v")
    dv_ref, dv_abs = O.lam_dv(k64, mx_in, sm_in, dlc_in.to(F64), dlp_in[..., :dv].to(F64), R64, dvpos64, H, W, dk, u,
                              dv, r)
    assert_within(dvo.t[..., :dv * u], dv_ref, dv_abs, "dv")
    _assert_zero(dvo.t, dv * u, "dv")

    if not r:
        return
    scratch, dR = Out((B, dk, u, rr), F32), Out((dk, u, rr), F32)
    _launch(lambda: L.hb_lambda_bwd_r_bf16(ptr(dlp_in), ptr(v), ptr(scratch.t), ptr(dR.t), *geom, st()),
            [scratch, dR], "bwd_r")
    part_ref, part_abs = O.lam_dr_partials(dlp_in[..., :dv].to(F64), v64, H, W, dk, u, dv, r)
    assert_within(scratch.t, part_ref, part_abs, "dR partials", bits=24)
    seq = torch.zeros(dk, u, rr, device=DEV, dtype=F32)
    for b in range(B):
        seq = seq + scratch.t[b]
    assert torch.equal(dR.t, seq), "dR is not the partials added in sample order"
    assert_within(dR.t, part_ref.sum(0), part_abs.sum(0), "dR", bits=24)


def _lam_calls(geom, bufs, null=frozenset()):
    """entry point -> a call of it on ``geom`` with every operand in one of ``bufs`` (NULL for the names in ``null``)."""
    L = lib()
    b16, f32 = bufs
    P = lambda i: ptr(b16[i])                                        # noqa: E731
    F = lambda i, name=None: ptr(None if name in null else f32[i])   # noqa: E731
    dlp = ptr(None if "dlp" in null else b16[4])
    return {
        "content_fwd": lambda: L.hb_lambda_content_fwd_bf16(P(0), P(1), F(0), F(1), *geom, stream_ptr()),
        "out_fwd": lambda: L.hb_lambda_out_fwd_bf16(P(0), P(1), F(2, "Rt"), F(1), F(3, "lp"), P(2), *geom, stream_ptr()),
        "bwd_content": lambda: L.hb_lambda_bwd_content_bf16(P(0), P(1), P(2), P(3), F(0), F(1), P(5), *geom,
                                                            stream_ptr()),
        "dlp": lambda: L.hb_lambda_dlp_bf16(P(0), P(3), P(4), *geom, stream_ptr()),
        "bwd_q": lambda: L.hb_lambda_bwd_q_bf16(P(3), P(1), F(2, "Rt"), F(1), F(3, "lp"), P(5), *geom, stream_ptr()),
        "bwd_v": lambda: L.hb_lambda_bwd_v_bf16(P(1), F(0), F(1), dlp, F(2, "Rt"), F(3, "dvpos"), P(5), *geom,
                                                stream_ptr()),
        "bwd_r": lambda: L.hb_lambda_bwd_r_bf16(dlp, P(1), F(4), F(5), *geom, stream_ptr()),
    }


def test_lambda_refusals_touch_nothing():
    gen = torch.Generator(device=DEV).manual_seed(6)
    bufs = ([_space(BF16, gen) for _ in range(6)], [_space(F32, gen) for _ in range(6)])
    flat = bufs[0] + bufs[1]
    n = 0
    for name, changes, want in O.LAM_ROWS:
        g = {**O.LAM_BASE, **changes}
        if g["B"] * max(g["H"], 1) * max(g["W"], 1) * max(g["Cqp"], g["Ckp"], g["Cvp"], g["Cop"]) > 1 << 16:
            continue        # the 2^31 and grid rows: a launch could reach past these buffers; checked without a GPU
        geom = [g[k] for k in O.LAM_KEYS]
        assert O.lam_refused(*geom) == want
        if not want:
            continue
        for entry, call in _lam_calls(geom, bufs).items():
            _refused(call, flat, f"{name} {entry}")
            n += 1
    for name, changes, null in O.LAM_POINTER_ROWS:
        g = {**O.LAM_BASE, **changes}
        geom = [g[k] for k in O.LAM_KEYS]
        for entry, call in _lam_calls(geom, bufs, frozenset(null)).items():
            if O.lam_pointer_refused(entry, g["r"], frozenset(null)):
                _refused(call, flat, f"{name} {entry}")
                n += 1
    g = {**O.LAM_BASE, "r": 0}
    _refused(_lam_calls([g[k] for k in O.LAM_KEYS], bufs)["bwd_r"], flat, "global bwd_r")
    assert n >= 7 * 18


def _check_torch(got, ref, abs_sum, what, rel=1e-5):
    """NaN exactly where torch's value is NaN; elsewhere the per-element bound."""
    got64 = got.to(F64)
    nan_ref = torch.isnan(ref)
    bad = torch.isnan(got64) != nan_ref
    if bool(bad.any()):
        i = tuple(int(j) for j in bad.nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} elements NaN where torch is not or the reverse, first at {i}: "
                             f"got {float(got64[i])}, torch {float(ref[i])}")
    z = torch.zeros_like(ref)
    assert_within(torch.where(nan_ref, z, got64), torch.where(nan_ref, z, ref), torch.where(nan_ref, z, abs_sum), what,
                  rel)


def test_lambda_neg_inf_keys():
    """Keys of -inf get weight 0, as in torch.softmax, and a row of -inf keys gives NaN where torch gives it. The keys
    at positions 0..255 of some rows are -inf, so every thread of the statistics pass meets one first; one row is -inf
    at every position. The kernels run as the layer chains them, each fed its upstream kernel's output."""
    B, H, W, dk, u, heads, dv, r = 2, 20, 20, 8, 2, 2, 16, 5
    geom = (B, H, W, dk, u, heads, dv, r, heads * dk, dk * u, dv * u, heads * dv)
    hw, dvp, ninf = H * W, O.round_up(dv, 8), -float("inf")
    q, k, v, dy, R, Rt, _, _ = _lam_inputs(geom, 11)
    k[0, :256, [0, 3, 5]] = ninf
    k[1, :256, 7] = ninf
    k[1, :, 2] = ninf
    L = lib()
    st = stream_ptr
    stats, lc = Out((B, dk * u, 2), F32), Out((B, dk, dv), F32)
    _launch(lambda: L.hb_lambda_content_fwd_bf16(ptr(k), ptr(v), ptr(stats.t), ptr(lc.t), *geom, st()), [stats, lc],
            "content_fwd")
    y = Out((B, hw, heads * dv), BF16)
    _launch(lambda: L.hb_lambda_out_fwd_bf16(ptr(q), ptr(v), ptr(Rt), ptr(lc.t), None, ptr(y.t), *geom, st()), [y],
            "out_fwd")
    dlc, dkt = Out((B, dk, dv), F32), Out((B, hw, dk * u), BF16)
    _launch(lambda: L.hb_lambda_bwd_content_bf16(ptr(q), ptr(k), ptr(v), ptr(dy), ptr(stats.t), ptr(dlc.t),
                                                  ptr(dkt.t), *geom, st()), [dlc, dkt], "bwd_content")
    dlp = Out((B, hw, dk, dvp), BF16)
    _launch(lambda: L.hb_lambda_dlp_bf16(ptr(q), ptr(dy), ptr(dlp.t), *geom, st()), [dlp], "dlp")
    dq = Out((B, hw, heads * dk), BF16)
    _launch(lambda: L.hb_lambda_bwd_q_bf16(ptr(dy), ptr(v), ptr(Rt), ptr(lc.t), None, ptr(dq.t), *geom, st()), [dq],
            "bwd_q")
    dvo = Out((B, hw, dv * u), BF16)
    _launch(lambda: L.hb_lambda_bwd_v_bf16(ptr(k), ptr(stats.t), ptr(dlc.t), ptr(dlp.t), ptr(Rt), None, ptr(dvo.t),
                                           *geom, st()), [dvo], "bwd_v")
    scratch, dR = Out((B, dk, u, r * r), F32), Out((dk, u, r * r), F32)
    _launch(lambda: L.hb_lambda_bwd_r_bf16(ptr(dlp.t), ptr(v), ptr(scratch.t), ptr(dR.t), *geom, st()), [scratch, dR],
            "bwd_r")

    def nchw(t):
        return t.to(F64).permute(0, 2, 1).reshape(B, t.shape[-1], H, W)

    def nhwc(t):
        return t.reshape(B, t.shape[1], hw).permute(0, 2, 1)

    q64, k64, v64, R64 = (nchw(q).requires_grad_(True), nchw(k).requires_grad_(True), nchw(v).requires_grad_(True),
                          R.to(F64).reshape(dk, u, 1, r, r).requires_grad_(True))
    ref = lambda_core(q64, k64, v64, R64, dk, u, heads, r)
    ref.backward(nchw(dy))
    qa, va, Ra = (nchw(q).abs().requires_grad_(True), nchw(v).abs().requires_grad_(True),
                  R.to(F64).abs().reshape(dk, u, 1, r, r).requires_grad_(True))
    refa = lambda_core(qa, nchw(k), va, Ra, dk, u, heads, r)
    refa.backward(nchw(dy).abs())
    mx, sm = O.lam_stats(k.to(F64), dk, u)
    dlc_ref, dlc_abs = O.lam_dlc(q.to(F64), dy.to(F64), dk, heads, dv)
    _, dk_abs = O.lam_dk(k.to(F64), v.to(F64), mx, sm, dlc_ref, dlc_abs, dk, u, dv)
    _check_torch(y.t, nhwc(ref.detach()), nhwc(refa.detach()), "y")
    _check_torch(dq.t, nhwc(q64.grad), nhwc(qa.grad), "dq")
    _check_torch(dkt.t, nhwc(k64.grad), dk_abs, "dk")
    # dv and dR take the per-position gradient of the position lambda through the bf16 dlp: 2^-8 of the terms
    _check_torch(dvo.t, nhwc(v64.grad), nhwc(va.grad), "dv", rel=4e-3)
    _check_torch(dR.t, R64.grad.reshape(dk, u, r * r), Ra.grad.reshape(dk, u, r * r), "dR", rel=4e-3)
    # the statistics: the max over the finite keys, the sum over them; (-inf, 0) for a row of -inf keys
    _assert_equal(stats.t[..., 0], mx, "stats max")
    _check_torch(stats.t[..., 1], sm, sm, "stats sum")
    assert float(stats.t[1, 2, 0]) == -float("inf") and float(stats.t[1, 2, 1]) == 0.0
    # the partly -inf rows are finite, as torch's are
    assert bool(torch.isfinite(y.t[0].float()).all()) and bool(torch.isfinite(lc.t[0]).all())
