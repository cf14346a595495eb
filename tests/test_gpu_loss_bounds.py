"""The loss kernels of csrc/losses.cu through their C entry points, checked per element against the fp64 references and
bounds of tests/_loss_oracle.py on every case of tests/_loss_cases.py: the per-position loss, {sum, count, mean}, the dice
value and coefficients, and dx for the three reductions. Outputs start as NaN between sentinel guard elements, so an
element left unwritten or written out of bounds fails. The mutual channel loss adds row_lse, lse_d and, per reduction,
rdot. The shifted-logit cases run the kernels on x + c (c = 16, 100, 1000, exact in the dtype) and hold them to the
reference and bound of x, plus the one rounding of lse + c that every fp32 kernel makes. Also: bit-identical reruns
(wrap cases included), every position ignored, and the autograd wrappers on contiguous, channels-last and offset
inputs."""
import ctypes

import pytest
import torch

import holocron_b200 as hb
import _loss_cases as D
import _loss_oracle as O
from holocron_b200._lib import lib

pytestmark = pytest.mark.gpu

SENTINEL = 12345.0
PAD = 16                    # guard elements (at least 32 bytes, so offset 0 keeps 16-byte alignment)
CODE = {"float32": 0, "bfloat16": 1, "float16": 2}
KIND = {"focal": 0, "poly": 1}
_cf = ctypes.c_float
CHECKED = list(D.CASES)


def _p(t):
    return ctypes.c_void_p(0 if t is None else t.data_ptr())


class Guarded:
    """A view of ``n`` elements ``offset`` elements into a buffer of sentinels, optionally filled."""

    def __init__(self, n, dtype, offset=0, fill=float("nan"), src=None):
        self.buf = torch.full((n + offset + 2 * PAD,), SENTINEL, dtype=dtype, device="cuda")
        self.o, self.n = PAD + offset, n
        self.v = self.buf[self.o:self.o + n]
        self.v.fill_(fill)
        if src is not None:
            self.v.copy_(src.reshape(-1))

    def guards_intact(self):
        return bool((self.buf[:self.o] == SENTINEL).all()) and bool((self.buf[self.o + self.n:] == SENTINEL).all())


def _st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def run(cs, sp):
    """Calls the entry points of the case's family; returns {output name: tensor} and the guarded outputs."""
    L = lib()
    n, k, s, dt = cs.n, cs.k, cs.s, CODE[cs.dtype]
    x = Guarded(n * k * s, sp.x.dtype, cs.offset, src=sp.x.cuda())
    w = None if sp.weight is None else sp.weight.cuda().float().contiguous()
    outs, guards = {}, []

    def out(size, dtype=torch.float32, offset=0):
        g = Guarded(size, dtype, offset)
        guards.append(g)
        return g

    if cs.family == "mcl":
        cnum, xi = cs.cnum, cs.xi
        tgt = sp.target.cuda().contiguous()
        mask = sp.mask.cuda().to(torch.uint8).reshape(-1).contiguous()
        row_lse, loss_pos, lse_d, fwd_out = out(n * k), out(n * s), out(n * s), out(3)
        parts = torch.full((3 * L.hb_loss_max_partials(),), float("nan"), dtype=torch.float64, device="cuda")
        assert L.hb_mcl_fwd(_p(x.v), _p(tgt), _p(w), _p(mask), _p(row_lse.v), _p(loss_pos.v), _p(lse_d.v), _p(parts),
                            _p(fwd_out.v), n, cnum, xi, s, sp.ignore_index, _cf(sp.alpha), dt, _st()) == 0
        outs.update(row_lse=row_lse.v, loss=loss_pos.v, lse_d=lse_d.v, sum=fwd_out.v[0:1], count=fwd_out.v[1:2],
                    mean=fwd_out.v[2:3])
        for red, code in (("none", 0), ("mean", 1), ("sum", 2)):
            gout = sp.gout.cuda().float() if red == "none" else torch.tensor([sp.gscalar], device="cuda")
            rdot, dx = out(n * k), out(n * k * s, sp.x.dtype, cs.offset)
            assert L.hb_mcl_bwd(_p(x.v), _p(tgt), _p(w), _p(mask), _p(row_lse.v), _p(lse_d.v), _p(gout), _p(fwd_out.v),
                                _p(rdot.v), _p(dx.v), n, cnum, xi, s, sp.ignore_index, _cf(sp.alpha), code, dt,
                                _st()) == 0
            outs[f"rdot_{red}"], outs[f"dx_{red}"] = rdot.v, dx.v.view(n, k, s)
        torch.cuda.synchronize()
        return outs, guards
    if cs.family == "dice":
        t = Guarded(n * k * s, sp.x.dtype, cs.offset, src=sp.target.cuda())
        scratch = torch.full((L.hb_dice_scratch_doubles(k),), float("nan"), dtype=torch.float64, device="cuda")
        val, coef = out(1), out(2 * k)
        assert L.hb_dice_fwd(_p(x.v), _p(t.v), _p(w), _p(scratch), _p(val.v), _p(coef.v), n, k, s, _cf(sp.gamma),
                             _cf(sp.eps), dt, _st()) == 0
        gout = torch.tensor([sp.gscalar], device="cuda")
        dx = out(n * k * s, sp.x.dtype, cs.offset)
        assert L.hb_dice_bwd(_p(t.v), _p(coef.v), _p(gout), _p(dx.v), n, k, s, dt, _st()) == 0
        torch.cuda.synchronize()
        return {"loss": val.v, "coef": coef.v, "dx": dx.v}, guards
    soft = cs.family == "soft"
    tgt = Guarded(n * k * s, sp.x.dtype, cs.offset, src=sp.target.cuda()).v if soft else sp.target.cuda().contiguous()
    loss_pos, fwd_out = out(n * s), out(3)
    parts = torch.full((3 * L.hb_loss_max_partials(),), float("nan"), dtype=torch.float64, device="cuda")
    if cs.family == "hard":
        rc = L.hb_cls_loss_hard_fwd(_p(x.v), _p(tgt), _p(w), _p(loss_pos.v), _p(parts), _p(fwd_out.v), n, k, s,
                                    sp.ignore_index, KIND[sp.kind], _cf(sp.gamma), _cf(sp.eps), dt, _st())
    elif soft:
        rc = L.hb_poly_soft_fwd(_p(x.v), _p(tgt), _p(w), _p(loss_pos.v), _p(parts), _p(fwd_out.v), n, k, s,
                                sp.ignore_index, _cf(sp.eps), dt, _st())
    else:
        rc = L.hb_cce_fwd(_p(x.v), _p(tgt), _p(w), _p(loss_pos.v), _p(parts), _p(fwd_out.v), n, k, s, sp.ignore_index,
                          _cf(sp.gamma), dt, _st())
    assert rc == 0
    outs.update(loss=loss_pos.v, sum=fwd_out.v[0:1], count=fwd_out.v[1:2], mean=fwd_out.v[2:3])
    for red, code in (("none", 0), ("mean", 1), ("sum", 2)):
        gout = sp.gout.cuda().float() if red == "none" else torch.tensor([sp.gscalar], device="cuda")
        dx = out(n * k * s, sp.x.dtype, cs.offset)
        if cs.family == "hard":
            rc = L.hb_cls_loss_hard_bwd(_p(x.v), _p(tgt), _p(w), _p(gout), _p(fwd_out.v), _p(dx.v), n, k, s,
                                        sp.ignore_index, KIND[sp.kind], _cf(sp.gamma), _cf(sp.eps), code, dt, _st())
        elif soft:
            rc = L.hb_poly_soft_bwd(_p(x.v), _p(tgt), _p(w), _p(gout), _p(dx.v), n, k, s, sp.ignore_index,
                                    _cf(sp.eps), code, dt, _st())
        else:
            rc = L.hb_cce_bwd(_p(x.v), _p(tgt), _p(w), _p(gout), _p(fwd_out.v), _p(dx.v), n, k, s, sp.ignore_index,
                              _cf(sp.gamma), code, dt, _st())
        assert rc == 0
        outs[f"dx_{red}"] = dx.v.view(n, k, s)
    torch.cuda.synchronize()
    if soft:
        assert float(fwd_out.v[1]) == n * s
    return outs, guards


@pytest.mark.parametrize("name", CHECKED)
def test_per_element_bounds(name):
    cs = D.CASES[name]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for i, prm in enumerate(O.params(cs)):
        sp = O.make_spec(cs, prm, seed=i, sms=sms)
        got, guards = run(cs, sp)
        ref = O.reference(cs.family, sp, device="cuda")
        what = f"{D.describe(cs, sms)} {prm}"
        for key, c in ref.items():
            O.assert_within(got[key], c, f"{what} {key}")
        assert all(g.guards_intact() for g in guards), f"{what}: wrote outside an output"


@pytest.mark.parametrize("name", [n for n in CHECKED if not D.CASES[n].light][::7]
                         + [n for n in CHECKED if D.CASES[n].wrap])
def test_bit_identical_reruns(name):
    cs = D.CASES[name]
    sp = O.make_spec(cs, O.params(cs)[-1], seed=5)
    a, _ = run(cs, sp)
    b, _ = run(cs, sp)
    for key in a:
        assert torch.equal(a[key].view(torch.uint8) if a[key].dtype != torch.float32 else a[key].view(torch.int32),
                           b[key].view(torch.uint8) if b[key].dtype != torch.float32 else b[key].view(torch.int32)), key


@pytest.mark.parametrize("name", ["hard_float32_n3k5s16", "hard_bfloat16_n37k33s1", "hard_float16_n3k33s16",
                                  "cce_float32_n3k5s16", "cce_bfloat16_n37k33s1"])
def test_every_position_ignored(name):
    """mean is NaN (0 / 0), sum is 0, and the mean / sum gradients are exactly 0 (complement CE without its
    complement term, which counts every position)."""
    cs = D.CASES[name]
    for prm in O.params(cs):
        if not 0 <= prm[4] < cs.k or prm[1] != 0 and cs.family == "cce":
            continue
        sp = O.make_spec(cs, prm, seed=3, all_ignored=True)
        got, _ = run(cs, sp)
        assert float(got["sum"]) == 0.0 and float(got["count"]) == 0.0 and torch.isnan(got["mean"]).all(), prm
        assert not got["dx_sum"].abs().any() and not got["dx_mean"].abs().any(), prm


@pytest.mark.parametrize("dtype", list(CODE))
def test_autograd_wrappers_agree_across_layouts(dtype):
    """nn/_losses.py: contiguous and channels-last inputs give bit-identical values and gradients. An input one element
    off its alignment takes the entry points' scalar paths (checked per element above), so it agrees within the
    dtype's rounding."""
    dt = O.DT[dtype]
    torch.manual_seed(0)
    x0 = (torch.randn(2, 12, 8, 8) * 2).to(dt).cuda()
    t = torch.randint(0, 12, (2, 8, 8), device="cuda")
    soft = torch.softmax(torch.randn(2, 12, 8, 8, device="cuda"), 1).to(dt)
    onehot = (torch.rand(2, 12, 8, 8, device="cuda") < 0.3).to(dt)
    t4 = torch.randint(0, 4, (2, 8, 8), device="cuda")

    def mcl(a):
        torch.manual_seed(1)        # the same channel mask for every layout
        return F.mutual_channel_loss(a, t4, xi=3, alpha=1.5)

    F = hb.nn.functional
    fns = [lambda a: F.focal_loss(a, t, gamma=2.0), lambda a: F.poly_loss(a, t, eps=1.0),
           lambda a: F.poly_loss(a, soft, eps=2.0), lambda a: F.multilabel_cross_entropy(a, soft),
           lambda a: F.complement_cross_entropy(a, t, gamma=-1), lambda a: F.dice_loss(a.sigmoid(), onehot), mcl]
    buf = torch.empty(x0.numel() + 1, dtype=dt, device="cuda")
    views = [x0.clone(), x0.clone().to(memory_format=torch.channels_last), buf[1:].view_as(x0).copy_(x0)]
    for j, fn in enumerate(fns):
        res = []
        for v in views:
            a = v.detach().requires_grad_(True)
            y = fn(a)
            (g,) = torch.autograd.grad(y, a)
            res.append((y.float(), g.contiguous().float()))
        assert torch.equal(res[1][0], res[0][0]) and torch.equal(res[1][1], res[0][1]), (dtype, j)
        tol = {"float32": 1e-5, "bfloat16": 1.6e-2, "float16": 2e-3}[dtype]
        torch.testing.assert_close(res[2][0], res[0][0], rtol=tol, atol=1e-6)
        torch.testing.assert_close(res[2][1], res[0][1], rtol=tol, atol=tol * float(res[0][1].abs().max()))
