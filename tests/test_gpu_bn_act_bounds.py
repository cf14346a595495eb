"""The fused BatchNorm / activation kernels (csrc/bn_act.cu) and the squeeze-excite gate (csrc/se_gate.cu) per element,
against the fp64 restatement and bounds of tests/_bn_oracle.py.

Each kernel is launched through the C ABI on its own inputs, so a failure names the kernel: statistics (stand-alone
partials + finalize, eval affine), forward, backward. Outputs are pre-filled with NaN so an unwritten element shows, and
sit in front of a guard band that must come back unchanged. Then the mode matrix end to end through ``bn_act`` /
``act_only``, the per-thread cp.async ring at sizes where every lane wraps it more than twice, non-finite inputs and the
gate kernels. fp64 references are computed on the GPU."""
import ctypes

import pytest
import torch

from holocron_b200._lib import lib, ptr, stream_ptr
from holocron_b200.nn import _fused as K
from holocron_b200.trainer import freeze_bn

import _bn_oracle as O
from _bounds import check_stats

pytestmark = pytest.mark.gpu
DEV = "cuda"
GUARD = 64
SENTINEL = 12345.0
EPS = 1e-5
SLOPE = 0.1


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def guarded(n, dtype=torch.float32, fill=float("nan")):
    """(view of n elements, whole buffer): the view is pre-filled with ``fill`` and followed by GUARD sentinels."""
    buf = torch.full((n + GUARD,), SENTINEL, device=DEV, dtype=dtype)
    buf[:n] = fill
    return buf[:n], buf


def assert_guard(buf, n, what):
    g = buf[n:]
    assert bool((g == SENTINEL).all()), f"{what}: guard band overwritten"


def bf16_rows(m, c, mu=0.0, sigma=1.0, gen=None):
    """[M, C] bf16 rows u = mu + sigma * randn (mu, sigma per channel or scalars)."""
    return (mu + sigma * torch.randn(m, c, device=DEV, generator=gen, dtype=torch.float64)).to(torch.bfloat16)


def _gen(seed):
    g = torch.Generator(device=DEV)
    g.manual_seed(seed)
    return g


def _f32(x):
    return x.to(torch.float32).contiguous()


def _d(x):
    return x.detach().to(torch.float64)


# ---------------------------------------------------------------------------------------------------------------------
# raw launches
# ---------------------------------------------------------------------------------------------------------------------
def stats_partials(u):
    m, c = u.shape
    cap = lib().hb_bn_stat_slots_max()
    parts, _ = guarded(cap * c * 2)
    sl = ctypes.c_int(-1)
    assert lib().hb_bn_stats_partials_bf16(ptr(u), m, c, ptr(parts), ctypes.byref(sl), stream_ptr()) == 0
    return parts.view(cap, c, 2), sl.value


def finalize(parts, slots, gammas, betas, rms, rvs, nbts, c, c_log, m, momentum):
    """Returns guarded [4][B][C] (mean, rstd, scale, shift) and its buffer."""
    nb = len(parts)
    out, buf = guarded(4 * nb * c)
    out = out.view(4, nb, c)
    rc = lib().hb_bn_finalize(K._arr3(parts), K._I3(*(slots + [0] * (3 - nb))), K._arr3(gammas), K._arr3(betas),
                              K._arr3(rms) if rms else None, K._arr3(rvs) if rvs else None,
                              K._arr3(nbts) if nbts else None, ptr(out[0]), ptr(out[1]), ptr(out[2]), ptr(out[3]),
                              nb, c, c_log, m, ctypes.c_float(EPS), ctypes.c_float(momentum), stream_ptr())
    assert rc == 0, rc
    return out, buf


def forward(us, sc, sh, res, m, c, act, res_after, stats):
    nb = len(us)
    out, obuf = guarded(m * c, torch.bfloat16)
    cap = lib().hb_bn_stat_slots_max()
    ost = guarded(cap * c * 2)[0] if stats else None
    sl = ctypes.c_int(-1)
    up = [ptr(us[i]) if i < nb else None for i in range(3)]
    rc = lib().hb_bn_act_fwd_bf16(up[0], up[1], up[2], nb, ptr(sc), ptr(sh), ptr(res), ptr(out), m, c, act,
                                  ctypes.c_float(SLOPE), int(res_after), ptr(ost), ctypes.byref(sl) if stats else None,
                                  stream_ptr())
    assert rc == 0, rc
    torch.cuda.synchronize()
    assert_guard(obuf, m * c, "forward output")
    return out.view(m, c), (ost.view(cap, c, 2) if stats else None), sl.value


def backward(d, us, sc, sh, mean, rstd, res, m, c, c_log, act, res_after, train, gacc=None, bacc=None):
    """Returns (du list, dres, dgamma [B][C], dbeta [B][C]); every output guarded and checked."""
    nb = len(us)
    dus = [guarded(m * c, torch.bfloat16) for _ in range(nb)]
    dres = guarded(m * c, torch.bfloat16) if res is not None else None
    dg, dgbuf = guarded(nb * c)
    db, dbbuf = guarded(nb * c)
    scratch = torch.full((lib().hb_bn_bwd_scratch_doubles(m, c, nb),), float("nan"), device=DEV, dtype=torch.float64)
    up = [ptr(us[i]) if i < nb else None for i in range(3)]
    dp = [ptr(dus[i][0]) if i < nb else None for i in range(3)]
    rc = lib().hb_bn_act_bwd_bf16(ptr(d), up[0], up[1], up[2], nb, ptr(sc), ptr(sh), ptr(mean), ptr(rstd), ptr(res),
                                  ptr(scratch), dp[0], dp[1], dp[2], ptr(dres[0]) if dres else None, ptr(dg), ptr(db),
                                  K._arr3(gacc) if gacc else None, K._arr3(bacc) if bacc else None, c_log, m, c, act,
                                  ctypes.c_float(SLOPE), int(train), int(res_after), stream_ptr())
    assert rc == 0, rc
    torch.cuda.synchronize()
    for i, (v, b) in enumerate(dus):
        assert_guard(b, m * c, f"du{i}")
    if dres:
        assert_guard(dres[1], m * c, "dres")
    assert_guard(dgbuf, nb * c, "dgamma")
    assert_guard(dbbuf, nb * c, "dbeta")
    return ([v.view(m, c) for v, _ in dus], dres[0].view(m, c) if dres else None, dg.view(nb, c), db.view(nb, c))


def reduce_rows(c, m):
    """Upper bound of R of the backward reduction (its grid has at least one block per SM and channel slab)."""
    return O.rows_per_lane(c, m, O.grid_rows(c, m, _sms(), 1))


# ---------------------------------------------------------------------------------------------------------------------
# fp64 references of the raw kernels (scale / shift / mean / rstd given)
# ---------------------------------------------------------------------------------------------------------------------
def affine_z(us, sc, sh):
    """(sum_b sc_b u_b + sh_b, sum_b |sc_b u_b|, sum_b |sh_b|) in fp64, [M, C]."""
    z = _d(sh).sum(0).expand(us[0].shape[0], -1).clone() if us else None
    a = torch.zeros_like(z) if us else None
    for b, u in enumerate(us):
        t = _d(sc[b]) * _d(u)
        z = z + t
        a = a + t.abs()
    return z, a, _d(sh).abs().sum(0) if us else None


def ref_forward(us, sc, sh, res, act, res_after):
    """(out, z, dz): fp64 output, pre-activation and the bound on the kernel's error in z."""
    nb = len(us)
    r = _d(res) if res is not None else None
    if nb:
        z, a, sha = affine_z(us, sc, sh)
    else:
        z, a, sha = torch.zeros_like(r), torch.zeros_like(r), torch.zeros(r.shape[1], device=DEV, dtype=torch.float64)
    inside = r is not None and not res_after
    dz = O.z_err(act, a, sha, r.abs() if inside else None, nb)
    zr = z
    if inside:
        zr = torch.maximum(z, r) if act == O.ACT_FRELU else z + r
    out = O.act_ref(act, zr, SLOPE)
    if r is not None and res_after:
        out = out + r
    return out, zr if act != O.ACT_FRELU else z, dz


def ref_backward(d, us, sc, sh, mean, rstd, res, act, res_after, train, r_red):
    """fp64 (du list, dres, dgamma, dbeta) with the slack of each, and the kink mask."""
    nb = len(us)
    m = d.shape[0]
    r = _d(res) if res is not None else None
    inside = r is not None and not res_after
    if nb:
        z0, a, sha = affine_z(us, sc, sh)
    else:
        z0, a, sha = torch.zeros_like(r), torch.zeros_like(r), 0
    dzb = O.z_err(act, a, sha, r.abs() if inside else None, nb)
    dd = _d(d)
    zv = z0.clone().requires_grad_(True)
    rv = r.clone().requires_grad_(True) if r is not None else None
    if inside and act == O.ACT_FRELU:
        y = torch.maximum(zv, rv)
        gz, gr = torch.autograd.grad(y, (zv, rv), dd)
        dz, dres = gz, gr
        mask = O.kink_mask(act, z0, dzb, r)
        zact = z0
    else:
        zin = zv + rv if inside else zv
        y = O.act_ref(act, zin, SLOPE)
        dz, = torch.autograd.grad(y, zv, dd)
        zact = (z0 + r) if inside else z0
        mask = O.kink_mask(act, zact, dzb)
        dres = dz if inside else (dd if r is not None else None)
    dz_err = dd.abs() * O.grad_act_err(act, zact, dzb)
    jump = dd.abs() * mask           # where the kernel may take the other side of a kink: dz off by at most |d|
    dz_abs = dz.abs()
    sums_dz_err = dz_err + jump
    dres_slack = (dz_err + O.EPS32 * dz_abs) if (dres is not None and dres is not dd) else torch.zeros_like(dd)
    dus, du_slack, dgs, dg_slack, dbs, db_slack = [], [], [], [], [], []
    db = dz.sum(0)
    db_err = O.sum_err(r_red, dz_abs.sum(0)) + sums_dz_err.sum(0) + 2 * O.EPS32 * db.abs()
    for b in range(nb):
        mu, rs, s = _d(mean[b]), _d(rstd[b]), _d(sc[b])
        u = _d(us[b])
        xh = (u - mu) * rs
        dg = rs * ((dz * u).sum(0) - mu * dz.sum(0))
        t_dzu = (dz_abs * u.abs()).sum(0) + (sums_dz_err * u.abs()).sum(0)
        t_dz = dz_abs.sum(0) + sums_dz_err.sum(0)
        dg_err = rs * (O.sum_err(r_red, t_dzu) + mu.abs() * O.sum_err(r_red, t_dz)
                       + (sums_dz_err * u.abs()).sum(0) + mu.abs() * sums_dz_err.sum(0)) + 2 * O.EPS32 * dg.abs()
        if train:
            mdz = dz.sum(0) / m
            mdzx = rs * ((dz * u).sum(0) / m - mu * mdz)
            du = s * dz + (-s * rs * mdzx) * u + (-s * mdz + s * rs * mdzx * mu)
            d_mdz = (O.sum_err(r_red, dz_abs.sum(0)) + sums_dz_err.sum(0)) / m
            d_mdzx = rs * ((O.sum_err(r_red, (dz_abs * u.abs()).sum(0)) + (sums_dz_err * u.abs()).sum(0)) / m
                           + mu.abs() * d_mdz)
            cu, c0 = -s * rs * mdzx, -s * mdz + s * rs * mdzx * mu
            slack = (s.abs() * (dz_err + d_mdz + xh.abs() * d_mdzx)
                     + O.FAST * ((s * dz).abs() + (cu * u).abs() + c0.abs()))
        else:
            du = s * dz
            slack = s.abs() * dz_err + O.FAST * (s * dz).abs()
        dus.append(du)
        du_slack.append(slack)
        dgs.append(dg)
        dg_slack.append(dg_err)
        dbs.append(db)
        db_slack.append(db_err)
    return dict(du=dus, du_slack=du_slack, dres=dres, dres_slack=dres_slack, dg=dgs, dg_slack=dg_slack, db=dbs,
                db_slack=db_slack, mask=mask)


# ---------------------------------------------------------------------------------------------------------------------
# a. statistics: stand-alone partials -> finalize, and the eval affine
# ---------------------------------------------------------------------------------------------------------------------
def check_statistics(us, c_log, momentum, what, seed=0):
    """Runs partials + finalize on the branches ``us`` ([M, C] bf16) and checks every output per channel."""
    m, c = us[0].shape
    nb = len(us)
    g = _gen(seed)
    gam = [guarded(c_log, fill=0.0) for _ in range(nb)]
    bet = [guarded(c_log, fill=0.0) for _ in range(nb)]
    rms = [guarded(c_log, fill=0.0) for _ in range(nb)]
    rvs = [guarded(c_log, fill=0.0) for _ in range(nb)]
    for i in range(nb):
        gam[i][0].copy_(torch.rand(c_log, device=DEV, generator=g) + 0.5)
        bet[i][0].copy_(torch.randn(c_log, device=DEV, generator=g))
        rms[i][0].copy_(torch.randn(c_log, device=DEV, generator=g))
        rvs[i][0].copy_(torch.rand(c_log, device=DEV, generator=g) + 0.5)
    nbt = [torch.full((1,), 5, device=DEV, dtype=torch.int64) for _ in range(nb)]
    rm0 = [_d(v[0]).clone() for v in rms]
    rv0 = [_d(v[0]).clone() for v in rvs]
    parts, slots = zip(*[stats_partials(u) for u in us])
    stats, sbuf = finalize(list(parts), list(slots), [v[0] for v in gam], [v[0] for v in bet], [v[0] for v in rms],
                           [v[0] for v in rvs], nbt, c, c_log, m, momentum)
    torch.cuda.synchronize()
    assert_guard(sbuf, 4 * nb * c, what + " stats")
    mom = float(torch.tensor(momentum, dtype=torch.float32))
    for b in range(nb):
        wb = f"{what} branch {b}"
        for v, nm in ((gam, "gamma"), (bet, "beta"), (rms, "running_mean"), (rvs, "running_var")):
            assert_guard(v[b][1], c_log, f"{wb} {nm}")
        assert int(nbt[b]) == 6, f"{wb}: num_batches_tracked {int(nbt[b])}"
        r = O.rows_per_lane(c, m, slots[b])
        u = us[b][:, :c_log]
        mu, var = O.batch_stats(u)
        dmean, dvar = O.stats_bounds(u, r)
        rstd = 1 / torch.sqrt(var + EPS)
        rel = O.rstd_rel_bound(var, dvar, EPS)
        gm, be = _d(gam[b][0]), _d(bet[b][0])
        sc = gm * rstd
        mean_k, rstd_k, sc_k, sh_k = (_d(stats[i][b]) for i in range(4))
        assert bool((stats[:, b, c_log:] == 0).all()), f"{wb}: padded channels not zero"
        cl = slice(0, c_log)
        O.within(mean_k[cl], mu, dmean, wb + " mean", bits=24)
        O.within(rstd_k[cl], rstd, rel * rstd, wb + " rstd", bits=24)
        O.within(sc_k[cl], sc, (rel + 2 * O.EPS32) * sc.abs(), wb + " scale", bits=24)
        O.within(sh_k[cl], be - mu * sc, sc.abs() * (dmean + mu.abs() * (rel + 2 * O.EPS32))
                 + 4 * O.EPS32 * (be.abs() + (mu * sc).abs()), wb + " shift", bits=24)
        unb = var * m / (m - 1)
        O.within(_d(rms[b][0]), (1 - mom) * rm0[b] + mom * mu,
                 mom * dmean + 4 * O.EPS32 * ((1 - mom) * rm0[b].abs() + mom * mu.abs()), wb + " running_mean", bits=24)
        O.within(_d(rvs[b][0]), (1 - mom) * rv0[b] + mom * unb,
                 mom * dvar * m / (m - 1) + 4 * O.EPS32 * ((1 - mom) * rv0[b] + mom * unb), wb + " running_var", bits=24)
    return stats, slots


STAT_CASES = [(48, 48, 5000), (152, 152, 3001), (264, 264, 2999), (304, 300, 4097), (1280, 1280, 777)]


@pytest.mark.parametrize("ratio", [0.0, 8.0, 64.0])
@pytest.mark.parametrize("c,c_log,m", STAT_CASES)
def test_statistics_partials_finalize(c, c_log, m, ratio):
    g = _gen(c + m + int(ratio))
    sigma = torch.rand(c, device=DEV, generator=g, dtype=torch.float64) + 0.5
    us = [bf16_rows(m, c, ratio * sigma * (1 - 2 * b), sigma, g) for b in range(2)]
    check_statistics(us, c_log, 0.1, f"C={c}/{c_log} M={m} mu/sigma={ratio}", seed=c)


@pytest.mark.parametrize("momentum", [0.0, 1.0])
def test_statistics_momentum_edges(momentum):
    g = _gen(7)
    us = [bf16_rows(3000, 64, 2.0, 1.5, g)]
    check_statistics(us, 64, momentum, f"momentum {momentum}")


@pytest.mark.parametrize("c,c_log,affine", [(48, 48, True), (304, 300, True), (304, 300, False)])
def test_eval_affine(c, c_log, affine):
    g = _gen(c)
    gam = torch.rand(c_log, device=DEV, generator=g) + 0.5 if affine else None
    bet = torch.randn(c_log, device=DEV, generator=g) if affine else None
    rm = torch.randn(c_log, device=DEV, generator=g) * 4
    rv = torch.rand(c_log, device=DEV, generator=g) + 0.1
    outs = [guarded(c) for _ in range(4)]
    assert lib().hb_bn_eval_affine(ptr(gam), ptr(bet), ptr(rm), ptr(rv), ctypes.c_float(EPS), c, c_log,
                                   *[ptr(v) for v, _ in outs], stream_ptr()) == 0
    torch.cuda.synchronize()
    for v, b in outs:
        assert_guard(b, c, "eval affine")
        assert bool((v[c_log:] == 0).all()), "eval affine: padded channels not zero"
    sc_k, sh_k, mean_k, rstd_k = (_d(v[:c_log]) for v, _ in outs)
    r = 1 / torch.sqrt(_d(rv) + EPS)
    gm = _d(gam) if affine else 1.0
    be = _d(bet) if affine else 0.0
    sc = gm * r
    O.within(rstd_k, r, 3 * O.EPS32 * r, "eval rstd", bits=24)
    O.within(sc_k, sc, 5 * O.EPS32 * sc.abs(), "eval scale", bits=24)
    O.within(sh_k, be - _d(rm) * sc, 4 * O.EPS32 * (abs(be) + 2 * (_d(rm) * sc).abs()), "eval shift", bits=24)
    assert torch.equal(mean_k, _d(rm)), "eval mean"


# ---------------------------------------------------------------------------------------------------------------------
# b. forward with scale / shift given
# ---------------------------------------------------------------------------------------------------------------------
def make_branches(nb, m, c, ratio, seed, c_log=None, gamma_hi=1.5):
    """bf16 branches u_b = mu + sigma randn, and fp32 (scale, shift, mean, rstd) [B][C] of their batch statistics."""
    c_log = c if c_log is None else c_log
    g = _gen(seed)
    us, sc, sh, mean, rstd = [], [], [], [], []
    for b in range(nb):
        sigma = torch.rand(c, device=DEV, generator=g, dtype=torch.float64) + 0.5
        u = bf16_rows(m, c, ratio * sigma * (1 if b % 2 == 0 else -1), sigma, g)
        mu, var = O.batch_stats(u)
        rs = 1 / torch.sqrt(var + EPS)
        gm = torch.rand(c, device=DEV, generator=g, dtype=torch.float64) * (gamma_hi - 0.5) + 0.5
        be = torch.randn(c, device=DEV, generator=g, dtype=torch.float64) * 0.5
        s = _f32(gm * rs)
        live = torch.arange(c, device=DEV) < c_log
        s = torch.where(live, s, 0)
        us.append(u)
        sc.append(s)
        sh.append(torch.where(live, _f32(be - mu * s.double()), 0))
        mean.append(_f32(mu))
        rstd.append(_f32(rs))
    stack = (lambda xs: torch.stack(xs).contiguous()) if nb else (lambda xs: torch.zeros(1, c, device=DEV))
    return us, stack(sc), stack(sh), stack(mean), stack(rstd)


FWD_CASES = ([(nb, act, res) for nb in (1, 2, 3) for act in range(7) for res in ("none", "inside", "after")]
             + [(0, act, "inside") for act in range(7)] + [(1, O.ACT_FRELU, "inside")])
CS = [8, 48, 64, 152, 256, 264, 304, 1280]


@pytest.mark.parametrize("nb,act,res", FWD_CASES)
def test_forward_per_element(nb, act, res):
    i = FWD_CASES.index((nb, act, res))
    c = CS[i % len(CS)]
    m = [3001, 2048 + 5, 777][i % 3]
    us, sc, sh, _, _ = make_branches(nb, m, c, 8.0 if i % 2 else 0.5, seed=100 + i, gamma_hi=3.0)
    r = bf16_rows(m, c, 0.0, 1.5, _gen(200 + i)) if res != "none" else None
    after = res == "after"
    what = f"fwd B={nb} act={act} res={res} C={c} M={m}"
    out, _, _ = forward(us, sc, sh, r, m, c, act, after, False)
    ref, z, dz = ref_forward(us, sc, sh, r, act, after)
    O.within(out, ref, O.fwd_bound(act, z, dz, r if after else None, SLOPE), what)
    # the statistics variant: same bits, partials that add up to the stored output, repeatable
    out2, ost, slots = forward(us, sc, sh, r, m, c, act, after, True)
    assert torch.equal(out, out2), what + ": statistics variant differs"
    check_stats(out2, ost, slots, what)
    out3, ost3, slots3 = forward(us, sc, sh, r, m, c, act, after, True)
    assert slots3 == slots and torch.equal(out3, out2) and torch.equal(ost3[:slots], ost[:slots]), what + ": not repeatable"


def test_forward_padded_channels_are_zero():
    c, c_log, m = 304, 300, 4097
    us, sc, sh, _, _ = make_branches(2, m, c, 8.0, seed=5, c_log=c_log)
    r = bf16_rows(m, c, 0.0, 1.0, _gen(6))
    r[:, c_log:] = 0
    out, _, _ = forward(us, sc, sh, r, m, c, O.ACT_SILU, False, True)
    assert bool((out[:, c_log:] == 0).all()), "padded channels of the output not zero"


# ---------------------------------------------------------------------------------------------------------------------
# c. backward with scale / shift / mean / rstd given
# ---------------------------------------------------------------------------------------------------------------------
def check_backward(us, sc, sh, mean, rstd, r, d, act, after, train, c_log, what, direct=True):
    m, c = d.shape
    nb = len(us)
    r_red = reduce_rows(c, m)
    ref = ref_backward(d, us, sc, sh, mean, rstd, r, act, after, train, r_red)
    O.mask_fraction_ok(ref["mask"][:, :c_log], what)
    outs = backward(d, us, sc, sh, mean, rstd, r, m, c, c_log, act, after, train)
    dus, dres, dg, db = outs
    cl = slice(0, c_log)
    for b in range(nb):
        O.within(dus[b][:, cl], ref["du"][b][:, cl], ref["du_slack"][b][:, cl], f"{what} du{b}", ref["mask"][:, cl])
        if c_log < c:
            assert bool((dus[b][:, c_log:] == 0).all()), f"{what} du{b}: padded channels not zero"
        O.within(dg[b][cl], ref["dg"][b][cl], ref["dg_slack"][b][cl], f"{what} dgamma{b}", bits=24)
        O.within(db[b][cl], ref["db"][b][cl], ref["db_slack"][b][cl], f"{what} dbeta{b}", bits=24)
    if dres is not None:
        O.within(dres[:, cl], ref["dres"][:, cl], ref["dres_slack"][:, cl], f"{what} dres", ref["mask"][:, cl])
    again = backward(d, us, sc, sh, mean, rstd, r, m, c, c_log, act, after, train)
    for x, y in zip(outs[0] + [outs[1], outs[2], outs[3]], again[0] + [again[1], again[2], again[3]]):
        assert x is None or torch.equal(x, y), what + ": not bit-reproducible"
    if direct and nb:
        # .grad buffers bound to a GradBucket: the kernel ADDS dgamma / dbeta into them, nothing past C_logical
        g = _gen(c + m)
        gacc = [guarded(c_log, fill=0.0) for _ in range(nb)]
        bacc = [guarded(c_log, fill=0.0) for _ in range(nb)]
        pre = []
        for v in gacc + bacc:
            v[0].copy_(torch.randn(c_log, device=DEV, generator=g) * 100)
            pre.append(_d(v[0]).clone())
        backward(d, us, sc, sh, mean, rstd, r, m, c, c_log, act, after, train, [v[0] for v in gacc],
                 [v[0] for v in bacc])
        for b in range(nb):
            for v, p, key in ((gacc[b], pre[b], "dg"), (bacc[b], pre[nb + b], "db")):
                want = p + ref[key][b][cl]
                O.within(v[0], want, ref[key + "_slack"][b][cl] + O.EPS32 * want.abs(), f"{what} {key}{b} accumulated",
                         bits=24)
                assert_guard(v[1], c_log, f"{what} {key}{b} accumulated")


BWD_CASES = ([(nb, act, res, train) for nb in (1, 2, 3) for act in range(7) for res in ("none", "inside", "after")
              for train in (1, 0) if (nb + act + len(res)) % 2 == train or act in (O.ACT_RELU6, O.ACT_SILU)]
             + [(0, act, "inside", 1) for act in range(7)] + [(1, O.ACT_FRELU, "inside", t) for t in (1, 0)])


@pytest.mark.parametrize("nb,act,res,train", BWD_CASES)
def test_backward_per_element(nb, act, res, train):
    i = BWD_CASES.index((nb, act, res, train))
    c, c_log = [(48, 48), (152, 152), (264, 264), (304, 300), (64, 64), (1280, 1280), (8, 8)][i % 7]
    m = [3001, 2500, 1023][i % 3]
    us, sc, sh, mean, rstd = make_branches(nb, m, c, 8.0 if i % 2 else 1.0, seed=300 + i, c_log=c_log, gamma_hi=4.0)
    g = _gen(400 + i)
    r = bf16_rows(m, c, 0.0, 1.5, g) if res != "none" else None
    d = bf16_rows(m, c, 0.3, 1.0, g)
    check_backward(us, sc, sh, mean, rstd, r, d, act, res == "after", train, c_log,
                   f"bwd B={nb} act={act} res={res} train={train} C={c}/{c_log} M={m}")


def test_frelu_exact_ties():
    """Eval branch with scale exactly 1 and shift exactly 0: z = u bit for bit, so planted ties r == u are exact and
    the gradient must split 1/2 : 1/2 there."""
    m, c = 2048, 64
    g = _gen(9)
    u = bf16_rows(m, c, 0.0, 1.0, g)
    r = bf16_rows(m, c, 0.0, 1.0, g)
    tie = torch.rand(m, c, device=DEV, generator=g) < 0.25
    r[tie] = u[tie]
    sc, sh = torch.ones(1, c, device=DEV), torch.zeros(1, c, device=DEV)
    mean, rstd = torch.zeros(1, c, device=DEV), torch.ones(1, c, device=DEV)
    d = bf16_rows(m, c, 0.0, 1.0, g)
    out, _, _ = forward([u], sc, sh, r, m, c, O.ACT_FRELU, False, False)
    assert torch.equal(out, torch.maximum(u, r)), "FReLU forward"
    dus, dres, _, _ = backward(d, [u], sc, sh, mean, rstd, r, m, c, c, O.ACT_FRELU, False, 0)
    gate = torch.where(u.double() > r.double(), 1.0, torch.where(u == r, 0.5, 0.0))
    assert torch.equal(dus[0].double(), (d.double() * gate).bfloat16().double()), "FReLU du"
    assert torch.equal(dres.double(), (d.double() - (d.double() * gate).bfloat16().double()).bfloat16().double()), "FReLU dres"


# ---------------------------------------------------------------------------------------------------------------------
# d. the mode matrix end to end: bn_act / act_only against F.batch_norm + activation in fp64 (autograd)
# ---------------------------------------------------------------------------------------------------------------------
E2E_CASES = [(nb, act, res) for nb in (1, 2, 3) for act in range(7) for res in ("none", "inside", "after")]
E2E_C = [(8, 8), (48, 48), (64, 64), (152, 152), (256, 256), (264, 264), (304, 300), (1280, 1280)]


def _e2e_m(c, i):
    rows_t = O.geometry(c).rows_t
    return [7, rows_t - 1, rows_t + 1, 3000][i % 4]


def _nchw(x2d, n, h, w):
    return x2d.view(n, h, w, -1).permute(0, 3, 1, 2)


@pytest.mark.parametrize("train", [True, False])
@pytest.mark.parametrize("nb,act,res", E2E_CASES)
def test_bn_act_end_to_end(nb, act, res, train):
    i = E2E_CASES.index((nb, act, res))
    c, c_log = E2E_C[(i + train) % len(E2E_C)]
    m = _e2e_m(c, i // 2 + train)
    trainable = (i + train) % 3 != 0
    after = res == "after"
    what = f"bn_act B={nb} act={act} res={res} train={train} C={c}/{c_log} M={m} trainable={trainable}"
    g = _gen(500 + i + 1000 * train)
    bns = []
    us = []
    for b in range(nb):
        bn = torch.nn.BatchNorm2d(c_log).to(DEV).train(train)
        with torch.no_grad():
            bn.weight.uniform_(0.5, 3.0, generator=g)
            bn.bias.normal_(0, 0.5, generator=g)
            bn.running_mean.normal_(0, 1, generator=g)
            bn.running_var.uniform_(0.5, 2.0, generator=g)
        bn.weight.requires_grad_(trainable)
        bn.bias.requires_grad_(trainable)
        bns.append(bn)
        u = bf16_rows(m, c, 0.5 * (b + 1), 1.0 + b, g)
        us.append(u)
    r = bf16_rows(m, c, 0.0, 1.0, g) if res != "none" else None
    if r is not None:
        r[:, c_log:] = 0
    d = bf16_rows(m, c, 0.2, 1.0, g)
    ud = [_nchw(u, 1, m, 1).requires_grad_(True) for u in us]
    rd = _nchw(r, 1, m, 1).requires_grad_(True) if r is not None else None
    out = K.bn_act(ud, bns, act, SLOPE, rd, res_after_act=after)
    out.backward(_nchw(d, 1, m, 1))
    rows = lambda t: t.detach().permute(0, 2, 3, 1).reshape(m, -1)   # noqa: E731
    cl = slice(0, c_log)
    # fp64 reference on the logical channels
    u64 = [_d(u[:, cl]).requires_grad_(True) for u in us]
    w64 = [_d(bn.weight).requires_grad_(trainable) for bn in bns]
    b64 = [_d(bn.bias).requires_grad_(trainable) for bn in bns]
    r64 = _d(r[:, cl]).requires_grad_(True) if r is not None else None
    running = None if train else [(_d(bn.running_mean), _d(bn.running_var)) for bn in bns]
    ref, z = O.bn_act_ref(u64, w64, b64, act, SLOPE, r64, after, running, EPS)
    leaves = u64 + ([r64] if r64 is not None else []) + ([*w64, *b64] if trainable else [])
    grads = torch.autograd.grad(ref, leaves, _d(d[:, cl]))
    # kernel-side constants and their error bounds
    sc_abs = torch.zeros(m, c_log, device=DEV, dtype=torch.float64)
    sh_abs = torch.zeros(c_log, device=DEV, dtype=torch.float64)
    dz_stats = torch.zeros_like(sc_abs)
    consts = []   # per branch: (scale, xhat, mean, rstd, bound on |xhat_kernel - xhat|, relative error of scale)
    r_fwd = O.rows_per_lane(c, m, O.grid_rows(c, m, _sms(), 1, 16))   # stand-alone statistics pass, smallest grid
    for b in range(nb):
        u = _d(us[b][:, cl])
        if train:
            mu, var = O.batch_stats(u)
            dmean, dvar = O.stats_bounds(u, r_fwd)
            rel = O.rstd_rel_bound(var, dvar, EPS) + 2 * O.EPS32
        else:
            mu, var = _d(bns[b].running_mean), _d(bns[b].running_var)
            dmean, rel = torch.zeros_like(mu), torch.full_like(mu, 5 * O.EPS32)
        rs = 1 / torch.sqrt(var + EPS)
        s = _d(bns[b].weight) * rs
        xh = (u - mu) * rs
        be = _d(bns[b].bias)
        sc_abs += (s * u).abs()
        sh_abs += (be - mu * s).abs()
        # the kernel's scale is off by rel, its shift by |sc| dmean + |mu sc| rel + four roundings
        dz_stats += s.abs() * (rel * (u - mu).abs() + dmean) + 4 * O.EPS32 * (be.abs() + (mu * s).abs())
        consts.append((s, xh, mu, rs, rel * xh.abs() + rs * dmean, rel))
    inside = r is not None and not after
    r64d = _d(r[:, cl]) if r is not None else None
    dzb = O.z_err(act, sc_abs, sh_abs, r64d.abs() if inside else None, nb) + dz_stats
    zk = z.detach()
    mask = O.kink_mask(act, zk, dzb)
    O.mask_fraction_ok(mask, what, 0.01 if m > 100 else 0.2)
    O.within(rows(out)[:, cl], ref.detach(), O.fwd_bound(act, zk, dzb, r64d if after else None, SLOPE), what + " out")
    if c_log < c:
        assert bool((rows(out)[:, c_log:] == 0).all()), what + ": padded output channels not zero"
    # gradients: dz (off by dz_err, and by up to |d| on the kink mask) and everything computed from it
    dd = _d(d[:, cl])
    zv = zk.clone().requires_grad_(True)
    dz, = torch.autograd.grad(O.act_ref(act, zv, SLOPE), zv, dd)
    dz_err = dd.abs() * (O.grad_act_err(act, zk, dzb) + mask)
    r_red = reduce_rows(c, m)
    dz_abs = dz.abs()
    e_sum_dz = O.sum_err(r_red, dz_abs.sum(0)) + dz_err.sum(0)
    off = len(u64) + (r64 is not None)
    for b in range(nb):
        s, xh, mu, rs, xe, rel = consts[b]
        ua = _d(us[b][:, cl]).abs()
        # sum dz * xhat as the kernel forms it, rstd * (sum dz u - mean sum dz), and its error
        e_dzx = (rs * (O.sum_err(r_red, (dz_abs * ua).sum(0)) + mu.abs() * e_sum_dz + (dz_err * ua).sum(0))
                 + (dz_abs * xe).sum(0))
        wb = f"{what} branch {b}"
        if train:
            mdz, mdzx = dz.mean(0), (dz * xh).mean(0)
            slack = (s.abs() * (dz_err + e_sum_dz / m + xh.abs() * e_dzx / m + xe * mdzx.abs())
                     + (rel + O.FAST) * s.abs() * (dz_abs + mdz.abs() + (xh * mdzx).abs()))
        else:
            slack = s.abs() * dz_err + (rel + O.FAST) * (s * dz).abs()
        O.within(rows(ud[b].grad)[:, cl], grads[b], slack, wb + " du", mask)
        if c_log < c:
            assert bool((rows(ud[b].grad)[:, c_log:] == 0).all()), wb + ": padded du channels not zero"
        if trainable:
            gw, gb = grads[off + b], grads[off + nb + b]
            O.within(_d(bns[b].weight.grad), gw, e_dzx + 2 * O.EPS32 * gw.abs(), wb + " dgamma", bits=24)
            O.within(_d(bns[b].bias.grad), gb, e_sum_dz + 2 * O.EPS32 * gb.abs(), wb + " dbeta", bits=24)
        else:
            assert bns[b].weight.grad is None and bns[b].bias.grad is None
    if r is not None:
        O.within(rows(rd.grad)[:, cl], grads[len(u64)], dz_err + O.EPS32 * dz_abs, what + " dres", mask)
    if train:
        for bn in bns:
            assert int(bn.num_batches_tracked) == 1, what + ": num_batches_tracked"


@pytest.mark.parametrize("act", range(7))
def test_act_only_end_to_end(act):
    m, c = 3000 + act, [8, 48, 64, 152, 264, 304, 1280][act]
    g = _gen(600 + act)
    x = bf16_rows(m, c, 0.0, 3.0, g)
    d = bf16_rows(m, c, 0.0, 1.0, g)
    xd = _nchw(x, 1, m, 1).requires_grad_(True)
    y = K.act_only(xd, act, SLOPE)
    y.backward(_nchw(d, 1, m, 1))
    rows = lambda t: t.detach().permute(0, 2, 3, 1).reshape(m, -1)   # noqa: E731
    x64 = _d(x).requires_grad_(True)
    ref = O.act_ref(act, x64, SLOPE)
    gx, = torch.autograd.grad(ref, x64, _d(d))
    z = _d(x)
    dz = 2 * O.EPS32 * z.abs()
    O.within(rows(y), ref.detach(), O.fwd_bound(act, z, dz, None, SLOPE), f"act_only {act}")
    mask = O.kink_mask(act, z, dz)
    O.within(rows(xd.grad), gx, _d(d).abs() * O.grad_act_err(act, z, dz) + O.EPS32 * gx.abs(), f"act_only {act} dx", mask)


def test_frelu_end_to_end_eval_ties():
    """The depth-wise FReLU path: eval branch whose folded scale is exactly 1 and shift exactly 0, residual equal to
    the branch on a quarter of the elements."""
    m, c = 2048, 48
    g = _gen(11)
    bn = torch.nn.BatchNorm2d(c).to(DEV).eval()
    with torch.no_grad():
        bn.running_mean.zero_()
        bn.running_var.fill_(1.0 - 2.0 ** -10)
        bn.weight.fill_(1.0)
        bn.bias.zero_()
    bn.eps = 2.0 ** -10                      # var + eps == 1 exactly in fp32: scale 1, shift 0
    u = bf16_rows(m, c, 0.0, 1.0, g)
    r = bf16_rows(m, c, 0.0, 1.0, g)
    tie = torch.rand(m, c, device=DEV, generator=g) < 0.25
    r[tie] = u[tie]
    d = bf16_rows(m, c, 0.0, 1.0, g)
    ud = _nchw(u, 1, m, 1).requires_grad_(True)
    rd = _nchw(r, 1, m, 1).requires_grad_(True)
    out = K.bn_act([ud], [bn], K.ACT_FRELU, 0.0, rd)
    out.backward(_nchw(d, 1, m, 1))
    rows = lambda t: t.detach().permute(0, 2, 3, 1).reshape(m, -1)   # noqa: E731
    assert torch.equal(rows(out), torch.maximum(u, r))
    u64, r64 = _d(u).requires_grad_(True), _d(r).requires_grad_(True)
    gu, gr = torch.autograd.grad(torch.maximum(u64, r64), (u64, r64), _d(d))
    assert torch.equal(rows(ud.grad).double(), gu.bfloat16().double()), "du at ties"
    assert torch.equal(rows(rd.grad).double(), gr.bfloat16().double()), "dres at ties"


# ---------------------------------------------------------------------------------------------------------------------
# module semantics nn.BatchNorm2d pins
# ---------------------------------------------------------------------------------------------------------------------
def test_untracked_running_stats_are_left_alone():
    torch.manual_seed(12)
    x = torch.randn(2, 16, 5, 5, device=DEV).bfloat16()
    bn = torch.nn.BatchNorm2d(16).to(DEV)
    bn.weight.requires_grad_(False)
    bn.bias.requires_grad_(False)
    freeze_bn(bn)       # clears track_running_stats; .train() afterwards brings back batch statistics only
    bn.train()
    before = [bn.running_mean.clone(), bn.running_var.clone(), bn.num_batches_tracked.clone()]
    out = K.bn_act([x], [bn], K.ACT_RELU)
    ref = torch.nn.functional.batch_norm(x.double(), None, None, bn.weight.double(), bn.bias.double(), True, 0.1,
                                         bn.eps).relu()
    assert (out.double() - ref).abs().max() < 0.05
    assert torch.equal(bn.running_mean, before[0]) and torch.equal(bn.running_var, before[1])
    assert torch.equal(bn.num_batches_tracked, before[2])


def test_one_value_per_channel_in_training_raises():
    bn = torch.nn.BatchNorm2d(16).to(DEV)
    x = torch.randn(1, 16, 1, 1, device=DEV)
    with pytest.raises(ValueError, match="Expected more than 1 value per channel when training"):
        bn(x)
    with pytest.raises(ValueError, match="Expected more than 1 value per channel when training"):
        K.bn_act([x], [bn], K.ACT_NONE)
    bn.eval()
    K.bn_act([x], [bn], K.ACT_NONE)       # eval with running statistics: fine, as in torch


# ---------------------------------------------------------------------------------------------------------------------
# e. the cp.async ring wrapped at the default grids
# ---------------------------------------------------------------------------------------------------------------------
WRAP_CASES = {
    "B1_C64": (1, 64, 64, 32 * 96 * 96, False),
    "B1_C1280": (1, 1280, 1280, 8 * 47 * 47, False),
    "B1_C304_300": (1, 304, 300, 16 * 63 * 63, False),
    "B3_res_C48": (3, 48, 48, 16 * 128 * 128, True),
}


@pytest.mark.parametrize("name", list(WRAP_CASES))
def test_ring_wrap(name):
    nb, c, c_log, m, has_res = WRAP_CASES[name]
    us, sc, sh, mean, rstd = make_branches(nb, m, c, 8.0, seed=len(name), c_log=c_log)
    g = _gen(700)
    r = bf16_rows(m, c, 0.0, 1.0, g) if has_res else None
    if r is not None:
        r[:, c_log:] = 0
    act = O.ACT_RELU if has_res else O.ACT_SILU
    out, ost, slots = forward(us, sc, sh, r, m, c, act, False, True)
    geo = O.geometry(c)
    lanes = slots * geo.rows_t
    rr = -(-m // lanes)
    kslots = O.ring_depth(nb + 1) + 1
    assert rr >= 2 * kslots + 1, f"{name}: R = {rr} rows per lane does not wrap the {kslots}-slot ring twice"
    assert m % lanes != 0, f"{name}: no lane ends one row early"
    print(f"{name}: forward slots {slots}, lanes {lanes}, R = {rr}, ring slots {kslots}")
    ref, z, dz = ref_forward(us, sc, sh, r, act, False)
    O.within(out, ref, O.fwd_bound(act, z, dz, None, SLOPE), name + " forward")
    check_stats(out, ost, slots, name)
    # a: the stand-alone statistics of the same tensors
    check_statistics(us, c_log, 0.1, name + " statistics")
    # c: backward, batch statistics
    d = bf16_rows(m, c, 0.3, 1.0, g)
    check_backward(us, sc, sh, mean, rstd, r, d, act, False, 1, c_log, name + " backward", direct=nb == 1)


# ---------------------------------------------------------------------------------------------------------------------
# f. non-finite inputs, eval
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("act", range(7))
def test_non_finite_inputs(act):
    m, c = 4096, 64
    us, sc, sh, _, _ = make_branches(1, m, c, 1.0, seed=800 + act)
    clean, _, _ = forward(us, sc, sh, None, m, c, act, False, False)
    bad = us[0].clone()
    idx = torch.tensor([[5, 3], [100, 17], [2047, 63], [4095, 0], [777, 40], [1234, 8]], device=DEV)
    vals = [float("nan"), float("inf"), float("-inf"), float("nan"), float("inf"), float("-inf")]
    for (i, j), v in zip(idx.tolist(), vals):
        bad[i, j] = v
    out, _, _ = forward([bad], sc, sh, None, m, c, act, False, False)
    hit = torch.zeros(m, c, dtype=torch.bool, device=DEV)
    hit[idx[:, 0], idx[:, 1]] = True
    assert torch.equal(out[~hit], clean[~hit]), f"act {act}: finite elements changed"
    z = _d(sc[0]) * _d(bad) + _d(sh[0])
    want = O.act_ref(act, z, SLOPE).to(torch.bfloat16)
    got, exp = out[hit].double(), want[hit].double()
    same = (got == exp) | (torch.isnan(got) & torch.isnan(exp))
    assert bool(same.all()), f"act {act}: non-finite elements {got.tolist()} vs torch {exp.tolist()}"


# ---------------------------------------------------------------------------------------------------------------------
# g. squeeze-excite gate + activation
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", [8, 304, 1280])
@pytest.mark.parametrize("hw", [1, 7, 3136])
@pytest.mark.parametrize("act", range(7))
def test_gate_act(act, hw, c):
    n = 2
    g = _gen(act * 100 + hw + c)
    x = bf16_rows(n * hw, c, 0.0, 2.0, g)
    gate = (torch.rand(n, c, device=DEV, generator=g) * 2).contiguous()
    d = bf16_rows(n * hw, c, 0.0, 1.0, g)
    out, obuf = guarded(n * hw * c, torch.bfloat16)
    assert lib().hb_gate_act_fwd_bf16(ptr(x), ptr(gate), ptr(out), n, hw, c, act, ctypes.c_float(SLOPE), stream_ptr()) == 0
    dx, dxbuf = guarded(n * hw * c, torch.bfloat16)
    dg, dgbuf = guarded(n * c)
    assert lib().hb_gate_act_bwd_bf16(ptr(d), ptr(x), ptr(gate), ptr(dx), ptr(dg), n, hw, c, act, ctypes.c_float(SLOPE),
                                      stream_ptr()) == 0
    torch.cuda.synchronize()
    for b, k, w in ((obuf, n * hw * c, "out"), (dxbuf, n * hw * c, "dx"), (dgbuf, n * c, "dgate")):
        assert_guard(b, k, f"gate {w}")
    what = f"gate act={act} HW={hw} C={c}"
    x3, g3, d3 = _d(x).view(n, hw, c), _d(gate).view(n, 1, c), _d(d).view(n, hw, c)
    z = x3 * g3
    dz_b = O.EPS32 * z.abs()
    O.within(out.view(n, hw, c), O.act_ref(act, z, SLOPE), O.fwd_bound(act, z, dz_b, None, SLOPE), what)
    zv = z.clone().requires_grad_(True)
    dz, = torch.autograd.grad(O.act_ref(act, zv, SLOPE), zv, d3)
    mask = O.kink_mask(act, z, dz_b)
    dz_err = d3.abs() * (O.grad_act_err(act, z, dz_b) + mask) + O.EPS32 * dz.abs()
    O.within(dx.view(n, hw, c), dz * g3, dz_err * g3 + O.EPS32 * (dz * g3).abs(), what + " dx", mask)
    # dgate: fp32 lane sums of R rows, then the rows_t lanes added in fp32
    geo = O.geometry(c)
    r = -(-hw // geo.rows_t)
    ref = (dz * x3).sum(1)
    terms = (dz.abs() * x3.abs()).sum(1)
    slack = (r + geo.rows_t + 2) * O.EPS32 * terms + (dz_err * x3.abs()).sum(1) + 2 * O.EPS32 * ref.abs()
    O.within(dg.view(n, c), ref, slack, what + " dgate", bits=24)


def test_gate_act_refuses_frelu():
    x = torch.zeros(1, 8, device=DEV, dtype=torch.bfloat16)
    gate = torch.ones(1, 8, device=DEV)
    out = torch.empty_like(x)
    assert lib().hb_gate_act_fwd_bf16(ptr(x), ptr(gate), ptr(out), 1, 1, 8, O.ACT_FRELU, ctypes.c_float(0), stream_ptr()) != 0
    assert lib().hb_gate_act_bwd_bf16(ptr(x), ptr(x), ptr(gate), ptr(out), ptr(gate), 1, 1, 8, O.ACT_FRELU,
                                      ctypes.c_float(0), stream_ptr()) != 0
