"""The synchronised-BatchNorm entry points of csrc/bn_act.cu per element, through the C ABI: partials -> fp64 sums,
finalisation from (all-reduced) sums, and the backward split into a reduce and an apply step.

Two "ranks" are emulated on one device by splitting the rows of one batch into two shards: each shard runs the local
step, the fp64 buffers are added (what a two-rank SUM all-reduce does) and the global step runs on the result. The outputs
are checked against the fp64 references and bounds of the whole batch (tests/_bn_oracle.py, the helpers of
tests/test_gpu_bn_act_bounds.py), and on one shard the split path must be bit-identical to the one-call path."""
import ctypes

import pytest
import torch

from holocron_b200._lib import lib, ptr, stream_ptr
from holocron_b200.nn import _fused as K

import _bn_oracle as O
from test_gpu_bn_act_bounds import (DEV, EPS, SLOPE, _d, _gen, assert_guard, backward, bf16_rows, finalize,
                                    guarded, make_branches, reduce_rows, ref_backward, stats_partials)

pytestmark = pytest.mark.gpu


def partials_sums(parts, slots, c, c_log, m):
    """Guarded fp64 [B][C][2] sums + count of hb_bn_partials_sums."""
    nb = len(parts)
    n = nb * c * 2 + 1
    sums, buf = guarded(n, torch.float64)
    rc = lib().hb_bn_partials_sums(K._arr3(parts), K._I3(*(list(slots) + [0] * (3 - nb))), nb, c, c_log, m, ptr(sums),
                                   stream_ptr())
    assert rc == 0, rc
    torch.cuda.synchronize()
    assert_guard(buf, n, "sums")
    return sums


def finalize_sums(sums, gammas, betas, rms, rvs, nbts, c, c_log, momentum):
    nb = len(gammas)
    out, buf = guarded(4 * nb * c)
    out = out.view(4, nb, c)
    rc = lib().hb_bn_finalize_sums(ptr(sums), K._arr3(gammas), K._arr3(betas), K._arr3(rms), K._arr3(rvs),
                                   K._arr3(nbts), ptr(out[0]), ptr(out[1]), ptr(out[2]), ptr(out[3]), nb, c, c_log,
                                   ctypes.c_float(EPS), ctypes.c_float(momentum), stream_ptr())
    assert rc == 0, rc
    torch.cuda.synchronize()
    assert_guard(buf, 4 * nb * c, "finalize_sums")
    return out


def _params(nb, c_log, seed):
    g = _gen(seed)
    gam = [torch.rand(c_log, device=DEV, generator=g) + 0.5 for _ in range(nb)]
    bet = [torch.randn(c_log, device=DEV, generator=g) for _ in range(nb)]
    rms = [torch.randn(c_log, device=DEV, generator=g) for _ in range(nb)]
    rvs = [torch.rand(c_log, device=DEV, generator=g) + 0.5 for _ in range(nb)]
    return gam, bet, rms, rvs


def _cast_parts(u, slots):
    """Partials of u [M, C] in exactly ``slots`` slots (row blocks of ceil(M / slots) rows), as a producer may write them."""
    m, c = u.shape
    rows = -(-m // slots)
    p = torch.zeros(slots, c, 2, device=DEV, dtype=torch.float32)
    for k in range(slots):
        blk = u[k * rows:(k + 1) * rows].float()
        p[k, :, 0] = blk.sum(0)
        p[k, :, 1] = (blk * blk).sum(0)
    return p, rows


# (C, C_logical, M of each shard, slot source): C not a multiple of 64, padded widths, one slot, many slots
STAT_CASES = [(48, 48, (3000, 3000), "pass"), (152, 152, (1000, 2999), "pass"), (200, 200, (37, 5000), "pass"),
              (304, 300, (4097, 777), "pass"), (1280, 1280, (512, 1500), "pass"), (48, 40, (999, 2), "one"),
              (96, 96, (2000, 2500), "many")]


@pytest.mark.parametrize("nb", [1, 2, 3])
@pytest.mark.parametrize("case", range(len(STAT_CASES)))
def test_partials_sums_and_finalize_sums(nb, case):
    c, c_log, shards, src = STAT_CASES[case]
    what = f"B={nb} C={c}/{c_log} shards={shards} slots={src}"
    g = _gen(case * 7 + nb)
    m = sum(shards)
    sigma = torch.rand(c, device=DEV, generator=g, dtype=torch.float64) + 0.5
    us = [bf16_rows(m, c, 8.0 * sigma * (1 - 2 * (b % 2)), sigma, g) for b in range(nb)]
    if c_log < c:
        us = [torch.where(torch.arange(c, device=DEV) < c_log, u, torch.zeros_like(u)) for u in us]
    gam, bet, rms, rvs = _params(nb, c_log, case)
    shard_sums, r_lane = [], 0
    lo = 0
    for ms in shards:
        parts, slots = [], []
        for u in us:
            su = u[lo:lo + ms].contiguous()
            if src == "pass":
                p, sl = stats_partials(su)
                r_lane = max(r_lane, O.rows_per_lane(c, ms, sl))
            else:
                p, rows = _cast_parts(su, 1 if src == "one" else lib().hb_bn_stat_slots_max())
                sl = p.shape[0]
                r_lane = max(r_lane, rows)
            parts.append(p)
            slots.append(sl)
        sums = partials_sums(parts, slots, c, c_log, ms)
        assert float(sums[-1]) == ms, f"{what}: count {float(sums[-1])}"
        # a single shard: finalising from its sums is hb_bn_finalize, bit for bit (every output and running statistic)
        rm_a, rv_a = [t.clone() for t in rms], [t.clone() for t in rvs]
        rm_b, rv_b = [t.clone() for t in rms], [t.clone() for t in rvs]
        nbt_a = [torch.full((1,), 3, device=DEV, dtype=torch.int64) for _ in range(nb)]
        nbt_b = [t.clone() for t in nbt_a]
        ref, _ = finalize(parts, slots, gam, bet, rm_a, rv_a, nbt_a, c, c_log, ms, 0.1)
        got = finalize_sums(sums, gam, bet, rm_b, rv_b, nbt_b, c, c_log, 0.1)
        assert torch.equal(ref, got), f"{what}: finalize_sums differs from finalize on one shard"
        for x, y in zip(rm_a + rv_a + nbt_a, rm_b + rv_b + nbt_b):
            assert torch.equal(x, y), f"{what}: running statistics differ from finalize on one shard"
        shard_sums.append(sums)
        lo += ms
    # the per-element sums against the fp64 column sums of each shard are covered through the statistics below
    total = shard_sums[0] + shard_sums[1]
    assert float(total[-1]) == m
    rm = [t.clone() for t in rms]
    rv = [t.clone() for t in rvs]
    nbt = [torch.full((1,), 5, device=DEV, dtype=torch.int64) for _ in range(nb)]
    stats = finalize_sums(total, gam, bet, rm, rv, nbt, c, c_log, 0.1)
    mom = float(torch.tensor(0.1, dtype=torch.float32))
    cl = slice(0, c_log)
    for b in range(nb):
        wb = f"{what} branch {b}"
        assert int(nbt[b]) == 6, wb
        assert bool((stats[:, b, c_log:] == 0).all()), f"{wb}: padded channels not zero"
        assert bool((total[b * c * 2:(b + 1) * c * 2].view(c, 2)[c_log:] == 0).all()), f"{wb}: padded sums not zero"
        u = us[b][:, :c_log]
        mu, var = O.batch_stats(u)
        dmean, dvar = O.stats_bounds(u, r_lane)
        rstd = 1 / torch.sqrt(var + EPS)
        rel = O.rstd_rel_bound(var, dvar, EPS)
        gm, be = _d(gam[b]), _d(bet[b])
        sc = gm * rstd
        mean_k, rstd_k, sc_k, sh_k = (_d(stats[i][b]) for i in range(4))
        O.within(mean_k[cl], mu, dmean, wb + " mean", bits=24)
        O.within(rstd_k[cl], rstd, rel * rstd, wb + " rstd", bits=24)
        O.within(sc_k[cl], sc, (rel + 2 * O.EPS32) * sc.abs(), wb + " scale", bits=24)
        O.within(sh_k[cl], be - mu * sc, sc.abs() * (dmean + mu.abs() * (rel + 2 * O.EPS32))
                 + 4 * O.EPS32 * (be.abs() + (mu * sc).abs()), wb + " shift", bits=24)
        unb = var * m / (m - 1)       # unbiased over the GLOBAL count, as nn.SyncBatchNorm
        rm0, rv0 = _d(rms[b]), _d(rvs[b])
        O.within(_d(rm[b]), (1 - mom) * rm0 + mom * mu,
                 mom * dmean + 4 * O.EPS32 * ((1 - mom) * rm0.abs() + mom * mu.abs()), wb + " running_mean", bits=24)
        O.within(_d(rv[b]), (1 - mom) * rv0 + mom * unb,
                 mom * dvar * m / (m - 1) + 4 * O.EPS32 * ((1 - mom) * rv0 + mom * unb), wb + " running_var", bits=24)


def bwd_reduce(d, us, sc, sh, mean, rstd, res, m, c, c_log, act, res_after, gacc=None, bacc=None):
    nb = len(us)
    scratch = torch.full((lib().hb_bn_bwd_scratch_doubles(m, c, nb),), float("nan"), device=DEV, dtype=torch.float64)
    dg, dgbuf = guarded(nb * c)
    db, dbbuf = guarded(nb * c)
    up = [ptr(us[i]) if i < nb else None for i in range(3)]
    rc = lib().hb_bn_act_bwd_reduce_bf16(ptr(d), up[0], up[1], up[2], nb, ptr(sc), ptr(sh), ptr(mean), ptr(rstd),
                                         ptr(res), ptr(scratch), ptr(dg), ptr(db), K._arr3(gacc) if gacc else None,
                                         K._arr3(bacc) if bacc else None, c_log, m, c, act, ctypes.c_float(SLOPE),
                                         int(res_after), stream_ptr())
    assert rc == 0, rc
    torch.cuda.synchronize()
    assert_guard(dgbuf, nb * c, "reduce dgamma")
    assert_guard(dbbuf, nb * c, "reduce dbeta")
    return scratch, dg.view(nb, c), db.view(nb, c)


def bwd_apply(d, us, sc, sh, mean, rstd, res, sums, count, m, c, act, res_after):
    nb = len(us)
    dus = [guarded(m * c, torch.bfloat16) for _ in range(nb)]
    dres = guarded(m * c, torch.bfloat16) if res is not None else None
    up = [ptr(us[i]) if i < nb else None for i in range(3)]
    dp = [ptr(dus[i][0]) if i < nb else None for i in range(3)]
    rc = lib().hb_bn_act_bwd_apply_bf16(ptr(d), up[0], up[1], up[2], nb, ptr(sc), ptr(sh), ptr(mean), ptr(rstd), ptr(res),
                                        ptr(sums), ptr(count), dp[0], dp[1], dp[2], ptr(dres[0]) if dres else None, m, c,
                                        act, ctypes.c_float(SLOPE), int(res_after), stream_ptr())
    assert rc == 0, rc
    torch.cuda.synchronize()
    for i, (_, b) in enumerate(dus):
        assert_guard(b, m * c, f"apply du{i}")
    if dres:
        assert_guard(dres[1], m * c, "apply dres")
    return [v.view(m, c) for v, _ in dus], dres[0].view(m, c) if dres else None


# (B, act, residual, C, C_logical, rows of each shard)
BWD_CASES = [(1, O.ACT_RELU, "none", 48, 48, (1500, 1501)), (1, O.ACT_SILU, "inside", 152, 152, (777, 2300)),
             (2, O.ACT_NONE, "none", 304, 300, (2000, 1023)), (2, O.ACT_LEAKY, "after", 200, 200, (1, 2999)),
             (3, O.ACT_RELU, "none", 64, 64, (1024, 1024)), (3, O.ACT_RELU6, "inside", 1280, 1280, (300, 700)),
             (1, O.ACT_FRELU, "inside", 96, 96, (900, 1100))]


@pytest.mark.parametrize("case", range(len(BWD_CASES)))
def test_backward_split(case):
    nb, act, res, c, c_log, shards = BWD_CASES[case]
    after = res == "after"
    what = f"split bwd B={nb} act={act} res={res} C={c}/{c_log} shards={shards}"
    m = sum(shards)
    us, sc, sh, mean, rstd = make_branches(nb, m, c, 4.0, seed=600 + case, c_log=c_log, gamma_hi=4.0)
    g = _gen(700 + case)
    r = bf16_rows(m, c, 0.0, 1.5, g) if res != "none" else None
    d = bf16_rows(m, c, 0.3, 1.0, g)
    # one shard: reduce + apply over the local count is hb_bn_act_bwd_bf16 (train = 1), bit for bit
    count = torch.tensor([float(m)], device=DEV, dtype=torch.float64)
    scratch, dg1, db1 = bwd_reduce(d, us, sc, sh, mean, rstd, r, m, c, c_log, act, after)
    dus1, dres1 = bwd_apply(d, us, sc, sh, mean, rstd, r, scratch, count, m, c, act, after)
    dus0, dres0, dg0, db0 = backward(d, us, sc, sh, mean, rstd, r, m, c, c_log, act, after, 1)
    for x, y in zip(dus0 + [dres0, dg0, db0], dus1 + [dres1, dg1, db1]):
        assert x is None or torch.equal(x, y), what + ": split differs from the one-call backward"
    # two shards: local reduce, fp64 sum of the [1+B][C] sums, apply with the global count
    lo, parts = 0, []
    for ms in shards:
        sl = slice(lo, lo + ms)
        sus = [u[sl].contiguous() for u in us]
        sr = r[sl].contiguous() if r is not None else None
        sd = d[sl].contiguous()
        parts.append((sus, sr, sd, ms) + bwd_reduce(sd, sus, sc, sh, mean, rstd, sr, ms, c, c_log, act, after))
        lo += ms
    n_sums = (1 + nb) * c
    total = parts[0][4][:n_sums] + parts[1][4][:n_sums]
    dus, dres = [[] for _ in range(nb)], []
    for sus, sr, sd, ms, _, _, _ in parts:
        du, dr = bwd_apply(sd, sus, sc, sh, mean, rstd, sr, total, count, ms, c, act, after)
        for b in range(nb):
            dus[b].append(du[b])
        dres.append(dr)
    r_red = max(reduce_rows(c, ms) for ms in shards)
    ref = ref_backward(d, us, sc, sh, mean, rstd, r, act, after, 1, r_red)
    O.mask_fraction_ok(ref["mask"][:, :c_log], what)
    cl = slice(0, c_log)
    for b in range(nb):
        du = torch.cat(dus[b])
        O.within(du[:, cl], ref["du"][b][:, cl], ref["du_slack"][b][:, cl], f"{what} du{b}", ref["mask"][:, cl])
        if c_log < c:
            assert bool((du[:, c_log:] == 0).all()), f"{what} du{b}: padded channels not zero"
        # parameter gradients stay local: their sum over the shards is the full-batch gradient
        for key, k in (("dg", 5), ("db", 6)):
            loc = [_d(p[k][b][cl]) for p in parts]
            O.within(loc[0] + loc[1], ref[key][b][cl], ref[key + "_slack"][b][cl] + O.EPS32 * (loc[0].abs() + loc[1].abs()),
                     f"{what} {key}{b} summed over shards", bits=24)
    if r is not None:
        dr = torch.cat(dres)
        O.within(dr[:, cl], ref["dres"][:, cl], ref["dres_slack"][:, cl], f"{what} dres", ref["mask"][:, cl])


def test_entry_points_reject_bad_arguments():
    L = lib()
    c = 48
    sums = torch.zeros(2 * c + 1, device=DEV, dtype=torch.float64)
    p = torch.zeros(4, c, 2, device=DEV)
    assert L.hb_bn_partials_sums(K._arr3([p]), K._I3(0, 0, 0), 1, c, c, 10, ptr(sums), stream_ptr()) != 0   # no slot
    assert L.hb_bn_partials_sums(K._arr3([p]), K._I3(4, 0, 0), 4, c, c, 10, ptr(sums), stream_ptr()) != 0   # B > 3
    assert L.hb_bn_partials_sums(K._arr3([p]), K._I3(4, 0, 0), 1, c, c, 10, None, stream_ptr()) != 0
    assert L.hb_bn_finalize_sums(None, None, None, None, None, None, None, None, None, None, 1, c, c,
                                 ctypes.c_float(EPS), ctypes.c_float(0.1), stream_ptr()) != 0
    assert L.hb_bn_act_bwd_apply_bf16(None, None, None, None, 1, None, None, None, None, None, ptr(sums), None, None,
                                      None, None, None, 10, c, 0, ctypes.c_float(0.0), 0, stream_ptr()) != 0   # no count
    assert L.hb_bn_act_bwd_reduce_bf16(None, None, None, None, 1, None, None, None, None, None, ptr(sums), None, None,
                                       None, None, c, 10, 44, 0, ctypes.c_float(0.0), 0, stream_ptr()) != 0   # C % 8
