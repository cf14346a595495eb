"""The fp64 optimizer steps of tests/_optim_oracle.py are right, their bound can fail, and the case tables of the GPU
tests hold what they promise. Runs without a GPU."""
import pytest
import torch

import _optim_oracle as O
from _bounds import FP32_BITS, ulp
from holocron_b200._lib import lib
from oracle import optim as OO

from conftest import load_golden


def _zero_state(name, p, kw):
    t = {k: torch.zeros_like(p) for k in O.state_keys(name, {**kw, "first": True} if name == "lars" else kw)}
    if name == "tadam":
        b1 = kw["betas"][0]
        t["W_t"] = b1 / (1 - b1) * torch.ones(1)
    return t


def _iterate(name, kw, p0, grad_of, steps, keep):
    """fp64 steps from zero state with the state rounded to fp32 between them, as the optimizers store it."""
    ps = [p.clone() for p in p0]
    states = [_zero_state(name, p, kw) for p in ps]
    traj, last = [], None
    for it in range(1, steps + 1):
        last = []
        for i, st in enumerate(states):
            out, info = O.STEPS[name]({"p": ps[i], "g": grad_of(i, it), **st}, it, kw)
            for k, e in out.items():
                if k == "p":
                    ps[i] = e.v.float()
                elif k not in ("g", "local_lr"):
                    st[k] = e.v.float()
            last.append((out, info))
        if it in keep:
            traj.append([p.clone() for p in ps])
    return traj, last


def _same(traj, ref, rtol, atol):
    assert len(traj) == len(ref)
    for ours, want in zip(traj, ref):
        for a, b in zip(ours, want):
            torch.testing.assert_close(a, b, rtol=rtol, atol=atol)


# the tolerances are those at which tests/test_oracle_golden.py pins the fp32 restatements to the same files: what fp32
# rounding leaves of agreement after three to six steps
@pytest.mark.parametrize("name,tol", [("adabelief", 2e-5), ("adabelief_wd_ams", 2e-5), ("lamb", 2e-5), ("lamb_wd", 2e-5),
                                      ("tadam", 5e-5), ("tadam_wd_ams_dof", 5e-5)])
def test_fp64_steps_reproduce_reference_trajectories(name, tol):
    g = load_golden("optim")
    traj, _ = _iterate(name.split("_")[0], g[name + "_kw"], g["p0"], lambda i, it: g["grads"][it - 1][i], 3, (1, 2, 3))
    _same(traj, g[name], tol, 1e-6)


@pytest.mark.parametrize("amsgrad,wd", [(False, 0.0), (True, 1e-2)])
def test_fp64_adamp_reproduces_reference(amsgrad, wd):
    g = load_golden("optim")["adamp"]
    kw = {"lr": 1e-2, "betas": (0.9, 0.99), "eps": 1e-8, "weight_decay": wd, "delta": 0.1, "amsgrad": amsgrad}
    traj, last = _iterate("adamp", kw, g["params"], lambda i, it: g["grads"][i] * it, 3, (3,))
    _same(traj, [g["after"][f"adamp_{int(amsgrad)}"]], 1e-6, 1e-8)


@pytest.mark.parametrize("name", ["adan", "adan_wd_ams", "ademamix", "ademamix_wd", "lars", "lars_mom_wd", "lars_nesterov",
                                  "ralars", "ralars_rect_wd", "ralars_force"])
def test_fp64_steps_reproduce_remaining_reference_trajectories(name):
    g = load_golden("optim2")
    kw = g[name]["kw"]
    fn = name.split("_")[0]

    if fn == "lars":        # the buffers appear on the first step and are read from the second on
        ps = [p.clone() for p in g["params"]]
        bufs, traj, grads = [None] * len(ps), [], None
        for it in range(1, 7):
            grads = []
            for i, p0 in enumerate(g["params"]):
                t = {"p": ps[i], "g": g["grads"][i] * it + 0.01 * p0}
                if bufs[i] is not None:
                    t["momentum_buffer"] = bufs[i]
                out, _ = O.lars(t, it, kw)
                ps[i] = out["p"].v.float()
                if "momentum_buffer" in out:
                    bufs[i] = out["momentum_buffer"].v.float()
                grads.append(out["g"].v.float() if "g" in out else t["g"])
            if it in (1, 3, 6):
                traj.append([p.clone() for p in ps])
        _same(traj, g[name]["traj"], 2e-6, 2e-6)
        if "grad_after" in g[name]:
            _same([grads], [g[name]["grad_after"]], 1e-6, 1e-7)
        return
    traj, last = _iterate(fn, kw, g["params"], lambda i, it: g["grads"][i] * it + 0.01 * g["params"][i], 6, (1, 3, 6))
    _same(traj, g[name]["traj"], 2e-6, 2e-6)
    if fn == "ralars":
        for (out, _), want in zip(last, g[name]["local_lr"]):
            assert abs(float(out["local_lr"].v) - want) <= 1e-5 * max(1.0, abs(want))


def test_fp64_lookahead_reproduces_reference():
    g = load_golden("optim2")
    ps = [torch.nn.Parameter(p.clone()) for p in g["params"]]
    slow = [p.detach().clone() for p in ps]
    base = torch.optim.SGD(ps, lr=0.1, momentum=0.9)
    traj = []
    for it in range(1, 8):
        for p, p0, gr in zip(ps, g["params"], g["grads"]):
            p.grad = gr * it + 0.01 * p0
        base.step()
        if it % 3 == 0:
            for i, f in enumerate(ps):
                out, _ = O.lookahead({"p": f.data, "slow": slow[i]}, it, {"sync_rate": 0.5})
                slow[i] = out["slow"].v.float()
                f.data.copy_(slow[i])
        if it in (2, 3, 7):
            traj.append([p.detach().clone() for p in ps])
    _same(traj, g["lookahead"]["traj"], 2e-6, 2e-6)
    _same([slow], [g["lookahead"]["slow"]], 2e-6, 2e-6)


def _fp32_restatement(name, t, step, kw):
    """One in-place step of oracle/optim.py on clones; returns the tensors it wrote, named as the fp64 step names them."""
    c = {k: v.clone() for k, v in t.items()}
    # hyper-parameters as the C ABI receives them: 1 - beta^step of a beta near 1 moves by 1e-5 with the beta's rounding
    kw = {k: O.f32(v) if isinstance(v, float) else tuple(O.f32(b) for b in v) if isinstance(v, tuple) else v
          for k, v in kw.items()}
    wd, ams = kw.get("weight_decay", 0.0), kw.get("amsgrad", False)
    if name == "adabelief":
        OO.adabelief_step(c["p"], c["g"], c["exp_avg"], c["exp_avg_sq"], step, kw["lr"], *kw["betas"], kw["eps"], wd, ams,
                          c.get("max_exp_avg_sq"))
    elif name == "lamb":
        c["local_lr"] = torch.tensor(OO.lamb_step(c["p"], c["g"], c["exp_avg"], c["exp_avg_sq"], kw["lr"], *kw["betas"],
                                                  kw["eps"], wd, kw["scale_clip"]))
    elif name == "tadam":
        OO.tadam_step(c["p"], c["g"], c["exp_avg"], c["exp_avg_sq"], c["W_t"], step, kw["lr"], *kw["betas"], kw["eps"], wd,
                      kw.get("dof"), ams, c.get("max_exp_avg_sq"))
    elif name == "adamp":
        OO.adamp_step(c["p"], c["g"], c["exp_avg"], c["exp_avg_sq"], step, kw["lr"], *kw["betas"], kw["eps"], wd, 0.1, ams,
                      c.get("max_exp_avg_sq"))
    elif name == "adan":
        OO.adan_step(c["p"], c["g"], c["prev_grad"], c["exp_avg"], c["exp_avg_sq"], c["exp_avg_delta"], step, kw["lr"],
                     *kw["betas"], kw["eps"], wd, ams, c.get("max_exp_avg_delta"))
    elif name == "ademamix":
        OO.ademamix_step(c["p"], c["g"], c["exp_avg"], c["exp_avg_slow"], c["exp_avg_sq"], step, kw["lr"], *kw["betas"],
                         kw["alpha"], kw["eps"], wd)
    elif name == "lars":
        buf = OO.lars_step(c["p"], c["g"], c.get("momentum_buffer"), kw["lr"], kw.get("momentum", 0.0),
                           kw.get("dampening", 0.0), wd, kw.get("nesterov", False))
        if buf is not None:
            c["momentum_buffer"] = buf
    elif name == "ralars":
        c["local_lr"] = torch.tensor(OO.ralars_step(c["p"], c["g"], c["exp_avg"], c["exp_avg_sq"], step, kw["lr"],
                                                    *kw["betas"], kw["eps"], wd, kw["force_adaptive_momentum"],
                                                    kw["scale_clip"]))
    else:
        OO.lookahead_sync(c["p"], c["slow"], kw["sync_rate"])
    return c


CASES = [(name, i) for name in O.STEPS for i in range(len(O.MODES[name]))]


@pytest.mark.parametrize("name,mode", CASES)
@pytest.mark.parametrize("numel", [1, 5, 4099])
def test_fp64_steps_agree_with_fp32_restatements_from_nonzero_state(name, mode, numel):
    """The eager fp32 restatement rounds as often as the kernel does, in another order and with python-double constants:
    it must sit inside twice the kernel's bound (REL counts the kernel's roundings; the restatement adds its own)."""
    kw, step = O.MODES[name][mode]
    gen = torch.Generator().manual_seed(numel * 100 + mode)
    t = O.random_tensors(name, (numel,), kw, gen, side=("project", "keep")[mode % 2] if name == "adamp" else None)
    out, info = O.STEPS[name](t, step, kw)
    got = _fp32_restatement(name, t, step, kw)
    if name == "adamp":
        assert abs(info["margin"]) > 100 * info["margin_err"]
    for key, e in out.items():
        O.assert_within(got[key], e.v, e.e, f"{name} {kw}: {key}", rel=2 * O.REL, bits=FP32_BITS)
    for key in set(t) - set(out):
        assert torch.equal(got[key], t[key]), key


def _rejects(got, out, what):
    with pytest.raises(AssertionError, match=what):
        O.check(got, out, "planted")


def test_bound_rejects_planted_errors():
    C = lib().hb_optim_chunk_elems()
    gen = torch.Generator().manual_seed(7)
    for name in ("adabelief", "lamb", "adan", "ademamix", "ralars", "tadam", "adamp"):
        kw, step = O.MODES[name][1]
        t = O.random_tensors(name, (2 * C + 3,), kw, gen)
        out, _ = O.STEPS[name](t, step, kw)
        exact = {k: e.v.float() for k, e in out.items()}
        O.check(exact, out, name)                                   # the correctly rounded result passes
        # one element of one state tensor off by 4 ulps
        for key in ("exp_avg", "exp_avg_sq"):
            bad = dict(exact)
            bad[key] = exact[key].clone()
            bad[key][C + 1] += 4 * ulp(out[key].v[C + 1], FP32_BITS).float()
            _rejects(bad, out, f"{key}: 1 of")
        # the bias corrections of the step before
        if name not in ("lamb",):
            prev, _ = O.STEPS[name](t, step - 1 if step > 1 else step + 1, kw)
            _rejects({**exact, "p": prev["p"].v.float()}, out, "planted: p")
        # a per-tensor reduction that only saw the first chunk
        first = {k: (v[:C] if v.numel() > 1 else v) for k, v in t.items()}
        part, _ = O.STEPS[name](first, step, kw)
        for key in O.SCALARS:
            if key in out:
                _rejects({**exact, key: part[key].v.float()}, out, f"planted: {key}")
    # an amsgrad maximum that is not stored
    kw, step = O.MODES["adabelief"][2]
    t = O.random_tensors("adabelief", (C + 5,), kw, gen)
    out, info = O.adabelief(t, step, kw)
    assert 0.2 < info["max_kept"] < 0.8
    _rejects({**{k: e.v.float() for k, e in out.items()}, "max_exp_avg_sq": t["max_exp_avg_sq"]}, out, "max_exp_avg_sq")
    # a LARS gradient that misses its weight decay, a Lookahead that forgets the fast weights
    kw, step = next((k, s) for k, s in O.MODES["lars"] if k["weight_decay"] and k.get("momentum"))
    t = O.random_tensors("lars", (C + 5,), kw, gen)
    out, _ = O.lars(t, step, kw)
    _rejects({**{k: e.v.float() for k, e in out.items()}, "g": t["g"]}, out, "planted: g")
    t = O.random_tensors("lookahead", (C + 5,), {}, gen)
    out, _ = O.lookahead(t, 1, {"sync_rate": 0.5})
    _rejects({"slow": out["slow"].v.float(), "p": t["p"]}, out, "planted: p")


def test_case_tables_hold_what_the_gpu_tests_promise():
    C = lib().hb_optim_chunk_elems()
    assert C % 4 == 0 and C >= 1024
    s = O.sizes(C)
    for edge in (4, C, 2 * C):                       # below, at and above the vector width and one and two chunks
        assert any(n < edge for n in s) and edge in s and any(edge < n < edge + 8 for n in s), edge
    assert {n % 4 for n in s} == {0, 1, 2, 3} and 1 in s and max(s) > 200 * C and any(3 * C < n < 4 * C for n in s)
    tab = O.table_sizes(C)
    assert len(tab) >= 190 and 0 in tab[1:-1] and tab.count(1) >= 40 and max(tab) >= 1_000_000
    for edge in (C, 2 * C):
        assert {edge - 1, edge, edge + 1} <= set(tab)
    big = tab.index(max(tab))
    assert tab[big - 1] < C and 0 < big < len(tab) - 1           # small tensors sit next to the large one
    scales = {O.table_scale(i) for i in range(len(tab))}
    assert min(scales) <= 1e-3 and max(scales) >= 1e2
    assert len({(n, O.table_scale(i)) for i, n in enumerate(tab)}) >= len(set(tab)) * len(scales) - len(scales)
    assert all(n > C and n % 4 for n in O.alignment_sizes(C)) and any(n > 2 * C for n in O.alignment_sizes(C))
    for name in O.STEPS:
        modes = O.MODES[name]
        if name not in ("lookahead",):
            assert {bool(k.get("weight_decay")) for k, _ in modes} == {False, True}, name
        if "max_exp_avg_sq" in O.STATE[name] or name == "adan":
            assert {bool(k.get("amsgrad")) for k, _ in modes} == {False, True}, name
        for kw, _ in modes:
            cases = O.alignment_cases(name, kw)
            keys = set(cases[0])
            assert keys >= {"p"} | set(O.state_keys(name, kw))
            assert {o for c in cases for o in c.values()} == {0, 1, 2, 3}
            assert any(not any(c.values()) for c in cases)
            for k in keys:                                       # each tensor alone off its boundary
                assert any(c[k] and not any(v for kk, v in c.items() if kk != k) for c in cases), (name, k)
            assert sum(len(set(c.values())) == 1 and c["p"] != 0 for c in cases) == 3
    assert {k.get("dof") for k, _ in O.MODES["tadam"]} == {None, 5.0}
    for name in ("lamb", "ralars"):
        assert {k["scale_clip"] for k, _ in O.MODES[name]} == {O.CLIP_BELOW, O.CLIP_ABOVE, O.CLIP_NONE}
    assert {O.ralars_mode(s, k["betas"][1], k["force_adaptive_momentum"])[0] for k, s in O.MODES["ralars"]} == {0, 1, 2}
    lars = {(bool(k.get("momentum")), bool(k.get("dampening")), bool(k.get("nesterov")), k["first"]) for k, _ in O.MODES["lars"]}
    assert lars == {(False, False, False, False), (True, True, False, False), (True, True, False, True),
                    (True, False, True, False), (True, False, True, True)}
    assert {k["sync_rate"] for k, _ in O.MODES["lookahead"]} == {0.0, 0.5, 1.0}
    # both sides of AdamP's projection, with a margin far above what rounding can move
    gen = torch.Generator().manual_seed(3)
    for side in ("project", "keep"):
        for n in s[:-1]:
            kw, step = O.MODES["adamp"][1]
            _, info = O.adamp(O.random_tensors("adamp", (n,), kw, gen, side=side), step, kw)
            assert info["project"] == (side == "project") and abs(info["margin"]) > 100 * info["margin_err"], (side, n)
