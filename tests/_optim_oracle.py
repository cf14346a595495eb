"""One step of each fused optimizer (holocron_b200/csrc/optim.cu) in fp64 from an ARBITRARY state, with a per-element
bound on what an fp32 evaluation of the same expression may differ by, and the case tables of the GPU tests.

Every quantity is an :class:`E`: its fp64 value and a first-order bound on the absolute error of the kernel's fp32 value,
counted in units of ``U = 2^-24`` (the unit roundoff of fp32). Exact inputs carry 0; every fp32 operation adds its operands'
errors, propagated through the operation, plus one rounding ``|value|``; a per-tensor sum adds ``17 |terms|`` (at most 16
fp32 additions per thread, fp64 from the block reduction on, one rounding back to fp32). The kernel must then lie within

    one fp32 ulp at the reference value  +  REL * error count                                   (REL = 2^-24)

per element, which is ``_bounds.assert_within`` with the count as its magnitude tensor. The count is the same expression
evaluated on absolute values wherever that is a bound; where it is not (a square root or a quotient of a cancelling
difference) the propagated form is what holds. Nothing in it is fitted to a run: a fused multiply-add the kernel performs
with one rounding is counted with two, so the bound is loose by a small factor and never tight by one.

Hyper-parameters are rounded to fp32 before use, as the C ABI receives them; the bias corrections are computed in fp64
from the rounded betas and rounded to fp32, as ``make_hyper`` and ``bias_corrections`` do."""
import math
from typing import Dict, Optional, Tuple

import numpy as np
import torch

from _bounds import FP32_BITS, assert_within

U = 2.0 ** -24
REL = U          # the bound's error counts are in units of one fp32 rounding
SUM_TERMS = 17   # per-tensor reductions: <= 16 fp32 additions per thread (4096 / 256), then fp64, then one rounding


def f32(x: float) -> float:
    return float(np.float32(x))


class E:
    """fp64 value ``v`` and error count ``e`` (absolute error bound of the fp32 evaluation, in units of U)."""
    __slots__ = ("v", "e")

    def __init__(self, v: torch.Tensor, e: Optional[torch.Tensor] = None) -> None:
        self.v = v
        self.e = torch.zeros_like(v) if e is None else e

    @staticmethod
    def exact(t: torch.Tensor, dev) -> "E":
        return E(t.detach().to(dev, torch.float64))

    def rnd(self) -> "E":
        """One more rounding to fp32 (a double narrowed to float)."""
        return E(self.v, self.e + self.v.abs())

    def __add__(self, o: "E") -> "E":
        return E(self.v + o.v, self.e + o.e).rnd()

    def __sub__(self, o: "E") -> "E":
        return E(self.v - o.v, self.e + o.e).rnd()

    def __mul__(self, o: "E") -> "E":
        return E(self.v * o.v, self.v.abs() * o.e + o.v.abs() * self.e).rnd()

    def __truediv__(self, o: "E") -> "E":
        q = self.v / o.v
        return E(q, (self.e + q.abs() * o.e) / o.v.abs()).rnd()

    def __neg__(self) -> "E":
        return E(-self.v, self.e)

    def sqrt(self) -> "E":
        # |sqrt(a + d) - sqrt(a)| = |d| / (sqrt(a + d) + sqrt(a)) <= min(|d| / sqrt(a), sqrt|d|): the second form is what is
        # left of the bound where a itself is (nearly) zero
        s = self.v.sqrt()
        d = self.e * U
        return E(s, torch.minimum(d / s.clamp_min(1e-300), d.sqrt()) / U).rnd()

    def sum(self) -> "E":
        return E(self.v.sum(), self.e.sum() + SUM_TERMS * self.v.abs().sum())

    def clamp(self, lo: float, hi: float) -> "E":
        # a value beyond a limit by more than its own error is the limit exactly
        c = self.v.clamp(lo, hi)
        return E(c, (self.e - (self.v - c).abs() / U).clamp_min(0))


def fma(a: E, b: E, c: E) -> E:
    return E(a.v * b.v + c.v, a.v.abs() * b.e + b.v.abs() * a.e + c.e).rnd()


def maximum(a: E, b: E) -> E:
    return E(torch.maximum(a.v, b.v), torch.maximum(a.e, b.e))


def where(cond: torch.Tensor, a: E, b: E) -> E:
    return E(torch.where(cond, a.v, b.v), torch.where(cond, a.e, b.e))


def bias_correction(beta: float, step: int) -> float:
    """1 - beta^step in fp64 from the fp32 beta, rounded to fp32 (make_hyper / bias_corrections of optim.cu)."""
    return f32(1.0 - f32(beta) ** step)


class _Ctx:
    """The fp32 tensors of one parameter as exact E's on one device, and fp32-rounded constants."""

    def __init__(self, t: Dict[str, torch.Tensor], dev) -> None:
        self.t, self.dev = t, dev

    def __call__(self, key: str) -> E:
        return E.exact(self.t[key], self.dev)

    def c(self, x: float) -> E:
        return E(torch.tensor(f32(x), dtype=torch.float64, device=self.dev))


def _adam_moments(x: _Ctx, g: E, kw) -> Tuple[E, E, E]:
    """The two Adam EMAs shared by LAMB / AdamP / AdEMAMix / RaLars (and the constant 1)."""
    one, b1, b2 = x.c(1), x.c(kw["betas"][0]), x.c(kw["betas"][1])
    m = fma(one - b1, g, b1 * x("exp_avg"))
    v = fma(one - b2, g * g, b2 * x("exp_avg_sq"))
    return m, v, one


def _decayed(x: _Ctx, p: E, g: E, kw) -> E:
    wd = kw.get("weight_decay", 0.0)
    return fma(x.c(wd), p, g) if f32(wd) != 0 else g


def _second(x: _Ctx, v: E, kw, key: str, out: Dict[str, E], info) -> E:
    """The amsgrad running maximum, when asked for."""
    if not kw.get("amsgrad", False):
        return v
    old = x(key)
    info["max_kept"] = float((old.v > v.v).double().mean()) if v.v.numel() else 0.0
    out[key] = maximum(old, v)
    return out[key]


def _trust_ratio(x: _Ctx, p: E, u: E, kw, info) -> E:
    """clamp(||p||, *scale_clip) / ||u||, 1 when either is zero (LAMB, RaLars)."""
    lo, hi = (f32(c) for c in kw.get("scale_clip") or (0.0, 10.0))
    pn, un = (p * p).sum().sqrt(), (u * u).sum().sqrt()
    phi = pn.clamp(lo, hi)
    info["clip"] = -1 if float(pn.v) < lo else (1 if float(pn.v) > hi else 0)
    return where((phi.v == 0) | (un.v == 0), x.c(1), phi / un)


def adabelief(t, step, kw, dev="cpu"):
    x = _Ctx(t, dev)
    out, info = {}, {}
    p = x("p")
    g = _decayed(x, p, x("g"), kw)
    one, b1, b2 = x.c(1), x.c(kw["betas"][0]), x.c(kw["betas"][1])
    m = fma(one - b1, g, b1 * x("exp_avg"))
    r = g - m
    s = fma(one - b2, r * r, b2 * x("exp_avg_sq"))
    out["exp_avg"], out["exp_avg_sq"] = m, s
    sec = _second(x, s, kw, "max_exp_avg_sq", out, info)
    bc1, bc2 = x.c(bias_correction(kw["betas"][0], step)), x.c(bias_correction(kw["betas"][1], step))
    denom = sec.sqrt() * (one / bc2.sqrt()) + x.c(kw["eps"])
    out["p"] = p - (x.c(kw["lr"]) / bc1) * (m / denom)
    return out, info


def lamb(t, step, kw, dev="cpu"):
    x = _Ctx(t, dev)
    out, info = {}, {}
    p, g = x("p"), x("g")
    m, v, _ = _adam_moments(x, g, kw)
    out["exp_avg"], out["exp_avg_sq"] = m, v
    u = m / (v.sqrt() + x.c(kw["eps"]))
    u = _decayed(x, p, u, kw)
    out["local_lr"] = _trust_ratio(x, p, u, kw, info)
    out["p"] = p - (x.c(kw["lr"]) * out["local_lr"]) * u
    return out, info


def tadam(t, step, kw, dev="cpu"):
    x = _Ctx(t, dev)
    out, info = {}, {}
    p = x("p")
    g = _decayed(x, p, x("g"), kw)
    one, b1, b2 = x.c(1), x.c(kw["betas"][0]), x.c(kw["betas"][1])
    m0, v0, W = x("exp_avg"), x("exp_avg_sq"), x("W_t")
    d = g - m0
    acc = ((d * d) / (v0 + x.c(kw["eps"]))).sum().rnd()
    n = float(t["p"].numel())
    dof = x.c(n if kw.get("dof") is None else kw["dof"])
    w = (dof + x.c(n)) / (acc + dof)
    m = m0 * (W / (W + w)) + (w * g) / (W + w)
    v = fma(one - b2, g * g, b2 * v0)
    out["exp_avg"], out["exp_avg_sq"] = m, v
    sec = _second(x, v, kw, "max_exp_avg_sq", out, info)
    bc1, bc2 = x.c(bias_correction(kw["betas"][0], step)), x.c(bias_correction(kw["betas"][1], step))
    denom = sec.sqrt() * (one / bc2.sqrt()) + x.c(kw["eps"])
    out["p"] = p - (x.c(kw["lr"]) / bc1) * (m / denom)
    out["W_t"] = W * ((x.c(2) * b1 - one) / b1) + w
    info["w"] = w
    return out, info


def adamp(t, step, kw, dev="cpu"):
    x = _Ctx(t, dev)
    out, info = {}, {}
    p = x("p")
    g = _decayed(x, p, x("g"), kw)
    m, v, one = _adam_moments(x, g, kw)
    out["exp_avg"], out["exp_avg_sq"] = m, v
    sec = _second(x, v, kw, "max_exp_avg_sq", out, info)
    bc1, bc2 = x.c(bias_correction(kw["betas"][0], step)), x.c(bias_correction(kw["betas"][1], step))
    eps = x.c(kw["eps"])
    pt = (m / bc1) / (sec.sqrt() * (one / bc2.sqrt()) + eps)
    pn, gn = (p * p).sum().sqrt(), (g * g).sum().sqrt()
    floor = x.c(1e-8)      # F.cosine_similarity clamps each norm
    cosv = (p * g).sum().rnd() / (maximum(pn, floor) * maximum(gn, floor))
    thr = x.c(kw.get("delta", 0.1)) / x.c(float(t["p"].numel())).sqrt()
    # the projection is a discontinuous decision: the caller keeps |margin| well above what fp32 can move it by
    info["margin"] = float(cosv.v - thr.v)
    info["margin_err"] = float((cosv.e + thr.e) * U)
    info["project"] = info["margin"] < 0
    if info["project"]:
        inv = one / (pn + eps)
        k = (p * pt).sum().rnd() * inv * inv
        pt = fma(-k, p, pt)
    out["p"] = fma(-x.c(kw["lr"]), pt, p)
    return out, info


def adan(t, step, kw, dev="cpu"):
    x = _Ctx(t, dev)
    out, info = {}, {}
    p = x("p")
    g = _decayed(x, p, x("g"), kw)
    one = x.c(1)
    b1, b2, b3 = (x.c(b) for b in kw["betas"])
    m = fma(one - b1, g, b1 * x("exp_avg"))
    dg = g - x("prev_grad")
    v = fma(one - b2, dg, b2 * x("exp_avg_sq"))
    tmp = fma(b2, dg, g)
    n = fma(one - b3, tmp * tmp, b3 * x("exp_avg_delta"))
    out["exp_avg"], out["exp_avg_sq"], out["exp_avg_delta"] = m, v, n
    sec = _second(x, n, kw, "max_exp_avg_delta", out, info)
    bc1, bc2, bc3 = (x.c(bias_correction(b, step)) for b in kw["betas"])
    denom = sec.sqrt() * (one / bc3.sqrt()) + x.c(kw["eps"])
    lr = x.c(kw["lr"])
    q = fma(-lr, (m / bc1 + b2 * v / bc2) / denom, p)
    wd = kw.get("weight_decay", 0.0)
    out["p"] = q / (one + x.c(wd) * lr) if f32(wd) != 0 else q
    return out, info


def ademamix(t, step, kw, dev="cpu"):
    x = _Ctx(t, dev)
    out, info = {}, {}
    p = x("p")
    g = _decayed(x, p, x("g"), kw)
    m1, nu, one = _adam_moments(x, g, kw)
    b3 = x.c(kw["betas"][2])
    m2 = fma(one - b3, g, b3 * x("exp_avg_slow"))
    out["exp_avg"], out["exp_avg_sq"], out["exp_avg_slow"] = m1, nu, m2
    bc1, bc2 = x.c(bias_correction(kw["betas"][0], step)), x.c(bias_correction(kw["betas"][1], step))
    denom = nu.sqrt() * (one / bc2.sqrt()) + x.c(kw["eps"])
    out["p"] = fma(-x.c(kw["lr"]), fma(x.c(kw.get("alpha", 5.0)), m2, m1 / bc1) / denom, p)
    return out, info


def lars(t, step, kw, dev="cpu"):
    """``momentum_buffer`` absent from ``t`` with a momentum: the launch that creates the buffers (a copy of g + wd p)."""
    x = _Ctx(t, dev)
    out, info = {}, {}
    p, g = x("p"), x("g")
    one = x.c(1)
    wd, mom = kw.get("weight_decay", 0.0), kw.get("momentum", 0.0)
    pn, gn = (p * p).sum().sqrt(), (g * g).sum().sqrt()
    denom = fma(x.c(wd), pn, gn) if f32(wd) != 0 else gn
    info["local_lr"] = where((pn.v == 0) | (denom.v == 0), one, pn / denom)
    if f32(wd) != 0:
        g = out["g"] = fma(x.c(wd), p, g)
    d = g
    if f32(mom) != 0:
        b = g if "momentum_buffer" not in t else \
            fma(x.c(mom), x("momentum_buffer"), (one - x.c(kw.get("dampening", 0.0))) * g)
        out["momentum_buffer"] = b
        d = fma(x.c(mom), b, g) if kw.get("nesterov", False) else b
    out["p"] = fma(-(x.c(kw["lr"]) * info["local_lr"]), d, p)
    return out, info


def ralars_mode(step: int, beta2: float, force_adaptive_momentum: bool) -> Tuple[int, float]:
    """The branch the host picks from the step count (optim/ralars.py): 0 rectified, 1 plain ratio, 2 momentum only."""
    sma_inf = 2 / (1 - beta2) - 1
    bc2 = 1 - beta2 ** step
    sma_t = sma_inf - 2 * step * (1 - bc2) / bc2
    if sma_t > 4:
        return 0, math.sqrt((sma_t - 4) * (sma_t - 2) * sma_inf / ((sma_inf - 4) * (sma_inf - 2) * sma_t))
    return (1 if force_adaptive_momentum else 2), 1.0


def ralars(t, step, kw, dev="cpu"):
    x = _Ctx(t, dev)
    out, info = {}, {}
    p, g = x("p"), x("g")
    m, v, _ = _adam_moments(x, g, kw)
    out["exp_avg"], out["exp_avg_sq"] = m, v
    bc1, bc2 = x.c(bias_correction(kw["betas"][0], step)), x.c(bias_correction(kw["betas"][1], step))
    info["mode"], r_t = ralars_mode(step, kw["betas"][1], kw.get("force_adaptive_momentum", False))
    u = m / bc1
    if info["mode"] != 2:
        u = x.c(r_t) * (u / ((v / bc2).sqrt() + x.c(kw["eps"])))
    u = _decayed(x, p, u, kw)
    out["local_lr"] = _trust_ratio(x, p, u, kw, info)
    out["p"] = fma(-(x.c(kw["lr"]) * out["local_lr"]), u, p)
    return out, info


def lookahead(t, step, kw, dev="cpu"):
    """``p`` the fast weights, ``slow`` the slow ones; both end up as slow + rate * (fast - slow)."""
    x = _Ctx(t, dev)
    f, s = x("p"), x("slow")
    rate = kw["sync_rate"]
    if f32(rate) > 0:
        s = fma(x.c(rate), f - s, s)
    return {"p": s, "slow": s}, {}


STEPS = {"adabelief": adabelief, "lamb": lamb, "tadam": tadam, "adamp": adamp, "adan": adan, "ademamix": ademamix,
         "lars": lars, "ralars": ralars, "lookahead": lookahead}

# full-size state tensors by optimizer (amsgrad maximum last, present only with amsgrad), as their state_dict names them
STATE = {"adabelief": ("exp_avg", "exp_avg_sq", "max_exp_avg_sq"), "lamb": ("exp_avg", "exp_avg_sq"),
         "tadam": ("exp_avg", "exp_avg_sq", "max_exp_avg_sq"), "adamp": ("exp_avg", "exp_avg_sq", "max_exp_avg_sq"),
         "adan": ("exp_avg", "exp_avg_sq", "exp_avg_delta", "prev_grad", "max_exp_avg_delta"),
         "ademamix": ("exp_avg", "exp_avg_slow", "exp_avg_sq"), "lars": ("momentum_buffer",), "ralars": ("exp_avg", "exp_avg_sq"),
         "lookahead": ("slow",)}
NON_NEGATIVE = ("exp_avg_sq", "exp_avg_delta", "max_exp_avg_sq", "max_exp_avg_delta")
SCALARS = ("local_lr", "W_t")      # per-tensor scalars the kernels store: compared on their own, before the parameters


def state_keys(name: str, kw) -> Tuple[str, ...]:
    keys = [k for k in STATE[name] if not k.startswith("max_") or kw.get("amsgrad", False)]
    if name == "lars" and (f32(kw.get("momentum", 0.0)) == 0 or kw.get("first", False)):
        keys = []
    return tuple(keys)


def random_tensors(name: str, shape, kw, gen: torch.Generator, scale: float = 1.0, side: Optional[str] = None
                   ) -> Dict[str, torch.Tensor]:
    """fp32 inputs of one step from a non-zero state (CPU). Second moments are non-negative and an amsgrad maximum is
    drawn around the second moment, so that the new moment lands above it on some elements and below it on others.
    ``side`` builds AdamP's gradient as a p + b q with q orthogonal to p: "project" (cosine far below the threshold) or
    "keep" (far above)."""
    def randn():
        return torch.randn(shape, generator=gen, dtype=torch.float32)

    def rand():
        return torch.rand(shape, generator=gen, dtype=torch.float32)

    t = {"p": randn() * scale}
    if name != "lookahead":
        t["g"] = randn() * (0.1 * scale)
    if side is not None:
        p64, q = t["p"].double(), randn().double() * scale
        if p64.numel() > 1:
            q = q - (q * p64).sum() / (p64 * p64).sum().clamp_min(1e-300) * p64
        else:
            q = q * 0
        a, b = (-0.5, 1.0) if side == "project" else (1.0, 0.5)
        t["g"] = (0.1 * (a * p64 + b * q)).float()
    for key in state_keys(name, kw):
        if key in ("max_exp_avg_sq", "max_exp_avg_delta"):
            t[key] = t["exp_avg_sq" if name != "adan" else "exp_avg_delta"] * (0.5 + rand())
        elif key in NON_NEGATIVE and not (name == "adan" and key == "exp_avg_sq"):     # Adan: EMA of a signed difference
            t[key] = (rand() * 0.01 + 1e-4) * scale * scale
        elif key == "slow":
            t[key] = t["p"] + randn() * (0.1 * scale)
        else:
            t[key] = randn() * (0.1 * scale)
    if name == "tadam":
        t["W_t"] = torch.rand(1, generator=gen, dtype=torch.float32) + 5.0
    return t


def check(got: Dict[str, torch.Tensor], out: Dict[str, E], what: str) -> None:
    """Every tensor the kernel writes against its bound: the per-tensor scalars first, so that a wrong reduction is
    reported as such and not as thousands of parameter failures (the parameter's own bound is built on the oracle's scalar
    and carries the scalar's error count)."""
    for key in sorted(out, key=lambda k: k not in SCALARS):
        assert_within(got[key], out[key].v, out[key].e, f"{what}: {key}", rel=REL, bits=FP32_BITS)


# ---------------------------------------------------------------------------------------------------------------------
# Case tables of tests/test_gpu_optim_bounds.py (walked by tests/test_optim_oracle_cpu.py so that they cannot be thinned
# unnoticed). C is the number of elements one CTA owns, lib().hb_optim_chunk_elems().
BIG = 1_000_003


def sizes(C: int):
    """Single-tensor tables: each side of the vector/tail split, of one and two chunk edges, and a real size."""
    return [1, 3, 4, 5, 6, 255, 1027, C - 1, C, C + 1, C + 4, 2 * C, 2 * C + 2, 2 * C + 3, 3 * C + 1029, BIG]


_AMS = [{}, {"weight_decay": 1e-2}, {"amsgrad": True}, {"weight_decay": 1e-2, "amsgrad": True}]
_B2 = {"lr": 1e-2, "betas": (0.9, 0.99), "eps": 1e-8}
CLIP_BELOW, CLIP_ABOVE, CLIP_NONE = (1e6, 1e7), (0.0, 1e-6), (0.0, 1e9)    # ||p|| is clamped up, down, not at all
# (constructor keywords, step the update is the ...th of). RaLars: its betas are exact in fp32 (7/8, 511/512), because the
# host derives r_t from the python doubles and the kernel its bias corrections from the fp32 values, and a restatement
# fed either kind alone would differ from both by 1e-5; with them the SMA length is 1 at step 1 (momentum only, or the plain
# ratio when forced) and ~9.9 at step 10 (rectified).
MODES = {
    "adabelief": [({**_B2, **m}, 4) for m in _AMS],
    "adamp": [({**_B2, **m}, 4) for m in _AMS],
    "tadam": [({**_B2, **m}, 4) for m in _AMS] + [({**_B2, "dof": 5.0}, 4),
                                                  ({**_B2, "dof": 5.0, "weight_decay": 1e-2, "amsgrad": True}, 4)],
    "adan": [({"lr": 1e-2, "betas": (0.98, 0.92, 0.99), "eps": 1e-8, **m}, 4) for m in _AMS],
    "ademamix": [({"lr": 1e-2, "betas": (0.9, 0.99, 0.999), "alpha": 5.0, "eps": 1e-8, **m}, 4) for m in _AMS[:2]],
    "lamb": [({**_B2, "scale_clip": c, **m}, 4) for c in (CLIP_NONE, CLIP_BELOW, CLIP_ABOVE) for m in _AMS[:2]],
    "lars": [({"lr": 0.1, "weight_decay": wd, "first": first, **m}, 4)
             for m in ({}, {"momentum": 0.9, "dampening": 0.1}, {"momentum": 0.9, "nesterov": True})
             for wd in (0.0, 1e-2) for first in ((False, True) if m else (False,))],
    "ralars": [({"lr": 1e-2, "betas": (0.875, 511 / 512), "eps": 1e-8, "weight_decay": wd, "scale_clip": c,
                 "force_adaptive_momentum": force}, step)
               for (force, step), wd, c in [((False, 1), 0.0, CLIP_NONE), ((False, 1), 1e-2, CLIP_BELOW),
                                            ((True, 1), 0.0, CLIP_ABOVE), ((True, 1), 1e-2, CLIP_NONE),
                                            ((False, 10), 0.0, CLIP_BELOW), ((False, 10), 1e-2, CLIP_ABOVE),
                                            ((False, 10), 1e-2, CLIP_NONE)]],
    "lookahead": [({"sync_rate": r}, 1) for r in (0.0, 0.5, 1.0)],
}
OPTIMIZERS = [n for n in MODES if n != "lookahead"]


def table_sizes(C: int):
    """One table of ~200 tensors: 1-element tensors and a zero-element one between tensors just under / at / over one
    and two chunks, and one of ~1 M elements in the middle."""
    unit = [1, C + 1, 3, 2 * C, 1, C - 1, 0, 2 * C + 3, 5, C, 1, 2 * C - 1, 2 * C + 1]
    out = unit * 15
    out.insert(len(out) // 2, BIG)
    return out


TABLE_SCALES = [1e-3, 1e-2, 0.1, 1.0, 3.0, 10.0, 100.0]     # 7 scales against a period of 13 sizes: every pairing occurs


def table_scale(i: int) -> float:
    return TABLE_SCALES[i % len(TABLE_SCALES)]


def alignment_sizes(C: int):
    return [C + 5, 2 * C + 3]


def alignment_cases(name: str, kw):
    """Element offsets (into 16-byte aligned flat buffers) of the parameter, the gradient and each state tensor: all
    aligned, each one alone off its 16-byte boundary, and everything off by the same 1, 2 and 3 elements."""
    keys = ("p",) + (("g",) if name != "lookahead" else ()) + state_keys(name, kw)
    cases = [{k: 0 for k in keys}]
    for i, k in enumerate(keys):
        cases.append({**cases[0], k: 1 + i % 3})
    cases += [{k: o for k in keys} for o in (1, 2, 3)]
    return cases
