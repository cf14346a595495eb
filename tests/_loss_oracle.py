"""fp64 references and per-element error bounds for the loss kernels of csrc/losses.cu (focal / poly-1 with hard targets,
poly-1 with soft targets and the multi-label cross entropy, dice, complement cross entropy).

The references are the repository's own restatements (oracle/functional.py, tests/_losses_extra_oracle.py) evaluated in
fp64 on the dtype-rounded inputs, on [P, K] rows (P = N * S positions); gradients come from fp64 autograd. Beside every
reference value sits a bound on the kernel's error: a kernel value must lie within

    one ulp of its output type at the reference value  +  E

where E propagates, to first order and per element, the fp32 rounding of every intermediate the kernel forms. With
u = 2^-24, a position with largest logit m, s = sum_k exp(x_k - m), p_k = exp(x_k - lse):

- log-sum-exp, lse = m + logf(s):  E_lse = u |lse| + 2u |log s| + E_s, with the relative error of s
  E_s = (K + 4) u + sum_k p_k e_k. Per exponential e_k = |x_k - m| u (the rounding of x - m) on the scalar paths
  (expf is exact to 2 ulp = 4u, counted in the K + 4); on the register-resident (vector) paths exp_shift computes
  ex2((x - m) log2e), so e_k = 8u (MUFU.EX2) + 2 |x_k - m| u (x - m and the product with the rounded log2e).
- logits shifted by c (the "shift" cases): the kernel runs on x + c (exact in its dtype), the reference and every
  term above are those of the unshifted x, and the one rounding no fp32 kernel avoids, that of lse + c, adds u |c|.
- log p_t = x_t - lse:  E_lse + u |log p_t|.
- focal's (1 - p_t)^gamma, poly's eps (1 - p_t) and their derivatives: evaluated in fp64 at log p_t +- E_lp, and
  separately at p_t (1 +- 4u) (expf's error of p_t), and the largest deviations added. This is first-order propagation where the
  function is smooth and stays a bound where 1 - p_t cancels (a confident prediction) or crosses 0, where it is not.
  powf adds 8u relative per call for non-integer gamma; the handful of products and sums after it add 8u of the sum
  of the absolute values of their terms.
- the gradient p_k is formed from the fp32 lse: relative E_lse + u |x_k - lse| + 4u (expf), or on the vector paths
  E_lse + 8u + 2 |x_k - lse| u. It multiplies the kernel's g dL/dlog p_t, which may lie anywhere within
  that factor's own bound: that bound is added to the factor's magnitude.
- soft targets: z_k = (x_k - lse) t_k, each term w_k (-z_k + eps (1 - e^z_k)) carries |w_k| |1 + eps e^z_k| E_z plus 8u
  of its terms, and the K-term fp32 sum adds (K + 2) u sum|terms|.
- dice: the fp32 partial sums that each thread flushes into fp64 every 32 vector (every 256 scalar) iterations are
  bounded by (chunk + 2) u sum|terms|, chunk being the number of fp32 additions between flushes; the fp64 rest and
  the class combination are exact to far below u.
- complement cross entropy: the same log-sum-exp terms for lse and for lse over the non-target classes, each
  w_k q_k log q_k term with its propagated E_lq, and the K-term sum.
- the reductions: partials are fp64 sums of the fp32 per-position values, so sum gets sum_p E_p + u |sum|, mean gets
  E_sum / count + 2u |mean| (the count is exact; the float division by it rounds once more).

Every term is computed from fp64 quantities per element; nothing is fitted to a run."""
import math
from dataclasses import dataclass
from typing import Dict, Optional

import torch

from oracle import functional as OF
import _losses_extra_oracle as OX

U = 2.0 ** -24
TINY = 2.0 ** -126      # ex2.approx.ftz and the fp32 products flush below this
BITS = {torch.float32: (24, -126), torch.bfloat16: (8, -126), torch.float16: (11, -14)}


def ulp(ref: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """One ulp of ``dtype`` at each reference value, subnormals included."""
    bits, emin = BITS[dtype]
    e = torch.floor(torch.log2(ref.abs().clamp_min(2.0 ** (emin - 1)))).clamp_min(emin)
    return torch.exp2(e - (bits - 1))


@dataclass
class Checked:
    """A reference and its bound E (the output type's ulp is added when the kernel value is compared)."""
    ref: torch.Tensor
    bound: torch.Tensor
    dtype: torch.dtype = torch.float32

    def excess(self, got: torch.Tensor) -> torch.Tensor:
        err = (got.detach().to(self.ref.device, torch.float64) - self.ref).abs()
        ok_nan = torch.isnan(self.ref) & torch.isnan(got.detach().to(self.ref.device, torch.float64))
        ex = err - (ulp(self.ref, self.dtype) + self.bound)
        return torch.where(ok_nan, torch.full_like(ex, -1.0), ex)


def assert_within(got: torch.Tensor, c: Checked, what: str) -> None:
    ex = c.excess(got.reshape(c.ref.shape))
    bad = ~(ex <= 0)        # NaN fails: an unwritten element of a NaN-filled output
    if bad.any():
        first = tuple(int(i) for i in bad.nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements off, worst excess "
                             f"{float(torch.nan_to_num(ex, nan=math.inf).max()):.3e}, first at {first}: got "
                             f"{float(got.reshape(c.ref.shape)[first]):.9g}, ref {float(c.ref[first]):.9g}, "
                             f"bound {float(c.bound[first]):.3e}")


def breaks(got: torch.Tensor, c: Checked) -> bool:
    return bool((~(c.excess(got.reshape(c.ref.shape)) <= 0)).any())


def rows(x: torch.Tensor) -> torch.Tensor:
    """[N, K, S] -> [N * S, K] (a view: gradients flow back to x)."""
    return x.permute(0, 2, 1).reshape(-1, x.shape[1])


def f32(v: float) -> float:
    return float(torch.tensor(v, dtype=torch.float32))


# ---- log-sum-exp -------------------------------------------------------------------------------------------------------
def lse_terms(X: torch.Tensor, vec: bool, exclude: Optional[torch.Tensor] = None, shift: float = 0.0):
    """(lse, p, E_lse) of the rows of X [P, K] as the kernel forms them from X + shift; ``exclude`` masks classes out
    (-inf)."""
    if exclude is not None:
        X = X.masked_fill(exclude, -math.inf)
    k = X.shape[1]
    m = X.amax(1, keepdim=True)
    d = (X - m).abs().nan_to_num(0.0, posinf=0.0)
    e = torch.exp(X - m)
    s = e.sum(1, keepdim=True)
    lse = m + torch.log(s)
    p = e / s
    per = d * U if not vec else 8 * U + 2 * d * U
    es = (k + 4) * U + (p * per).sum(1, keepdim=True)
    e_lse = U * (lse.abs() + abs(shift)) + 2 * U * torch.log(s).abs() + es
    return lse, torch.exp(X - lse), e_lse


def p_rel(X: torch.Tensor, lse: torch.Tensor, e_lse: torch.Tensor, vec: bool) -> torch.Tensor:
    """Relative error of the kernel's p_k = exp(x_k - lse)."""
    d = (X - lse).abs().nan_to_num(0.0, posinf=0.0)
    return e_lse + (d * U + 4 * U if not vec else 8 * U + 2 * d * U)


def _spread(fn, at: torch.Tensor, d: torch.Tensor) -> torch.Tensor:
    """max |fn(at +- d) - fn(at)|, elementwise (p_t = exp(log p_t) moves with log p_t)."""
    f0 = fn(at)
    return torch.maximum((fn(at + d) - f0).abs(), (fn(at - d) - f0).abs()).nan_to_num(0.0)


def _spread_pt(fn, lp: torch.Tensor) -> torch.Tensor:
    """The same for expf's own error of p_t (4u relative) at a fixed log p_t."""
    f0 = fn(lp)
    pt = torch.exp(lp)
    return torch.maximum((fn(lp, pt * (1 + 4 * U)) - f0).abs(), (fn(lp, pt * (1 - 4 * U)) - f0).abs()).nan_to_num(0.0)


# ---- hard targets ------------------------------------------------------------------------------------------------------
def _focal_pieces(lp, gamma, pt=None):
    pt = torch.exp(lp) if pt is None else pt
    om = (1 - pt).clamp_min(0)
    mod = om ** gamma if gamma != 0 else torch.ones_like(om)
    dmod = gamma * om ** (gamma - 1) * pt if gamma != 0 else torch.zeros_like(om)
    return om, mod, torch.where(om > 0, dmod, torch.zeros_like(dmod))


def hard_fns(kind: str, gamma: float, eps: float):
    """(loss, d loss / d log p_t) per unit weight as functions of log p_t and p_t (exp(log p_t) unless given), in the
    kernel's form."""
    if kind == "focal":
        def F(lp, pt=None):
            return -_focal_pieces(lp, gamma, pt)[1] * lp

        def D(lp, pt=None):
            if gamma == 0:
                return -torch.ones_like(lp)
            _, mod, dmod = _focal_pieces(lp, gamma, pt)
            return -(mod - dmod * lp)
    else:
        def F(lp, pt=None):
            return -lp + eps * (1 - (torch.exp(lp) if pt is None else pt))

        def D(lp, pt=None):
            return -1 - eps * (torch.exp(lp) if pt is None else pt)
    return F, D


@dataclass
class Spec:
    """One call: x [N, K, S] (dtype-rounded), targets, optional class weights, ignore_index and loss parameters."""
    x: torch.Tensor
    target: torch.Tensor            # hard: [N, S] int64; soft / dice: [N, K, S] in x's dtype
    weight: Optional[torch.Tensor]
    ignore_index: int
    kind: str                       # "focal", "poly", "soft", "dice", "cce"
    gamma: float = 0.0
    eps: float = 0.0
    vec: bool = False               # the register-resident path / dice vec flag
    chunk: int = 1                  # dice: fp32 additions between fp64 flushes
    gout: Optional[torch.Tensor] = None     # reduction none: [N * S]
    gscalar: float = 1.0                    # reduction mean / sum
    shift: float = 0.0                      # x holds the logits of the reference plus this (exactly)
    mask: Optional[torch.Tensor] = None     # mutual channel loss: [cnum, xi] 0/1
    xi: int = 1
    alpha: float = 0.0


def _prep(sp: Spec, device):
    x64 = sp.x.detach().to(device, torch.float64) - sp.shift
    w64 = None if sp.weight is None else sp.weight.detach().to(device, torch.float64)
    return x64, w64


def _reduce(loss, e_loss, keep, dtype=torch.float32):
    """fwd_out {sum, count, mean} of the per-position values."""
    cnt = keep.sum().to(loss.dtype)
    s = torch.where(keep, loss, 0).sum()
    es = torch.where(keep, e_loss, 0).sum() + U * s.abs()
    mean = s / cnt
    return {"sum": Checked(s.reshape(1), es.reshape(1)), "count": Checked(cnt.reshape(1), torch.zeros(1, device=s.device, dtype=s.dtype)),
            "mean": Checked(mean.reshape(1), (es / cnt + 2 * U * mean.abs()).reshape(1))}


def _grads(fn, x64, sp: Spec):
    """fp64 autograd gradients of the reference for the three reductions ({none: with gout, mean, sum})."""
    out = {}
    for red in ("none", "mean", "sum"):
        a = x64.clone().requires_grad_(True)
        y = fn(a, red)
        if red == "none":
            y = (y.reshape(-1) * sp.gout.to(y.device, torch.float64)).sum()
        else:
            y = y * sp.gscalar
        (g,) = torch.autograd.grad(y, a)
        out[red] = g
    return out


def _g_per_pos(sp: Spec, red: str, denom, P, device):
    if red == "none":
        return sp.gout.to(device, torch.float64).reshape(P, 1)
    d = denom if red == "mean" else 1.0
    return torch.full((P, 1), sp.gscalar / d if d else math.inf, device=device, dtype=torch.float64)


def _to_nks(t: torch.Tensor, n: int, k: int, s: int) -> torch.Tensor:
    return t.reshape(n, s, k).permute(0, 2, 1)


def hard(sp: Spec, device="cpu") -> Dict[str, Checked]:
    x64, w64 = _prep(sp, device)
    n, k, s = x64.shape
    P = n * s
    t = sp.target.reshape(-1).to(device)
    ign = 0 <= sp.ignore_index < k
    keep = ~(t == sp.ignore_index) if ign else torch.ones_like(t, dtype=torch.bool)
    X = rows(x64)
    lse, p, e_lse = lse_terms(X, sp.vec, shift=sp.shift)
    lse, e_lse = lse[:, 0], e_lse[:, 0]
    lp = X.gather(1, t[:, None])[:, 0] - lse
    e_lp = e_lse + U * lp.abs()
    w = w64[t] if w64 is not None else torch.ones_like(lp)
    F, D = hard_fns(sp.kind, sp.gamma, sp.eps)
    pw = 8 * U if sp.kind == "focal" and sp.gamma not in (0.0, 1.0, 2.0) else 0.0
    loss = w * F(lp)
    if sp.kind == "focal":
        om, mod, dmod = _focal_pieces(lp, sp.gamma)
        terms = (w * mod * lp).abs()
        dterms = w.abs() * (mod + (dmod * lp).abs())
    else:
        terms = w.abs() * (lp.abs() + abs(sp.eps) * (1 - torch.exp(lp)).abs())
        dterms = w.abs() * (1 + abs(sp.eps) * torch.exp(lp))
    e_loss = w.abs() * (_spread(F, lp, e_lp) + _spread_pt(F, lp)) + (8 * U + pw) * terms
    # the repository's restatement gives the values; the kernel-form F above only sizes the bound
    if sp.kind == "focal":
        ref = OF.focal_loss(X, t, w64, sp.ignore_index, "none", sp.gamma)
        fn = lambda a, red: OF.focal_loss(rows(a), t, w64, sp.ignore_index, red, sp.gamma)      # noqa: E731
    else:
        ref = OF.poly_loss(X, t, sp.eps, w64, sp.ignore_index, "none")
        fn = lambda a, red: OF.poly_loss(rows(a), t, sp.eps, w64, sp.ignore_index, red)          # noqa: E731
    out = {"loss": Checked(ref.detach(), e_loss)}
    out.update(_reduce(ref.detach(), e_loss, keep))
    # backward: dx_k = g D(lp) (delta_kt - p_k)
    grads = _grads(fn, x64, sp)
    # with one class log p_t = 0 and focal's (1 - p_t)^gamma has no derivative for gamma < 1: the kernel takes 0
    flat = _to_nks((lp == 0)[:, None].expand(-1, k), n, k, s)
    grads = {red: torch.where(flat & torch.isnan(g), 0.0, g) for red, g in grads.items()}
    Dv = (w * D(lp))[:, None]
    e_D = (w.abs() * (_spread(D, lp, e_lp) + _spread_pt(D, lp)) + (8 * U + 2 * pw) * dterms)[:, None]
    onehot = torch.zeros_like(X).scatter_(1, t[:, None], 1.0)
    e_p = p_rel(X, lse[:, None], e_lse[:, None], sp.vec)
    cnt = float(keep.sum())
    for red in ("none", "mean", "sum"):
        g = _g_per_pos(sp, red, cnt, P, device)
        if red != "none":
            g = torch.where(keep[:, None], g, 0)
        c = g * Dv
        cmax = c.abs() + g.abs() * e_D      # p_k's error meets the kernel's c, which may be far from the reference's
        e = g.abs() * e_D * (onehot - p).abs() + cmax * p * e_p + 4 * U * cmax * (onehot + p) + cmax * TINY
        out[f"dx_{red}"] = Checked(grads[red], _to_nks(e, n, k, s), sp.x.dtype)
    return out


# ---- soft targets ------------------------------------------------------------------------------------------------------
def soft(sp: Spec, device="cpu") -> Dict[str, Checked]:
    x64, w64 = _prep(sp, device)
    n, k, s = x64.shape
    P = n * s
    X, T = rows(x64), rows(sp.target.detach().to(device, torch.float64))
    lse, p, e_lse = lse_terms(X, sp.vec, shift=sp.shift)
    lp = X - lse
    e_lp = e_lse + U * lp.abs()
    z = lp * T
    e_z = T.abs() * e_lp + U * z.abs()
    ez = torch.exp(z)
    eexp = (8 * U + U * z.abs()) if sp.vec else 4 * U          # exp_mufu rounds z log2e first
    w = (w64 if w64 is not None else torch.ones(k, device=device, dtype=torch.float64))[None, :]
    valid = torch.ones(k, device=device, dtype=torch.float64)
    if 0 <= sp.ignore_index < k:
        valid[sp.ignore_index] = 0
    valid = valid[None, :]
    term = w * (-z + sp.eps * (1 - ez))
    e_term = w.abs() * ((1 + sp.eps * ez).abs() * e_z + abs(sp.eps) * ez * eexp) + 8 * U * w.abs() * (z.abs() + abs(sp.eps) * (1 + ez))
    e_loss = (valid * (e_term + (k + 2) * U * term.abs())).sum(1)
    if sp.eps == 0.0:
        ref = OX.multilabel_cross_entropy(X, T, w64, sp.ignore_index, "none")
        fn = lambda a, red: OX.multilabel_cross_entropy(rows(a), T, w64, sp.ignore_index, red)   # noqa: E731
    else:
        ref = OF.poly_loss(X, T, sp.eps, w64, sp.ignore_index, "none")
        fn = lambda a, red: OF.poly_loss(rows(a), T, sp.eps, w64, sp.ignore_index, red)         # noqa: E731
    out = {"loss": Checked(ref.detach(), e_loss)}
    keep = torch.ones(P, dtype=torch.bool, device=device)
    out.update(_reduce(ref.detach(), e_loss, keep))
    out.pop("count")        # the soft forward reports P
    # backward: dx_j = g (c_j t_j - p_j tot), c_k = valid_k w_k (-1 - eps e^z_k), tot = sum_k c_k t_k
    grads = _grads(fn, x64, sp)
    c = valid * w * (-1 - sp.eps * ez)
    e_c = valid * w.abs() * abs(sp.eps) * ez * (e_z + eexp) + 4 * U * c.abs()
    tot = (c * T).sum(1, keepdim=True)
    e_tot = (T.abs() * e_c).sum(1, keepdim=True) + (k + 2) * U * (c * T).abs().sum(1, keepdim=True)
    e_p = p_rel(X, lse, e_lse, sp.vec) if not sp.vec else e_lp + 8 * U + U * lp.abs()
    for red in ("none", "mean", "sum"):
        g = _g_per_pos(sp, red, float(P), P, device)
        d = c * T - p * tot
        e = g.abs() * (T.abs() * e_c + p * e_tot + p * tot.abs() * e_p + 4 * U * ((c * T).abs() + p * tot.abs())) \
            + 2 * U * (g * d).abs() + g.abs() * TINY
        out[f"dx_{red}"] = Checked(grads[red], _to_nks(e, n, k, s), sp.x.dtype)
    return out


# ---- dice --------------------------------------------------------------------------------------------------------------
def dice(sp: Spec, device="cpu") -> Dict[str, Checked]:
    x64, w64 = _prep(sp, device)
    t64 = sp.target.detach().to(device, torch.float64)
    n, k, s = x64.shape
    gamma, eps = f32(sp.gamma), f32(sp.eps)
    xs, ts = x64.transpose(0, 1).reshape(k, -1), t64.transpose(0, 1).reshape(k, -1)
    inter = (xs * ts).sum(1)
    card = (xs + gamma * ts).sum(1)
    ch = sp.chunk + 2
    e_i = ch * U * (xs * ts).abs().sum(1)
    e_c = ch * U * (xs.abs() + abs(gamma) * ts.abs()).sum(1)
    num, den = gamma * inter + eps, card + eps
    dk = num / den
    e_dk = (abs(gamma) * e_i + dk.abs() * e_c) / den.abs()
    w = w64 if w64 is not None else torch.ones(k, device=device, dtype=torch.float64)
    wn = w / w.sum()
    f = 1 + 1 / gamma
    a = x64.clone().requires_grad_(True)
    ref = OF.dice_loss(a, t64, w64, gamma, eps)
    (gx,) = torch.autograd.grad(ref * sp.gscalar, a)
    out = {"loss": Checked(ref.detach().reshape(1), (abs(f) * (wn.abs() * e_dk).sum() + 2 * U * (1 + f * (wn * dk).abs().sum())).reshape(1))}
    coef0 = -f * wn * gamma / den
    coef1 = f * wn * num / den ** 2
    e0 = coef0.abs() * e_c / den.abs()
    e1 = coef1.abs() * (abs(gamma) * e_i / num.abs() + 2 * e_c / den.abs())
    out["coef"] = Checked(torch.stack([coef0, coef1], 1).reshape(-1), torch.stack([e0, e1], 1).reshape(-1))
    g = sp.gscalar
    tt = t64.transpose(0, 1)                        # [K, N, S]
    c0, c1 = coef0.view(k, 1, 1), coef1.view(k, 1, 1)
    e = abs(g) * (tt.abs() * (e0.view(k, 1, 1) + U * c0.abs()) + e1.view(k, 1, 1) + U * c1.abs()) \
        + 4 * U * abs(g) * ((c0 * tt).abs() + c1.abs()) + TINY
    out["dx"] = Checked(gx, e.transpose(0, 1), sp.x.dtype)
    return out


# ---- complement cross entropy ------------------------------------------------------------------------------------------
def cce(sp: Spec, device="cpu") -> Dict[str, Checked]:
    x64, w64 = _prep(sp, device)
    n, k, s = x64.shape
    P = n * s
    t = sp.target.reshape(-1).to(device)
    inr = (t >= 0) & (t < k)
    tc = torch.where(inr, t, 0)
    drop = t == sp.ignore_index                             # the CE part drops the row for any ignore_index
    X = rows(x64)
    w = w64 if w64 is not None else torch.ones(k, device=device, dtype=torch.float64)
    lse, p, e_lse = lse_terms(X, False, shift=sp.shift)
    xt = X.gather(1, tc[:, None])
    ce = (lse - xt)[:, 0]
    wt = torch.where(drop, 0, w[tc])
    e_wce = wt * (e_lse[:, 0] + U * ce.abs()) + U * (wt * ce).abs()
    onehot = torch.zeros_like(X).scatter_(1, tc[:, None], 1.0) * inr[:, None]
    comp = sp.gamma != 0.0
    A = torch.ones_like(X) - onehot
    if 0 <= sp.ignore_index < k:
        A[:, sp.ignore_index] = 0
    inv = 1.0 / (k - 1) if k > 1 else 0.0
    if comp:
        lsen, q, e_lsen = lse_terms(X, False, exclude=onehot.bool(), shift=sp.shift)
        lq = (X - lsen).masked_fill(onehot.bool(), 0.0)
        q = q.masked_fill(onehot.bool(), 0.0)
        e_lq = e_lsen + U * lq.abs()
        wa = A * w[None, :]
        term = wa * q * lq
        e_acc = (wa.abs() * q * ((1 + lq).abs() * e_lq + 4 * U * lq.abs())).sum(1) + (k + 2) * U * term.abs().sum(1)
        cpos = -inv * term.sum(1)
        e_cpos = inv * e_acc + 2 * U * cpos.abs()
    else:
        cpos = e_cpos = torch.zeros(P, device=device, dtype=torch.float64)
    e_loss = e_wce + abs(sp.gamma) * e_cpos + 2 * U * ((wt * ce).abs() + abs(sp.gamma) * cpos.abs())
    fn = lambda a, red: OX.complement_cross_entropy(rows(a), t, w64, sp.ignore_index, red, sp.gamma)  # noqa: E731
    ref = fn(x64, "none").detach()
    out = {"loss": Checked(ref, e_loss)}
    A_sum, B = (wt * ce).sum(), wt.sum()
    tot = ref.sum()
    e_sum = e_loss.sum() + U * tot.abs()
    mean = A_sum / B + sp.gamma * cpos.sum() / P
    e_mean = e_wce.sum() / B + abs(sp.gamma) * e_cpos.sum() / P + 2 * U * mean.abs() + U * (A_sum / B).abs()
    out.update({"sum": Checked(tot.reshape(1), e_sum.reshape(1)), "count": Checked(B.reshape(1), U * B.reshape(1)),
                "mean": Checked(mean.reshape(1), e_mean.reshape(1))})
    grads = _grads(fn, x64, sp)
    e_p = p_rel(X, lse, e_lse, False)
    for red in ("none", "mean", "sum"):
        g = _g_per_pos(sp, red, 1.0, P, device)
        gce = g / (B if red == "mean" else 1.0)
        gc = g / (P if red == "mean" else 1.0)
        cw = gce * wt[:, None]
        e = cw.abs() * p * e_p + 4 * U * cw.abs() * (p + onehot)
        if comp:
            cc = -sp.gamma * gc * inv
            Bk = A * w[None, :] * (1 + lq)
            accb = (wa * q * (1 + lq)).sum(1, keepdim=True)
            e_accb = (wa.abs() * q * ((2 + lq).abs() * e_lq + 4 * U * (1 + lq).abs())).sum(1, keepdim=True) \
                + (k + 2) * U * (wa * q * (1 + lq)).abs().sum(1, keepdim=True)
            e_q = e_lq + 4 * U
            e = e + cc.abs() * q * ((Bk - accb).abs() * e_q + (A * w[None, :]).abs() * e_lq + e_accb) \
                + 4 * U * cc.abs() * q * (Bk.abs() + accb.abs())
        d = grads[red]
        e = _to_nks(e, n, k, s) + 4 * U * d.abs() + TINY * (g.abs().max() + 1)
        out[f"dx_{red}"] = Checked(d, e, sp.x.dtype)
    return out


# ---- mutual channel loss -----------------------------------------------------------------------------------------------
def _online_lse_err(lse, z, rng, depth):
    """Error of a log-sum-exp merged online (lse_merge) over ``depth`` levels: each level rescales z by two expf of
    arguments within ``rng`` of each other and adds, 10u + u rng relative."""
    return U * lse.abs() + 2 * U * torch.log(z).abs() + depth * (10 * U + U * rng)


def mcl(sp: Spec, device="cpu") -> Dict[str, Checked]:
    """Per position: d_c = max_j x_{c,j} mask_{c,j}, torch's cross entropy of d over the classes, minus alpha times the
    mean over classes of max_j softmax_S(x_{c,j}). Outputs: row_lse (log sum_s exp of every channel row), the loss,
    lse_d, fwd_out and, per reduction, rdot and dx. Evaluated on the CPU, where torch's max takes the first index on
    ties as the kernels do."""
    import _loss_cases as D
    x64, w64 = _prep(sp, "cpu")
    n, c, s = x64.shape
    xi = sp.xi
    cnum = c // xi
    P = n * s
    t = sp.target.reshape(n, s).cpu()
    mask = sp.mask.double().cpu()
    G = x64.view(n, cnum, xi, s)
    gmax, gmin = G.amax(-1, keepdim=True), G.amin(-1, keepdim=True)
    z = torch.exp(G - gmax).sum(-1, keepdim=True)
    rlse = gmax + torch.log(z)
    depth = -(-s // D.THREADS) + 16 + D.vec16_width(str(sp.x.dtype).split(".")[1])
    e_row = _online_lse_err(rlse, z, gmax - gmin, depth)
    pr = torch.exp(G - rlse)
    e_pr = e_row + U * (G - rlse).abs() + 4 * U
    pv, jv = pr.max(2)                                            # [n, cnum, s]
    dm = G * mask.view(1, cnum, xi, 1)
    d, jd = dm.max(2)
    dmax, dmin = d.amax(1, keepdim=True), d.amin(1, keepdim=True)
    zd = torch.exp(d - dmax).sum(1, keepdim=True)
    lsed = dmax + torch.log(zd)                                   # [n, 1, s]
    e_lsed = _online_lse_err(lsed, zd, dmax - dmin, cnum)
    ign = t == sp.ignore_index
    tc = t.clamp(0, cnum - 1)
    w = w64 if w64 is not None else torch.ones(cnum, dtype=torch.float64)
    wt = torch.where(ign, 0.0, w[tc])
    dt_ = d.gather(1, tc[:, None])[:, 0]
    ce = lsed[:, 0] - dt_
    wce = wt * ce
    e_wce = wt * (e_lsed[:, 0] + U * ce.abs()) + U * wce.abs()
    e_pv = pv * e_pr.gather(2, jv[:, :, None]).squeeze(2)
    div = pv.sum(1) / cnum
    e_div = e_pv.sum(1) / cnum + (cnum + 2) * U * div
    a = abs(sp.alpha)
    e_loss = e_wce + a * e_div + 2 * U * (wce.abs() + a * div)
    fn = lambda q, red: OX.mutual_channel_loss(q, t, mask, w64, sp.ignore_index, red, xi, sp.alpha)     # noqa: E731
    ref = fn(x64, "none").detach().reshape(-1)
    A, B = wce.sum(), wt.sum()
    mean = A / B - sp.alpha * div.sum() / P
    out = {"row_lse": Checked(rlse.reshape(-1), e_row.reshape(-1)),
           "loss": Checked(ref, e_loss.reshape(-1)),
           "lse_d": Checked(lsed.reshape(-1), e_lsed.reshape(-1)),
           "sum": Checked(ref.sum().reshape(1), (e_loss.sum() + U * ref.sum().abs()).reshape(1)),
           "count": Checked(B.reshape(1), (U * B).reshape(1)),
           "mean": Checked(mean.reshape(1), (e_wce.sum() / B + a * e_div.sum() / P + 2 * U * mean.abs()
                                             + U * (A / B).abs()).reshape(1))}
    grads = _grads(fn, x64, _with_device(sp))
    f = -sp.alpha / cnum
    selv = torch.zeros_like(pr).scatter_(2, jv[:, :, None, :], 1.0)
    seld = torch.zeros_like(pr).scatter_(2, jd[:, :, None, :], 1.0) * mask.view(1, cnum, xi, 1)
    pd = torch.exp(d - lsed)                                      # [n, cnum, s]
    onehot = torch.zeros_like(d).scatter_(1, tc[:, None, :], 1.0)
    rt = D.mcl_rdot_threads(xi)
    for red in ("none", "mean", "sum"):
        g = sp.gout.double().cpu().view(n, 1, 1, s) if red == "none" else torch.full((n, 1, 1, s), sp.gscalar, dtype=torch.float64)
        gdiv = g / (P if red == "mean" else 1)
        gce = (g[:, :, 0] / (B if red == "mean" else 1)) * wt[:, None, :]            # [n, 1, s]
        terms = selv * gdiv * pr
        rdot = f * terms.sum(-1, keepdim=True)                                       # [n, cnum, xi, 1]
        e_rdot = abs(f) * (terms.abs() * (e_pr + (-(-s // rt) + 2) * U)).sum(-1, keepdim=True) + 2 * U * rdot.abs()
        out[f"rdot_{red}"] = Checked(rdot.reshape(-1), e_rdot.reshape(-1))
        dd = gce * (pd - onehot)                                                     # [n, cnum, s]
        e_dd = gce.abs() * pd * (e_lsed + U * (d - lsed).abs() + 4 * U) + 2 * U * dd.abs()
        h = selv * f * gdiv - rdot
        e = pr * e_pr * h.abs() + pr * e_rdot + seld * e_dd[:, :, None, :] \
            + 4 * U * (pr * (selv * (f * gdiv).abs() + rdot.abs()) + seld * dd.abs()[:, :, None, :]) + TINY
        out[f"dx_{red}"] = Checked(grads[red], e.reshape(n, c, s), sp.x.dtype)
    return out


def _with_device(sp: Spec) -> Spec:
    d = dict(sp.__dict__)
    d["gout"] = sp.gout.cpu()
    return Spec(**d)


ORACLES = {"hard": hard, "soft": soft, "dice": dice, "cce": cce, "mcl": mcl}


def reference(family: str, sp: Spec, device="cpu") -> Dict[str, Checked]:
    return ORACLES[family](sp, device)


# ---- inputs ------------------------------------------------------------------------------------------------------------
DT = {"float32": torch.float32, "bfloat16": torch.bfloat16, "float16": torch.float16}


def params(cs) -> list:
    """The parameter sets a case runs: (kind, gamma, eps, weighted, ignore_index, soft-target kind). Weights and the
    ignore index rotate over the loss parameters so that each combination appears with every kernel."""
    k = cs.k
    ii_in = min(1, k - 1)
    rot = [(False, -100), (True, ii_in), (False, ii_in), (True, -100)]
    if cs.family == "hard":
        ps = [("focal", g, 0.0) for g in (0.0, 0.5, 1.0, 2.0, 3.5)] + [("poly", 0.0, e) for e in (2.0, 0.0, -1.0)]
        out = [(kind, g, e) + rot[i % 4] + ("",) for i, (kind, g, e) in enumerate(ps)]
    elif cs.family == "soft":
        out = [("soft", 0.0, e) + rot[i % 4] + (tk,) for i, (e, tk) in enumerate(
            [(2.0, "sum1"), (0.0, "multilabel"), (2.0, "multilabel"), (0.0, "sum1")])]
    elif cs.family == "dice":
        out = [("dice", g, 1e-8, wt, -100, "") for g in (0.5, 1.0, 2.0) for wt in (False, True)]
    elif cs.family == "mcl":
        ii_in = 1 if cs.cnum > 1 else -100     # with one class an in-range ignore_index would drop every position
        out = [("mcl", a, 0.0, wt, ii, "") for a, wt, ii in ((1.5, False, -100), (0.0, True, ii_in), (1.5, True, ii_in))]
    else:
        out = [("cce", g, 0.0) + rot[i % 4] + ("",) for i, g in enumerate((0.0, -1.0, 0.5, -1.0, 0.0, 0.5))]
        out.append(("cce", 0.0, 0.0, True, 255, ""))
    return out[:2] if cs.light else out


def make_spec(cs, prm, seed: int, device="cpu", all_ignored: bool = False, sms: int = 132) -> Spec:
    """The inputs of one parameter set of a case; ``sms`` is the SM count of the device that runs it."""
    import _loss_cases as D
    kind, gamma, eps, weighted, ii, tk = prm
    gen = torch.Generator().manual_seed(seed)
    dt = DT[cs.dtype]
    n, k, s = cs.n, cs.k, cs.s
    if kind == "mcl":
        cnum, xi = cs.cnum, cs.xi
        x = torch.randn(n, k, s, generator=gen) * 2
        if cs.logits == "equal":        # every channel of a class alike: both argmaxes must take the first
            x = x.view(n, cnum, xi, s)[:, :, :1].expand(n, cnum, xi, s).reshape(n, k, s).clone()
        target = torch.randint(0, cnum, (n, s), generator=gen)
        if 0 <= ii < cnum:
            target.view(-1)[:: 3] = ii
        mask = torch.zeros(cnum, xi)
        for c in range(cnum):
            mask[c, torch.randperm(xi, generator=gen)[: (xi + 1) // 2]] = 1
        weight = torch.rand(cnum, generator=gen) * 1.5 + 0.5 if weighted else None
        gout = torch.randn(n * s, generator=gen)
        return Spec(x.to(dt).to(device), target.to(device), None if weight is None else weight.to(device), ii, kind,
                    gout=gout.to(device), gscalar=0.75, mask=mask.to(device), xi=xi, alpha=gamma)
    if kind == "dice":
        x = torch.rand(n, k, s, generator=gen)
        target = (torch.rand(n, k, s, generator=gen) < 0.3).float()
        target[0, :, 0] = 1         # every class present
    else:
        x = torch.randn(n, k, s, generator=gen) * 2
        if cs.logits == "uniform":
            x.zero_()
        if kind == "soft":
            if tk == "sum1":
                target = torch.softmax(torch.randn(n, k, s, generator=gen) * 2, 1)
            else:
                target = (torch.rand(n, k, s, generator=gen) < 0.3).float()
                target[0, :, 0] = 0         # an all-zero row
            if cs.logits == "confident":
                x.scatter_add_(1, target.argmax(1, keepdim=True), torch.full((n, 1, s), 30.0))
        else:
            target = torch.randint(0, k, (n, s), generator=gen)
            if 0 <= ii < k:
                target.view(-1)[:: 3] = ii           # ignored positions
            if ii == 255:
                target.view(-1)[:: 4] = 255
            if all_ignored:
                target.fill_(ii)
            if cs.logits == "confident":
                x.scatter_add_(1, target.clamp(0, k - 1)[:, None, :], torch.full((n, 1, s), 30.0))
    weight = torch.rand(k, generator=gen) * 1.5 + 0.5 if weighted else None
    P = n * s
    gout = torch.randn(P, generator=gen)
    vec = D.vec_eligible(cs) if kind in ("focal", "poly", "soft") else D.dice_vec(cs)
    chunk = 1
    if kind == "dice":
        route = D.route(cs, sms)["fwd"]
        per = D.vec16_width(cs.dtype) if vec else 1
        chunk = per * min(route.max_iters, 32 if vec else 256)
    shift = float(cs.logits[5:]) if cs.logits.startswith("shift") else 0.0
    return Spec((x + shift).to(dt).to(device), (target.to(dt) if kind in ("soft", "dice") else target).to(device),
                None if weight is None else weight.to(device), ii, kind, gamma, eps, vec, chunk, gout.to(device), 0.75,
                shift)
