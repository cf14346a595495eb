"""Plain fp64 restatement of the fused BatchNorm / branch-sum / activation kernels (csrc/bn_act.cu) and of the squeeze-
excite gate (csrc/se_gate.cu), with the per-element error bounds the kernels must meet and the geometry they run on.

Tensors are [M, C] (rows = N*H*W pixels, channels last), the layout the kernels stream; ``F.batch_norm`` normalises a
2-D input per column, so the reference is ``nn.BatchNorm2d``'s own arithmetic. Everything differentiates with autograd.

Bounds. Inputs are bf16, so each product of a bf16 value and an fp32 constant is one fp32 rounding, and a kernel's error
is the fp32 rounding of its few additions plus, for the reductions, the fp32 per-lane sums. A lane adds R rows in fp32
(R = ceil(M / lanes)) before its block adds the lanes in fp64 and stores an fp32 partial: the sum of n values carries at
most (R + 2) * 2^-24 * sum|values|. Statistics therefore satisfy, per channel,
    |mean - mu| <= 2^-23 |mu| + (R+2) 2^-24 mean|u|
    |var - v|   <= (R+2) 2^-24 (mean u^2 + 2 |mu| mean|u|)
and every bf16 output lies within one ulp at the fp64 reference plus the fp32 error of what was rounded."""
from typing import Optional, Sequence

import torch
import torch.nn.functional as F

from _bounds import ulp
from _slab import geometry, grid_rows  # noqa: F401  (re-exported: the geometry the BatchNorm tests run on)

ACT_NONE, ACT_RELU, ACT_RELU6, ACT_SILU, ACT_LEAKY, ACT_MISH, ACT_HARDMISH, ACT_FRELU = range(8)
EPS32 = 2.0 ** -24          # unit roundoff of fp32
FAST = 2.0 ** -20           # relative error allowed to the fast-math SiLU / Mish (act.cuh)
SMOOTH = (ACT_SILU, ACT_MISH)
# sup |act''| (0 for the piecewise-linear ones away from their kinks): how far act' moves with an error in z
CURVATURE = {ACT_SILU: 0.5, ACT_MISH: 0.7, ACT_HARDMISH: 1.0}


# ---------------------------------------------------------------------------------------------------------------------
# reference arithmetic
# ---------------------------------------------------------------------------------------------------------------------
def act_ref(code: int, z: torch.Tensor, slope: float = 0.0) -> torch.Tensor:
    """act(z) for the kernels' activation codes; FReLU (7) is the identity here, its max is taken on the residual."""
    if code == ACT_RELU:
        return torch.relu(z)
    if code == ACT_RELU6:
        return F.hardtanh(z, 0.0, 6.0)
    if code == ACT_SILU:
        return F.silu(z)
    if code == ACT_LEAKY:
        return F.leaky_relu(z, slope)
    if code == ACT_MISH:
        return F.mish(z)
    if code == ACT_HARDMISH:
        return 0.5 * z * (z + 2).clamp(0, 2)
    return z


def bn_act_ref(us: Sequence[torch.Tensor], weights, biases, act: int, slope: float = 0.0,
               residual: Optional[torch.Tensor] = None, res_after: bool = False, running=None, eps: float = 1e-5):
    """(out, z): out = act(sum_b BN_b(u_b) [+ residual]) [+ residual] on [M, C] inputs, in their dtype. ``weights`` /
    ``biases`` entries may be None (no affine). ``running``: None for batch statistics, else [(mean, var)] per branch.
    FReLU: z = max(sum_b BN_b(u_b), residual) with torch.maximum, whose backward splits ties 1/2 : 1/2 like the kernel.
    No branch (act_only): z = residual."""
    z = None
    for b, u in enumerate(us):
        rm, rv = (None, None) if running is None else running[b]
        y = F.batch_norm(u, rm, rv, weights[b], biases[b], running is None, 0.0, eps)
        z = y if z is None else z + y
    if z is None:
        z = residual
    elif residual is not None and not res_after:
        z = torch.maximum(z, residual) if act == ACT_FRELU else z + residual
    out = act_ref(act, z, slope)
    if residual is not None and res_after:
        out = out + residual
    return out, z


def batch_stats(u: torch.Tensor):
    """fp64 (mean, biased variance) per column of [M, C]."""
    u = u.double()
    mean = u.mean(0)
    return mean, (u - mean).square().mean(0)


# ---------------------------------------------------------------------------------------------------------------------
# geometry (tests/_slab.py mirrors SlabGeo of slab.cuh; RowRing of bn_act.cu)
# ---------------------------------------------------------------------------------------------------------------------
def ring_depth(tensors: int) -> int:
    """Rows in flight per thread with ``tensors`` streamed inputs; a ring has depth + 1 slots."""
    return 7 if tensors <= 2 else 3


def rows_per_lane(c: int, m: int, grid_x: int) -> int:
    """R: rows the busiest lane walks."""
    return -(-m // (grid_x * geometry(c).rows_t))


# ---------------------------------------------------------------------------------------------------------------------
# bounds
# ---------------------------------------------------------------------------------------------------------------------
def sum_err(r: int, abs_sum: torch.Tensor) -> torch.Tensor:
    """Error of an fp32 per-lane sum of R rows, combined in fp64 and stored in fp32 (see the module docstring)."""
    return (r + 2) * EPS32 * abs_sum


def stats_bounds(u: torch.Tensor, r: int):
    """(mean error, variance error) bounds per channel of the statistics of [M, C] ``u`` from fp32 lane sums of R rows."""
    u = u.double()
    mu = u.mean(0)
    ma = u.abs().mean(0)
    dmean = 2 * EPS32 * mu.abs() + sum_err(r, ma)
    dvar = sum_err(r, u.square().mean(0) + 2 * mu.abs() * ma)
    return dmean, dvar


def rstd_rel_bound(var: torch.Tensor, dvar: torch.Tensor, eps: float) -> torch.Tensor:
    """Relative error of rstd = fp32(1 / sqrt(var + eps)) when var is off by at most dvar."""
    x = (dvar / (var + eps)).clamp(max=0.5)
    return 0.5 * x / (1 - x) + 2 * EPS32


def z_err(code: int, sc_u_abs: torch.Tensor, sh_abs: torch.Tensor, r_abs, nb: int) -> torch.Tensor:
    """Bound on the fp32 error of z = sum_b fma(sc_b, u_b, .) + sum_b sh_b (+ r): 2B + 2 roundings of partial sums that
    are each at most sum|terms|."""
    terms = sc_u_abs + sh_abs + (0 if r_abs is None else r_abs)
    return (2 * nb + 2) * EPS32 * terms


def fwd_bound(code: int, z: torch.Tensor, dz: torch.Tensor, res_after_r: Optional[torch.Tensor] = None,
              slope: float = 0.0) -> torch.Tensor:
    """Slack of a forward output beyond one bf16 ulp: act's Lipschitz constant (<= 2) times the error of z, the fast-math
    error of SiLU / Mish, and one fp32 rounding of act(z) + r when the residual is added after the activation."""
    lip = max(1.0, abs(slope)) if code == ACT_LEAKY else (2.0 if code in SMOOTH + (ACT_HARDMISH,) else 1.0)
    a = act_ref(code, z, slope).abs()
    b = lip * dz
    if code in SMOOTH:
        b = b + FAST * a
    if res_after_r is not None:
        b = b + EPS32 * (a + res_after_r.abs())
    return b


def grad_act_err(code: int, z: torch.Tensor, dz: torch.Tensor) -> torch.Tensor:
    """Bound on |act'_kernel(z_kernel) - act'(z)| away from the kinks: the curvature of act times the error of z, plus
    the fast-math error of the SiLU / Mish derivatives (relative to their terms, which grow like 1 + |z|)."""
    e = CURVATURE.get(code, 0.0) * dz
    if code in SMOOTH:
        e = e + FAST * (1 + z.abs())
    return e


def kink_mask(code: int, z: torch.Tensor, dz: torch.Tensor, r: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Elements whose fp64 pre-activation lies within the forward error ``dz`` of a discontinuity of act' (FReLU: of
    z = r). There the kernel may take either side, and its gradient is not bounded by the reference's."""
    if code == ACT_FRELU:
        return (z - r).abs() <= dz if r is not None else torch.zeros_like(z, dtype=torch.bool)
    kinks = {ACT_RELU: (0.0,), ACT_LEAKY: (0.0,), ACT_RELU6: (0.0, 6.0), ACT_HARDMISH: (-2.0, 0.0)}.get(code, ())
    m = torch.zeros_like(z, dtype=torch.bool)
    for k in kinks:
        m |= (z - k).abs() <= dz
    return m


def within(got: torch.Tensor, ref: torch.Tensor, slack: torch.Tensor, what: str, mask: Optional[torch.Tensor] = None,
           bits: int = 8) -> None:
    """|got - ref| <= ulp(ref) + slack per element (outside ``mask``); NaNs in ``got`` fail."""
    g = got.detach().to(ref.device, torch.float64)
    err = (g - ref).abs()
    bad = ~(err <= ulp(ref, bits) + slack)
    if mask is not None:
        bad &= ~mask
    if bool(bad.any()):
        idx = tuple(int(i) for i in bad.nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements off; first at {idx}: got {float(g[idx]):.8g}, "
                             f"ref {float(ref[idx]):.8g}, allowed {float((ulp(ref, bits) + slack)[idx]):.3e}")


def mask_fraction_ok(mask: torch.Tensor, what: str, limit: float = 0.01) -> None:
    frac = float(mask.double().mean()) if mask.numel() else 0.0
    assert frac < limit, f"{what}: kink mask covers {frac:.2%} of the elements"
