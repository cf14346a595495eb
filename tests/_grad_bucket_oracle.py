"""Oracles of the gradient-bucket plumbing of the training step: the launch planning of the weight-gradient entry points,
the filter packing and the gradient clipping.

* :func:`route_wgrad` / :func:`route_repvgg_wgrad` restate ``plan_wgrad`` (csrc/conv_wgrad.cu), ``plan_wrows``
  (csrc/conv_wgrad_rows.cu) and the path choice of ``hb_conv2d_wgrad[_acc]_bf16`` / ``hb_repvgg_wgrad[_acc]_bf16``: which
  path a shape takes for a given CTA count and workspace, how many partial slices it reduces, and the workspace bytes the
  size queries return.
* :func:`pack_wf`, :func:`pack_wd` and :func:`pack_dgrad_s2` restate ``pack_element`` and ``pack_dgrad_s2_kernel``
  (csrc/conv_aux.cu) with torch's round-to-nearest-even ``.bfloat16()``.
* :func:`clip_ref` restates ``hb_grad_clip_norm`` (csrc/train_ctl.cu) as ``torch.nn.utils.clip_grad_norm_`` computes it.

The case tables at the end are the ones tests/test_gpu_grad_bucket_bounds.py runs; tests/test_grad_bucket_oracle_cpu.py
checks that they reach every path for every SM count an H100 can have."""
from typing import NamedTuple, Optional

import torch

SMS_RANGE = range(100, 145)

# ---------------------------------------------------------------------------------------------------------------------
# weight-gradient planning
# ---------------------------------------------------------------------------------------------------------------------
ROWS, PARTIALS, SINGLE, ATOMICS, REFUSED = "rows", "partials", "single", "atomics", "refused"
NOT_SUPPORTED = 801     # cudaErrorNotSupported


class Route(NamedTuple):
    path: str            # ROWS, PARTIALS, SINGLE, ATOMICS or REFUSED
    slices: int          # partial slices the reduction pass sums (rows: members, partials: k_splits), else 1
    ws_bytes: int        # what the workspace-size query returns for the shape


def window_out(h: int, k: int, stride: int, pad: int, dil: int = 1) -> Optional[int]:
    if h <= 0 or k <= 0 or stride <= 0 or pad < 0 or dil <= 0:
        return None
    span = dil * (k - 1) + 1
    if h + 2 * pad < span:
        return None
    return (h + 2 * pad - span) // stride + 1


def plan_wgrad(n, h, w, cin, cout, k, stride, pad, ctas):
    """(k_splits, partial workspace bytes) of the generic kernel, or None for a malformed window."""
    ho, wo = window_out(h, k, stride, pad), window_out(w, k, stride, pad)
    if ho is None or wo is None:
        return None
    m_total = n * ho * wo
    ci_tile = cin
    if cin > 128:
        ci_tile = 64 if (cin % 128 != 0 and cin % 64 == 0) else 128
    base_units = ((cout + 127) // 128) * ((cin + ci_tile - 1) // ci_tile) * (k * k)
    kblocks = (m_total + 63) // 64
    k_splits = 1 if base_units >= ctas else (2 * ctas + base_units - 1) // base_units
    k_splits = max(1, min(k_splits, (kblocks + 7) // 8))
    return k_splits, (k_splits * cout * k * k * cin * 4 if k_splits > 1 else 0)


def plan_wrows(n, h, w, cin, cout, ctas, has_b1):
    """(members, workspace bytes) of the row-window kernel, or None when the shape does not fit it."""
    if cin % 8 or cout % 8 or w < 8 or w + 2 > 128:
        return None
    wp = w + 2
    n_cig = (cin + 63) // 64
    nslots = 9 + has_b1
    n_cog = (cout + 63) // 64
    co_group = ((cout + n_cog - 1) // n_cog + 15) & ~15
    tpw = min(8, 128 // co_group)
    n_sg = (nslots + 2 * tpw - 1) // (2 * tpw)
    ngroups = n_cig * n_cog * n_sg
    if ngroups > 32:
        return None
    tro = min(h, 16)
    while tro >= 1:
        ks = (tro * wp + 15) // 16
        xrows = 2 * wp + 2 + ks * 16
        xbytes = (max(xrows, (tro + 2) * wp) * 128 + 1023) & ~1023
        ybytes = (ks * 16 * 128 + 1023) & ~1023
        if 2 * (xbytes + (1 + has_b1) * ybytes) <= 220 * 1024:
            break
        tro -= 1
    if tro < 1:
        return None
    num_tiles = n * ((h + tro - 1) // tro)
    members = min(ctas // ngroups, num_tiles)
    if members < 1:
        return None
    slice_elems = cout * 9 * cin + (cout * cin if has_b1 else 0)
    return members, members * slice_elems * 4


def rows_eligible(k, stride, pad):
    return k == 3 and stride == 1 and pad == 1


def wgrad_workspace_bytes(n, h, w, cin, cout, k, stride, pad, ctas):
    """hb_conv2d_wgrad_workspace_bytes: the larger of the two kernels' wants (0 for a malformed window)."""
    g = plan_wgrad(n, h, w, cin, cout, k, stride, pad, ctas)
    if g is None:
        return 0
    r = plan_wrows(n, h, w, cin, cout, ctas, 0) if rows_eligible(k, stride, pad) else None
    return max(g[1], r[1] if r else 0)


def route_wgrad(n, h, w, cin, cout, k, stride, pad, num_ctas, acc, ws_bytes, sms=132):
    """The path of hb_conv2d_wgrad_bf16 (``acc`` False) or hb_conv2d_wgrad_acc_bf16 (``acc`` True) with a workspace of
    ``ws_bytes`` (0: no workspace). ``sms`` stands for the device's SM count when ``num_ctas`` is 0."""
    ctas = num_ctas if num_ctas > 0 else sms
    want = wgrad_workspace_bytes(n, h, w, cin, cout, k, stride, pad, ctas)
    if ws_bytes > 0 and rows_eligible(k, stride, pad):
        r = plan_wrows(n, h, w, cin, cout, ctas, 0)
        if r is not None and ws_bytes >= r[1]:
            return Route(ROWS, r[0], want)
    k_splits, part_bytes = plan_wgrad(n, h, w, cin, cout, k, stride, pad, ctas)
    fits = ws_bytes > 0 and ws_bytes >= part_bytes
    if acc and not (k_splits > 1 and fits):
        return Route(REFUSED, 1, want)
    if k_splits == 1:
        return Route(SINGLE, 1, want)
    return Route(PARTIALS, k_splits, want) if fits else Route(ATOMICS, k_splits, want)


def route_repvgg_wgrad(n, h, w, cin, cout, num_ctas, ws_bytes, sms=132):
    """The path of hb_repvgg_wgrad[_acc]_bf16: the row-window kernel with both branches, or the 801 refusal."""
    ctas = num_ctas if num_ctas > 0 else sms
    r = plan_wrows(n, h, w, cin, cout, ctas, 1)
    want = r[1] if r else 0
    if r is None or ws_bytes <= 0 or ws_bytes < r[1]:
        return Route(REFUSED, 1, want)
    return Route(ROWS, r[0], want)


# ---------------------------------------------------------------------------------------------------------------------
# filter packing
# ---------------------------------------------------------------------------------------------------------------------
def pack_wf(w_krsc: torch.Tensor, cout_f: int, cin_p: int) -> torch.Tensor:
    """wf [CoutF][R][S][CinP] bf16: the KRSC fp32 master rounded to nearest even, zero rows and channels beyond it."""
    cout, r, s, cin = w_krsc.shape
    out = torch.zeros((cout_f, r, s, cin_p), dtype=torch.bfloat16)
    out[:cout, :, :, :cin] = w_krsc.cpu().bfloat16()
    return out


def pack_wd(w_krsc: torch.Tensor, cin_d: int, cout_p: int) -> torch.Tensor:
    """wd [CinD][R][S][CoutP] bf16 with wd[ci][r][s][co] = w[co][R-1-r][S-1-s][ci] (the data-gradient filter)."""
    cout, r, s, cin = w_krsc.shape
    out = torch.zeros((cin_d, r, s, cout_p), dtype=torch.bfloat16)
    out[:cin, :, :, :cout] = w_krsc.cpu().flip(1, 2).permute(3, 1, 2, 0).bfloat16()
    return out


def pack_dgrad_s2(w_krsc: torch.Tensor, cin_d: int, cout_p: int) -> torch.Tensor:
    """The four parity-class filters of the stride-2 3x3 data gradient back to back, classes (0,0), (0,1), (1,0), (1,1):
    class (a, b) is [CinD][1+a][1+b][CoutP] with filter row 1 for a = 0 and rows (2, 0) for a = 1 (columns likewise)."""
    cout, _, _, cin = w_krsc.shape
    taps = {0: [1], 1: [2, 0]}
    parts = []
    for a in (0, 1):
        for b in (0, 1):
            sub = w_krsc.cpu()[:, taps[a]][:, :, taps[b]]                # [Cout][1+a][1+b][Cin]
            out = torch.zeros((cin_d, 1 + a, 1 + b, cout_p), dtype=torch.bfloat16)
            out[:cin, :, :, :cout] = sub.permute(3, 1, 2, 0).bfloat16()
            parts.append(out.reshape(-1))
    return torch.cat(parts)


def edge_values() -> torch.Tensor:
    """fp32 masters where bf16 rounding goes wrong: signed zeros, exact ties (both parities), values one ulp either side
    of a tie, the largest finite value (rounds to inf), infinities, NaN and subnormals (ties among them too)."""
    bits = [0x00000000, 0x80000000,                     # +-0
            0x3F808000, 0x3F818000, 0xBF808000,         # ties: to even down, to even up, negative
            0x3F807FFF, 0x3F808001, 0xBF807FFF,         # just below / above a tie
            0x7F7FFFFF, 0x7F7F7FFF, 0xFF7FFFFF,         # max finite (-> inf), just below its tie, negative
            0x7F800000, 0xFF800000, 0x7FC00000,         # +-inf, NaN
            0x00000001, 0x80000001, 0x00008000,         # smallest subnormals, a subnormal tie (to even: 0)
            0x00018000, 0x007FFFFF, 0x807F8000,         # a subnormal tie rounding up, largest subnormal, negative tie
            0x00800000, 0x3F7FFFFF]                     # smallest normal, just below 1 (rounds to 1)
    return torch.tensor(bits, dtype=torch.int64).to(torch.int32).view(torch.float32)


def masters(shape, gen: torch.Generator, edges: bool = True) -> torch.Tensor:
    """Random fp32 filter masters of ``shape`` (on the CPU), with :func:`edge_values` planted at the start."""
    w = torch.randn(shape, generator=gen) * 0.5
    if edges:
        e = edge_values()
        k = min(e.numel(), w.numel())
        w.view(-1)[:k] = e[:k]
    return w


def bf16_equal(got: torch.Tensor, want: torch.Tensor):
    """(equal, number of differing elements): bit-equal bf16 except that NaN only needs to be NaN (the device conversion
    and torch write different NaN payloads)."""
    g, w = got.cpu().reshape(-1), want.cpu().reshape(-1)
    gb, wb = g.view(torch.int16), w.view(torch.int16)
    same = (gb == wb) | (torch.isnan(g) & torch.isnan(w))
    return bool(same.all()), int((~same).sum())


# ---------------------------------------------------------------------------------------------------------------------
# gradient clipping
# ---------------------------------------------------------------------------------------------------------------------
def norm_ref(g: torch.Tensor) -> float:
    """fp64 L2 norm of the fp32 values."""
    return float(g.detach().cpu().double().norm())


def clip_coef(norm32: float, max_norm: float) -> torch.Tensor:
    """torch.nn.utils.clip_grad_norm_'s coefficient in fp32: min(1, fl(max_norm / fl(norm + 1e-6))), NaN kept."""
    n = torch.tensor(norm32, dtype=torch.float32)
    c = torch.tensor(max_norm, dtype=torch.float32) / (n + torch.tensor(1e-6, dtype=torch.float32))
    return torch.clamp(c, max=1.0)


def clip_ref(g: torch.Tensor, norm32: float, max_norm: float) -> torch.Tensor:
    """The clipped gradients fl32(g * coef) for the norm ``norm32`` the kernel formed (NaN and inf propagate)."""
    return g.detach().cpu() * clip_coef(norm32, max_norm)


# ---------------------------------------------------------------------------------------------------------------------
# case tables of tests/test_gpu_grad_bucket_bounds.py
# ---------------------------------------------------------------------------------------------------------------------
# accumulating weight gradient: name -> ((N, H, W, Cin, Cout, k, stride, pad), num_ctas, workspace, expected path).
# workspace: "full" (what the size query returns), "short" (one byte less), "none"
WGRAD_ACC_CASES = {
    "rows-c1": ((2, 12, 10, 16, 16, 3, 1, 1), 1, "full", ROWS),
    "rows-c7": ((2, 20, 14, 32, 48, 3, 1, 1), 7, "full", ROWS),
    "rows-c0": ((4, 24, 22, 48, 64, 3, 1, 1), 0, "full", ROWS),
    "partials-1x1-c2": ((2, 20, 18, 48, 16, 1, 1, 0), 2, "full", PARTIALS),
    "partials-1x1-c7": ((4, 20, 20, 40, 24, 1, 1, 0), 7, "full", PARTIALS),
    "partials-3x3s2-c0": ((2, 33, 31, 16, 32, 3, 2, 1), 0, "full", PARTIALS),
    "partials-3x3s1-narrow-w-c0": ((16, 32, 6, 32, 64, 3, 1, 1), 0, "full", PARTIALS),
    "partials-1x1s2-c0": ((8, 28, 28, 64, 128, 1, 2, 0), 0, "full", PARTIALS),
    "partials-rows-ws-short-c0": ((4, 24, 22, 48, 64, 3, 1, 1), 0, "short", PARTIALS),
    "refused-single-c1": ((2, 16, 16, 16, 32, 3, 2, 1), 1, "full", REFUSED),
    "refused-single-c0": ((2, 8, 8, 256, 256, 3, 1, 1), 0, "full", REFUSED),
    "refused-ws-short-c0": ((2, 33, 31, 16, 32, 3, 2, 1), 0, "short", REFUSED),
    "refused-no-ws-c2": ((4, 20, 20, 40, 24, 1, 1, 0), 2, "none", REFUSED),
}

# RepVGG one-pass accumulation: name -> ((N, H, W, Cin, Cout), num_ctas, workspace, expected path)
REPVGG_ACC_CASES = {
    "rows-c1": ((2, 12, 10, 16, 16), 1, "full", ROWS),
    "rows-c2": ((2, 18, 12, 16, 16), 2, "full", ROWS),
    "rows-c7": ((2, 20, 22, 24, 32), 7, "full", ROWS),
    "rows-c0": ((4, 28, 28, 48, 48), 0, "full", ROWS),
    "rows-wide-c0": ((2, 14, 14, 128, 128), 0, "full", ROWS),
    "refused-ws-short-c0": ((2, 14, 14, 48, 48), 0, "short", REFUSED),
    "refused-narrow-w-c0": ((2, 14, 6, 48, 48), 0, "full", REFUSED),
    "refused-groups-c2": ((2, 14, 14, 128, 128), 2, "full", REFUSED),
}


def case_route(case, sms=132):
    """Route of a WGRAD_ACC_CASES entry (accumulating form) with its workspace rule."""
    (n, h, w, cin, cout, k, stride, pad), ctas, ws_rule, _ = case
    want = route_wgrad(n, h, w, cin, cout, k, stride, pad, ctas, False, 1 << 40, sms).ws_bytes
    ws = {"full": want, "short": want - 1, "none": 0}[ws_rule]
    return route_wgrad(n, h, w, cin, cout, k, stride, pad, ctas, True, ws, sms), ws


def repvgg_case_route(case, sms=132):
    (n, h, w, cin, cout), ctas, ws_rule, _ = case
    want = route_repvgg_wgrad(n, h, w, cin, cout, ctas, 1 << 40, sms).ws_bytes
    ws = {"full": want, "short": want - 1, "none": 0}[ws_rule]
    return route_repvgg_wgrad(n, h, w, cin, cout, ctas, ws, sms), ws


# Routes a parameter gradient takes into a direct GradBucket (tests/test_gpu_grad_bucket_bounds.py, part d): the one-pass
# RepVGG accumulation, the generic / row-window accumulation, the 801 refusal (overwriting form + AccumulateGrad), a
# channel-padded filter (overwriting form), the im2col stem and the BatchNorm parameters added by the bn_act backward.
R_REPVGG, R_ACC, R_801, R_PADDED, R_STEM, R_BN = "repvgg_acc", "wgrad_acc", "refused_801", "padded", "stem", "bn_direct"
ALL_ROUTES = frozenset({R_REPVGG, R_ACC, R_801, R_PADDED, R_STEM, R_BN})
PLANNED_ROUTES = frozenset({R_REPVGG, R_ACC, R_801})     # the ones the launch planning (and so the SM count) decides

# case -> routes its direct arm takes. Blocks (N, C, H, W inputs as in the GPU table) and whole models at 4 x 3 x 64 x 64.
DIRECT_ROUTES = {
    "repblock-s1-identity": {R_REPVGG, R_BN},
    "repblock-s1": {R_REPVGG, R_BN},
    "repblock-s2": {R_ACC, R_BN},
    "repblock-s2-single-range": {R_801, R_BN},
    "repblock-s1-padded": {R_PADDED, R_BN},
    "repblock-stem": {R_STEM, R_BN},
    "repvgg_a0": {R_STEM, R_REPVGG, R_ACC, R_801, R_BN},
    "rexnet1_0x": {R_STEM, R_ACC, R_801, R_PADDED, R_BN},
    "resnet18": {R_PADDED, R_ACC, R_801, R_BN},
}

# case -> (planned route, weight-gradient call) pairs that the case runs: ("repvgg", (N, H, W, Cin, Cout)) for the one-pass
# RepVGG kernel, ("wgrad", (N, H, W, Cin, Cout, k, stride, pad)) for the single-filter one. The GPU test checks that each
# call is made and takes its route; the CPU test that it takes that route for every SM count.
DIRECT_WITNESSES = {
    "repblock-s1-identity": [(R_REPVGG, ("repvgg", (4, 16, 16, 48, 48)))],
    "repblock-s1": [(R_REPVGG, ("repvgg", (2, 24, 20, 32, 64)))],
    "repblock-s2": [(R_ACC, ("wgrad", (4, 32, 32, 48, 64, 3, 2, 1))), (R_ACC, ("wgrad", (4, 32, 32, 48, 64, 1, 2, 0)))],
    "repblock-s2-single-range": [(R_801, ("wgrad", (2, 4, 4, 128, 256, 3, 2, 1))),
                                 (R_801, ("wgrad", (2, 4, 4, 128, 256, 1, 2, 0)))],
    "repblock-s1-padded": [],
    "repblock-stem": [],
    # features.0.1 (48 -> 48 at 32 x 32), features.1.0 (stride 2), features.4.0 (192 -> 1280, 4 x 4 -> 2 x 2)
    "repvgg_a0": [(R_REPVGG, ("repvgg", (4, 32, 32, 48, 48))), (R_ACC, ("wgrad", (4, 32, 32, 48, 48, 3, 2, 1))),
                  (R_801, ("wgrad", (4, 4, 4, 192, 1280, 3, 2, 1)))],
    # block 2's 16 -> 96 expansion at 32 x 32; block 12's 128 -> 768 expansion at 4 x 4
    "rexnet1_0x": [(R_ACC, ("wgrad", (4, 32, 32, 16, 96, 1, 1, 0))), (R_801, ("wgrad", (4, 4, 4, 128, 768, 1, 1, 0)))],
    # layer1's 3x3 at 16 x 16; layer4's 3x3 at 2 x 2
    "resnet18": [(R_ACC, ("wgrad", (4, 16, 16, 64, 64, 3, 1, 1))), (R_801, ("wgrad", (4, 2, 2, 512, 512, 3, 1, 1)))],
}


def witness_route(kind, shape, sms):
    """The route a direct bucket's call of ``kind`` on ``shape`` takes with the workspace the size query asks for."""
    if kind == "repvgg":
        n, h, w, cin, cout = shape
        want = route_repvgg_wgrad(n, h, w, cin, cout, 0, 1 << 40, sms).ws_bytes
        r = route_repvgg_wgrad(n, h, w, cin, cout, 0, want, sms)
        return R_REPVGG if r.path == ROWS else R_PADDED if r.path == REFUSED else r.path
    n, h, w, cin, cout, k, stride, pad = shape
    want = route_wgrad(n, h, w, cin, cout, k, stride, pad, 0, False, 0, sms).ws_bytes
    r = route_wgrad(n, h, w, cin, cout, k, stride, pad, 0, True, want, sms)
    return R_801 if r.path == REFUSED else R_ACC
