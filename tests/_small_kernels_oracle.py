"""fp64 restatements, error magnitudes and launch routes of four small kernel families: DropBlock
(csrc/dropblock.cu), global average pooling (csrc/se_gate.cu gap_fwd_kernel, csrc/conv_aux.cu gap_bwd_kernel), the
HardMish / NLReLU activations (csrc/pointwise.cu) and the pairwise box backward (csrc/boxes.cu pairwise_bwd_kernel).

``route_*`` restate each family's launch arithmetic in Python and name the code paths a case takes, so the case
tables can state the path they are meant to reach and a CPU test can show that every path is reached. The oracles run
on whatever device their inputs are on."""
from typing import FrozenSet, Tuple

import torch
import torch.nn.functional as TF

U32 = 2.0 ** -24          # unit roundoff of fp32
THREADS = 256             # kThreads of pointwise.cu, the block size of the DropBlock and GAP kernels
MAX_WAVES = 8             # stream_grid's default cap: num_sms * 8 blocks
H100_SMS = 132

HM, NL, NL_OUT = "hard_mish", "nl_relu", "nl_relu_from_out"


def _cdiv(a: int, b: int) -> int:
    return -(-a // b)


def stream_grid(work: int, per_block: int, sms: int, max_waves: int = MAX_WAVES) -> Tuple[int, bool]:
    """(blocks, capped) of common.cuh stream_grid: enough blocks for the work, at most sms * max_waves."""
    need = max(1, _cdiv(work, per_block))
    cap = sms * max_waves
    return min(need, cap), need > cap


def vec_width(dtype: torch.dtype) -> int:
    """Vec16<T>::N: elements of one 128-bit vector."""
    return 16 // torch.empty((), dtype=dtype).element_size()


# ---------------------------------------------------------------------------------------------------------------------
# activations (pointwise.cu)
# ---------------------------------------------------------------------------------------------------------------------
ACT_PATHS = ("unrolled", "remainder", "tail", "capped", "unaligned")


def route_act(n: int, dtype: torch.dtype, binary: bool, aligned: bool, sms: int) -> FrozenSet[str]:
    """Loops of unary_kernel (forward; kUnroll = 4) or binary_kernel (backward; U = 2) that run for n elements:
    'unrolled' (the kUnroll / U vectors-per-trip body), 'remainder' (the one-vector loop after it), 'tail' (the scalar
    loop over the last n % V elements), 'capped' (stream_grid hit num_sms * 8 blocks, so threads stride), and
    'unaligned' (a pointer not 16-byte aligned: everything in the scalar loop)."""
    v = vec_width(dtype)
    u = 2 if binary else 4
    grid, capped = stream_grid(n, THREADS * v * u, sms)
    nt = grid * THREADS
    nvec = n // v if aligned else 0
    taken = set()
    if nvec > (u - 1) * nt:         # thread 0 has all u vectors of its first trip in range
        taken.add("unrolled")
    if nvec % (u * nt) != 0:        # some thread leaves the unrolled loop with a vector left
        taken.add("remainder")
    if n - nvec * v > 0:
        taken.add("tail" if aligned else "unaligned")
    if capped:
        taken.add("capped")
    return frozenset(taken)


# (name, vectors, tail elements, aligned, route): n = vectors * V + tail elements for every dtype, and one route for the
# forward (unary_kernel) and both backwards (binary_kernel) at any SM count from 100 to 144
ACT_CASES = [
    ("remainder_only", 250, 0, True, {"remainder"}),
    ("remainder_tail", 250, 3, True, {"remainder", "tail"}),
    ("unrolled_only", 3072, 0, True, {"unrolled"}),
    ("unrolled_remainder_tail", 3077, 3, True, {"unrolled", "remainder", "tail"}),
    ("capped", 1_250_001, 3, True, {"capped", "unrolled", "remainder", "tail"}),
    ("unaligned", 625, 1, False, {"unaligned"}),
]


def hard_mish_ref(x64: torch.Tensor) -> torch.Tensor:
    return 0.5 * x64 * (x64 + 2).clamp(0, 2)


def hard_mish_grad_ref(x64: torch.Tensor, dy64: torch.Tensor) -> torch.Tensor:
    """Autograd of the reference composition: clamp's gradient passes at both ends (x = -2 and x = 0 included) and is
    selected, not multiplied, elsewhere (x = +-inf gives dy or 0); a NaN input gives NaN."""
    t = x64 + 2
    inner = torch.where((t >= 0) & (t <= 2), 0.5 * x64, torch.zeros_like(x64))
    return dy64 * (0.5 * t.clamp(0, 2) + inner)


def nl_relu_ref(x64: torch.Tensor, beta: float) -> torch.Tensor:
    return torch.log1p(beta * torch.relu(x64))


def nl_relu_grad_ref(x64: torch.Tensor, dy64: torch.Tensor, beta: float) -> torch.Tensor:
    """relu'(0) = 0 and a NaN input gives NaN, as autograd of the reference gives them."""
    return torch.where(x64 <= 0, torch.zeros_like(x64), dy64 * beta / (1 + beta * x64))


def nl_relu_grad_from_out_ref(y64: torch.Tensor, dy64: torch.Tensor, beta: float) -> torch.Tensor:
    """The in-place gradient, from the stored output y: beta * exp(-y) where y > 0, else 0."""
    return torch.where(y64 <= 0, torch.zeros_like(y64), dy64 * beta * torch.exp(-y64))


# ---------------------------------------------------------------------------------------------------------------------
# DropBlock (dropblock.cu)
# ---------------------------------------------------------------------------------------------------------------------
DB_PATHS = ("nchw_scalar", "nhwc_vec", "nhwc_scalar_cvec", "nhwc_scalar_unaligned", "mask_capped")


def route_dropblock(n: int, c: int, h: int, w: int, dtype: torch.dtype, channels_last: bool, aligned: bool,
                    sms: int) -> FrozenSet[str]:
    """Kernels hb_dropblock_apply picks: the NHWC vector kernel when the layout is channels_last, C % V == 0 and both
    pointers are 16-byte aligned; otherwise the scalar kernel, in NCHW or NHWC indexing. 'mask_capped': the mask kernel's
    grid hit the num_sms * 8 cap."""
    v = vec_width(dtype)
    total = n * c * h * w
    taken = set()
    if not channels_last:
        taken.add("nchw_scalar")
    elif c % v != 0:
        taken.add("nhwc_scalar_cvec")
    elif not aligned:
        taken.add("nhwc_scalar_unaligned")
    elif total // v < 0xFFFFFFFF:
        taken.add("nhwc_vec")
    if stream_grid(n * h * w, THREADS, sms)[1]:
        taken.add("mask_capped")
    return frozenset(taken)


# (name, N, C, H, W, channels_last, storage offset in elements, in place, route); the C % V case uses
# C = 10, which no vector width (4 for fp32, 8 for 16-bit) divides
DB_APPLY_CASES = [
    ("nchw", 2, 5, 9, 11, False, 0, False, {"nchw_scalar"}),
    ("nchw_inplace", 2, 5, 9, 11, False, 0, True, {"nchw_scalar"}),
    ("nhwc_vec", 2, 16, 9, 11, True, 0, False, {"nhwc_vec"}),
    ("nhwc_vec_inplace", 2, 16, 9, 11, True, 0, True, {"nhwc_vec"}),
    ("nhwc_c_not_vec", 2, 10, 9, 11, True, 0, False, {"nhwc_scalar_cvec"}),
    ("nhwc_unaligned", 2, 16, 9, 11, True, 1, False, {"nhwc_scalar_unaligned"}),
    ("nchw_unaligned_inplace", 2, 5, 9, 11, False, 1, True, {"nchw_scalar"}),
]
# one mask of just over 2^24 cells, counted through the capped grid-stride loop
DB_BIG = (1, 1, 4100, 4100, {"nchw_scalar", "mask_capped"})


def dropblock_mask_ref(noise: torch.Tensor, gamma: float, block_size: int) -> Tuple[torch.Tensor, int]:
    """(mask [N, H, W] in fp64, exact kept count): 1 - max over the block_size window (stride 1, zero padding
    block_size // 2) of the seeds noise <= gamma, with gamma the fp32 value the kernel compares against."""
    g32 = torch.tensor(gamma, dtype=torch.float32).item()
    seeds = (noise.to(torch.float32) <= g32).to(torch.float64)
    p = block_size // 2
    pooled = TF.max_pool2d(seeds[:, None], block_size, stride=1, padding=p)[:, 0]
    mask = 1 - pooled
    return mask, int(mask.sum().item())


def dropblock_out_ref(x: torch.Tensor, mask64: torch.Tensor, kept: int) -> torch.Tensor:
    """fp64 x * mask * numel / kept with the exact count (scale 1 when nothing is kept)."""
    scale = mask64.numel() / kept if kept > 0 else 1.0
    return x.to(torch.float64) * mask64[:, None] * scale


def dropblock_reference_ops(x: torch.Tensor, noise: torch.Tensor, gamma: float, block_size: int) -> torch.Tensor:
    """The reference's op sequence (holocron/nn/functional.py:465-500) in x.dtype, given its noise."""
    mask = (noise <= gamma).to(dtype=x.dtype)
    mask = 1 - TF.max_pool2d(mask, kernel_size=(block_size, block_size), stride=(1, 1), padding=block_size // 2)
    one_count = mask.sum()
    out = x * mask.unsqueeze(1)
    if one_count > 0:
        out *= mask.numel() / one_count
    return out


# ---------------------------------------------------------------------------------------------------------------------
# global average pooling (se_gate.cu gap_fwd_kernel, conv_aux.cu gap_bwd_kernel)
# ---------------------------------------------------------------------------------------------------------------------
GAP_PATHS = ("pairs", "tail", "multi_slab", "partial_slab", "spare_lanes", "bwd_capped")


def slab_geo(c: int) -> Tuple[int, int, int, int]:
    """SlabGeo::make (slab.cuh): (cg_total, cg_t, rows_t, slabs)."""
    cg_total = c // 8
    nslab = _cdiv(cg_total, 32)
    cg_t = _cdiv(cg_total, nslab)
    rows_t = 256 // cg_t
    return cg_total, cg_t, rows_t, _cdiv(cg_total, cg_t)


# (N, HW, C, route)
GAP_CASES = [
    (3, 1, 8, {"tail"}),
    (2, 49, 8, {"tail"}),
    (2, 1, 24, {"tail", "spare_lanes"}),
    (2, 49, 1280, {"pairs", "tail", "multi_slab"}),
    (2, 3136, 2048, {"pairs", "multi_slab", "bwd_capped"}),
    (2, 3136, 24, {"pairs", "tail", "spare_lanes"}),
    (3, 3136, 264, {"pairs", "tail", "multi_slab", "partial_slab", "spare_lanes", "bwd_capped"}),
    (2, 256, 8, {"tail"}),
    (2, 512, 8, {"pairs"}),
]


def gap_chain(hw: int, c: int) -> int:
    """L: the most fp32 roundings on the way from one input to the mean. A row lane ty walks rows ty, ty + rows_t, ...
    two at a time: each pair costs a rounding for a + b and one for acc += (a + b), a lone last row one; the block fold
    adds rows_t lane sums in order (rows_t - 1 roundings); then 1 / HW and the product round once each."""
    _, _, rows_t, _ = slab_geo(c)
    rows0 = _cdiv(hw, rows_t)                   # rows of lane 0, the longest
    pairs, tail = rows0 // 2, rows0 % 2
    return 2 * pairs + tail + (rows_t - 1) + 2


def route_gap(n: int, hw: int, c: int, sms: int) -> FrozenSet[str]:
    cg_total, cg_t, rows_t, slabs = slab_geo(c)
    taken = set()
    if hw > rows_t:
        taken.add("pairs")
    # a lane's last row is alone when it owns an odd number of rows
    if any(_cdiv(hw - ty, rows_t) % 2 == 1 for ty in range(min(rows_t, hw))):
        taken.add("tail")
    if slabs > 1:
        taken.add("multi_slab")
    if slabs * cg_t > cg_total:
        taken.add("partial_slab")
    if rows_t * cg_t < 256:
        taken.add("spare_lanes")
    if stream_grid(n * hw * (c // 8), 256, sms)[1]:
        taken.add("bwd_capped")
    return frozenset(taken)


# ---------------------------------------------------------------------------------------------------------------------
# pairwise box backward (boxes.cu pair_grad / pairwise_bwd_kernel)
# ---------------------------------------------------------------------------------------------------------------------
IOU, GIOU, PENALTY, DIOU = 0, 1, 2, 3
BOX_PATHS = ("g1", "g2", "multi_block", "empty")


def route_box(m: int, n: int, want1: bool, want2: bool) -> FrozenSet[str]:
    """One thread per gradient row (M rows of boxes1, then N of boxes2), 128 per block; a NULL gradient pointer makes its
    threads return."""
    taken = set()
    if want1 and m > 0:
        taken.add("g1")
    if want2 and n > 0:
        taken.add("g2")
    if m + n > 128:
        taken.add("multi_block")
    if m == 0 or n == 0:
        taken.add("empty")
    return frozenset(taken)


# (name, M, N, gradients wanted (g1, g2), route)
BOX_SIZES = [
    ("small_both", 9, 7, (True, True), {"g1", "g2"}),
    ("only_g1", 9, 7, (True, False), {"g1"}),
    ("only_g2", 9, 7, (False, True), {"g2"}),
    ("multi_block", 150, 170, (True, True), {"g1", "g2", "multi_block"}),
    ("multi_block_only_g1", 300, 40, (True, False), {"g1", "multi_block"}),
    ("m_zero", 0, 5, (True, True), {"g2", "empty"}),
    ("n_zero", 5, 0, (True, True), {"g1", "empty"}),
]


class Mag:
    """A value and a magnitude that bounds the fp32 rounding error of computing it: |fl(v) - v| <= k * u * mag for a k
    that grows by at most one per operation. Sums add magnitudes, products multiply them, quotients follow
    d(a / b) = da / b - a db / b^2. Comparisons and max / min of input coordinates are exact."""

    def __init__(self, v, m=None):
        self.v = v
        self.m = v.abs() if m is None else m

    def __add__(self, o):
        o = _mag(o, self.v)
        return Mag(self.v + o.v, self.m + o.m)

    __radd__ = __add__

    def __sub__(self, o):
        o = _mag(o, self.v)
        return Mag(self.v - o.v, self.m + o.m)

    def __rsub__(self, o):
        return _mag(o, self.v) - self

    def __neg__(self):
        return Mag(-self.v, self.m)

    def __mul__(self, o):
        o = _mag(o, self.v)
        return Mag(self.v * o.v, self.m * o.m)

    __rmul__ = __mul__

    def __truediv__(self, o):
        o = _mag(o, self.v)
        return Mag(self.v / o.v, self.m / o.v.abs() + self.v.abs() * o.m / (o.v * o.v))

    def __rtruediv__(self, o):
        return _mag(o, self.v) / self


def _mag(o, like):
    return o if isinstance(o, Mag) else Mag(torch.full_like(like, float(o)))


def _mx(a, b):
    return Mag(torch.maximum(a.v, b.v))


def _mn(a, b):
    return Mag(torch.minimum(a.v, b.v))


def _relu(a):
    """fmaxf(a, 0): its magnitude stays a's (the computed a may be off by its own error)."""
    return Mag(a.v.clamp_min(0), a.m)


def _dmax(a, b):
    da = torch.where(a > b, 1.0, torch.where(a == b, 0.5, 0.0)).to(a.dtype)
    return da, 1 - da


def _dmin(a, b):
    da = torch.where(a < b, 1.0, torch.where(a == b, 0.5, 0.0)).to(a.dtype)
    return da, 1 - da


def pair_grad(mode: int, b1: torch.Tensor, b2: torch.Tensor):
    """fp64 restatement of boxes.cu pair_grad for every pair: (t, tmag), each [M, N, 8] with the derivative of the pair's
    value with respect to (ax1, ay1, ax2, ay2, bx1, by1, bx2, by2), and the magnitude of its terms. The kernel returns
    g1[i] = sum_j gout[i, j] * t[i, j, :4] and g2[j] = sum_i gout[i, j] * t[i, j, 4:]."""
    b1 = b1.to(torch.float64)
    b2 = b2.to(torch.float64)
    A = [Mag(b1[:, None, k].expand(b1.shape[0], b2.shape[0]).clone()) for k in range(4)]
    B = [Mag(b2[None, :, k].expand(b1.shape[0], b2.shape[0]).clone()) for k in range(4)]
    ax1, ay1, ax2, ay2 = A
    bx1, by1, bx2, by2 = B
    zero = Mag(torch.zeros_like(ax1.v))
    wa, ha, wb, hb = ax2 - ax1, ay2 - ay1, bx2 - bx1, by2 - by1
    ltx, lty, rbx, rby = _mx(ax1, bx1), _mx(ay1, by1), _mn(ax2, bx2), _mn(ay2, by2)
    wr, hr = rbx - ltx, rby - lty
    w, h = _relu(wr), _relu(hr)
    inter = w * h
    uni = wa * ha + wb * hb - inter
    c_inter, c_area, g_cw, g_ch, g_dx, g_dy = zero, zero, zero, zero, zero, zero
    cwr = _mx(ax2, bx2) - _mn(ax1, bx1)
    chr_ = _mx(ay2, by2) - _mn(ay1, by1)
    if mode in (IOU, GIOU, DIOU):
        s = -1.0 if mode == DIOU else 1.0
        c_inter = c_inter + s * ((uni + inter) / (uni * uni))
        c_area = c_area + s * (-inter / (uni * uni))
    if mode == GIOU:
        cw, ch = _relu(cwr), _relu(chr_)
        area_c = cw * ch
        c_area = c_area + 1.0 / area_c
        c_inter = c_inter + (-1.0) / area_c
        g_area_c = -uni / (area_c * area_c)
        g_cw = g_cw + g_area_c * ch * Mag((cwr.v >= 0).to(torch.float64))
        g_ch = g_ch + g_area_c * cw * Mag((chr_.v >= 0).to(torch.float64))
    if mode in (PENALTY, DIOU):
        c2 = cwr * cwr + chr_ * chr_
        dx = (ax1 + ax2) - (bx1 + bx2)
        dy = (ay1 + ay2) - (by1 + by2)
        r2 = (dx * dx + dy * dy) * 0.25
        g_dx = g_dx + 0.5 * dx / c2
        g_dy = g_dy + 0.5 * dy / c2
        g_c2 = -r2 / (c2 * c2)
        g_cw = g_cw + g_c2 * 2.0 * cwr
        g_ch = g_ch + g_c2 * 2.0 * chr_
    gi_w = c_inter * h * Mag((wr.v >= 0).to(torch.float64))
    gi_h = c_inter * w * Mag((hr.v >= 0).to(torch.float64))
    t = [zero] * 8
    da, db = _dmax(ax1.v, bx1.v); t[0] = t[0] - gi_w * Mag(da); t[4] = t[4] - gi_w * Mag(db)
    da, db = _dmax(ay1.v, by1.v); t[1] = t[1] - gi_h * Mag(da); t[5] = t[5] - gi_h * Mag(db)
    da, db = _dmin(ax2.v, bx2.v); t[2] = t[2] + gi_w * Mag(da); t[6] = t[6] + gi_w * Mag(db)
    da, db = _dmin(ay2.v, by2.v); t[3] = t[3] + gi_h * Mag(da); t[7] = t[7] + gi_h * Mag(db)
    t[0] = t[0] + c_area * (-ha); t[2] = t[2] + c_area * ha; t[1] = t[1] + c_area * (-wa); t[3] = t[3] + c_area * wa
    t[4] = t[4] + c_area * (-hb); t[6] = t[6] + c_area * hb; t[5] = t[5] + c_area * (-wb); t[7] = t[7] + c_area * wb
    da, db = _dmax(ax2.v, bx2.v); t[2] = t[2] + g_cw * Mag(da); t[6] = t[6] + g_cw * Mag(db)
    da, db = _dmin(ax1.v, bx1.v); t[0] = t[0] - g_cw * Mag(da); t[4] = t[4] - g_cw * Mag(db)
    da, db = _dmax(ay2.v, by2.v); t[3] = t[3] + g_ch * Mag(da); t[7] = t[7] + g_ch * Mag(db)
    da, db = _dmin(ay1.v, by1.v); t[1] = t[1] - g_ch * Mag(da); t[5] = t[5] - g_ch * Mag(db)
    t[0] = t[0] + g_dx; t[2] = t[2] + g_dx; t[4] = t[4] - g_dx; t[6] = t[6] - g_dx
    t[1] = t[1] + g_dy; t[3] = t[3] + g_dy; t[5] = t[5] - g_dy; t[7] = t[7] - g_dy
    return torch.stack([e.v for e in t], -1), torch.stack([e.m for e in t], -1)


# the longest chain of fp32 operations inside pair_grad, each of which may add one rounding (counted generously)
PAIR_GRAD_DEPTH = 32


def box_grads_ref(mode: int, b1: torch.Tensor, b2: torch.Tensor, gout: torch.Tensor):
    """(g1, g2, bound1, bound2) in fp64: the gradients of sum(gout * value(b1, b2)) and per-element bounds on the fp32
    kernel's error, rel * sum_j |gout_ij| * tmag_ij with rel = (PAIR_GRAD_DEPTH + terms summed) * 2^-24."""
    t, tm = pair_grad(mode, b1, b2)
    g = gout.to(torch.float64)[..., None]
    m, n = gout.shape
    g1 = (g * t[..., :4]).sum(1)
    g2 = (g * t[..., 4:]).sum(0)
    bound1 = (PAIR_GRAD_DEPTH + n) * U32 * (g.abs() * tm[..., :4]).sum(1)
    bound2 = (PAIR_GRAD_DEPTH + m) * U32 * (g.abs() * tm[..., 4:]).sum(0)
    return g1, g2, bound1, bound2


def box_value(mode: int, b1: torch.Tensor, b2: torch.Tensor) -> torch.Tensor:
    """The reference's pairwise value (oracle/boxes.py) of a mode, for autograd."""
    from oracle import boxes as OB
    if mode == IOU:
        return OB.box_iou(b1, b2)
    if mode == GIOU:
        return OB.box_giou(b1, b2)
    if mode == PENALTY:
        # oracle/boxes.py casts to fp32 as the reference does; keep the caller's dtype for an fp64 autograd
        dw = torch.max(b1[:, None, 2], b2[None, :, 2]) - torch.min(b1[:, None, 0], b2[None, :, 0])
        dh = torch.max(b1[:, None, 3], b2[None, :, 3]) - torch.min(b1[:, None, 1], b2[None, :, 1])
        c2 = dw ** 2 + dh ** 2
        cx = (b1[:, 0] + b1[:, 2])[:, None] - (b2[:, 0] + b2[:, 2])[None, :]
        cy = (b1[:, 1] + b1[:, 3])[:, None] - (b2[:, 1] + b2[:, 3])[None, :]
        return (cx ** 2 + cy ** 2) / 4 / c2
    return 1 - OB.box_iou(b1, b2) + box_value(PENALTY, b1, b2)


def box_autograd(mode: int, b1: torch.Tensor, b2: torch.Tensor, gout: torch.Tensor):
    """Gradients of sum(gout * value) by torch autograd of the reference's composition, in the inputs' dtype."""
    a = b1.detach().clone().requires_grad_(True)
    b = b2.detach().clone().requires_grad_(True)
    (box_value(mode, a, b) * gout).sum().backward()
    return a.grad, b.grad


def integer_boxes(n: int, gen: torch.Generator, span: int = 6, border: int = 0) -> torch.Tensor:
    """n boxes with small integer corners in [0, span]: full of ties, touching edges, identical and contained pairs.
    With border > 0 the corners are clipped to [0, border] (boxes cut by a common image border)."""
    xy = torch.randint(0, span + 1, (n, 2), generator=gen)
    wh = torch.randint(0, span // 2 + 1, (n, 2), generator=gen)
    b = torch.cat([xy, xy + wh], 1).to(torch.float64)
    if border:
        b = b.clamp(0, border)
    return b


def f32_ulp(x: torch.Tensor) -> torch.Tensor:
    """One fp32 ulp at each |x| (fp64 result; subnormal spacing below 2^-126)."""
    a = x.to(torch.float64).abs().clamp_min(2.0 ** -126)
    return torch.exp2(torch.floor(torch.log2(a)) - 23)


LOG_FAST_ABS = 2.0 ** -21.4    # __logf absolute error for arguments >= 1 (CUDA C Programming Guide, intrinsic functions)

