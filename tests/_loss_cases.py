"""The loss kernel cases and a Python mirror of the dispatch and grid geometry of csrc/losses.cu (no GPU).

``route`` names, for each entry point a case calls, the kernel instantiation launched and its grid: the launcher
conditions of ``hb_cls_loss_hard_*``, ``hb_poly_soft_*`` (``class_loss``), ``hb_dice_*``, ``hb_cce_*`` and ``hb_mcl_*``,
and ``vec_eligible``, ``dispatch_kmax``, ``grid_for``, ``dice_blocks_per_class`` and ``mcl_rdot_threads``. A kernel's
branch on ``S == 1`` (one warp or one thread per position) and on its ``vec`` flag is part of the name after a ``/``.
Every kernel except the row / group / finalize kernels is grid-stride: a thread starting at item ``i0 < stride`` runs
``ceil((total - i0) / stride)`` iterations, at least ``total // stride`` and at most ``ceil(total / stride)``. The SM
count sizes the grids, so the mirror takes it as an argument (H100 SXM: 132, H100 PCIe: 114)."""
from dataclasses import dataclass, field
from typing import Dict, List, Tuple

THREADS = 256
TYPES = {"float32": ("float", 4), "bfloat16": ("__nv_bfloat16", 2), "float16": ("__half", 2)}
DTYPES = tuple(TYPES)
KMAXES = (4, 8, 12, 16, 20, 24, 28, 32)
RDOT_BLOCKS = (256, 224, 32)            # mcl_rdot_kernel block sizes the cases must reach


def _cdiv(a: int, b: int) -> int:
    return -(-a // b)


def _instantiations() -> Tuple[str, ...]:
    out = []
    for dt in DTYPES:
        T = TYPES[dt][0]
        for kern in ("hard_vec_kernel", "poly_soft_vec_kernel"):
            out += [f"{kern}<{T},{km},{str(bwd).lower()}>" for km in KMAXES for bwd in (False, True)]
        out += [f"hard_kernel<{T},{str(bwd).lower()}>/{b}" for bwd in (False, True) for b in ("warp", "thread")]
        out += [f"poly_soft_kernel<{T},{str(bwd).lower()}>" for bwd in (False, True)]
        out += [f"dice_{d}_kernel<{T}>/{v}" for d in ("sums", "bwd") for v in ("vec", "scalar")]
        out += [f"cce_kernel<{T},{str(bwd).lower()}>/{b}" for bwd in (False, True) for b in ("warp", "thread")]
        out += [f"mcl_row_lse_kernel<{T}>/{v}" for v in ("vec", "scalar")]
        out += [f"mcl_{k}_kernel<{T}>" for k in ("fwd", "rdot", "bwd")]
    return tuple(out) + ("finalize_kernel<2>", "finalize_kernel<3>", "dice_finalize_kernel")


# every kernel instantiation in losses.cu, one entry per side of a kernel's S == 1 / vec branch
INSTANTIATIONS = _instantiations()


@dataclass(frozen=True)
class Case:
    """One loss call: x is [N, K, S] (MCL: K = cnum * xi) in ``dtype``, placed ``offset`` elements past an aligned
    address; for soft targets and dice the targets and dx sit at the same offset."""
    family: str             # "hard", "soft", "dice", "cce", "mcl"
    dtype: str
    n: int
    k: int
    s: int
    offset: int = 0
    xi: int = 1             # MCL channels per class
    logits: str = "randn"   # "randn", "confident" (target logit +30), "uniform", "shift16", "shift100", "shift1000"
    wrap: bool = False      # every thread of every grid-stride launch runs at least two iterations
    light: bool = False     # large: run with one parameter set only
    tags: Tuple[str, ...] = field(default=())

    @property
    def positions(self) -> int:
        return self.n * self.s

    @property
    def cnum(self) -> int:
        return self.k // self.xi

    @property
    def name(self) -> str:
        extra = "".join(f"_{t}" for t in (self.logits,) if t != "randn")
        extra += f"_off{self.offset}" if self.offset else ""
        extra += f"_xi{self.xi}" if self.family == "mcl" else ""
        return f"{self.family}_{self.dtype}_n{self.n}k{self.k}s{self.s}{extra}"


@dataclass(frozen=True)
class Launch:
    kernel: str
    total: int          # grid-stride items (positions, vector positions, elements); 0: not grid-stride
    stride: int         # items the whole grid takes per iteration
    grid: int
    block: int = THREADS

    @property
    def min_iters(self) -> int:
        return self.total // self.stride if self.total else 0

    @property
    def max_iters(self) -> int:
        return _cdiv(self.total, self.stride) if self.total else 0


def grid_for(work: int, per_block: int, sms: int) -> int:
    return max(min(_cdiv(work, per_block), sms * 8), 1)


def vec_width(dtype: str) -> int:
    """V of Vec8<T>: elements per 8-byte vector."""
    return 8 // TYPES[dtype][1]


def vec16_width(dtype: str) -> int:
    return 16 // TYPES[dtype][1]


def _aligned(cs: Case, nbytes: int) -> bool:
    return (cs.offset * TYPES[cs.dtype][1]) % nbytes == 0


def vec_eligible(cs: Case) -> bool:
    v = vec_width(cs.dtype)
    return cs.s > 1 and cs.s % v == 0 and cs.k <= 32 and cs.k * cs.s < 0x7FFFFFFF and _aligned(cs, 8)


def kmax(k: int) -> int:
    return min(max((k + 3) // 4, 1), 8) * 4


def dice_blocks_per_class(per_class: int, k: int, sms: int) -> int:
    gx = max(min(_cdiv(per_class, THREADS * 16), sms * 8), 1)
    if gx * k > sms * 16:
        gx = _cdiv(sms * 16, k)
    return max(gx, 1)


def mcl_rdot_threads(xi: int) -> int:
    return min((47 * 1024 // 4 // xi) // 32 * 32, THREADS)


def dice_vec(cs: Case) -> bool:
    """The vec flag of both dice kernels (x, target and dx share the case's offset)."""
    return cs.s % vec16_width(cs.dtype) == 0 and _aligned(cs, 16)


def _lanes(cs: Case, name: str, sms: int) -> Launch:
    """A scalar kernel with a warp per position when S == 1, a thread per position otherwise."""
    p = cs.positions
    if cs.s == 1:
        gx = grid_for(p, THREADS // 32, sms)
        return Launch(f"{name}/warp", p, gx * (THREADS // 32), gx)
    gx = grid_for(p, THREADS, sms)
    return Launch(f"{name}/thread", p, gx * THREADS, gx)


def route(cs: Case, sms: int) -> Dict[str, Launch]:
    T = TYPES[cs.dtype][0]
    p = cs.positions
    if cs.family in ("hard", "soft"):
        out = {}
        for d, bwd in (("fwd", False), ("bwd", True)):
            if vec_eligible(cs):
                v = vec_width(cs.dtype)
                kern = "hard_vec_kernel" if cs.family == "hard" else "poly_soft_vec_kernel"
                gx = grid_for(p // v, THREADS, sms)
                out[d] = Launch(f"{kern}<{T},{kmax(cs.k)},{str(bwd).lower()}>", p // v, gx * THREADS, gx)
            elif cs.family == "hard":
                out[d] = _lanes(cs, f"hard_kernel<{T},{str(bwd).lower()}>", sms)
            else:
                gx = grid_for(p, THREADS, sms)
                out[d] = Launch(f"poly_soft_kernel<{T},{str(bwd).lower()}>", p, gx * THREADS, gx)
        out["finalize"] = Launch("finalize_kernel<2>", 0, 1, 1, 32)
        return out
    if cs.family == "dice":
        vec, v = dice_vec(cs), vec16_width(cs.dtype)
        gx = dice_blocks_per_class(p, cs.k, sms)
        tag = "vec" if vec else "scalar"
        items = p // v if vec else p
        total = p * cs.k
        bgrid = grid_for(total, THREADS * (v * 2 if vec else 4), sms)
        btotal = total // v if vec else total
        return {"fwd": Launch(f"dice_sums_kernel<{T}>/{tag}", items, gx * THREADS, gx),
                "finalize": Launch("dice_finalize_kernel", 0, 1, 1),
                "bwd": Launch(f"dice_bwd_kernel<{T}>/{tag}", btotal, bgrid * THREADS, bgrid)}
    if cs.family == "cce":
        return {"fwd": _lanes(cs, f"cce_kernel<{T},false>", sms), "bwd": _lanes(cs, f"cce_kernel<{T},true>", sms),
                "finalize": Launch("finalize_kernel<3>", 0, 1, 1, 32)}
    if cs.family == "mcl":
        vec = cs.s % vec16_width(cs.dtype) == 0 and _aligned(cs, 16)
        gx = grid_for(p, THREADS, sms)
        return {"row_lse": Launch(f"mcl_row_lse_kernel<{T}>/{'vec' if vec else 'scalar'}", 0, 1, cs.n * cs.k),
                "fwd": Launch(f"mcl_fwd_kernel<{T}>", p, gx * THREADS, gx),
                "finalize": Launch("finalize_kernel<3>", 0, 1, 1, 32),
                "rdot": Launch(f"mcl_rdot_kernel<{T}>", 0, 1, cs.n * cs.cnum, mcl_rdot_threads(cs.xi)),
                "bwd": Launch(f"mcl_bwd_kernel<{T}>", p, gx * THREADS, gx)}
    raise ValueError(cs.family)


def kernels_taken(cs: Case, sms: int) -> List[str]:
    return [launch.kernel for launch in route(cs, sms).values()]


def describe(cs: Case, sms: int) -> str:
    parts = [f"{d}: {v.kernel} grid={v.grid}x{v.block} iters {v.min_iters}..{v.max_iters}" for d, v in route(cs, sms).items()]
    return f"{cs.name} @ {sms} SMs: " + "; ".join(parts)


# ---- the case table ---------------------------------------------------------------------------------------------------
def _hard_soft(family: str) -> List[Case]:
    out = []
    for dt in DTYPES:
        # the vector path at both edges of every KMAX bucket (S = 16 is a multiple of V in every dtype)
        out += [Case(family, dt, 3, k, 16) for k in (1, 4, 5, 8, 9, 12, 13, 16, 17, 20, 21, 24, 25, 28, 29, 32)]
        out += [Case(family, dt, 3, 33, 16),            # K > 32: one thread per position
                Case(family, dt, 5, 7, 6),              # S % V != 0 in bf16 / fp16, vector in fp32
                Case(family, dt, 3, 5, 7), Case(family, dt, 2, 29, 9),      # odd S
                Case(family, dt, 3, 12, 16, offset=1)]  # logits (and targets, dx) one element off the vector alignment
        out += [Case(family, dt, 37, k, 1) for k in (1, 2, 31, 32, 33, 1000, 4099)]     # S == 1
        for logits in ("confident", "uniform", "shift16", "shift100") + (("shift1000",) if dt == "float32" else ()):
            out += [Case(family, dt, 3, 12, 16, logits=logits), Case(family, dt, 3, 33, 5, logits=logits),
                    Case(family, dt, 19, 40, 1, logits=logits)]
    out += [Case(family, "bfloat16", 4, 5, 1 << 21, wrap=True, light=True),       # vector path
            Case(family, "float32", 3, 5, 200003, wrap=True, light=True)]          # one thread per position
    if family == "hard":
        out.append(Case(family, "float16", 40000, 33, 1, wrap=True, light=True))   # one warp per position
    return out


def _dice() -> List[Case]:
    out = []
    for dt in DTYPES:
        out += [Case("dice", dt, 3, 4, 64), Case("dice", dt, 3, 4, 63), Case("dice", dt, 2, 5, 1),
                Case("dice", dt, 2, 3, 1 << 18),        # several blocks per class
                Case("dice", dt, 2, 2200, 3),           # K > 16 * SMs: one block per class
                Case("dice", dt, 3, 4, 64, offset=1)]   # target / dx off the 16-byte alignment
    out.append(Case("dice", "bfloat16", 2, 21, 1 << 16, wrap=True, light=True))
    return out


def _cce() -> List[Case]:
    out = []
    for dt in DTYPES:
        out += [Case("cce", dt, 37, k, 1) for k in (2, 33, 1000)]
        out += [Case("cce", dt, 3, 5, 16), Case("cce", dt, 2, 40, 7), Case("cce", dt, 3, 12, 16, offset=1)]
        for logits in ("confident", "uniform", "shift16", "shift100") + (("shift1000",) if dt == "float32" else ()):
            out += [Case("cce", dt, 3, 12, 16, logits=logits), Case("cce", dt, 19, 40, 1, logits=logits)]
    out += [Case("cce", "float32", 3, 5, 200003, wrap=True, light=True),
            Case("cce", "bfloat16", 40000, 33, 1, wrap=True, light=True)]
    return out


def _mcl() -> List[Case]:
    out = []
    for dt in DTYPES:
        for xi, cnum, s in ((1, 4, 7), (2, 4, 64), (3, 21, 7), (47, 1, 64), (48, 4, 1), (376, 1, 7), (2, 21, 1)):
            out.append(Case("mcl", dt, 3, cnum * xi, s, xi=xi))
        out.append(Case("mcl", dt, 3, 8, 64, xi=2, offset=1))
        out.append(Case("mcl", dt, 3, 12, 7, xi=3, logits="equal"))
    out.append(Case("mcl", "float32", 3, 8, 200003, xi=2, wrap=True, light=True))
    return out


CASES: Dict[str, Case] = {cs.name: cs for cs in _hard_soft("hard") + _hard_soft("soft") + _dice() + _cce() + _mcl()}
