"""Launch routes, refusals and fp64 oracles of the involution and lambda kernels (csrc/involution.cu,
csrc/lambda_layer.cu), the two families that stage a shared-memory halo box (nhwc.cuh stage_box).

``route_*`` restate each entry point's launch arithmetic in Python and name the code paths a case takes for a given SM
count, so the case tables below can state the path each case is meant to reach and a CPU test can show that every path
is reached. ``*_refused`` restate the shape checks of ``make_params`` and the pointer checks of the entry points.

The oracles take the kernels' operands in their NHWC layouts ([B, HW, C] with the logical channels only), promoted to
fp64, and return the fp64 value of one entry point's output together with the same computation on absolute values (the
sum |terms| of _bounds.py). Each kernel is checked on its own: an oracle takes the intermediate a kernel is fed (the
softmax statistics, lc, dlc, dlp) as that kernel sees it, not as the upstream oracle would have computed it. They run
on whatever device their inputs are on."""
from typing import Dict, FrozenSet, Optional, Tuple

import torch
import torch.nn.functional as TF

THREADS = 256              # kThreads of both files
GRID_WAVES = 16            # stream_grid(..., kThreads, 16) of the grid-stride kernels
INDEX_LIMIT = 0x7fffffff   # element counts of the 32-bit grid-stride indices must stay below this
MAX_GRID_Z = 65535         # N (involution) and B (lambda) are a grid's y / z dimension
OPTIN = 48 * 1024          # dynamic shared memory above this needs allow_smem


def cdiv(a: int, b: int) -> int:
    return -(-a // b)


def round_up(v: int, m: int) -> int:
    return cdiv(v, m) * m


def stream_grid(work: int, sms: int, per_block: int = THREADS, waves: int = GRID_WAVES) -> Tuple[int, bool]:
    """(blocks, capped) of common.cuh stream_grid: enough blocks for the work, at most sms * waves; when capped, the
    grid-stride loops run more than once for some threads."""
    need = max(1, cdiv(work, per_block))
    cap = sms * waves
    return min(need, cap), need > cap


def window_out(n: int, k: int, stride: int, pad: int, dil: int) -> Optional[int]:
    """common.cuh window_out: the output extent, or None where the entry points refuse the window."""
    if n < 1 or k < 1 or stride < 1 or dil < 1 or pad < 0:
        return None
    span = n + 2 * pad - dil * (k - 1) - 1
    if span < 0 or span // stride >= INDEX_LIMIT:
        return None
    return span // stride + 1


# ---------------------------------------------------------------------------------------------------------------------
# involution (involution.cu)
# ---------------------------------------------------------------------------------------------------------------------
INV_TILE_W = 8                 # kTileW
INV_SMEM_MAX = 112 * 1024      # kSmemMax
INV_K = (1, 3, 5, 7)

INV_PATHS = ("uniform", "mixed", "fwd_nv1", "fwd_nv2", "fwd_nv4", "fwd_th_full", "fwd_th_halved", "fwd_th_one",
             "fwd_smem", "fwd_smem_optin", "fwd_global", "bwk_vg1", "bwk_vg2", "bwk_vg4", "bwk_vg8", "bwk_th_halved",
             "bwk_generic", "data_capped", "generic_capped")


def inv_refused(N, H, W, C, Cp, Kp, K, G, stride, pad, dil) -> bool:
    """make_params of involution.cu: True where all three entry points return cudaErrorInvalidValue."""
    if N <= 0 or C <= 0 or G <= 0 or C % G != 0 or Cp < C or Cp % 8 != 0 or Kp < G * K * K or K not in INV_K:
        return True
    ho, wo = window_out(H, K, stride, pad, dil), window_out(W, K, stride, pad, dil)
    if ho is None or wo is None or N > MAX_GRID_Z:
        return True
    return N * H * W * Cp >= INDEX_LIMIT or N * ho * wo * max(Cp, Kp) >= INDEX_LIMIT


def uniform_vectors(C: int, Cp: int, G: int) -> bool:
    return (C // G) % 8 == 0 and Cp == C


def make_tile(K: int, stride: int, dil: int, nv: int) -> Dict[str, int]:
    """make_tile: th rows of kTileW output pixels, halved while the halo box exceeds kSmemMax and th > 1."""
    th0 = th = THREADS // (nv * INV_TILE_W)
    reach = dil * (K - 1) + 1
    in_w = (INV_TILE_W - 1) * stride + reach
    while True:
        in_h = (th - 1) * stride + reach
        smem = in_h * in_w * nv * 16
        if smem <= INV_SMEM_MAX or th == 1:
            break
        th //= 2
    return dict(th0=th0, th=th, in_h=in_h, in_w=in_w, smem=smem)


def _th_tag(tile) -> str:
    if tile["th"] == tile["th0"]:
        return "th_full"
    return "th_one" if tile["th"] == 1 else "th_halved"


def route_involution(N, H, W, C, Cp, Kp, K, G, stride, pad, dil, sms) -> FrozenSet[str]:
    """Paths of the three entry points for an accepted shape: uniform or mixed vectors; the forward's vectors per pixel
    (nv), its th halving and whether its halo box fits shared memory (above 48 KiB with allow_smem) or the taps come
    from global memory; the kernel-gradient tile kernel per vg (with its own tile) or the generic kernel; and the
    grid-stride kernels whose stream_grid(..., 16) grid is capped."""
    ho, wo = window_out(H, K, stride, pad, dil), window_out(W, K, stride, pad, dil)
    uni = uniform_vectors(C, Cp, G)
    cv = Cp // 8
    nv = 4 if cv >= 4 else (2 if cv >= 2 else 1)
    taken = {"uniform" if uni else "mixed", f"fwd_nv{nv}"}
    ft = make_tile(K, stride, dil, nv)
    taken.add("fwd_" + _th_tag(ft))
    if ft["smem"] > INV_SMEM_MAX:
        taken.add("fwd_global")
    else:
        taken.add("fwd_smem_optin" if ft["smem"] > OPTIN else "fwd_smem")
    vg = C // G // 8 if uni else 0
    generic = True
    if vg in (1, 2, 4, 8):
        bt = make_tile(K, stride, dil, max(nv, vg))
        if bt["smem"] <= INV_SMEM_MAX:
            generic = False
            taken.add(f"bwk_vg{vg}")
            if bt["th"] != bt["th0"]:
                taken.add("bwk_th_halved")
    if generic:
        taken.add("bwk_generic")
        if stream_grid(N * ho * wo * Kp, sms)[1]:
            taken.add("generic_capped")
    if stream_grid(N * H * W * cv, sms)[1]:
        taken.add("data_capped")
    return frozenset(taken)


def inv_case_geom(case) -> Tuple[int, ...]:
    """(N, H, W, C, Cp, Kp, K, G, stride, pad, dil) of an INV_CASES row."""
    name, N, H, W, C, G, K, s, p, d, kp_extra, want = case
    return (N, H, W, C, round_up(C, 8), G * K * K + kp_extra, K, G, s, p, d)


# (name, N, H, W, C, G, K, stride, pad, dil, Kp - G*K^2, paths it witnesses at every SM count from 100 to 144)
INV_CASES = [
    ("c8_vg1_nv1", 2, 9, 7, 8, 1, 3, 1, 1, 1, 7, {"uniform", "fwd_nv1", "fwd_th_full", "fwd_smem", "bwk_vg1"}),
    ("c16_vg2_nv2", 2, 11, 9, 16, 1, 5, 2, 2, 1, 0, {"fwd_nv2", "bwk_vg2"}),
    ("c32_vg4", 1, 10, 13, 32, 1, 7, 1, 3, 1, 3, {"fwd_nv4", "bwk_vg4"}),
    ("c64_vg8", 2, 9, 9, 64, 1, 3, 1, 1, 1, 0, {"bwk_vg8"}),
    ("c64_vg8_halved", 1, 40, 44, 64, 1, 3, 3, 8, 8, 0, {"bwk_vg8", "bwk_th_halved", "fwd_smem_optin"}),
    ("c128_g2_fwd_halved", 1, 40, 38, 128, 2, 5, 2, 14, 7, 2, {"fwd_th_halved", "fwd_smem_optin", "bwk_generic"}),
    ("c12_g6_mixed", 2, 11, 9, 12, 6, 3, 1, 1, 2, 1, {"mixed", "bwk_generic"}),
    ("c20_g5_mixed_k1", 1, 7, 8, 20, 5, 1, 1, 0, 1, 0, {"mixed", "fwd_nv2"}),
    ("c24_g1_vg3", 2, 8, 8, 24, 1, 5, 1, 2, 1, 4, {"uniform", "bwk_generic"}),
    ("c32_th_one_global", 1, 40, 40, 32, 4, 7, 3, 5, 6, 0, {"fwd_th_one", "fwd_global", "bwk_generic"}),
    ("c32_th_one_smem", 1, 36, 37, 32, 4, 5, 3, 16, 8, 0, {"fwd_th_one", "fwd_smem_optin", "bwk_vg1"}),
    ("c256_g2_capped", 8, 56, 56, 256, 2, 7, 1, 3, 1, 14, {"data_capped", "generic_capped", "bwk_generic"}),
]


# ---------------------------------------------------------------------------------------------------------------------
# lambda (lambda_layer.cu)
# ---------------------------------------------------------------------------------------------------------------------
LAM_TILE = 8          # kTile: 8 x 8 output positions per CTA of the halo kernels
LAM_MAX_R = 23        # kMaxR
LAM_DK = (8, 16, 32)
LAM_CHUNK_M = 256     # positions per m-chunk of the content kernels (kThreads)
LAM_CHUNK_V = 128     # dim_v values per v0 chunk of the content kernels
DR_TILE = 8           # kDrTile
DR_V = 8              # kDrV
LAM_ENTRIES = ("content_fwd", "out_fwd", "bwd_content", "dlp", "bwd_q", "bwd_v", "bwd_r")

LAM_PATHS = tuple(
    [f"outdq_dk{dk}_u{u}_local" for dk in LAM_DK for u in (1, 2, 3, 4)]
    + [f"outdq_dk{dk}_u1_global" for dk in LAM_DK]
    + [f"dv_dk{dk}_u{u}_{kind}" for dk in LAM_DK for u in (1, 2, 3, 4) for kind in ("local", "global")]
    + ["halo_le48k", "halo_gt48k", "y_vec", "y_scalar", "content_mchunks", "global_mchunks", "content_v0chunks",
       "dr_le48k", "dr_gt48k", "dr_sliced", "dr_one_slice", "dv_capped", "dlp_capped"])


def lam_refused(B, H, W, dk, u, heads, dv, r, Cqp, Ckp, Cvp, Cop) -> bool:
    """make_params of lambda_layer.cu: True where all seven entry points return cudaErrorInvalidValue."""
    if (B <= 0 or H <= 0 or W <= 0 or dk not in LAM_DK or not 1 <= u <= 4 or not 1 <= heads <= 8 or dv < 1 or r < 0
            or r > LAM_MAX_R or (r > 0 and r % 2 == 0) or Cqp < heads * dk or Ckp < dk * u or Cvp < dv * u
            or Cop < heads * dv or Cqp % 8 or Ckp % 8 or Cvp % 8 or Cop % 8 or B > MAX_GRID_Z):
        return True
    dvp = round_up(dv, 8)
    return B * H * W * max(Cqp, Ckp, Cvp, Cop) >= INDEX_LIMIT or B * H * W * dk * dvp >= INDEX_LIMIT


def lam_pointer_refused(entry: str, r: int, null: FrozenSet[str]) -> bool:
    """The pointer checks after make_params: out_fwd / bwd_q need Rt (local) or lp (global), bwd_v needs Rt and dlp
    (local) or dvpos (global), bwd_r has no global variant."""
    if entry in ("out_fwd", "bwd_q"):
        return ("Rt" if r > 0 else "lp") in null
    if entry == "bwd_v":
        return bool({"Rt", "dlp"} & null) if r > 0 else "dvpos" in null
    if entry == "bwd_r":
        return r == 0
    return False


def halo_smem(r: int, u: int) -> int:
    """halo_grid's dynamic shared memory of the output and dq kernels: the (8 + r - 1)^2 box of u vectors."""
    box = LAM_TILE + r - 1
    return box * box * u * 16 if r > 0 else 0


def dr_smem_bytes(dk: int, u: int, r: int) -> int:
    stage = DR_TILE * DR_TILE * DR_V * dk + DR_TILE * (DR_TILE + r + 2) * DR_V * u
    return max(stage, THREADS * 16) * 4


def dr_microtiles(dk: int, u: int, r: int) -> int:
    """mt of lam_dr_partial_kernel: one thread per 4 k x 4 taps of one u'; the kernel needs mt <= kThreads."""
    return (dk // 4) * u * cdiv(r, 4)


def route_lambda(B, H, W, dk, u, heads, dv, r, sms) -> FrozenSet[str]:
    """Paths of the seven entry points for an accepted shape: the (DK, U, local) instantiation of the output / dq kernels
    (U = 1 for the global variant) and of the dv kernel (the layer's u either way); the halo box below or above 48 KiB;
    the vector or scalar store of y; several m-chunks (HW > 256) and v0 chunks (dv > 128) in the content kernels; the dR
    partial kernel's shared memory and slice count; and the dv / dlp grids capped by stream_grid(..., 16)."""
    hw = H * W
    loc = "local" if r else "global"
    taken = {f"outdq_dk{dk}_u{u if r else 1}_{loc}", f"dv_dk{dk}_u{u}_{loc}", "y_vec" if dv % 8 == 0 else "y_scalar"}
    if r:
        taken.add("halo_gt48k" if halo_smem(r, u) > OPTIN else "halo_le48k")
        taken.add("dr_gt48k" if dr_smem_bytes(dk, u, r) > OPTIN else "dr_le48k")
        taken.add("dr_sliced" if THREADS // dr_microtiles(dk, u, r) > 1 else "dr_one_slice")
    if hw > LAM_CHUNK_M:
        taken.add("content_mchunks" if r else "global_mchunks")
    if dv > LAM_CHUNK_V:
        taken.add("content_v0chunks")
    if stream_grid(B * hw * cdiv(dv, 8), sms)[1]:
        taken.add("dv_capped")
    if stream_grid(B * hw * dk * round_up(dv, 8) // 8, sms)[1]:
        taken.add("dlp_capped")
    return frozenset(taken)


def lam_case_geom(case) -> Tuple[int, ...]:
    """(B, H, W, dk, u, heads, dv, r, Cqp, Ckp, Cvp, Cop) of a LAM_CASES row: each width is its logical channels rounded
    up to 8, plus the row's extra padding."""
    name, B, H, W, dk, u, heads, dv, r, extra, want = case
    return (B, H, W, dk, u, heads, dv, r, round_up(heads * dk, 8) + extra, round_up(dk * u, 8) + extra,
            round_up(dv * u, 8) + extra, round_up(heads * dv, 8) + extra)


# (name, B, H, W, dk, u, heads, dv, r, extra padding channels, paths it witnesses at every SM count from 100 to 144):
# every (dk, u) local and global, so every instantiation of the output, dq and dv kernels runs
LAM_CASES = [
    ("dk8u1_r1", 2, 9, 11, 8, 1, 1, 8, 1, 0, {"outdq_dk8_u1_local", "dv_dk8_u1_local", "dr_le48k", "dr_sliced"}),
    ("dk8u2_r5_pad", 2, 11, 9, 8, 2, 3, 12, 5, 8, {"outdq_dk8_u2_local", "dv_dk8_u2_local", "y_scalar"}),
    ("dk8u3_r7", 1, 13, 10, 8, 3, 2, 5, 7, 0, {"outdq_dk8_u3_local", "dv_dk8_u3_local"}),
    ("dk8u4_r23", 1, 10, 12, 8, 4, 2, 8, 23, 0, {"outdq_dk8_u4_local", "dv_dk8_u4_local", "halo_gt48k"}),
    ("dk16u1_r3", 2, 9, 9, 16, 1, 4, 24, 3, 0, {"outdq_dk16_u1_local", "dv_dk16_u1_local", "halo_le48k", "y_vec"}),
    ("dk16u2_r9_mchunks", 1, 17, 16, 16, 2, 2, 16, 9, 0, {"outdq_dk16_u2_local", "dv_dk16_u2_local",
                                                         "content_mchunks"}),
    ("dk16u3_r11_pad", 2, 8, 8, 16, 3, 1, 7, 11, 8, {"outdq_dk16_u3_local", "dv_dk16_u3_local"}),
    ("dk16u4_r21", 1, 12, 9, 16, 4, 2, 6, 21, 0, {"outdq_dk16_u4_local", "dv_dk16_u4_local", "halo_gt48k"}),
    ("dk32u1_r3_h8", 2, 7, 13, 32, 1, 8, 8, 3, 0, {"outdq_dk32_u1_local", "dv_dk32_u1_local", "dr_gt48k"}),
    ("dk32u2_r5_v0chunks", 1, 9, 9, 32, 2, 2, 136, 5, 0, {"outdq_dk32_u2_local", "dv_dk32_u2_local",
                                                          "content_v0chunks"}),
    ("dk32u3_r13", 1, 10, 10, 32, 3, 1, 10, 13, 0, {"outdq_dk32_u3_local", "dv_dk32_u3_local"}),
    ("dk32u4_r23", 1, 11, 12, 32, 4, 3, 16, 23, 0, {"outdq_dk32_u4_local", "dv_dk32_u4_local", "dr_one_slice",
                                                    "halo_gt48k"}),
    ("dk8u1_global", 2, 5, 6, 8, 1, 4, 8, 0, 0, {"outdq_dk8_u1_global", "dv_dk8_u1_global"}),
    ("dk8u2_global_mchunks_pad", 1, 17, 16, 8, 2, 2, 12, 0, 8, {"dv_dk8_u2_global", "global_mchunks"}),
    ("dk8u3_global", 2, 4, 7, 8, 3, 1, 5, 0, 0, {"dv_dk8_u3_global"}),
    ("dk8u4_global", 1, 6, 6, 8, 4, 3, 16, 0, 0, {"dv_dk8_u4_global"}),
    ("dk16u1_global", 2, 5, 5, 16, 1, 2, 9, 0, 0, {"outdq_dk16_u1_global", "dv_dk16_u1_global"}),
    ("dk16u2_global_v0chunks", 1, 7, 5, 16, 2, 1, 130, 0, 0, {"dv_dk16_u2_global", "content_v0chunks"}),
    ("dk16u3_global_pad", 2, 3, 9, 16, 3, 2, 8, 0, 8, {"dv_dk16_u3_global"}),
    ("dk16u4_global", 1, 6, 4, 16, 4, 4, 4, 0, 0, {"dv_dk16_u4_global"}),
    ("dk32u1_global", 2, 5, 6, 32, 1, 1, 16, 0, 0, {"outdq_dk32_u1_global", "dv_dk32_u1_global"}),
    ("dk32u2_global", 1, 4, 4, 32, 2, 2, 3, 0, 0, {"dv_dk32_u2_global"}),
    ("dk32u3_global", 2, 6, 5, 32, 3, 3, 8, 0, 0, {"dv_dk32_u3_global"}),
    ("dk32u4_global", 1, 5, 7, 32, 4, 1, 24, 0, 0, {"dv_dk32_u4_global"}),
    ("capped", 16, 48, 48, 16, 1, 1, 136, 3, 0, {"dv_capped", "dlp_capped", "content_mchunks", "content_v0chunks"}),
]


# ---------------------------------------------------------------------------------------------------------------------
# refusal tables: geometries the C ABI must refuse (or accept), each a change to a valid base geometry
# ---------------------------------------------------------------------------------------------------------------------
LAM_BASE = dict(B=2, H=9, W=7, dk=16, u=2, heads=2, dv=12, r=5, Cqp=32, Ckp=32, Cvp=24, Cop=24)
LAM_KEYS = ("B", "H", "W", "dk", "u", "heads", "dv", "r", "Cqp", "Ckp", "Cvp", "Cop")
INV_BASE = dict(N=2, H=9, W=7, C=16, Cp=16, Kp=48, K=3, G=4, stride=1, pad=1, dil=1)
INV_KEYS = ("N", "H", "W", "C", "Cp", "Kp", "K", "G", "stride", "pad", "dil")

# (name, changes to LAM_BASE, expected refusal): the rows at a 2^31 limit come with the shape one step below it
LAM_ROWS = [
    ("B0", dict(B=0), True), ("H0", dict(H=0), True), ("W_negative", dict(W=-3), True), ("dk12", dict(dk=12), True),
    ("dk64", dict(dk=64, Cqp=128, Ckp=128), True), ("u0", dict(u=0), True), ("u5", dict(u=5, Ckp=80, Cvp=64), True),
    ("heads0", dict(heads=0), True), ("heads9", dict(heads=9, Cqp=144, Cop=112), True), ("dv0", dict(dv=0), True),
    ("r_negative", dict(r=-1), True), ("r_even", dict(r=4), True), ("r25", dict(r=25), True),
    ("Cqp_narrow", dict(Cqp=24), True), ("Cqp_unaligned", dict(Cqp=36), True), ("Ckp_narrow", dict(Ckp=24), True),
    ("Ckp_unaligned", dict(Ckp=36), True), ("Cvp_narrow", dict(Cvp=16), True), ("Cvp_unaligned", dict(Cvp=28), True),
    ("Cop_narrow", dict(Cop=16), True), ("Cop_unaligned", dict(Cop=28), True),
    ("B_over_grid", dict(B=65536, H=1, W=1), True), ("B_at_grid", dict(B=65535, H=1, W=1), False),
    # B * H * W * max(C): 2 * 2^30 = 2^31 at the limit, 2 * (2^30 - 8) below it
    ("channels_at_limit", dict(B=1, H=1, W=2, Cqp=1 << 30), True),
    ("channels_below_limit", dict(B=1, H=1, W=2, Cqp=(1 << 30) - 8), False),
    # B * H * W * dk * round_up(dv, 8): 2^25 positions * 8 * 8 = 2^31 at the limit
    ("dlp_at_limit", dict(B=1, H=1 << 12, W=1 << 13, dk=8, u=1, heads=1, dv=8, r=1, Cqp=8, Ckp=8, Cvp=8, Cop=8), True),
    ("dlp_below_limit", dict(B=1, H=1, W=(1 << 25) - 1, dk=8, u=1, heads=1, dv=8, r=1, Cqp=8, Ckp=8, Cvp=8, Cop=8),
     False),
    ("dlp_at_limit_by_dv", dict(B=1, H=1, W=1 << 21, dk=16, u=1, heads=1, dv=57, r=0, Cqp=16, Ckp=16, Cvp=64,
                                Cop=64), True),
    ("dlp_below_limit_by_dv", dict(B=1, H=1, W=(1 << 21) - 1, dk=16, u=1, heads=1, dv=57, r=0, Cqp=16, Ckp=16, Cvp=64,
                                   Cop=64), False),
]

# (name, changes to INV_BASE, expected refusal)
INV_ROWS = [
    ("N0", dict(N=0), True), ("C0", dict(C=0), True), ("G0", dict(G=0), True), ("C_not_multiple_of_G", dict(G=5), True),
    ("Cp_below_C", dict(Cp=8), True), ("Cp_unaligned", dict(C=12, G=4, Cp=12), True), ("Kp_below", dict(Kp=35), True),
    ("K2", dict(K=2, Kp=16), True), ("K9", dict(K=9, Kp=324), True), ("stride0", dict(stride=0), True),
    ("N_over_grid", dict(N=65536, H=3, W=3), True), ("N_at_grid", dict(N=65535, H=3, W=3), False),
    # N * H * W * Cp: 2^28 * 8 = 2^31 at the limit
    ("x_at_limit", dict(N=1, H=1, W=1 << 28, C=8, Cp=8, G=1, K=1, Kp=8, pad=0), True),
    ("x_below_limit", dict(N=1, H=1, W=(1 << 28) - 1, C=8, Cp=8, G=1, K=1, Kp=8, pad=0), False),
    # N * Ho * Wo * max(Cp, Kp): one output pixel and Kp = 2^31 - 1 is at the limit
    ("ker_at_limit", dict(N=1, H=1, W=1, C=8, Cp=8, G=1, K=1, Kp=INDEX_LIMIT, pad=0), True),
    ("ker_below_limit", dict(N=1, H=1, W=1, C=8, Cp=8, G=1, K=1, Kp=INDEX_LIMIT - 1, pad=0), False),
]

# (name, changes to LAM_BASE, NULL operands): lam_pointer_refused names the entry points that must refuse
LAM_POINTER_ROWS = [
    ("local_no_Rt", {}, ["Rt"]),
    ("local_no_dlp", {}, ["dlp"]),
    ("local_no_lp_needed", {}, ["lp", "dvpos"]),
    ("global_no_lp", dict(r=0), ["lp"]),
    ("global_no_dvpos", dict(r=0), ["dvpos"]),
    ("global_no_Rt_needed", dict(r=0), ["Rt", "dlp"]),
]

# ---------------------------------------------------------------------------------------------------------------------
# fp64 oracles
# ---------------------------------------------------------------------------------------------------------------------
def inv_oracle(x64, ker64, dy64, K, G, stride, pad, dil):
    """(y, dx, dker) of the involution and the same on absolute values, all NHWC: x [N,H,W,C], ker [N,Ho,Wo,G*K^2],
    dy [N,Ho,Wo,C], fp64. dx and dker are autograd of the reference restatement in tests/_involution_oracle.py."""
    from _involution_oracle import involution2d

    def run(x, k, d):
        xs = x.permute(0, 3, 1, 2).detach().requires_grad_(True)
        ks = k.permute(0, 3, 1, 2).detach().requires_grad_(True)
        y = involution2d(xs, ks, K, stride, pad, dil, G)
        y.backward(d.permute(0, 3, 1, 2))
        nhwc = lambda t: t.detach().permute(0, 2, 3, 1)   # noqa: E731
        return nhwc(y), nhwc(xs.grad), nhwc(ks.grad)

    return run(x64, ker64, dy64), run(x64.abs(), ker64.abs(), dy64.abs())


def _img(t, H, W):
    """[B, HW, ...] -> [B, H, W, ...]"""
    return t.reshape(t.shape[0], H, W, *t.shape[2:])


def _windows(v5, r):
    """The r*r zero-padded windows of v5 [B, H, W, ...]: yields (i, j, window [B, HW, ...]) with window[b, (y, x)] =
    v5[b, y + i - r//2, x + j - r//2] (zero outside the image)."""
    b, h, w = v5.shape[:3]
    rest = v5.shape[3:]
    p = r // 2
    flat = v5.reshape(b, h, w, -1).permute(0, 3, 1, 2)
    vp = TF.pad(flat, (p, p, p, p)).permute(0, 2, 3, 1)
    for i in range(r):
        for j in range(r):
            yield i, j, vp[:, i:i + h, j:j + w].reshape(b, h * w, *rest)


def lam_stats(k64, dk, u):
    """(row max, sum over the finite keys of exp(x - max)) of each key row k*u+u' over the positions: k [B, HW, dk*u]
    -> two [B, dk*u]. A row whose keys are all -inf gives (-inf, 0); torch.softmax gives that row NaN."""
    mx = k64.amax(1)
    e = torch.where(k64 == -float("inf"), torch.zeros_like(k64), torch.exp(k64 - mx[:, None]))
    return mx, e.sum(1)


def lam_sigma(k64, mx, sm, dk, u):
    """sigma [B, dk, u, HW] = exp(k - max) / sum with the statistics the kernels are given (NaN for a row of -inf)."""
    b, hw, _ = k64.shape
    return (torch.exp(k64 - mx[:, None]) / sm[:, None]).permute(0, 2, 1).reshape(b, dk, u, hw)


def lam_lc(sig, v64, dv, u):
    """(lc [B, dk, dv], the same on |v|) = sum_{m,u'} sigma * v[m, v*u+u']."""
    vv = v64.reshape(v64.shape[0], v64.shape[1], dv, u)
    return torch.einsum("bkum,bmvu->bkv", sig, vv), torch.einsum("bkum,bmvu->bkv", sig.abs(), vv.abs())


def lam_y(q64, v64, R64, lc64, lp64, H, W, dk, u, heads, dv, r):
    """(y [B, HW, heads*dv], the same on absolute values) of the output kernel: sum_k q (lc + lp), with lp the local
    correlation of v with R [dk, u, r, r] or the given global lp [B, HW, dk, dv]."""
    b, hw, _ = q64.shape
    qh = q64.reshape(b, hw, heads, dk)
    outs = []
    for sgn in (lambda t: t, torch.abs):
        qs = sgn(qh)
        y = torch.einsum("bnhk,bkv->bnhv", qs, sgn(lc64))
        if r:
            v5 = _img(sgn(v64).reshape(b, hw, dv, u), H, W)
            Rs = sgn(R64)
            for i, j, win in _windows(v5, r):
                qr = torch.einsum("bnhk,ku->bnhu", qs, Rs[:, :, i, j])
                y = y + torch.einsum("bnhu,bnvu->bnhv", qr, win)
        else:
            y = y + torch.einsum("bnhk,bnkv->bnhv", qs, sgn(lp64))
        outs.append(y.reshape(b, hw, heads * dv))
    return tuple(outs)


def lam_dq(dy64, v64, R64, lc64, lp64, H, W, dk, u, heads, dv, r):
    """(dq [B, HW, heads*dk], the same on absolute values) = sum_v dy[h, v] (lc[k, v] + lp[k, v, n])."""
    b, hw, _ = dy64.shape
    gh = dy64.reshape(b, hw, heads, dv)
    outs = []
    for sgn in (lambda t: t, torch.abs):
        gs = sgn(gh)
        dq = torch.einsum("bnhv,bkv->bnhk", gs, sgn(lc64))
        if r:
            v5 = _img(sgn(v64).reshape(b, hw, dv, u), H, W)
            Rs = sgn(R64)
            for i, j, win in _windows(v5, r):
                d = torch.einsum("bnhv,bnvu->bnhu", gs, win)
                dq = dq + torch.einsum("bnhu,ku->bnhk", d, Rs[:, :, i, j])
        else:
            dq = dq + torch.einsum("bnhv,bnkv->bnhk", gs, sgn(lp64))
        outs.append(dq.reshape(b, hw, heads * dk))
    return tuple(outs)


def lam_dlc(q64, dy64, dk, heads, dv):
    """(dlc [B, dk, dv], the same on absolute values) = sum_{n,h} q[n, h*dk+k] dy[n, h*dv+v]."""
    b, hw, _ = q64.shape
    qh, gh = q64.reshape(b, hw, heads, dk), dy64.reshape(b, hw, heads, dv)
    return torch.einsum("bnhk,bnhv->bkv", qh, gh), torch.einsum("bnhk,bnhv->bkv", qh.abs(), gh.abs())


def lam_dk(k64, v64, mx, sm, dlc64, dlc_abs, dk, u, dv):
    """(dk [B, HW, dk*u], its sum |terms|) of the backward content kernel: sigma (dsigma - sum_m sigma dsigma) with
    dsigma[m] = sum_v dlc[k, v] v[m, v*u+u'] and sigma from the given statistics; the terms bound takes dlc over |q| |dy|
    (``dlc_abs``): sigma (a + sum_m sigma a) with a = sum_v |dlc| |v|."""
    b, hw, _ = k64.shape
    sig = lam_sigma(k64, mx, sm, dk, u)
    vv = v64.reshape(b, hw, dv, u)
    ds = torch.einsum("bkv,bmvu->bkum", dlc64, vv)
    g = sig * (ds - (sig * ds).sum(-1, keepdim=True))
    a = torch.einsum("bkv,bmvu->bkum", dlc_abs, vv.abs())
    ga = sig * (a + (sig * a).sum(-1, keepdim=True))
    flat = lambda t: t.reshape(b, dk * u, hw).permute(0, 2, 1)   # noqa: E731
    return flat(g), flat(ga)


def lam_dlp(q64, dy64, dk, heads, dv):
    """(dlp [B, HW, dk, dv], the same on absolute values) = sum_h q[n, h*dk+k] dy[n, h*dv+v]."""
    b, hw, _ = q64.shape
    qh, gh = q64.reshape(b, hw, heads, dk), dy64.reshape(b, hw, heads, dv)
    return torch.einsum("bnhk,bnhv->bnkv", qh, gh), torch.einsum("bnhk,bnhv->bnkv", qh.abs(), gh.abs())


def lam_dv(k64, mx, sm, dlc64, dlp64, R64, dvpos64, H, W, dk, u, dv, r):
    """(dv [B, HW, dv*u], the same on absolute values) of the dv kernel: sum_k sigma[u', k, m] dlc[k, v], plus the
    correlation of dlp [B, HW, dk, dv] with the flipped R (local) or the given dvpos [B, HW, dv*u] (global)."""
    b, hw, _ = k64.shape
    sig = lam_sigma(k64, mx, sm, dk, u)
    outs = []
    for sgn in (lambda t: t, torch.abs):
        g = torch.einsum("bkum,bkv->bmvu", sig.abs() if sgn is torch.abs else sig, sgn(dlc64))
        if r:
            # dv[m] += sum_{k,(i,j)} R[k,u',i,j] dlp[m - (i, j) + r//2]: the windows of dlp taken at tap (r-1-i, r-1-j)
            Rs = sgn(R64)
            d5 = _img(sgn(dlp64), H, W)
            for i, j, win in _windows(d5, r):
                g = g + torch.einsum("ku,bnkv->bnvu", Rs[:, :, r - 1 - i, r - 1 - j], win)
            outs.append(g.reshape(b, hw, dv * u))
        else:
            outs.append(g.reshape(b, hw, dv * u) + sgn(dvpos64))
    return tuple(outs)


def lam_dr_partials(dlp64, v64, H, W, dk, u, dv, r):
    """(part [B, dk, u, r*r], the same on absolute values): part[b,k,u',i*r+j] = sum_n sum_v dlp[b,n,k,v] *
    v[b, n + (i, j) - r//2, v*u+u']."""
    b, hw = dlp64.shape[:2]
    v5 = _img(v64.reshape(b, hw, dv, u), H, W)
    part = torch.zeros(b, dk, u, r * r, dtype=dlp64.dtype, device=dlp64.device)
    pa = torch.zeros_like(part)
    for i, j, win in _windows(v5, r):
        part[..., i * r + j] = torch.einsum("bnkv,bnvu->bku", dlp64, win)
    for i, j, win in _windows(v5.abs(), r):
        pa[..., i * r + j] = torch.einsum("bnkv,bnvu->bku", dlp64.abs(), win)
    return part, pa
