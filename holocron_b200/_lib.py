"""ctypes binding of the C-ABI CUDA library ``libholocron_b200.so`` (declared in ``include/holocron_b200.h``).

The library is the product: there is no Python/PyTorch fallback for any op it implements. ``lib()`` raises
``RuntimeError`` when the shared object is missing or a kernel launch reports an error.
"""
import ctypes
import os
from pathlib import Path
from typing import Optional

import torch

_LIB_PATH = Path(__file__).resolve().parent / "csrc" / "libholocron_b200.so"
_lib: Optional[ctypes.CDLL] = None

DTYPE_CODE = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}


class HolocronB200Error(RuntimeError):
    pass


def lib_path() -> Path:
    return _LIB_PATH


# Argument signatures of every entry point declared in include/holocron_b200.h
# (p = pointer, i = int, z = size_t, q = long long, f = float). Kept in sync with the header by tests/test_cabi.py.
SIGNATURES = {
    "hb_hard_mish_fwd": "ppzip",
    "hb_hard_mish_bwd": "pppzip",
    "hb_nl_relu_fwd": "ppzfip",
    "hb_nl_relu_bwd": "pppzfip",
    "hb_nl_relu_bwd_from_out": "pppzfip",
    "hb_conv2d_fprop_bf16": "ppppp" + "i" * 12 + "p",
    "hb_conv3x3_accum_bf16": "pppppp" + "i" + "p" + "i" * 6 + "p",
    "hb_conv2d_wgrad_bf16": "ppppz" + "i" * 11 + "p",
    "hb_conv2d_wgrad_workspace_bytes": "i" * 11,
    "hb_repvgg_wgrad_workspace_bytes": "i" * 6,
    "hb_repvgg_wgrad_bf16": "pppppz" + "i" * 6 + "p",
    "hb_conv2d_wgrad_acc_bf16": "ppppz" + "i" * 11 + "p",
    "hb_repvgg_wgrad_acc_bf16": "ppppppz" + "i" * 6 + "p",
    "hb_pack_conv_weights": "ppp" + "i" * 8 + "p",
    "hb_zero_insert_bf16": "pp" + "i" * 7 + "p",
    "hb_pack_conv_weights_multi": "ppip",
    "hb_pack_chunk_elems": "",
    "hb_pack_meta_bytes": "",
    "hb_conv2d_dgrad_s2_bf16": "ppppp" + "i" * 8 + "p",
    "hb_pack_dgrad_s2_weights": "pp" + "i" * 4 + "p",
    "hb_nchw_to_nhwc_pad_bf16": "pp" + "i" * 6 + "p",
    "hb_im2col_smallc_bf16": "pp" + "i" * 10 + "p",
    "hb_conv2d_fused_bf16": "ppp",
    "hb_conv_stat_slots_max": "",
    "hb_patch_stats_bf16": "pppp" + "i" * 10 + "fp",
    "hb_bn_stats_partials_bf16": "piippp",
    "hb_bn_stat_slots_max": "",
    "hb_bn_finalize": "ppppppp" + "pppp" + "iiiiffp",
    "hb_bn_partials_sums": "ppiiiipp",
    "hb_bn_finalize_sums": "p" * 10 + "iiiffp",
    "hb_bn_eval_affine": "ppppfiippppp",
    "hb_bn_act_fwd_bf16": "pppipppp" + "iiifi" + "ppp",
    "hb_bn_bwd_scratch_doubles": "iii",
    "hb_bn_act_bwd_bf16": "ppppi" + "pppppp" + "pppppp" + "pp" + "iiiifiip",
    "hb_bn_act_bwd_reduce_bf16": "ppppi" + "pppppp" + "pppp" + "iiiifip",
    "hb_bn_act_bwd_apply_bf16": "ppppi" + "pppppp" + "ppppp" + "iiifip",
    "hb_dwconv_fwd_bf16": "pppp" + "iiiiiiip",
    "hb_dwconv_bwd_data_bf16": "ppp" + "iiiiiiip",
    "hb_dwconv_wgrad_scratch_doubles": "ii",
    "hb_dwconv_bwd_weight_bf16": "ppppp" + "iiiiiiip",
    "hb_involution_fwd_bf16": "ppp" + "i" * 11 + "p",
    "hb_involution_bwd_data_bf16": "ppp" + "i" * 11 + "p",
    "hb_involution_bwd_kernel_bf16": "ppp" + "i" * 11 + "p",
    "hb_lambda_content_fwd_bf16": "pppp" + "i" * 12 + "p",
    "hb_lambda_out_fwd_bf16": "pppppp" + "i" * 12 + "p",
    "hb_lambda_bwd_content_bf16": "ppppppp" + "i" * 12 + "p",
    "hb_lambda_dlp_bf16": "ppp" + "i" * 12 + "p",
    "hb_lambda_bwd_q_bf16": "pppppp" + "i" * 12 + "p",
    "hb_lambda_bwd_v_bf16": "ppppppp" + "i" * 12 + "p",
    "hb_lambda_bwd_r_bf16": "pppp" + "i" * 12 + "p",
    "hb_gap_fwd_bf16": "ppiiip",
    "hb_gap_bwd_bf16": "ppiiip",
    "hb_blurpool_fwd": "ppp" + "i" * 8 + "p",
    "hb_blurpool_bwd": "ppp" + "i" * 8 + "p",
    "hb_pool_mid_fwd": "ppp" + "i" * 7 + "p",
    "hb_pool_mid_bwd": "ppp" + "i" * 7 + "p",
    "hb_pool_last_fwd": "ppp" + "iiii" + "p",
    "hb_pool_last_bwd": "ppp" + "iiii" + "p",
    "hb_sam_bwd_slots": "iiii",
    "hb_sam_fwd": "ppppp" + "iiii" + "p",
    "hb_sam_bwd": "ppppppp" + "iiii" + "p",
    "hb_triplet_row_block": "iiii",
    "hb_triplet_pool_fwd": "p" * 10 + "i" * 6 + "p",
    "hb_triplet_pool_bwd": "p" * 6 + "i" * 6 + "p",
    "hb_triplet_conv_fwd": "p" * 7 + "i" + "p",
    "hb_triplet_gate": "p" * 5 + "i" + "p",
    "hb_triplet_bn_bwd": "p" * 10 + "i" + "f" + "i" + "p",
    "hb_triplet_conv_bwd": "p" * 8 + "i" + "p",
    "hb_triplet_apply": "p" * 5 + "i" * 6 + "p",
    "hb_triplet_dx": "p" * 11 + "i" * 6 + "p",
    "hb_gate_act_fwd_bf16": "ppp" + "iiii" + "f" + "p",
    "hb_gate_act_bwd_bf16": "ppppp" + "iiii" + "f" + "p",
    "hb_box_pairwise": "pppiiip",
    "hb_box_degenerate": "pipp",
    "hb_box_pairwise_bwd": "pppppiiip",
    "hb_xcorr2d_fwd": "pppppp" + "i" * 12 + "fp",
    "hb_xcorr2d_wgrad": "pppppp" + "i" * 12 + "fp",
    "hb_add2d_dgrad": "pppp" + "i" * 10 + "p",
    "hb_dropblock_mask": "pppiiiifp",
    "hb_dropblock_apply": "ppppiiiiiip",
    "hb_loss_max_partials": "",
    "hb_cls_loss_hard_fwd": "pppppp" + "iiiiiffip",
    "hb_cls_loss_hard_bwd": "pppppp" + "iiiiiffiip",
    "hb_poly_soft_fwd": "pppppp" + "iiiifip",
    "hb_poly_soft_bwd": "ppppp" + "iiiifiip",
    "hb_dice_scratch_doubles": "i",
    "hb_dice_fwd": "pppppp" + "iiqffip",
    "hb_dice_bwd": "pppp" + "iiqip",
    "hb_cce_fwd": "pppppp" + "iiii" + "f" + "ip",
    "hb_cce_bwd": "pppppp" + "iiii" + "f" + "iip",
    "hb_mcl_fwd": "p" * 9 + "iiiii" + "f" + "ip",
    "hb_mcl_bwd": "p" * 10 + "iiiii" + "f" + "iip",
    "hb_optim_chunk_elems": "",
    "hb_adabelief_step": "ppifffffiippp",
    "hb_adamp_step": "ppiifffffifipppp",
    "hb_train_ctl_bytes": "",
    "hb_train_ctl_observe": "ppip",
    "hb_train_ctl_step": "ppiip",
    "hb_train_ctl_tick": "pp",
    "hb_grad_clip_partials_max": "",
    "hb_grad_clip_norm": "pqfppp",
    "hb_lamb_step": "ppiifffffffpp",
    "hb_tadam_step": "ppiifffffifipp" + "p",
    "hb_step_increment": "ppp",
    "hb_adan_step": "ppi" + "ffffff" + "ii" + "ppp",
    "hb_ademamix_step": "ppi" + "fffffff" + "i" + "ppp",
    "hb_lars_step": "ppii" + "ffff" + "ii" + "pp",
    "hb_ralars_step": "ppii" + "fffffff" + "ifi" + "pp",
    "hb_lookahead_sync": "ppi" + "f" + "p",
    "hb_resample_batch": "p" + "i" * 8 + "p",
    "hb_erase_batch": "pp" + "i" * 4 + "p",
    "hb_image_tail_batch": "pp" + "i" * 6 + "p",
    "hb_autoaugment_batch": "pppp" + "i" * 5 + "p",
    "hb_color_jitter_batch": "pppp" + "i" * 6 + "p",
    "hb_box_transform_batch": "ppp" + "iii" + "pppp",
    "hb_assign_iou_batch": "pifpppp",
    "hb_detect_scratch_bytes": "piii",
    "hb_detect": "piii" + "p" * 6,
}
_CTYPE = {"p": ctypes.c_void_p, "i": ctypes.c_int, "z": ctypes.c_size_t, "f": ctypes.c_float, "q": ctypes.c_longlong}


def lib() -> ctypes.CDLL:
    """Returns the loaded C-ABI library, loading it on first use. Fails loudly if it has not been built."""
    global _lib
    if _lib is None:
        if not _LIB_PATH.exists():
            raise HolocronB200Error(
                f"{_LIB_PATH} is missing: build it with `python -m holocron_b200.csrc.build` "
                "(there is no CPU / PyTorch fallback for the holocron_b200 kernels)"
            )
        handle = ctypes.CDLL(os.fspath(_LIB_PATH))
        for name, sig in SIGNATURES.items():
            fn = getattr(handle, name)  # AttributeError here = the library is stale: rebuild it
            fn.argtypes = [_CTYPE[c] for c in sig]
            fn.restype = ctypes.c_size_t if name.endswith(("_bytes", "_doubles")) else ctypes.c_int
        handle.hb_launch_count.argtypes = []
        handle.hb_launch_count.restype = ctypes.c_longlong
        handle.hb_launch_count_reset.argtypes = []
        handle.hb_launch_count_reset.restype = None
        handle.hb_version.argtypes = []
        handle.hb_version.restype = ctypes.c_char_p
        _lib = handle
    return _lib


class ConvArgs(ctypes.Structure):
    """``hb_conv_args`` of include/holocron_b200.h (argument block of hb_conv2d_fused_bf16)."""
    _fields_ = ([(n, ctypes.c_void_p) for n in ("x", "w", "y", "bias", "residual")]
                + [(n, ctypes.c_int) for n in ("N", "H", "W", "Cin", "Cout", "R", "S", "stride", "pad", "dil", "act", "num_ctas")]
                + [("xe", ctypes.c_void_p), ("we", ctypes.c_void_p), ("Ce", ctypes.c_int), ("w2", ctypes.c_void_p),
                   ("y2", ctypes.c_void_p), ("stats", ctypes.c_void_p), ("stats2", ctypes.c_void_p),
                   ("norm_mean", ctypes.c_void_p), ("norm_rstd", ctypes.c_void_p), ("norm_wsum", ctypes.c_void_p)])


def check(rc: int, what: str) -> None:
    if rc != 0:
        raise HolocronB200Error(f"{what} failed with CUDA error code {rc}")


def ptr(t: Optional[torch.Tensor]) -> ctypes.c_void_p:
    return ctypes.c_void_p(0 if t is None else t.data_ptr())


def stream_ptr() -> ctypes.c_void_p:
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def dtype_code(t: torch.Tensor) -> int:
    try:
        return DTYPE_CODE[t.dtype]
    except KeyError:
        raise TypeError(f"unsupported dtype {t.dtype}: expected float32, bfloat16 or float16") from None


def require_cuda(*tensors: torch.Tensor) -> None:
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise HolocronB200Error(
                "holocron_b200 ops run on CUDA tensors only (no CPU fallback); "
                "use the reference implementation / oracle for CPU tensors"
            )
