"""Coverage of the NormConv2d / Add2d cases (tests/_xcorr_cases.py), the geometry checks of their C ABI and the geometry
errors of ``_XcorrFn``, without a GPU.

The mirror must send the cases through every path of csrc/xcorr.cu, the norm epilogue of csrc/conv_fprop.cu and the
routing of nn/_xcorr.py at the SM counts of both H100 variants. The four entry points must refuse malformed geometry with
cudaErrorInvalidValue before they divide by the stride or touch a device: they are called with dummy pointers in a
child process that sees no CUDA device, so nothing can be written anywhere, and a host-side crash (stride 0 divides by
zero) fails the test instead of the run. A valid geometry in the same child must get past the checks (and then fail for
want of a device), so the refusals are not a blanket error."""
import json
import os
import subprocess
import sys
from pathlib import Path

import pytest
import torch

import _xcorr_cases as D
from holocron_b200.nn import functional as F
from oracle import functional as OF

ROOT = Path(__file__).resolve().parents[1]
SMS = [132, 114]            # H100 SXM, H100 PCIe
INVALID_VALUE = 1           # cudaErrorInvalidValue

FP32_PATHS = {"xcorr_fwd_kernel<false>", "xcorr_fwd_kernel<false>+patch_stats_kernel", "xcorr_fwd_kernel<true>",
              "xcorr_fwd_kernel<true>+patch_stats_kernel",
              "ragged_L", "ragged_Cout", "ragged_K", "K<32", "Cout>32_ragged",
              "wgrad_cps>1", "wgrad_cps=1", "wgrad_several_splits", "wgrad_partial_last_split", "wgrad_straddling_chunk",
              "dgrad_stride1", "dgrad_stride2_uncovered", "dgrad_stride3_uncovered", "dgrad_dilated",
              "rectangular_filter"}
TC_PATHS = {"narrow_whole", "narrow_masked", "wide192", "wide256", "narrow_1x1_at_wide_size", "cin_padded",
            "cout_padded_sliced"}


def fp32_paths(cs, sms):
    f = D.fwd_geo(cs)
    out = set(D.fwd_kernels(cs)) | {f"ragged_{d}" for d in f.ragged}
    if cs.k < D.TK:
        out.add("K<32")
    if cs.cout > D.TC and "Cout" in f.ragged:
        out.add("Cout>32_ragged")
    if cs.kh != cs.kw:
        out.add("rectangular_filter")
    return out | D.wgrad_paths(cs, sms) | D.dgrad_paths(cs)


@pytest.mark.parametrize("sms", SMS)
def test_every_fp32_path_is_reached(sms):
    taken = set().union(*(fp32_paths(cs, sms) for cs in D.CASES.values()))
    assert FP32_PATHS <= taken, f"not reached at {sms} SMs: {sorted(FP32_PATHS - taken)}"


@pytest.mark.parametrize("sms", SMS)
def test_every_tensor_core_tile_kind_is_reached(sms):
    taken = set().union(*(D.tc_paths(cs, sms) for cs in D.TC_CASES.values()))
    assert TC_PATHS <= taken, f"not reached at {sms} SMs: {sorted(TC_PATHS - taken)}"
    assert D.tc_launch(D.TC_CASES["tc_rgb_stem"], sms).cin_p == 8


def test_wgrad_split_geometry_covers_every_row_once():
    for name, cs in D.CASES.items():
        for sms in SMS:
            g = D.wgrad_geo(cs, sms)
            # the splits [z * cps * 32, min(M, (z + 1) * cps * 32)) tile [0, M) and none is empty
            assert (g.splits - 1) * g.cps * D.TL < cs.m <= g.splits * g.cps * D.TL, D.describe(name, sms)
            assert 0 < g.last_rows <= g.cps * D.TL, D.describe(name, sms)


def test_routing():
    rect, sq = D.CASES["rect_3x1"], D.TC_CASES["tc_rgb_stem"]
    assert D.route(sq, 0, True) == "tensor_cores"
    assert D.route(rect, 0, True) == "xcorr_fwd_kernel<false>"        # non-square NormConv2d: fp32 kernel
    assert D.route(sq, 0, False) == "xcorr_fwd_kernel<false>"
    assert D.route(sq, 1, True) == D.route(sq, 1, False) == "xcorr_fwd_kernel<true>"
    for cs in D.TC_CASES.values():
        assert cs.kh == cs.kw


def test_tile_rule_at_forced_grids():
    # one to three CTAs: the wide-tile condition holds on any shape, so Cout = 144 takes one 144-column tile
    cs = D.TC_CASES["tc_masked144"]
    for g in (1, 2, 3):
        assert D.tc_launch(cs, 132, g).bn == 144
    assert D.tc_launch(D.TC_CASES["tc_1x1_cout192"], 132, 1).bn == 96


# (N, Cin, H, W, Cout, kh, kw, stride, pad, dil): each refused by all four entry points (hb_patch_stats_bf16 has no Cout)
BAD_GEOMETRY = {
    "stride0": (2, 8, 9, 9, 16, 3, 3, 0, 1, 1),
    "stride_negative": (2, 8, 9, 9, 16, 3, 3, -1, 1, 1),
    "dil0": (2, 8, 9, 9, 16, 3, 3, 1, 1, 0),
    "dil_negative": (2, 8, 9, 9, 16, 3, 3, 1, 1, -2),
    "pad_negative": (2, 8, 9, 9, 16, 3, 3, 1, -1, 1),
    "n0": (0, 8, 9, 9, 16, 3, 3, 1, 1, 1),
    "n_negative": (-2, 8, 9, 9, 16, 3, 3, 1, 1, 1),
    "cin0": (2, 0, 9, 9, 16, 3, 3, 1, 1, 1),
    "cin_negative": (2, -8, 9, 9, 16, 3, 3, 1, 1, 1),
    "cout0": (2, 8, 9, 9, 0, 3, 3, 1, 1, 1),
    "h0": (2, 8, 0, 9, 16, 3, 3, 1, 1, 1),
    "w_negative": (2, 8, 9, -9, 16, 3, 3, 1, 1, 1),
    "kh0": (2, 8, 9, 9, 16, 0, 3, 1, 1, 1),
    "kw_negative": (2, 8, 9, 9, 16, 3, -3, 1, 1, 1),
    "filter_exceeds_both": (2, 8, 2, 2, 16, 7, 7, 1, 0, 1),           # Ho, Wo < 0: N * Ho * Wo > 0 again
    "filter_exceeds_h": (2, 8, 2, 16, 16, 7, 7, 1, 0, 1),
    "filter_exceeds_w_by_one_stride2": (2, 8, 16, 2, 16, 3, 3, 2, 0, 1),   # (2 - 3) / 2 truncates to 0: Wo = 1 in C
    "dilated_filter_exceeds": (2, 8, 9, 9, 16, 3, 3, 1, 0, 5),
    "pixels_exceed_int": (2, 8, 8, 8, 16, 1, 1, 1, 1 << 15, 1),      # Ho = Wo = 65544: N * Ho * Wo > 2^31 - 1
    "output_exceeds_int": (2, 8, 8, 8, 16, 1, 1, 1, 1 << 30, 1),     # Ho = 2^31 + 8 does not fit an int
    "patch_exceeds_int": (2, 1 << 28, 9, 9, 16, 3, 3, 1, 1, 1),      # Cin * 9 > 2^31 - 1
}
VALID = (2, 8, 9, 9, 16, 3, 3, 1, 1, 1)

_CHILD = """
import ctypes, json, sys
sys.path.insert(0, sys.argv[1])
from holocron_b200._lib import lib
L = lib()
f = ctypes.c_float(1e-5)
dummy = ctypes.c_void_p(256)                 # 16-byte aligned and never dereferenced
out = {}
for name, (n, cin, h, w, co, kh, kw, s, p, d) in json.loads(sys.argv[2]).items():
    out[name] = [L.hb_xcorr2d_fwd(dummy, dummy, None, dummy, dummy, dummy, n, cin, h, w, co, kh, kw, s, p, d, 1, 1, f, None),
                 L.hb_xcorr2d_wgrad(dummy, dummy, dummy, dummy, dummy, dummy, n, cin, h, w, co, kh, kw, s, p, d, 1, 1, f,
                                    None),
                 L.hb_add2d_dgrad(dummy, dummy, dummy, dummy, n, cin, h, w, co, kh, kw, s, p, d, None),
                 L.hb_patch_stats_bf16(dummy, dummy, dummy, dummy, n, h, w, cin, kh, kw, s, p, d,
                                       min(max(cin * kh * kw, 1), 2**31 - 1), f, None)]
    print(name, out[name], flush=True)
n, cin, h, w, co, kh, kw, s, p, d = json.loads(sys.argv[3])
out["fwd_grid_z"] = [L.hb_xcorr2d_fwd(dummy, dummy, None, dummy, dummy, dummy, 65536, cin, h, w, co, kh, kw, s, p, d, 0, 0,
                                      f, None)]
out["k_logical"] = [L.hb_patch_stats_bf16(dummy, dummy, dummy, dummy, n, h, w, cin, kh, kw, s, p, d, k, f, None)
                    for k in (0, -1, cin * kh * kw + 1)]
out["valid"] = [L.hb_xcorr2d_fwd(dummy, dummy, None, dummy, dummy, dummy, n, cin, h, w, co, kh, kw, s, p, d, 1, 0, f, None),
                L.hb_add2d_dgrad(dummy, dummy, dummy, dummy, n, cin, h, w, co, kh, kw, s, p, d, None),
                L.hb_patch_stats_bf16(dummy, dummy, dummy, dummy, n, h, w, cin, kh, kw, s, p, d, cin * kh * kw, f, None)]
print("RESULT " + json.dumps(out))
"""


def test_abi_refuses_malformed_geometry():
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    proc = subprocess.run([sys.executable, "-c", _CHILD, str(ROOT), json.dumps(BAD_GEOMETRY), json.dumps(VALID)], env=env,
                          capture_output=True, text=True, timeout=300)
    assert proc.returncode == 0, (f"the child exited with {proc.returncode} (a negative code is the signal that killed "
                                  f"it):\n{proc.stdout[-2000:]}\n{proc.stderr[-2000:]}")
    line = next(ln for ln in proc.stdout.splitlines() if ln.startswith("RESULT "))
    got = json.loads(line[len("RESULT "):])
    for name in BAD_GEOMETRY:
        want = [INVALID_VALUE] * 4 if name != "cout0" else [INVALID_VALUE] * 3 + got[name][3:]
        assert got[name] == want, f"{name}: (fwd, wgrad, dgrad, patch stats) returned {got[name]}"
    assert got["fwd_grid_z"] == [INVALID_VALUE]
    assert got["k_logical"] == [INVALID_VALUE] * 3
    # past the checks: the launch fails for want of a device, with an error other than the refusal
    assert all(rc not in (0, INVALID_VALUE) for rc in got["valid"]), got["valid"]


# ---------------------------------------------------------------------------------------------------------------------
# _XcorrFn: the geometry errors of F.unfold, which the reference's forward calls
# ---------------------------------------------------------------------------------------------------------------------
BAD_ARGS = {
    "stride0": (dict(stride=0), "stride should be greater than zero"),
    "stride_negative": (dict(stride=-2), "stride should be greater than zero"),
    "dilation0": (dict(dilation=0), "dilation should be greater than zero"),
    "dilation_negative": (dict(dilation=-1), "dilation should be greater than zero"),
    "padding_negative": (dict(padding=-1), "padding should be non-negative"),
    "window_exceeds_input": (dict(dilation=5), "must be at least one"),
}


@pytest.mark.parametrize("name", list(BAD_ARGS))
@pytest.mark.parametrize("op", ["norm_conv2d", "add2d"])
def test_geometry_errors_match_the_oracle(op, name):
    kw, msg = BAD_ARGS[name]
    x, w = torch.rand(2, 3, 9, 9), torch.rand(4, 3, 3, 3)
    with pytest.raises(RuntimeError, match=msg):
        getattr(OF, op)(x, w, None, **kw)
    # the check comes before the device check, so it is the same error on CPU tensors
    with pytest.raises(RuntimeError, match=msg):
        getattr(F, op)(x, w, None, **kw)
