"""Coverage of the depth-wise convolution cases (tests/_dwconv_cases.py) and the geometry checks of its C ABI, without a
GPU.

The routing mirror must send the cases through every kernel instantiation of csrc/dwconv.cu at the SM counts of both
H100 variants, and the cases tagged ``wrap`` must give every thread of every launch a second grid-stride iteration.
The entry points must refuse malformed geometry with cudaErrorInvalidValue before they launch or query a device: they
are called with null pointers in a child process that sees no CUDA device, so nothing can be written anywhere, and a
host-side crash (stride 0 divides by zero) fails the test instead of the run."""
import json
import os
import subprocess
import sys
from pathlib import Path

import pytest

import _dwconv_cases as D

ROOT = Path(__file__).resolve().parents[1]
SMS = [132, 114]            # H100 SXM, H100 PCIe
INVALID_VALUE = 1           # cudaErrorInvalidValue


@pytest.mark.parametrize("sms", SMS)
def test_every_instantiation_is_reached(sms):
    taken = {}
    for name, cs in D.CASES.items():
        for kern in D.kernels_taken(cs, sms):
            taken.setdefault(kern, name)
    missing = [k for k in D.INSTANTIATIONS + (D.FINALIZE_UNROLLED,) if k not in taken]
    assert not missing, f"not reached at {sms} SMs: {missing}"
    assert set(taken) <= set(D.INSTANTIATIONS + (D.FINALIZE_UNROLLED,)), set(taken)


@pytest.mark.parametrize("sms", SMS)
def test_wrap_cases_wrap(sms):
    wraps = [n for n, cs in D.CASES.items() if cs.wrap]
    assert wraps
    for name in wraps:
        for d, launch in D.route(D.CASES[name], sms).items():
            assert launch.min_iters >= 2, D.describe(name, sms)


def test_quad_switch_reaches_the_one_output_kernels():
    taken = {k for n in D.QUAD_CASES for k in D.kernels_taken(D.CASES[n], 132, quad=False)}
    assert {"dw3x3_kernel<false,1>", "dw3x3_kernel<false,2>", "dw3x3_kernel<true,1>", "dw3x3_kernel<true,2>",
            "dw_bwd_weight_kernel<3>"} <= taken
    assert not any("quad" in k for k in taken)
    wide = D.route(D.CASES["rexnet_s1_wrap"], 114, quad=False)
    assert all(v.min_iters >= 2 for v in wide.values())


def test_cases_are_valid_shapes():
    for name, cs in D.CASES.items():
        assert cs.c % 8 == 0 and cs.ho >= 1 and cs.wo >= 1, name
        assert cs.k in (1, 3, 5, 7), name


# (N, H, W, C, K, stride, pad): each refused by all three entry points
BAD_GEOMETRY = {
    "stride0": (2, 8, 8, 16, 3, 0, 1),
    "stride_negative": (2, 8, 8, 16, 3, -1, 1),
    "pad_negative": (2, 8, 8, 16, 3, 1, -1),
    "n0": (0, 8, 8, 16, 3, 1, 1),
    "n_negative": (-2, 8, 8, 16, 3, 1, 1),
    "h0": (2, 0, 8, 16, 3, 1, 1),
    "w0": (2, 8, 0, 16, 3, 1, 1),
    "k0": (2, 8, 8, 16, 0, 1, 1),
    "k_negative": (2, 8, 8, 16, -3, 1, 1),
    "c0": (2, 8, 8, 0, 3, 1, 1),
    "c_negative": (2, 8, 8, -16, 3, 1, 1),
    "c_not_multiple_of_8": (2, 8, 8, 12, 3, 1, 1),
    "filter_exceeds_both": (2, 2, 2, 16, 7, 1, 0),             # Ho, Wo < 0: N * Ho * Wo > 0 again
    "filter_exceeds_h": (2, 2, 16, 16, 7, 1, 0),
    "filter_exceeds_w_by_one_stride2": (2, 16, 2, 16, 3, 2, 0),  # (2 - 3) / 2 truncates to 0: Wo = 1 in C
    "filter_exceeds_k5_stride3": (2, 3, 3, 16, 5, 3, 0),
    "output_exceeds_int": (2, 8, 8, 16, 1, 1, 1 << 30),          # Ho = 2^31 + 8 does not fit an int
}

_CHILD = """
import json, sys
sys.path.insert(0, sys.argv[1])
from holocron_b200._lib import lib
L = lib()
out = {}
for name, (n, h, w, c, k, s, p) in json.loads(sys.argv[2]).items():
    out[name] = [L.hb_dwconv_fwd_bf16(None, None, None, None, n, h, w, c, k, s, p, None),
                 L.hb_dwconv_bwd_data_bf16(None, None, None, n, h, w, c, k, s, p, None),
                 L.hb_dwconv_bwd_weight_bf16(None, None, None, None, None, n, h, w, c, k, s, p, None)]
    print(name, out[name], flush=True)
out["wgrad_k9"] = [L.hb_dwconv_bwd_weight_bf16(None, None, None, None, None, 2, 16, 16, 16, 9, 1, 4, None)]
out["scratch"] = [L.hb_dwconv_wgrad_scratch_doubles(16, 0), L.hb_dwconv_wgrad_scratch_doubles(16, -3),
                  L.hb_dwconv_wgrad_scratch_doubles(0, 3), L.hb_dwconv_wgrad_scratch_doubles(12, 3),
                  L.hb_dwconv_wgrad_scratch_doubles(16, 9), L.hb_dwconv_wgrad_scratch_doubles(16, 1 << 30)]
print("RESULT " + json.dumps(out))
"""


def test_abi_refuses_malformed_geometry():
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    proc = subprocess.run([sys.executable, "-c", _CHILD, str(ROOT), json.dumps(BAD_GEOMETRY)], env=env,
                          capture_output=True, text=True, timeout=300)
    assert proc.returncode == 0, (f"the child exited with {proc.returncode} (a negative code is the signal that killed "
                                  f"it):\n{proc.stdout[-2000:]}\n{proc.stderr[-2000:]}")
    line = next(ln for ln in proc.stdout.splitlines() if ln.startswith("RESULT "))
    got = json.loads(line[len("RESULT "):])
    for name in BAD_GEOMETRY:
        assert got[name] == [INVALID_VALUE] * 3, f"{name}: (fwd, dgrad, wgrad) returned {got[name]}"
    assert got["wgrad_k9"] == [INVALID_VALUE]
    assert got["scratch"] == [0] * 6
