"""The window geometry checks of the convolution, involution and stem im2col entry points of the C ABI, without a GPU.

Every entry point that slides a window computes its output size with one rule (``hb::window_out`` in csrc/common.cuh).
These entry points must refuse a malformed window with cudaErrorInvalidValue (the workspace-size query with 0) before
they divide by the stride or touch a device. In particular a window up to stride - 1 pixels too large, which C's
truncating division alone would give one output row, must be refused as ``F.conv2d`` and ``F.unfold`` refuse it. The
calls take aligned dummy pointers in a child process that sees no CUDA device, so nothing can be written anywhere, and
a host-side crash (stride 0 divides by zero) fails the test instead of the run. A valid geometry in the same child must
get past the checks (and then fail for want of a device), so the refusals are not a blanket error."""
import json
import os
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
INVALID_VALUE = 1           # cudaErrorInvalidValue

# (N, H, W, kh, kw, stride, pad, dil): each refused by every entry point that can express it. Entry points with one
# square K take the rows with kh == kw, those without dilation the rows with dil == 1.
BAD_GEOMETRY = {
    "stride0": (2, 9, 9, 3, 3, 0, 1, 1),
    "stride_negative": (2, 9, 9, 3, 3, -1, 1, 1),
    "dil0": (2, 9, 9, 3, 3, 1, 1, 0),
    "dil_negative": (2, 9, 9, 3, 3, 1, 1, -2),
    "pad_negative": (2, 9, 9, 3, 3, 1, -1, 1),
    "h0": (2, 0, 9, 3, 3, 1, 1, 1),
    "w_negative": (2, 9, -9, 3, 3, 1, 1, 1),
    "kh0": (2, 9, 9, 0, 3, 1, 1, 1),
    "kw_negative": (2, 9, 9, 3, -3, 1, 1, 1),
    "filter_exceeds_both": (2, 2, 2, 7, 7, 1, 0, 1),
    "filter_exceeds_h": (2, 2, 16, 7, 7, 1, 0, 1),
    "filter_exceeds_w_by_one_stride2": (2, 16, 2, 3, 3, 2, 0, 1),   # (2 - 3) / 2 truncates to 0: Wo = 1 in C
    "filter_exceeds_by_two_stride3": (2, 3, 3, 5, 5, 3, 0, 1),      # (3 - 5) / 3 truncates to 0
    "dilated_filter_exceeds": (2, 9, 9, 3, 3, 1, 0, 5),
    "output_exceeds_int": (2, 8, 8, 1, 1, 1, 1 << 30, 1),           # Ho = 2^31 + 8 does not fit an int
}
VALID = (2, 32, 32, 3, 3, 1, 1, 1)

_CHILD = """
import ctypes, json, sys
sys.path.insert(0, sys.argv[1])
from holocron_b200._lib import ConvArgs, lib
L = lib()
dummy = ctypes.c_void_p(256)                 # 16-byte aligned and never dereferenced
CIN, COUT, C = 16, 32, 8

def conv(n, h, w, kh, kw, s, p, d):
    a = ConvArgs(x=256, w=256, y=256, N=n, H=h, W=w, Cin=CIN, Cout=COUT, R=kh, S=kw, stride=s, pad=p, dil=d)
    return [L.hb_conv2d_fused_bf16(ctypes.byref(a), None, None),
            L.hb_conv2d_fprop_bf16(dummy, dummy, dummy, None, None, n, h, w, CIN, COUT, kh, kw, s, p, d, 0, 0, None),
            L.hb_conv2d_wgrad_bf16(dummy, dummy, dummy, dummy, 1 << 30, n, h, w, CIN, COUT, kh, kw, s, p, d, 0, None),
            L.hb_conv2d_wgrad_acc_bf16(dummy, dummy, dummy, dummy, 1 << 30, n, h, w, CIN, COUT, kh, kw, s, p, d, 0, None),
            L.hb_conv2d_wgrad_workspace_bytes(n, h, w, CIN, COUT, kh, kw, s, p, d, 0)]

def involution(n, h, w, k, s, p, d):
    kp = max(8, (k * k + 7) // 8 * 8)
    return [f(dummy, dummy, dummy, n, h, w, C, C, kp, k, 1, s, p, d, None)
            for f in (L.hb_involution_fwd_bf16, L.hb_involution_bwd_data_bf16, L.hb_involution_bwd_kernel_bf16)]

def im2col(n, h, w, kh, kw, s, p):
    kp = max(8, (3 * kh * kw + 7) // 8 * 8)
    return [L.hb_im2col_smallc_bf16(dummy, dummy, n, 3, h, w, kh, kw, s, p, kp, 0, None)]

def run(g):
    n, h, w, kh, kw, s, p, d = g
    out = {"conv": conv(*g)}
    if kh == kw:
        out["involution"] = involution(n, h, w, kh, s, p, d)
    if d == 1:
        out["im2col"] = im2col(n, h, w, kh, kw, s, p)
    return out

res = {}
for name, g in json.loads(sys.argv[2]).items():
    res[name] = run(g)
    print(name, res[name], flush=True)
res["valid"] = run(json.loads(sys.argv[3]))
print("RESULT " + json.dumps(res))
"""


def _run_child(rows):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    proc = subprocess.run([sys.executable, "-c", _CHILD, str(ROOT), json.dumps(rows), json.dumps(VALID)], env=env,
                          capture_output=True, text=True, timeout=300)
    assert proc.returncode == 0, (f"the child exited with {proc.returncode} (a negative code is the signal that killed "
                                  f"it):\n{proc.stdout[-2000:]}\n{proc.stderr[-2000:]}")
    line = next(ln for ln in proc.stdout.splitlines() if ln.startswith("RESULT "))
    return json.loads(line[len("RESULT "):])


def test_abi_refuses_malformed_windows():
    got = _run_child(BAD_GEOMETRY)
    for name in BAD_GEOMETRY:
        # (fused, fprop, wgrad, wgrad_acc, workspace bytes): the size query refuses with 0
        assert got[name]["conv"] == [INVALID_VALUE] * 4 + [0], f"{name}: conv returned {got[name]['conv']}"
        for entry in ("involution", "im2col"):
            if entry in got[name]:
                assert all(rc == INVALID_VALUE for rc in got[name][entry]), f"{name}: {entry} returned {got[name][entry]}"
    # past the checks: the workspace query sizes a workspace and the launchers fail for want of a device
    valid = got["valid"]
    assert valid["conv"][4] > 0, valid
    for rc in valid["conv"][:4] + valid["involution"] + valid["im2col"]:
        assert rc not in (0, INVALID_VALUE), valid
