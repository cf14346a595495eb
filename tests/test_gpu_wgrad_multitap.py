"""The generic weight-gradient kernel (conv_wgrad.cu) gives the same dW whatever number of taps a CTA runs together.

A CTA runs up to three units of the same (co tile, ci tile, pixel range) that differ only in tap. Every tap's
accumulators take the same k-steps in the same order as in a one-tap unit, so dW must be bit-identical between
HB_WGRAD_TAPS_PER_UNIT = 1, 2 and 3 on every deterministic path: a single pixel range stored directly, per-range
partials reduced in a fixed order (hb_conv2d_wgrad_bf16 and hb_conv2d_wgrad_acc_bf16), at CTA counts from 1 to 144, so
that there are more tap groups than CTAs and fewer. Filters of 1, 9, 25 and 49 taps (and a 1x5 one) give tap groups of
1, 2 and 3 taps with every remainder; Cin 48 and 192 (64-wide tiles) and Cout not a multiple of 128 reach the partial
tiles. The atomics path (several pixel ranges, no workspace) adds in no fixed order: it is held to the fp64 oracle, as
is one deterministic result per shape (tests/_bounds.py).

The switch is read once per process, so each execution runs in a child process (this file run as a script) that
writes its results to a file."""
import os
import subprocess
import sys
from pathlib import Path

import pytest
import torch
from torch.nn.grad import conv2d_weight

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent
for p in (str(ROOT), str(HERE)):
    if p not in sys.path:
        sys.path.insert(0, p)

from _bounds import FP32_BITS, assert_within  # noqa: E402

pytestmark = pytest.mark.gpu

# name: (N, H, W, Cin, Cout, R, S, stride, pad). None of them is a stride-1 3x3 pad-1 filter, which the row-window kernel
# would take.
CASES = {
    "1x1": (2, 20, 20, 64, 96, 1, 1, 1, 0),
    "3x3_s2_cin48": (8, 33, 33, 48, 32, 3, 3, 2, 1),
    "3x3_p0_cin192_cout200": (8, 12, 12, 192, 200, 3, 3, 1, 0),
    "3x3_s2_cin256_cout136": (4, 14, 14, 256, 136, 3, 3, 2, 1),
    "5x5_p2": (8, 16, 16, 64, 64, 5, 5, 1, 2),
    "7x7_s2_p3": (8, 30, 30, 32, 48, 7, 7, 2, 3),
    "1x5_p0": (8, 10, 14, 128, 64, 1, 5, 1, 0),
}
GRIDS = [0, 1, 2, 3, 7, 33, 144]   # 0 = one CTA per SM
TAPS = ["1", "2", "3"]


def _inputs(name):
    n, h, w, cin, cout, r, s, stride, pad = CASES[name]
    ho, wo = (h + 2 * pad - r) // stride + 1, (w + 2 * pad - s) // stride + 1
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    x = (torch.randn(n, cin, h, w, generator=g)).bfloat16()
    dy = (torch.randn(n, cout, ho, wo, generator=g)).bfloat16()
    base = torch.randn(cout, r, s, cin, generator=g)
    return x, dy, base


def _run_all(out_path):
    """Every case x grid x path with the switch as this process has it -> {key: dW or return code} saved to out_path."""
    from holocron_b200._lib import lib, ptr, stream_ptr
    L = lib()
    res = {}
    for name, (n, h, w, cin, cout, r, s, stride, pad) in CASES.items():
        x, dy, base = _inputs(name)
        xg = x.permute(0, 2, 3, 1).contiguous().cuda()
        dg = dy.permute(0, 2, 3, 1).contiguous().cuda()
        for g in GRIDS:
            wsb = L.hb_conv2d_wgrad_workspace_bytes(n, h, w, cin, cout, r, s, stride, pad, 1, g)
            for path in ("store", "acc", "atomics"):
                ws = torch.empty(max(wsb // 4, 1), device="cuda") if wsb and path != "atomics" else None
                if path == "acc":
                    dw = base.cuda()
                    fn = L.hb_conv2d_wgrad_acc_bf16
                else:
                    dw = torch.full((cout, r, s, cin), float("nan"), device="cuda")
                    fn = L.hb_conv2d_wgrad_bf16
                rc = fn(ptr(xg), ptr(dg), ptr(dw), ptr(ws), wsb if ws is not None else 0, n, h, w, cin, cout, r, s,
                        stride, pad, 1, g, stream_ptr())
                torch.cuda.synchronize()
                res[(name, g, path)] = dw.cpu() if rc == 0 else rc
    torch.save(res, out_path)


@pytest.fixture(scope="module")
def executions(tmp_path_factory):
    out = {}
    tmp = tmp_path_factory.mktemp("wgrad_multitap")
    for taps in TAPS:
        path = tmp / f"taps{taps}.pt"
        env = dict(os.environ, HB_WGRAD_TAPS_PER_UNIT=taps)
        proc = subprocess.run([sys.executable, "-s", __file__, str(path)], env=env, cwd=ROOT, capture_output=True,
                              text=True, timeout=900)
        assert proc.returncode == 0, f"taps {taps}: child failed\n{proc.stdout[-2000:]}\n{proc.stderr[-4000:]}"
        out[taps] = torch.load(path, weights_only=False)
    return out


def _ref(name):
    n, h, w, cin, cout, r, s, stride, pad = CASES[name]
    x, dy, _ = _inputs(name)
    x64, d64 = x.double(), dy.double()
    ref = conv2d_weight(x64, (cout, cin, r, s), d64, stride, pad)
    abs_sum = conv2d_weight(x64.abs(), (cout, cin, r, s), d64.abs(), stride, pad)
    return ref.permute(0, 2, 3, 1), abs_sum.permute(0, 2, 3, 1)


@pytest.mark.parametrize("name", list(CASES))
def test_wgrad_taps_bit_identical(executions, name):
    one = executions["1"]
    _, _, base = _inputs(name)
    for g in GRIDS:
        for path in ("store", "acc"):
            key = (name, g, path)
            ref = one[key]
            for taps in TAPS[1:]:
                got = executions[taps][key]
                if isinstance(ref, int) or isinstance(got, int):
                    # acc on a single pixel range: cudaErrorNotSupported (801) from every execution, dW untouched
                    assert ref == got == 801, (key, taps, ref, got)
                    continue
                assert torch.equal(got, ref), f"{key}: {taps} taps per unit differ from one tap per unit"
            if path == "acc" and not isinstance(ref, int):
                # the reduction adds the same fixed-order sum onto the buffer
                assert torch.equal(ref, base + one[(name, g, "store")]), f"{key}: acc != base + store"


@pytest.mark.parametrize("name", list(CASES))
def test_wgrad_taps_oracle(executions, name):
    ref, abs_sum = _ref(name)
    for taps in TAPS:
        res = executions[taps]
        assert_within(res[(name, 0, "store")], ref, abs_sum, f"{name} taps {taps}", bits=FP32_BITS)
        for g in GRIDS:
            got = res[(name, g, "atomics")]
            assert not isinstance(got, int), (name, g, got)
            assert_within(got, ref, abs_sum, f"{name} taps {taps} grid {g} atomics", bits=FP32_BITS)


if __name__ == "__main__":
    _run_all(sys.argv[1])
