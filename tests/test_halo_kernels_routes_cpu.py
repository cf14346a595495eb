"""The launch routes and refusals of the involution and lambda entry points, without a GPU.

The case tables of tests/_halo_kernels_oracle.py must reach every path of both families (tests/
test_gpu_halo_kernels_bounds.py runs each table row) at every SM count from 100 to 144, and the dR partial kernel's
microtiles must fit its 256 threads for every accepted (dim_k, dim_u, r). Every refusal the oracle predicts must come
back as cudaErrorInvalidValue through the C ABI, from every entry point it applies to, including the shapes at each
2^31 index limit; the accepted shapes one step below each limit must get past the checks. The calls take aligned dummy
pointers in a child process that sees no CUDA device, so nothing can be written anywhere: an accepted shape fails for
want of a device instead."""
import json
import os
import subprocess
import sys
from pathlib import Path

import pytest

import _halo_kernels_oracle as O

ROOT = Path(__file__).resolve().parents[1]
INVALID_VALUE = 1           # cudaErrorInvalidValue
SMS = range(100, 145)


def test_involution_case_routes():
    reached = set()
    for sms in SMS:
        for case in O.INV_CASES:
            geom = O.inv_case_geom(case)
            assert not O.inv_refused(*geom), case[0]
            got = O.route_involution(*geom, sms)
            assert case[-1] <= got, (case[0], sms, sorted(case[-1] - got))
            reached |= got
        assert reached == set(O.INV_PATHS), (sms, sorted(set(O.INV_PATHS) - reached))


def test_lambda_case_routes():
    reached = set()
    for sms in SMS:
        for case in O.LAM_CASES:
            geom = O.lam_case_geom(case)
            assert not O.lam_refused(*geom), case[0]
            got = O.route_lambda(*geom[:8], sms)
            assert case[-1] <= got, (case[0], sms, sorted(case[-1] - got))
            reached |= got
        assert reached == set(O.LAM_PATHS), (sms, sorted(set(O.LAM_PATHS) - reached))


def test_capped_cases_run_their_grid_stride_loops_twice():
    """The capped rows give some threads a second trip of every grid-stride loop they are meant to cap; every other row
    gives no thread one."""
    for sms in SMS:
        for case in O.INV_CASES:
            n, h, w, c, cp, kp, k, g, s, p, d = O.inv_case_geom(case)
            ho, wo = O.window_out(h, k, s, p, d), O.window_out(w, k, s, p, d)
            capped = "capped" in case[0]
            assert O.stream_grid(n * h * w * cp // 8, sms)[1] == capped
            if "bwk_generic" in case[-1]:
                assert O.stream_grid(n * ho * wo * kp, sms)[1] == capped
        for case in O.LAM_CASES:
            b, h, w, dk, u, heads, dv, r = O.lam_case_geom(case)[:8]
            capped = case[0] == "capped"
            assert O.stream_grid(b * h * w * O.cdiv(dv, 8), sms)[1] == capped
            assert O.stream_grid(b * h * w * dk * O.round_up(dv, 8) // 8, sms)[1] == capped


def test_halo_above_48k_needs_u4_and_r21():
    """allow_smem raises the output and dq kernels' limit only for a halo box above 48 KiB: dim_u = 4 with r = 21 or
    23 and nothing else the checks accept."""
    above = {(u, r) for u in (1, 2, 3, 4) for r in range(1, O.LAM_MAX_R + 1, 2) if O.halo_smem(r, u) > O.OPTIN}
    assert above == {(4, 21), (4, 23)}


def test_dr_microtiles_fit_the_block():
    for dk in O.LAM_DK:
        for u in (1, 2, 3, 4):
            for r in range(1, O.LAM_MAX_R + 1, 2):
                mt = O.dr_microtiles(dk, u, r)
                assert mt <= O.THREADS, (dk, u, r, mt)
                # the slices' partial sums reuse the dlp stage: it must hold slices * mt * 16 floats
                assert (O.THREADS // mt) * mt * 16 * 4 <= O.dr_smem_bytes(dk, u, r)
    assert O.dr_microtiles(32, 4, 23) == 192


# ---------------------------------------------------------------------------------------------------------------------
# refusals through the C ABI
# ---------------------------------------------------------------------------------------------------------------------
_CHILD = """
import ctypes, json, sys
sys.path.insert(0, sys.argv[1])
from holocron_b200._lib import lib
L = lib()
D = 256                                      # 16-byte aligned and never dereferenced

def p(name, null):
    return None if name in null else D

def lam(g, null):
    geom = [g[k] for k in %r]
    return {
        "content_fwd": L.hb_lambda_content_fwd_bf16(D, D, D, D, *geom, None),
        "out_fwd": L.hb_lambda_out_fwd_bf16(D, D, p("Rt", null), D, p("lp", null), D, *geom, None),
        "bwd_content": L.hb_lambda_bwd_content_bf16(D, D, D, D, D, D, D, *geom, None),
        "dlp": L.hb_lambda_dlp_bf16(D, D, D, *geom, None),
        "bwd_q": L.hb_lambda_bwd_q_bf16(D, D, p("Rt", null), D, p("lp", null), D, *geom, None),
        "bwd_v": L.hb_lambda_bwd_v_bf16(D, D, D, p("dlp", null), p("Rt", null), p("dvpos", null), D, *geom, None),
        "bwd_r": L.hb_lambda_bwd_r_bf16(p("dlp", null), D, D, D, *geom, None),
    }

def inv(g):
    geom = [g[k] for k in %r]
    return {name: getattr(L, "hb_involution_" + name + "_bf16")(D, D, D, *geom, None)
            for name in ("fwd", "bwd_data", "bwd_kernel")}

rows = json.loads(sys.argv[2])
res = {"lam": {n: lam(g, set(null)) for n, g, null in rows["lam"]}, "inv": {n: inv(g) for n, g in rows["inv"]}}
print("RESULT " + json.dumps(res))
""" % (O.LAM_KEYS, O.INV_KEYS)


def _lam_geom(changes):
    return {**O.LAM_BASE, **changes}


def _inv_geom(changes):
    return {**O.INV_BASE, **changes}


@pytest.fixture(scope="module")
def abi_results():
    rows = {"lam": [(n, _lam_geom(c), []) for n, c, _ in O.LAM_ROWS]
                   + [(n, _lam_geom(c), null) for n, c, null in O.LAM_POINTER_ROWS]
                   + [("base", O.LAM_BASE, []), ("base_global", _lam_geom(dict(r=0)), [])],
            "inv": [(n, _inv_geom(c)) for n, c, _ in O.INV_ROWS] + [("base", O.INV_BASE)]}
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    proc = subprocess.run([sys.executable, "-c", _CHILD, str(ROOT), json.dumps(rows)], env=env, capture_output=True,
                          text=True, timeout=300)
    assert proc.returncode == 0, (f"the child exited with {proc.returncode} (a negative code is the signal that killed "
                                  f"it):\n{proc.stdout[-2000:]}\n{proc.stderr[-2000:]}")
    line = next(ln for ln in proc.stdout.splitlines() if ln.startswith("RESULT "))
    return json.loads(line[len("RESULT "):])


def _expect(rc, refused, what):
    if refused:
        assert rc == INVALID_VALUE, f"{what}: returned {rc}, the checks should refuse it"
    else:
        # past the checks: the launch fails for want of a device
        assert rc not in (0, INVALID_VALUE), f"{what}: returned {rc}, the checks should accept it"


def test_lambda_abi_refusals(abi_results):
    got = abi_results["lam"]
    for name, changes, want in O.LAM_ROWS:
        g = _lam_geom(changes)
        refused = O.lam_refused(*(g[k] for k in O.LAM_KEYS))
        assert refused == want, f"{name}: the oracle predicts refused={refused}"
        for entry in O.LAM_ENTRIES:
            # bwd_r has no global variant; every row here is local unless it is refused by the shape checks
            _expect(got[name][entry], refused or O.lam_pointer_refused(entry, g["r"], frozenset()), f"{name} {entry}")
    for name, changes, null in O.LAM_POINTER_ROWS + [("base", {}, []), ("base_global", dict(r=0), [])]:
        g = _lam_geom(changes)
        assert not O.lam_refused(*(g[k] for k in O.LAM_KEYS))
        for entry in O.LAM_ENTRIES:
            _expect(got[name][entry], O.lam_pointer_refused(entry, g["r"], frozenset(null)), f"{name} {entry}")
    # each pointer rule refuses something, and lets the operand of the other variant be NULL
    assert got["local_no_Rt"]["out_fwd"] == got["global_no_lp"]["bwd_q"] == got["global_no_dvpos"]["bwd_v"] == 1
    assert got["local_no_dlp"]["bwd_v"] == got["base_global"]["bwd_r"] == 1
    assert got["global_no_Rt_needed"]["out_fwd"] != 1 and got["local_no_lp_needed"]["bwd_v"] != 1


def test_involution_abi_refusals(abi_results):
    got = abi_results["inv"]
    for name, changes, want in O.INV_ROWS + [("base", {}, False)]:
        g = _inv_geom(changes)
        refused = O.inv_refused(*(g[k] for k in O.INV_KEYS))
        assert refused == want, f"{name}: the oracle predicts refused={refused}"
        for entry, rc in got[name].items():
            _expect(rc, refused, f"{name} {entry}")
