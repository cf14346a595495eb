"""The oracles of tests/_grad_bucket_oracle.py on the CPU.

The library's two weight-gradient workspace queries, called with an explicit CTA count in a child process that sees no
CUDA device, return exactly the bytes the restated planning predicts over a sweep of shapes and CTA counts 1 .. 144. The
case tables of tests/test_gpu_grad_bucket_bounds.py reach every path for every SM count from 100 to 144. The packing
restatements reproduce small cases written out by hand, edge values included, and the clip oracle follows
``torch.nn.utils.clip_grad_norm_`` on NaN and inf norms. Every route of the bucket test's blocks and models that the
launch planning decides is reached, for every SM count from 100 to 144, by a weight-gradient call the GPU test sees made."""
import itertools
import json
import os
import subprocess
import sys
from pathlib import Path

import pytest
import torch

import _grad_bucket_oracle as O

ROOT = Path(__file__).resolve().parents[1]

_CHILD = """
import json, sys
sys.path.insert(0, sys.argv[1])
from holocron_b200._lib import lib
L = lib()
out = []
for n, h, w, cin, cout, k, stride, pad, ctas in json.loads(sys.argv[2]):
    out.append([int(L.hb_conv2d_wgrad_workspace_bytes(n, h, w, cin, cout, k, k, stride, pad, 1, ctas)),
                int(L.hb_repvgg_wgrad_workspace_bytes(n, h, w, cin, cout, ctas))])
print("RESULT " + json.dumps(out))
"""

SHAPES = [  # (N, H, W, Cin, Cout, k, stride, pad)
    (2, 12, 10, 16, 16, 3, 1, 1), (2, 20, 14, 32, 48, 3, 1, 1), (4, 24, 22, 48, 64, 3, 1, 1), (2, 14, 14, 128, 128, 3, 1, 1),
    (2, 14, 6, 48, 48, 3, 1, 1), (16, 32, 6, 32, 64, 3, 1, 1), (2, 8, 8, 256, 256, 3, 1, 1), (1, 7, 7, 512, 512, 3, 1, 1),
    (2, 33, 31, 16, 32, 3, 2, 1), (8, 56, 56, 64, 64, 3, 1, 1), (8, 28, 127, 64, 96, 3, 1, 1), (2, 9, 126, 16, 16, 3, 1, 1),
    (4, 20, 20, 40, 24, 1, 1, 0), (8, 28, 28, 64, 128, 1, 2, 0), (2, 112, 112, 8, 48, 7, 2, 3), (4, 56, 56, 192, 320, 1, 1, 0),
    (2, 16, 16, 16, 32, 3, 2, 1), (3, 17, 23, 24, 40, 5, 1, 2),
]
CTAS = [1, 2, 3, 7, 12, 31, 64, 100, 114, 132, 144]


def _run_child(rows):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    proc = subprocess.run([sys.executable, "-c", _CHILD, str(ROOT), json.dumps(rows)], env=env, capture_output=True,
                          text=True, timeout=300)
    assert proc.returncode == 0, (f"the child exited with {proc.returncode} (a negative code is the signal that killed "
                                  f"it):\n{proc.stdout[-2000:]}\n{proc.stderr[-2000:]}")
    line = next(ln for ln in proc.stdout.splitlines() if ln.startswith("RESULT "))
    return json.loads(line[len("RESULT "):])


def test_workspace_queries_match_the_restated_planning():
    rows = [list(s) + [c] for s, c in itertools.product(SHAPES, CTAS)]
    rows += [list(c[0]) + [c[1]] for c in O.WGRAD_ACC_CASES.values() if c[1] > 0]
    rows += [list(c[0]) + [3, 1, 1, c[1]] for c in O.REPVGG_ACC_CASES.values() if c[1] > 0]
    got = _run_child(rows)
    bad = []
    for (n, h, w, cin, cout, k, stride, pad, ctas), (g, r) in zip(rows, got):
        want_g = O.route_wgrad(n, h, w, cin, cout, k, stride, pad, ctas, False, 0).ws_bytes
        want_r = O.route_repvgg_wgrad(n, h, w, cin, cout, ctas, 0).ws_bytes
        if (g, r) != (want_g, want_r):
            bad.append(((n, h, w, cin, cout, k, stride, pad, ctas), (g, r), (want_g, want_r)))
    assert not bad, f"{len(bad)} of {len(rows)} queries differ (shape+ctas, library, oracle): {bad[:5]}"
    # the sweep is not trivially all-zero: both kernels size a workspace somewhere, and some shapes need none
    assert any(g for g, _ in got) and any(r for _, r in got) and any(g == 0 for g, _ in got)


@pytest.mark.parametrize("sms", list(O.SMS_RANGE))
def test_case_tables_reach_every_path(sms):
    seen = set()
    for name, case in O.WGRAD_ACC_CASES.items():
        route, _ = O.case_route(case, sms)
        assert route.path == case[3], (name, sms, route)
        assert name.startswith(route.path)
        seen.add(route.path)
    assert seen == {O.ROWS, O.PARTIALS, O.REFUSED}
    seen = set()
    for name, case in O.REPVGG_ACC_CASES.items():
        route, _ = O.repvgg_case_route(case, sms)
        assert route.path == case[3], (name, sms, route)
        assert name.startswith(route.path)
        seen.add(route.path)
    assert seen == {O.ROWS, O.REFUSED}
    # the overwriting form on the same tables also takes the single-range and atomics paths
    over = set()
    for case in O.WGRAD_ACC_CASES.values():
        (n, h, w, cin, cout, k, stride, pad), ctas, _, _ = case
        full = O.route_wgrad(n, h, w, cin, cout, k, stride, pad, ctas, False, 0, sms).ws_bytes
        over.add(O.route_wgrad(n, h, w, cin, cout, k, stride, pad, ctas, False, full, sms).path)
        over.add(O.route_wgrad(n, h, w, cin, cout, k, stride, pad, ctas, False, 0, sms).path)
    assert over == {O.ROWS, O.PARTIALS, O.SINGLE, O.ATOMICS}
    # every CTA count the GPU test forces appears in both tables
    assert {c[1] for c in O.WGRAD_ACC_CASES.values()} >= {0, 1, 2, 7}
    assert {c[1] for c in O.REPVGG_ACC_CASES.values()} >= {0, 1, 2, 7}


def _bits(vals):
    return torch.tensor(vals, dtype=torch.int32).to(torch.int16)


def test_bf16_rounding_of_the_edge_values():
    """torch's .bfloat16() is the round-to-nearest-even that __float2bfloat16_rn performs, subnormals included."""
    want = [0x0000, 0x8000, 0x3F80, 0x3F82, 0xBF80, 0x3F80, 0x3F81, 0xBF80, 0x7F80, 0x7F7F, 0xFF80, 0x7F80, 0xFF80, None,
            0x0000, 0x8000, 0x0000, 0x0002, 0x0080, 0x807F + 1, 0x0080, 0x3F80]
    got = O.edge_values().bfloat16().view(torch.int16).to(torch.int32) & 0xFFFF
    for i, wv in enumerate(want):
        if wv is None:
            assert torch.isnan(O.edge_values()[i].bfloat16())
        else:
            assert int(got[i]) == wv, (i, hex(int(got[i])), hex(wv))


def test_pack_restatements_on_a_hand_written_filter():
    # w[co][r][s][ci], Cout 2, 2x2 taps, Cin 3: value = 100 co + 10 (2 r + s) + ci (exact in bf16 up to 256: use small)
    w = torch.tensor([[[[0., 1, 2], [3, 4, 5]], [[6, 7, 8], [9, 10, 11]]],
                      [[[-0., -1, -2], [-3, -4, -5]], [[-6, -7, -8], [-9, -10, -11]]]])
    wf = O.pack_wf(w, 3, 4).float()
    assert wf.shape == (3, 2, 2, 4)
    assert wf[0, 1, 0].tolist() == [6, 7, 8, 0] and wf[1, 0, 1].tolist() == [-3, -4, -5, 0]
    assert bool((wf[2] == 0).all()) and bool((wf[..., 3] == 0).all())
    assert torch.signbit(wf[1, 0, 0, 0]) and not torch.signbit(wf[2, 0, 0, 0])     # -0 kept, padding +0
    wd = O.pack_wd(w, 4, 3).float()
    assert wd.shape == (4, 2, 2, 3)
    # wd[ci][r][s][co] = w[co][1-r][1-s][ci]
    assert wd[0, 0, 0].tolist() == [9, -9, 0] and wd[2, 1, 0].tolist() == [5, -5, 0] and wd[1, 1, 1].tolist() == [1, -1, 0]
    assert bool((wd[3] == 0).all())
    # stride-2 classes of a 3x3 filter: class (0,0) = tap (1,1); (0,1) = taps (1,2), (1,0); (1,0) = (2,1), (0,1);
    # (1,1) = (2,2), (2,0), (0,2), (0,0)
    w3 = torch.arange(9.).view(1, 3, 3, 1) + 1                                       # w[0][r][s][0] = 3 r + s + 1
    cls = O.pack_dgrad_s2(w3, 2, 2).float()
    assert cls.numel() == 9 * 2 * 2
    c00, c01, c10, c11 = cls[:4].view(2, 1, 1, 2), cls[4:12].view(2, 1, 2, 2), cls[12:20].view(2, 2, 1, 2), cls[20:].view(2, 2, 2, 2)
    assert c00[0, 0, 0].tolist() == [5, 0]
    assert c01[0, 0, :, 0].tolist() == [6, 4]
    assert c10[0, :, 0, 0].tolist() == [8, 2]
    assert c11[0, :, :, 0].tolist() == [[9, 7], [3, 1]]
    assert bool((cls.view(-1)[[1, 3]] == 0).all())
    # edge values survive the restatement with their rounding
    e = O.edge_values()
    we = e[:20].view(1, 2, 2, 5)
    got = O.pack_wf(we, 1, 8)[0, :, :, :5].reshape(-1)
    ok, nbad = O.bf16_equal(got, e[:20].bfloat16())
    assert ok, nbad


def test_clip_oracle_follows_clip_grad_norm_on_special_norms():
    for vals, max_norm in (([3.0, 4.0, -0.0], 1.0), ([3.0, float("inf"), 1.0, -2.0], 1.0), ([1.0, float("nan"), 2.0], 5.0),
                           ([1e-3, 2e-3], 1.0)):
        g = torch.tensor(vals)
        p = torch.nn.Parameter(torch.zeros_like(g))
        p.grad = g.clone()
        norm = torch.nn.utils.clip_grad_norm_([p], max_norm)
        want = O.clip_ref(g, float(norm), max_norm)
        same = (p.grad.view(torch.int32) == want.view(torch.int32)) | (torch.isnan(p.grad) & torch.isnan(want))
        assert bool(same.all()), (vals, p.grad, want)
    assert torch.isnan(O.clip_coef(float("nan"), 1.0))
    assert float(O.clip_coef(float("inf"), 1.0)) == 0.0


@pytest.mark.parametrize("sms", list(O.SMS_RANGE))
def test_direct_cases_reach_their_planned_routes(sms):
    """Every route of the bucket test's cases that the launch planning decides is reached through a witness call whose
    route is the same for every SM count; the structural routes (stem, padded, BatchNorm) do not depend on it."""
    assert set().union(*O.DIRECT_ROUTES.values()) == O.ALL_ROUTES
    assert set(O.DIRECT_WITNESSES) == set(O.DIRECT_ROUTES)
    for name, witnesses in O.DIRECT_WITNESSES.items():
        for route, (kind, shape) in witnesses:
            assert O.witness_route(kind, shape, sms) == route, (name, kind, shape, sms)
        assert {r for r, _ in witnesses} == O.DIRECT_ROUTES[name] & O.PLANNED_ROUTES, name
