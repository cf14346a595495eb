"""Coverage of the loss cases (tests/_loss_cases.py), the argument checks of the loss entry points, and the power of the
per-element bounds of tests/_loss_oracle.py, without a GPU.

The routing mirror must send the cases through every kernel instantiation of csrc/losses.cu at the SM counts of both
H100 variants, its list of instantiations must be the set of kernels the compiler built from losses.cu, and the cases tagged ``wrap`` must give every thread of every grid-stride launch a second iteration. The
entry points must refuse malformed shapes with cudaErrorInvalidValue before they launch or query a device: they are
called with null pointers in a child process that sees no CUDA device. And the bounds must not be vacuous: each planted
fault, applied to the fp64 reference, must break the bound of at least one element of every case it applies to."""
import json
import os
import re
import shutil
import subprocess
import sys
from pathlib import Path

import pytest
import torch

import _loss_cases as D
import _loss_oracle as O

ROOT = Path(__file__).resolve().parents[1]
SMS = [132, 114]            # H100 SXM, H100 PCIe
INVALID_VALUE = 1           # cudaErrorInvalidValue


@pytest.mark.parametrize("sms", SMS)
def test_every_instantiation_is_reached(sms):
    taken = {}
    for name, cs in D.CASES.items():
        for kern in D.kernels_taken(cs, sms):
            taken.setdefault(kern, name)
    missing = [k for k in D.INSTANTIATIONS if k not in taken]
    assert not missing, f"not reached at {sms} SMs: {missing}"
    assert set(taken) <= set(D.INSTANTIATIONS), set(taken) - set(D.INSTANTIATIONS)
    assert len([k for k in D.INSTANTIATIONS if "_vec_kernel<" in k]) == 96
    blocks = {D.route(cs, sms)["rdot"].block for cs in D.CASES.values() if cs.family == "mcl"}
    assert set(D.RDOT_BLOCKS) <= blocks


@pytest.mark.parametrize("sms", SMS)
def test_wrap_cases_wrap(sms):
    wraps = [cs for cs in D.CASES.values() if cs.wrap]
    assert {cs.family for cs in wraps} == {"hard", "soft", "dice", "cce", "mcl"}
    for cs in wraps:
        for launch in D.route(cs, sms).values():
            if launch.total:
                assert launch.min_iters >= 2, D.describe(cs, sms)
    paths = {D.route(cs, sms)["fwd"].kernel.split("<")[0] + D.route(cs, sms)["fwd"].kernel.split(">")[-1]
             for cs in wraps if cs.family == "hard"}
    assert paths == {"hard_vec_kernel", "hard_kernel/thread", "hard_kernel/warp"}


def test_mirror_lists_the_compiled_kernels():
    """The mirror's instantiations, without their /warp /thread /vec /scalar branch names, are exactly the entry functions
    in the -Xptxas -v output that holocron_b200/csrc/build.py keeps in csrc/build/losses.log."""
    log = ROOT / "holocron_b200" / "csrc" / "build" / "losses.log"
    if not log.exists():
        pytest.skip(f"{log.name} absent: build the library first (python -m holocron_b200.csrc.build)")
    mangled = re.findall(r"Compiling entry function '(\w+)'", log.read_text())
    assert mangled, f"{log.name} holds no ptxas -v output"
    tool = shutil.which("cu++filt") or shutil.which("c++filt")
    if tool is None:
        pytest.skip("no demangler (cu++filt or c++filt) on PATH")
    lines = subprocess.run([tool], input="\n".join(mangled), capture_output=True, text=True, check=True).stdout.split("\n")
    compiled = []
    for line in lines[:len(mangled)]:
        # c++filt: "void (anonymous namespace)::k<float, 4, false>(...)"; cu++filt: "void <unnamed>::k<float, (int)4, (bool)0>(...)"
        name = re.sub(r"\(anonymous namespace\)::|<unnamed>::|\(int\)", "", line).removeprefix("void ")
        name = name.replace("(bool)0", "false").replace("(bool)1", "true")
        compiled.append(name.split("(")[0].replace(" ", ""))
    assert len(set(compiled)) == len(compiled), compiled
    mirror = {k.split("/")[0] for k in D.INSTANTIATIONS}
    assert set(compiled) == mirror, (f"compiled, not in the mirror: {sorted(set(compiled) - mirror)}; "
                                     f"in the mirror, not compiled: {sorted(mirror - set(compiled))}")


def test_case_geometry():
    for cs in D.CASES.values():
        assert cs.k % cs.xi == 0 and cs.positions > 0, cs.name
    # each K sits on both edges of its KMAX bucket in every dtype
    for dt in D.DTYPES:
        ks = {cs.k for cs in D.CASES.values() if cs.family == "hard" and cs.dtype == dt and D.vec_eligible(cs)}
        for km in D.KMAXES:
            assert {km - 3 if km > 4 else 1, km} <= ks, (dt, km)
        # S = 6 is vector-eligible in fp32 only
        assert D.vec_eligible(D.CASES[f"hard_{dt}_n5k7s6"]) == (dt == "float32")
        assert not D.vec_eligible(D.CASES[f"hard_{dt}_n3k12s16_off1"])


# (N, K, S, extra): refused by every entry point of the family
BAD = {
    "n_negative": (-1, 4, 8), "k0": (2, 0, 8), "k_negative": (2, -3, 8), "s0": (2, 4, 0), "s_negative": (2, 4, -8),
}
_CHILD = """
import json, sys, ctypes
sys.path.insert(0, sys.argv[1])
from holocron_b200._lib import lib
L = lib()
f = ctypes.c_float
out = {}
def each(n, k, s):
    return [L.hb_cls_loss_hard_fwd(None, None, None, None, None, None, n, k, s, -100, 0, f(2), f(0), 0, None),
            L.hb_cls_loss_hard_bwd(None, None, None, None, None, None, n, k, s, -100, 0, f(2), f(0), 1, 0, None),
            L.hb_poly_soft_fwd(None, None, None, None, None, None, n, k, s, -100, f(2), 1, None),
            L.hb_poly_soft_bwd(None, None, None, None, None, n, k, s, -100, f(2), 1, 1, None),
            L.hb_dice_fwd(None, None, None, None, None, None, n, k, s, f(1), f(1e-8), 2, None),
            L.hb_dice_bwd(None, None, None, None, n, k, s, 2, None),
            L.hb_cce_fwd(None, None, None, None, None, None, n, k, s, -100, f(-1), 0, None),
            L.hb_cce_bwd(None, None, None, None, None, None, n, k, s, -100, f(-1), 1, 0, None)]
def mcl(n, cnum, xi, s):
    return [L.hb_mcl_fwd(*([None] * 9), n, cnum, xi, s, -100, f(1), 0, None),
            L.hb_mcl_bwd(*([None] * 10), n, cnum, xi, s, -100, f(1), 1, 0, None)]
for name, (n, k, s) in json.loads(sys.argv[2]).items():
    out[name] = each(n, k, s)
    out["mcl_" + name] = mcl(n, k, 2, s)
    print(name, out[name], flush=True)
out["cce_k1"] = [L.hb_cce_fwd(None, None, None, None, None, None, 4, 1, 8, -100, f(0.5), 0, None),
                 L.hb_cce_bwd(None, None, None, None, None, None, 4, 1, 8, -100, f(-1), 1, 0, None)]
out["mcl_xi0"] = mcl(2, 4, 0, 8)
out["mcl_xi_negative"] = mcl(2, 4, -2, 8)
out["mcl_xi377"] = mcl(2, 1, 377, 8)
print("RESULT " + json.dumps(out))
"""


def test_abi_refuses_malformed_shapes():
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    proc = subprocess.run([sys.executable, "-c", _CHILD, str(ROOT), json.dumps(BAD)], env=env, capture_output=True,
                          text=True, timeout=300)
    assert proc.returncode == 0, (f"the child exited with {proc.returncode} (a negative code is the signal that killed "
                                  f"it):\n{proc.stdout[-2000:]}\n{proc.stderr[-2000:]}")
    got = json.loads(next(ln for ln in proc.stdout.splitlines() if ln.startswith("RESULT "))[len("RESULT "):])
    for name, codes in got.items():
        assert codes == [INVALID_VALUE] * len(codes), f"{name}: returned {codes}"
    assert len(got) == 2 * len(BAD) + 4


# ---- planted faults ----------------------------------------------------------------------------------------------------
# not where the loss is identically 0 (one class) or where the target's probability is 1 - O(e^-30): there the
# loss and its gradient lie below fp32's resolution, and the faults change nothing a fp32 kernel could show
FAULT_CASES = [n for n, cs in D.CASES.items() if not cs.light and cs.cnum > 1 and cs.logits != "confident"]


def _faults(cs, prm, sp, ref):
    """{fault: (outputs as the faulty kernel would give them)} for the faults that apply to this parameter set."""
    fam = cs.family
    fn = lambda spec: O.reference(fam, spec)        # noqa: E731
    out = {}
    k = cs.cnum
    base = {key: c.ref.clone() for key, c in ref.items()}
    hard_t = fam in ("hard", "cce", "mcl")
    if hard_t and k > 1:
        t2 = torch.where((sp.target >= 0) & (sp.target < k), (sp.target + 1) % k, sp.target)
        out["target swapped with its neighbour"] = {key: c.ref for key, c in fn(_with(sp, target=t2)).items()}
    if sp.weight is not None:
        out["class weight dropped"] = {key: c.ref for key, c in fn(_with(sp, weight=None)).items()}
    if hard_t and 0 <= sp.ignore_index < k:
        out["ignored position counted"] = {key: c.ref for key, c in fn(_with(sp, ignore_index=-100)).items()}
        m = dict(base)
        m["mean"] = base["sum"] / (cs.n * cs.s)
        out["mean over P instead of the valid count"] = m
    if fam == "soft" and prm[5] == "multilabel":
        m = dict(base)
        labelled = float((sp.target.double().sum(1) > 0).sum())
        m["mean"] = base["sum"] / labelled
        out["mean over the labelled positions instead of P"] = m
    if fam == "dice" and sp.weight is not None:
        w = sp.weight.double()
        m = dict(base)
        m["loss"] = 1 - (1 - base["loss"]) * w.sum() / w.numel()
        out["mean over K instead of the weight sum"] = m
        lo = fn(_with(sp, weight=None))["loss"].ref
        out["class weight dropped"] = dict(base, loss=lo)
    key0 = "loss" if fam != "dice" else "dx"
    m = dict(base)
    m[key0] = base[key0].clone()
    m[key0][(0,) * m[key0].ndim] = float("nan")
    out["one position left unwritten"] = m
    if k > 1 and fam != "mcl":
        x2 = sp.x.clone()
        x2[:, k - 1] = -1e30 if fam != "dice" else 0
        t2 = sp.target
        if fam == "dice":
            t2 = sp.target.clone()
            t2[:, k - 1] = 0
        drop = {key: c.ref for key, c in fn(_with(sp, x=x2, target=t2)).items()}
        for key in drop:
            if key.startswith("dx"):
                drop[key] = drop[key].clone()
                drop[key][:, k - 1] = 0
        out["last class column dropped"] = drop
    return out


def _with(sp, **kw):
    d = dict(sp.__dict__)
    d.update(kw)
    return O.Spec(**d)


@pytest.mark.parametrize("name", FAULT_CASES)
def test_planted_faults_break_the_bound(name):
    cs = D.CASES[name]
    for i, prm in enumerate(O.params(cs)):
        sp = O.make_spec(cs, prm, seed=i)
        ref = O.reference(cs.family, sp)
        for key, c in ref.items():
            assert not O.breaks(c.ref, c), f"{name} {prm}: the reference breaks its own bound on {key}"
        for fault, got in _faults(cs, prm, sp, ref).items():
            broken = [key for key, v in got.items() if O.breaks(v, ref[key])]
            assert broken, f"{name} {prm}: '{fault}' stays within every bound"
