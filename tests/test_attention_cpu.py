"""CPU checks of SAM, DimAttention and TripletAttention against tests/golden/attention.pt (written by
make_golden_attention.py from the unmodified reference): the torch restatement (tests/_attention_oracle.py) against the
reference's outputs, gradients and running statistics, the module trees, signatures, reprs, state_dict layouts and
seeded initialisation, conv_sequence's attention layer, and the ptxas report of the attention kernels."""
import inspect
import re
from pathlib import Path

import pytest
import torch
from torch import nn

import holocron_b200 as hb
from holocron_b200.models.utils import conv_sequence

import _attention_oracle as O
from conftest import load_golden

LOG = Path(__file__).resolve().parents[1] / "holocron_b200" / "csrc" / "build" / "attention.log"
ATT = hb.nn.modules.attention


@pytest.fixture(scope="module")
def g():
    return load_golden("attention")


@pytest.fixture(autouse=True)
def _global_rng_untouched():
    """These tests seed and draw from the global generator (module construction); later tests that draw unseeded
    inputs see the same generator state whether or not this file ran."""
    with torch.random.fork_rng(devices=[]):
        yield


def _describe(obj):
    target = obj.__init__ if inspect.isclass(obj) else obj
    return [[n, p.kind.name, None if p.default is inspect.Parameter.empty else repr(p.default)]
            for n, p in inspect.signature(target).parameters.items() if n != "self"]


def test_signatures_and_exports(g):
    assert list(ATT.__all__) == g["all"]
    for name, sig in g["signatures"].items():
        assert _describe(getattr(ATT, name)) == sig, name
    for name in g["all"]:
        assert getattr(hb.nn, name) is getattr(ATT, name)


def test_module_trees_and_seeded_init(g):
    for rec in g["modules"]:
        torch.manual_seed(0)
        mod = getattr(ATT, rec["ctor"])(*rec["args"])
        assert repr(mod) == rec["repr"]
        assert [(n, repr(m)) for n, m in mod.named_children()] == rec["children"]
        sd = mod.state_dict()
        assert [(k, tuple(v.shape), str(v.dtype)) for k, v in sd.items()] == rec["state_dict_layout"]
        for k, v in rec["state_dict"].items():
            assert torch.equal(sd[k], v), (rec["ctor"], k)
        # the reference's checkpoints load unchanged
        mod.load_state_dict(rec["state_dict"])


def test_conv_sequence_attention_layer(g):
    torch.manual_seed(0)
    layers = conv_sequence(4, 8, nn.ReLU(inplace=True), nn.BatchNorm2d, kernel_size=3, padding=1,
                           attention_layer=ATT.SAM)
    assert [repr(m) for m in layers] == g["conv_sequence"]
    assert isinstance(layers[-1], ATT.SAM)


def _params(mod):
    return {k: O.branch_params(getattr(mod, f"{k}_branch")) for k in "chw"}


def _oracle_step(fn, step):
    x = step["x"].clone().requires_grad_(True)
    y = fn(x, step["training"])
    (y * step["w"]).sum().backward()
    return y.detach(), x.grad


def test_oracle_reproduces_sam(g):
    for case in g["sam"]:
        w = case["state_dict"]["conv.weight"].clone().requires_grad_(True)
        b = case["state_dict"]["conv.bias"].clone().requires_grad_(True)
        x = case["x"].clone().requires_grad_(True)
        y = O.sam(x, w, b)
        (y * case["w"]).sum().backward()
        assert torch.equal(y, case["y"])
        assert torch.equal(x.grad, case["dx"])
        assert torch.equal(w.grad, case["dweight"]) and torch.equal(b.grad, case["dbias"])


def _check_steps(case, fn_of_params, params, grad_names):
    for step in case["steps"]:
        for p in params.values():
            for t in p.values():
                t.grad = None
        y, dx = _oracle_step(fn_of_params, step)
        torch.testing.assert_close(y, step["y"], rtol=1e-6, atol=1e-6, equal_nan=True)
        torch.testing.assert_close(dx, step["dx"], rtol=1e-6, atol=1e-6, equal_nan=True)
        for name, (k, key) in grad_names.items():
            torch.testing.assert_close(params[k][key].grad, step["grads"][name], rtol=1e-5, atol=1e-6)


_KEYS = {"compress.1.weight": "conv_weight", "compress.2.weight": "bn_weight", "compress.2.bias": "bn_bias"}


def test_oracle_reproduces_triplet_two_steps(g):
    for case in g["triplet"]:
        mod = ATT.TripletAttention()
        mod.load_state_dict(case["state_dict"])
        ps = _params(mod)
        names = {f"{k}_branch.{n}": (k, key) for k in "chw" for n, key in _KEYS.items()}
        _check_steps(case, lambda x, t: O.triplet_attention(x, ps, t), ps, names)
        for k in "chw":
            for key in ("running_mean", "running_var"):
                torch.testing.assert_close(ps[k][key], case["buffers_after"][f"{k}_branch.compress.2.{key}"],
                                           rtol=1e-6, atol=1e-7)
        assert int(case["buffers_after"]["c_branch.compress.2.num_batches_tracked"]) == 2


def test_oracle_reproduces_dim_attention(g):
    for case in g["dim"]:
        mod = ATT.DimAttention(case["dim"])
        mod.load_state_dict(case["state_dict"])
        p = O.branch_params(mod)
        names = {n: ("b", key) for n, key in _KEYS.items()}
        _check_steps(case, lambda x, t: O.dim_attention(x, case["dim"], p, t), {"b": p}, names)
        for key in ("running_mean", "running_var"):
            torch.testing.assert_close(p[key], case["buffers_after"][f"compress.2.{key}"], rtol=1e-6, atol=1e-7)


def test_oracle_reproduces_nan_routing(g):
    case = g["nan"]
    mod = ATT.TripletAttention()
    mod.load_state_dict(case["state_dict"])
    ps = _params(mod)
    y, dx = _oracle_step(lambda x, t: O.triplet_attention(x, ps, t), case["step"])
    assert y.isnan().any() and not y.isnan().all()
    torch.testing.assert_close(y, case["step"]["y"], rtol=1e-6, atol=1e-6, equal_nan=True)
    torch.testing.assert_close(dx, case["step"]["dx"], rtol=1e-6, atol=1e-6, equal_nan=True)


def test_forward_needs_cuda():
    with pytest.raises(RuntimeError):
        ATT.SAM(4)(torch.randn(1, 4, 3, 3))
    with pytest.raises(NotImplementedError):
        ATT.TripletAttention()(torch.randn(4, 3, 3))


def test_attention_kernels_build_without_spills():
    if not LOG.exists():
        pytest.skip(f"{LOG.name} absent: build the library first (python -m holocron_b200.csrc.build)")
    text = LOG.read_text()
    assert "Compiling entry function" in text
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", text)
    assert spills and all(s == ("0", "0") for s in spills)
    frames = re.findall(r"(\d+) bytes stack frame", text)
    assert all(f == "0" for f in frames)
