"""CPU checks of LambdaLayer against tests/golden/lambda_layer.pt (written by make_golden_lambda.py from the unmodified
reference): the torch restatement against the reference's outputs, gradients and eval outputs, the signature, repr
strings, state_dict layout and seeded init of the module, the constructions and inputs it must refuse, and the ptxas
report of its kernels."""
import inspect
import re
from pathlib import Path

import pytest
import torch

import holocron_b200 as hb
from holocron_b200._lib import HolocronB200Error

import _lambda_oracle as O
from conftest import load_golden

LOG = Path(__file__).resolve().parents[1] / "holocron_b200" / "csrc" / "build" / "lambda_layer.log"


@pytest.fixture(scope="module")
def g():
    return load_golden("lambda_layer")


def _ours(cfg):
    c, o, dk, n, r, heads, u = cfg
    return hb.nn.LambdaLayer(c, o, dk, n=n, r=r, num_heads=heads, dim_u=u)


def _rel_l2(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_oracle_matches_reference(g, dtype):
    assert len(g["cases"]) == 7
    tol = 1e-5 if dtype == torch.float32 else 1e-6
    for case in g["cases"]:
        torch.manual_seed(case["seed"])
        mod = _ours(case["cfg"]).to(dtype)
        x = case["x"].clone().to(dtype).requires_grad_(True)
        y = O.lambda_module(x, mod)
        torch.manual_seed(case["w_seed"])
        w = torch.randn(case["y"].shape).to(dtype)
        (y * w).sum().backward()
        assert _rel_l2(y.detach(), case["y"]) <= tol, case["cfg"]
        assert _rel_l2(x.grad, case["dx"]) <= tol, case["cfg"]
        for name, p in mod.named_parameters():
            assert _rel_l2(p.grad, case["grads"][name]) <= 10 * tol, (case["cfg"], name)
        mod.load_state_dict({**mod.state_dict(), **case["running"]})
        with torch.no_grad():
            ye = O.lambda_module(case["x"][:1].to(dtype), mod, training=False)
        assert _rel_l2(ye, case["y_eval"]) <= tol, case["cfg"]


def test_conv3d_formulation_matches_reference(g):
    for case in g["cases"]:
        torch.manual_seed(case["seed"])
        mod = _ours(case["cfg"])
        y = O.lambda_module(case["x"], mod, core=O.lambda_core_conv3d)
        assert _rel_l2(y.detach(), case["y"]) <= 1e-5, case["cfg"]


def test_signature_repr_state_dict_and_init(g):
    ours = [[n, p.kind.name, None if p.default is inspect.Parameter.empty else repr(p.default)]
            for n, p in inspect.signature(hb.nn.LambdaLayer.__init__).parameters.items() if n != "self"]
    assert ours == g["signature"]
    assert "LambdaLayer" in hb.nn.modules.lambda_layer.__all__
    for case in g["cases"]:
        torch.manual_seed(case["seed"])
        mod = _ours(case["cfg"])
        assert repr(mod) == case["repr"]
        assert [(k, tuple(v.shape)) for k, v in mod.state_dict().items()] == case["state_dict"]
        for k, v in mod.state_dict().items():
            assert torch.equal(v, case["init"][k]), k
        c, o, dk, n, r, heads, u = case["cfg"]
        assert (mod.u, mod.num_heads, mod.local_contexts) == (u, heads, r is not None)
        if r is not None:
            assert mod.padding == r // 2


def test_refused_constructions(g):
    for ref in g["refused_constructions"]:
        assert ref["raised"] == "AssertionError"
        with pytest.raises(AssertionError) as info:
            hb.nn.LambdaLayer(**ref["kwargs"])
        assert str(info.value) == ref["message"]


def test_refused_inputs(g):
    for err in g["errors"]:
        assert err["raised"] == "RuntimeError"
        x = torch.randn(*err["shape"])
        with pytest.raises(RuntimeError) as info:
            _ours(err["cfg"])(x)
        assert not isinstance(info.value, HolocronB200Error), "the shape is refused before the device check"
        with pytest.raises(RuntimeError):
            O.lambda_module(x, _ours(err["cfg"]))


@pytest.mark.parametrize("kwargs", [dict(dim_k=4, r=3), dict(dim_k=16, r=25), dict(dim_k=16, r=3, dim_u=5),
                                    dict(dim_k=16, r=3, num_heads=16)])
def test_unsupported_configurations(kwargs):
    with pytest.raises(NotImplementedError):
        hb.nn.LambdaLayer(8, 32, **kwargs)(torch.randn(1, 8, 8, 8))


def test_cpu_tensor_raises():
    with pytest.raises(HolocronB200Error):
        hb.nn.LambdaLayer(8, 32, 16, r=3)(torch.randn(1, 8, 8, 8))


def test_no_spills():
    if not LOG.exists():
        pytest.skip(f"{LOG.name} absent: build the library first (python -m holocron_b200.csrc.build)")
    text = LOG.read_text()
    assert "Compiling entry function" in text, f"{LOG.name} holds no ptxas -v output"
    spills = [m.group(0) for m in re.finditer(r"(\d+) bytes spill stores, (\d+) bytes spill loads", text)
              if m.group(1) != "0" or m.group(2) != "0"]
    assert not spills, spills
