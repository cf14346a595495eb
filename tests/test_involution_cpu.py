"""CPU checks of Involution2d against tests/golden/involution.pt (written by make_golden_involution.py from the unmodified
reference): the torch restatement against the reference's outputs and gradients, the signature, repr strings,
state_dict layout and seeded init of the module, the shapes it must refuse, and the ptxas report of its kernels."""
import inspect
import re
from pathlib import Path

import pytest
import torch

import holocron_b200 as hb
from holocron_b200._lib import HolocronB200Error

import _involution_oracle as O
from conftest import load_golden

LOG = Path(__file__).resolve().parents[1] / "holocron_b200" / "csrc" / "build" / "involution.log"


@pytest.fixture(scope="module")
def g():
    return load_golden("involution")


def _ours(cfg):
    c, k, p, s, d, gr, r = cfg
    return hb.nn.Involution2d(c, k, padding=p, stride=s, groups=gr, dilation=d, reduction_ratio=r)


def test_oracle_matches_reference(g):
    assert len(g["cases"]) == 7
    for case in g["cases"]:
        torch.manual_seed(case["seed"])
        mod = _ours(case["cfg"])
        x = case["x"].clone().requires_grad_(True)
        y = O.involution_module(x, mod)
        (y * case["w"]).sum().backward()
        torch.testing.assert_close(y.detach(), case["y"], rtol=1e-5, atol=1e-5)
        torch.testing.assert_close(x.grad, case["dx"], rtol=1e-5, atol=1e-5)
        for name, p in mod.named_parameters():
            torch.testing.assert_close(p.grad, case["grads"][name], rtol=1e-5, atol=1e-5, msg=lambda m: f"{name}: {m}")


def test_signature_repr_state_dict_and_init(g):
    ours = [[n, p.kind.name, None if p.default is inspect.Parameter.empty else repr(p.default)]
            for n, p in inspect.signature(hb.nn.Involution2d.__init__).parameters.items() if n != "self"]
    assert ours == g["signature"]
    assert "Involution2d" in hb.nn.modules.conv.__all__
    for case in g["cases"]:
        torch.manual_seed(case["seed"])
        mod = _ours(case["cfg"])
        assert repr(mod) == case["repr"]
        assert [(k, tuple(v.shape)) for k, v in mod.state_dict().items()] == case["state_dict"]
        for k, v in mod.state_dict().items():
            assert torch.equal(v, case["init"][k]), k
        assert (mod.pool is None) == (case["cfg"][3] == 1)


def test_refused_shapes(g):
    for err in g["errors"]:
        assert err["raised"] == "RuntimeError"
        c, k, p, s, d, gr, r = err["cfg"]
        mod = hb.nn.Involution2d(c, k, padding=p, stride=s, groups=gr, dilation=d, reduction_ratio=r)
        x = torch.randn(*err["shape"])
        with pytest.raises(RuntimeError) as info:
            mod(x)
        assert not isinstance(info.value, HolocronB200Error), "the shape is refused before the device check"
        with pytest.raises(RuntimeError):
            O.involution_module(x, mod)


@pytest.mark.parametrize("k", [2, 9])
def test_unsupported_kernel_size(k):
    with pytest.raises(NotImplementedError):
        hb.nn.Involution2d(8, k, padding=(k - 1) // 2 if k % 2 else 0)(torch.randn(1, 8, 8, 8))


def test_cpu_tensor_raises():
    with pytest.raises(HolocronB200Error):
        hb.nn.Involution2d(8, 3, padding=1)(torch.randn(1, 8, 8, 8))
    with pytest.raises(HolocronB200Error):
        hb.nn._involution.involution2d(torch.randn(1, 8, 8, 8), torch.randn(1, 9, 8, 8), 3, 1, 1, 1, 1)


def test_no_spills():
    if not LOG.exists():
        pytest.skip(f"{LOG.name} absent: build the library first (python -m holocron_b200.csrc.build)")
    text = LOG.read_text()
    assert "Compiling entry function" in text, f"{LOG.name} holds no ptxas -v output"
    spills = [m.group(0) for m in re.finditer(r"(\d+) bytes spill stores, (\d+) bytes spill loads", text)
              if m.group(1) != "0" or m.group(2) != "0"]
    assert not spills, spills
