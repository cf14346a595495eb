"""CPU checks of BlurPool2d, GlobalMaxPool2d, ZPool and z_pool against tests/golden/downsample.pt (written by
make_golden_downsample.py from the unmodified reference): the torch restatement against the reference's outputs and
gradients, the signatures, reprs, children and state_dict layouts, the errors the reference raises, and the ptxas report
of the pooling kernels."""
import inspect
import re
from pathlib import Path

import pytest
import torch

import holocron_b200 as hb
from holocron_b200._lib import HolocronB200Error
from holocron_b200.nn import _pooling

import _downsample_oracle as O
from conftest import load_golden

LOG = Path(__file__).resolve().parents[1] / "holocron_b200" / "csrc" / "build" / "pooling.log"
DS = hb.nn.modules.downsample


@pytest.fixture(scope="module")
def g():
    return load_golden("downsample")


def _describe(obj):
    target = obj.__init__ if inspect.isclass(obj) else obj
    return [[n, p.kind.name, None if p.default is inspect.Parameter.empty else repr(p.default)]
            for n, p in inspect.signature(target).parameters.items() if n != "self"]


def _ulp_bf16(t):
    return torch.exp2(torch.floor(torch.log2(t.double().abs().clamp_min(2.0 ** -126))) - 7)


def test_signatures(g):
    for name, sig in g["signatures"].items():
        assert _describe(getattr(DS, name)) == sig, name
        assert name in DS.__all__ and getattr(hb.nn, name) is getattr(DS, name)
    assert _describe(hb.nn.functional.z_pool) == g["z_pool_signature"]
    assert "z_pool" in hb.nn.functional.__all__


def test_repr_children_state_dict_and_filter(g):
    for rec in g["modules"]:
        mod = getattr(DS, rec["ctor"])(*rec["args"])
        assert repr(mod) == rec["repr"]
        assert [(n, repr(m)) for n, m in mod.named_children()] == rec["children"]
        assert [(k, tuple(v.shape)) for k, v in mod.state_dict().items()] == rec["state_dict"]
        if rec["ctor"] == "BlurPool2d":
            assert mod._coeffs.dtype == torch.float64 and torch.equal(mod._coeffs, rec["coeffs"])
            k = rec["args"][1] if len(rec["args"]) > 1 else 3
            # the taps handed to the kernel are the reference's filter, rounded to the input dtype
            for dtype, key in ((torch.bfloat16, "filter_bf16"), (torch.float32, "filter_fp32")):
                taps = torch.tensor(list(_pooling.blur_taps(mod._coeffs, dtype))).view(k, k)
                assert torch.equal(taps, rec[key].float()), (rec["args"], dtype)
                assert torch.equal(O.blur_filter(k, dtype), rec[key])
    k8 = next(r for r in g["modules"] if r["args"] == (16, 8, 2))
    assert k8["filter_bf16"][3, 3].item() == 0.07470703125


def test_reference_errors(g):
    for err in g["errors"]:
        channels, k, s = err["ctor"]
        if err["shape"] is None:
            assert err["raised"] == "AssertionError"
            with pytest.raises(AssertionError):
                DS.BlurPool2d(channels, k, s)
            continue
        assert err["raised"] == "RuntimeError", err
        mod = DS.BlurPool2d(channels, k, s)
        with pytest.raises(RuntimeError) as info:
            mod(torch.randn(*err["shape"]))
        assert not isinstance(info.value, HolocronB200Error), f"{err['case']}: refused before the device check"


def test_documented_deviations():
    mod = DS.BlurPool2d(4, 8, 2)        # builds like the reference; the kernel stops at 7 taps
    with pytest.raises(NotImplementedError):
        mod(torch.randn(1, 4, 16, 16))
    for shape, dim in (((4, 8, 8), 1), ((1, 4, 8, 8), 0), ((1, 4, 8, 8), 4), ((1, 4, 8, 8), -4)):
        with pytest.raises(NotImplementedError):
            hb.nn.functional.z_pool(torch.randn(*shape), dim)
    with pytest.raises(NotImplementedError):
        DS.ZPool(0)(torch.randn(1, 4, 8, 8))


def test_cpu_tensor_raises():
    for mod in (DS.BlurPool2d(4), DS.GlobalMaxPool2d(), DS.GlobalMaxPool2d(True), DS.ZPool(), DS.ZPool(-2)):
        with pytest.raises(HolocronB200Error):
            mod(torch.randn(2, 4, 8, 8))


def test_conv_sequence_blurpool_message():
    with pytest.raises(NotImplementedError) as info:
        hb.models.utils.conv_sequence(3, 32, blurpool=True, kernel_size=3, stride=2)
    assert "outside" not in str(info.value)


def test_oracle_blur_matches_reference(g):
    assert len(g["blur"]) == 60
    for case in g["blur"]:
        x, k, s = case["x"], case["k"], case["s"]
        y = O.blur_pool2d(x, k, s)
        dx = O.blur_pool2d_backward(case["w"], x.shape, k, s)
        assert y.dtype == case["y"].dtype and y.shape == case["y"].shape
        if x.dtype == torch.float32:
            torch.testing.assert_close(y, case["y"], rtol=0, atol=1e-6)
            torch.testing.assert_close(dx, case["dx"], rtol=0, atol=1e-6)
        else:
            # bf16: the same fp32 sums rounded once. The reference's y is within one bf16 ulp; its dx rounds the conv's
            # input gradient to bf16 before the reflection adjoint adds the border terms, so it also carries a bf16
            # rounding of the summed terms
            assert ((y.double() - case["y"].double()).abs() <= _ulp_bf16(case["y"])).all(), (k, s)
            terms = O.blur_pool2d_backward(case["w"].double().abs(), x.shape, k, s)
            err = (dx.double() - case["dx"].double()).abs()
            assert (err <= _ulp_bf16(case["dx"]) + 2.0 ** -8 * terms).all(), (k, s)


def _same_bits(a, b):
    """torch.equal with NaN equal to NaN and -0.0 different from +0.0."""
    return (torch.equal(a.isnan(), b.isnan()) and torch.equal(a.nan_to_num(), b.nan_to_num())
            and torch.equal(torch.signbit(a), torch.signbit(b)))


def _check_max_mean(y, ref):
    mx, mean = y
    rmx, rmean = ref
    assert _same_bits(mx, rmx), "max values (a selected zero keeps its sign)"
    tol = 1e-6 if mean.dtype == torch.float32 else _ulp_bf16(rmean)
    assert (((mean.double() - rmean.double()).abs() <= tol) | (mean.isnan() & rmean.isnan())).all()


def test_oracle_global_max_pool_matches_reference(g):
    assert len(g["gmp"]) == 8
    for case in g["gmp"]:
        x = case["x"]
        y, idx = O.global_max_pool2d(x)
        ref = case["y"].view(y.shape)
        assert _same_bits(y, ref)
        dx = O.global_max_pool2d_backward(case["w"], idx, x.shape)
        assert torch.equal(dx, case["dx"]), (case["tag"], x.dtype)


def test_oracle_z_pool_matches_reference(g):
    assert len(g["zpool"]) == 16
    for case in g["zpool"]:
        x, dim = case["x"], case["dim"]
        y, idx = O.z_pool(x, dim)
        _check_max_mean(y.split(1, dim), case["y"].split(1, dim))
        dx = O.z_pool_backward(case["w"], idx, x.shape, dim)
        assert torch.equal(dx, case["dx"]), (case["tag"], dim, x.dtype)


def test_planted_ties_route_as_recorded(g):
    """The planted cases hold what they are for: a NaN row, +-0.0 pairs and ties."""
    case = next(c for c in g["gmp"] if c["tag"] == "planted" and c["x"].dtype == torch.float32)
    y = case["y"].view(2, 5)
    assert y[0, 1].isnan() and y[1, 2].item() == 0.0 and not torch.signbit(y[1, 2])
    assert torch.signbit(y[1, 3]), "-0.0 comes first in (1, 3) and is the value returned"
    assert case["dx"][0, 1].flatten().nonzero().flatten().tolist() == [2 * 7 + 3]
    assert case["dx"][1, 3].flatten().nonzero().flatten().tolist() == [1 * 7 + 1]


def test_no_spills():
    if not LOG.exists():
        pytest.skip(f"{LOG.name} absent: build the library first (python -m holocron_b200.csrc.build)")
    text = LOG.read_text()
    assert "Compiling entry function" in text, f"{LOG.name} holds no ptxas -v output"
    spills = [m.group(0) for m in re.finditer(r"(\d+) bytes spill stores, (\d+) bytes spill loads", text)
              if m.group(1) != "0" or m.group(2) != "0"]
    assert not spills, spills
