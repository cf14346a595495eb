"""Per-element error bounds for kernels that multiply bf16 operands and accumulate in fp32.

The operands are exact bf16 values, so every product is exact in fp32 and the only errors are the fp32 summation and the
final rounding. For each output element the kernel must then lie within

    one ulp of the output type at the reference value  +  rel * sum|terms|

of an fp64 reference fed the same operands, where sum|terms| is the same operation on the absolute values of the
operands (it bounds the summation error, cancellation included). A whole-tensor relative L2 norm cannot see a fault
confined to a few elements; this bound sees it on the element it touches.

Where a kernel rounds an intermediate to bf16 (the convolution epilogue rounds acc + bias into its staging tile before
it adds the residual), the caller passes half an ulp of that intermediate as ``slack``."""
from typing import Optional

import torch
import torch.nn.functional as TF
from torch.nn.grad import conv2d_input, conv2d_weight

BF16_BITS = 8      # significant bits of bf16
FP32_BITS = 24     # significant bits of fp32


def ulp(ref: torch.Tensor, bits: int = BF16_BITS) -> torch.Tensor:
    """One ulp at each reference value for a format with ``bits`` significant bits (bf16 by default)."""
    a = ref.abs().clamp_min(2.0 ** -126)
    return torch.exp2(torch.floor(torch.log2(a)) - (bits - 1))


def excess(got: torch.Tensor, ref: torch.Tensor, abs_sum: torch.Tensor, rel: float = 1e-5, bits: int = BF16_BITS,
           slack: Optional[torch.Tensor] = None) -> torch.Tensor:
    """|got - ref| minus the bound, per element, in fp64 on ``ref``'s device: positive where the bound is broken."""
    err = (got.detach().to(ref.device, torch.float64) - ref).abs()
    bound = ulp(ref, bits) + rel * abs_sum
    if slack is not None:
        bound = bound + slack
    return err - bound


def assert_within(got: torch.Tensor, ref: torch.Tensor, abs_sum: torch.Tensor, what: str, rel: float = 1e-5,
                  bits: int = BF16_BITS, slack: Optional[torch.Tensor] = None) -> None:
    ex = excess(got, ref, abs_sum, rel, bits, slack)
    bad = ~(ex <= 0)        # NaN fails too: an element left unwritten in a NaN-filled output
    if bad.any():
        first = tuple(int(i) for i in bad.nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements off, worst excess {float(ex.max()):.3e}, "
                             f"first at {first}: got {float(got.detach().double().cpu()[first]):.6g}, "
                             f"ref {float(ref.cpu()[first]):.6g}")


def _f64(t: torch.Tensor, device="cpu") -> torch.Tensor:
    return t.detach().to(device, torch.float64)


def conv_ref(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, stride: int = 1, padding: int = 0,
             dilation: int = 1, groups: int = 1, device="cpu"):
    """(fp64 conv2d, the same conv2d on |x| and |w|) of NCHW ``x`` and OIHW ``w`` (``[Cout, Cin / groups, k, k]``), on
    ``device`` (the CPU by default)."""
    x64, w64 = _f64(x, device), _f64(w, device)
    b64 = None if bias is None else _f64(bias, device)
    ref = TF.conv2d(x64, w64, b64, stride, padding, dilation, groups)
    abs_sum = TF.conv2d(x64.abs(), w64.abs(), None if b64 is None else b64.abs(), stride, padding, dilation, groups)
    return ref, abs_sum


def dgrad_ref(input_shape, w: torch.Tensor, dy: torch.Tensor, stride: int = 1, padding: int = 0, dilation: int = 1,
              groups: int = 1, device="cpu"):
    """(fp64 data gradient of a conv2d with filter ``w`` (OIHW) and output gradient ``dy``, the same on |w| and |dy|)."""
    d64, w64 = _f64(dy, device), _f64(w, device)
    return (conv2d_input(input_shape, w64, d64, stride, padding, dilation, groups),
            conv2d_input(input_shape, w64.abs(), d64.abs(), stride, padding, dilation, groups))


def wgrad_ref(x: torch.Tensor, dy: torch.Tensor, k: int, stride: int = 1, padding: int = 0, dilation: int = 1,
              groups: int = 1, device="cpu"):
    """(fp64 weight gradient [Cout, Cin / groups, k, k], the same on |x| and |dy|) of a conv2d with NCHW input ``x`` and
    output gradient ``dy``."""
    x64, d64 = _f64(x, device), _f64(dy, device)
    shape = (dy.shape[1], x.shape[1] // groups, k, k)
    return (conv2d_weight(x64, shape, d64, stride, padding, dilation, groups),
            conv2d_weight(x64.abs(), shape, d64.abs(), stride, padding, dilation, groups))


def epilogue_ref(acc: torch.Tensor, abs_sum: torch.Tensor, residual: Optional[torch.Tensor] = None, relu: bool = False):
    """Reference, sum|terms| and slack of the convolution epilogue y = act(bf16(acc + bias) + residual): ``acc`` already
    holds the bias. The kernel rounds acc + bias to bf16 before adding the residual: half an ulp of that value is slack."""
    slack = None
    ref = acc
    if residual is not None:
        slack = 0.5 * ulp(acc)
        r64 = _f64(residual)
        ref = acc + r64
        abs_sum = abs_sum + r64.abs()
    if relu:
        ref = ref.clamp_min(0)
    return ref, abs_sum, slack


def check_stats(y, parts, slots, what):
    """The first ``slots`` partials are all written and add up (fp64) to the per-channel sum and sum of squares of the
    stored output within 1e-5 of the sums of their absolute values."""
    c = y.shape[-1]
    p = parts[:slots].double().cpu()
    assert not torch.isnan(p).any(), f"{what}: unwritten statistics slot"
    tot = p.sum(0)
    yf = y.double().cpu().reshape(-1, c)
    for j, v in enumerate((yf, yf * yf)):
        err = (tot[:, j] - v.sum(0)).abs()
        assert bool((err <= 1e-5 * v.abs().sum(0)).all()), f"{what}: statistics {j} off by {float(err.max()):.3e}"
