"""Native-dtype NHWC plumbing shared by the pooling and attention bindings (holocron_b200/csrc/pooling.cu,
holocron_b200/csrc/attention.cu): bf16 and fp32 tensors run natively (fp32 is not rounded through bf16: that would
create ties and move the gradient of a max), other float dtypes are computed in fp32 and cast back. Rows are
channels_last with the channel pitch rounded up to one 16-byte vector."""
import torch
from torch import Tensor

from ._fused import _empty_cl


def compute_dtype(dtype: torch.dtype) -> torch.dtype:
    """The dtype the kernels run a tensor of ``dtype`` in."""
    return dtype if dtype in (torch.float32, torch.bfloat16) else torch.float32


def pitch(c: int, dtype: torch.dtype) -> int:
    """Channels per NHWC row: C rounded up to one 16-byte vector."""
    v = 16 // torch.tensor([], dtype=dtype).element_size()
    return (c + v - 1) // v * v


def nhwc(x: Tensor, cp: int) -> Tensor:
    """x as channels_last with a row pitch of ``cp`` channels. The padding channels are left uninitialised: the kernels
    never read them into a result."""
    n, c, h, w = x.shape
    if cp == c:
        return x.contiguous(memory_format=torch.channels_last)
    out = _empty_cl(n, cp, h, w, x.device, x.dtype)
    out[:, :c] = x
    return out


def require_4d(name: str, x: Tensor) -> None:
    if x.ndim != 4:
        raise NotImplementedError(f"{name}: 4-D (N, C, H, W) inputs only, got shape {tuple(x.shape)}")


def crop(t: Tensor, c: int) -> Tensor:
    """The first ``c`` channels of ``t``, a view unless ``t`` has exactly ``c``."""
    return t if t.shape[1] == c else t[:, :c]


def run_native(fn, x: Tensor, *args, crop_channels: bool = True) -> Tensor:
    """Runs ``fn`` in the compute dtype of ``x``, drops the padding channels and casts back to the input dtype."""
    if not x.is_floating_point():
        raise RuntimeError(f"pooling: floating-point input expected, got {x.dtype}")
    dt = compute_dtype(x.dtype)
    y = fn.apply(x if x.dtype == dt else x.to(dt), *args)
    if crop_channels:
        y = crop(y, x.shape[1])
    return y if y.dtype == x.dtype else y.to(x.dtype)
