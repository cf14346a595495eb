"""fp64 CPU restatement of holocron_b200.transforms: torchvision's tensor resize (torch's upsample filters with
align_corners=False) followed by torchvision's pad, per image.

Each axis is a dense [n_out, n_in] matrix of filter weights, so an image resamples as My @ X @ Mx^T in fp64. Which
source pixels a filter reads, and its weights, are computed in the precision torch computes them in (fp32 for every
dtype but fp64, whose filters are fp64; nearest always uses an fp32 scale): an fp64 position would pick other
neighbours for nearest, and move bilinear / bicubic positions by more than the rounding the kernels are held to. The
weights and sums are fp64. ``magnitude`` is the same sum over absolute values, the scale of the rounding error of any
summation order."""
import numpy as np
import torch

FILTERS = ("nearest", "nearest-exact", "bilinear", "bicubic")
PAD_MODES = ("constant", "edge", "reflect", "symmetric")


def _aa_filter(x, name):
    x = np.abs(x)
    if name == "bilinear":
        return np.where(x < 1, 1 - x, 0.0)
    a = -0.5
    return np.where(x < 1, ((a + 2) * x - (a + 3)) * x * x + 1,
                    np.where(x < 2, (((x - 5) * x + 8) * x - 4) * a, 0.0))


def _cubic(t):
    """Weights of the taps at -1, 0, 1, 2 around a position with fraction t (a = -0.75)."""
    a = -0.75

    def c1(x):
        return ((a + 2) * x - (a + 3)) * x * x + 1

    def c2(x):
        return ((a * x - 5 * a) * x + 8 * a) * x - 4 * a
    return np.stack([c2(t + 1), c1(t), c1(1 - t), c2(2 - t)], -1)


def axis_matrix(n_in: int, n_out: int, name: str, antialias: bool, fp64: bool = False) -> np.ndarray:
    """[n_out, n_in] fp64 weights of resampling one axis from n_in to n_out samples."""
    m = np.zeros((n_out, n_in))
    rows = np.arange(n_out)
    if name in ("nearest", "nearest-exact"):
        scale = np.float32(n_in) / np.float32(n_out)
        pos = rows.astype(np.float32)
        if name == "nearest-exact":
            pos = pos + np.float32(0.5)
        idx = np.minimum(np.floor(pos * scale).astype(np.int64), n_in - 1)
        m[rows, idx] = 1.0
        return m
    wt = np.float64 if fp64 else np.float32
    scale = wt(n_in) / wt(n_out)
    if antialias:
        half = 1.0 if name == "bilinear" else 2.0
        support = wt(half * float(scale)) if scale >= 1 else wt(half)
        invscale = wt(1.0 / float(scale)) if scale >= 1 else wt(1.0)
        center = scale * (rows.astype(wt) + wt(0.5))
        lo = np.maximum(np.trunc(center - support + wt(0.5)).astype(np.int64), 0)
        hi = np.minimum(np.trunc(center + support + wt(0.5)).astype(np.int64), n_in)
        for r in rows:
            j = np.arange(hi[r] - lo[r])
            x = (j.astype(wt) + (wt(lo[r]) - center[r]) + wt(0.5)) * invscale
            w = _aa_filter(x.astype(np.float64), name)
            m[r, lo[r]:hi[r]] = w / w.sum() if w.sum() != 0 else w
        return m
    real = scale * (rows.astype(wt) + wt(0.5)) - wt(0.5)
    if name == "bilinear":
        real = np.maximum(real, wt(0))
        i0 = np.trunc(real).astype(np.int64)
        l1 = (real - i0.astype(wt)).astype(np.float64)
        np.add.at(m, (rows, i0), 1 - l1)
        np.add.at(m, (rows, np.minimum(i0 + 1, n_in - 1)), l1)
        return m
    fl = np.floor(real)
    w = _cubic((real - fl).astype(np.float64))
    for k in range(4):
        np.add.at(m, (rows, np.clip(fl.astype(np.int64) - 1 + k, 0, n_in - 1)), w[:, k])
    return m


def fold(t: np.ndarray, n: int, mode: str) -> np.ndarray:
    """Box coordinates of canvas rows / columns folded into [0, n) by the pad mode, -1 where the canvas is 0."""
    inside = (t >= 0) & (t < n)
    if mode == "constant":
        return np.where(inside, t, -1)
    if mode == "edge":
        return np.clip(t, 0, n - 1)
    if mode == "reflect":
        return np.where(t < 0, -t, np.where(t >= n, 2 * (n - 1) - t, t))
    return np.where(t < 0, -t - 1, np.where(t >= n, 2 * n - 1 - t, t))


def placement(inner, canvas):
    """(top, left) of an inner box on a canvas as torchvision's pad places it (negative: the box is cropped)."""
    return (canvas[0] - inner[0]) // 2, (canvas[1] - inner[1]) // 2


def resize_pad(x: torch.Tensor, inner, canvas, name: str, antialias: bool, pad_mode: str = "constant"):
    """(value, magnitude): fp64 [C, Hc, Wc] arrays of resizing x [C, H, W] to inner = (h, w) and placing it on canvas."""
    fp64 = x.dtype == torch.float64
    xs = x.detach().cpu().double().numpy()
    _, H, W = xs.shape
    h, w = inner
    aa = antialias and name in ("bilinear", "bicubic")
    my, mx = axis_matrix(H, h, name, aa, fp64), axis_matrix(W, w, name, aa, fp64)
    val = np.einsum("yi,cij,xj->cyx", my, xs, mx)
    mag = np.einsum("yi,cij,xj->cyx", np.abs(my), np.abs(xs), np.abs(mx))
    top, left = placement(inner, canvas)
    ry = fold(np.arange(canvas[0]) - top, h, pad_mode)
    rx = fold(np.arange(canvas[1]) - left, w, pad_mode)
    live = (ry[:, None] >= 0) & (rx[None, :] >= 0)
    out = np.where(live, val[:, np.maximum(ry, 0)][:, :, np.maximum(rx, 0)], 0.0)
    mag = np.where(live, mag[:, np.maximum(ry, 0)][:, :, np.maximum(rx, 0)], 0.0)
    return out, mag


def to_uint8(value: np.ndarray) -> np.ndarray:
    """torchvision's cast back to uint8: clamp, round half to even."""
    return np.rint(np.clip(value, 0, 255)).astype(np.uint8)


def tie_distance(value: np.ndarray) -> np.ndarray:
    """Distance of each value to the nearest .5 rounding tie."""
    return np.abs(value - np.floor(value) - 0.5)
