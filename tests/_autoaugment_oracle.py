"""fp64 / fp32-emulating oracle of the fourteen TrivialAugmentWide ops on uint8 images (torchvision's
``autoaugment._apply_op`` on a tensor), in numpy.

The value-map and blend ops (everything but the affine ops) restate torchvision's tensor arithmetic step by step with
numpy fp32 scalars and arrays, whose operations round like torch's separate elementwise kernels; they are exact.

The affine ops are computed in fp64 from the fp32 matrix and the fp32 grid scale, and each output pixel comes with a
flag: ambiguous when an fp32 evaluation may land on the other side of a rounding decision than the exact value.
Derivation of the band, with u = 2^-24 the fp32 unit roundoff: torch forms the grid as g = x*a + y*b + c (x, y
half-integer pixel centres, a, b, c the fp32 coefficients of theta^T / [w/2, h/2]) with an unspecified order and FMA
use, then ix = ((g + 1)*W - 1) / 2. Whatever the order, the two roundings of partial sums and the final one are each
within u of a magnitude at most T = |x*a| + |y*b| + |c| (the last within u|g|); (g + 1) adds u|g + 1|; the product
with W, with or without an FMA for the -1, adds at most 2u|2 ix + 1| / 2; the halving is exact. So an fp32 ix is
within e_x = u ((W/2)(2T + |g| + |g + 1|) + 2|ix| + 1) of the exact one (likewise e_y), and a result can differ from
the exact one's rounding decision only when the exact value is within that distance of the decision point. The band
is taken as 2 e_x to cover the slack in this tally. Nearest sampling is ambiguous when ix or iy is within its band of
a half-integer (the nearest tap and the in-bounds test both change there). The bilinear value v (out-of-image taps
zero) moves by at most G_x eps_x when ix moves by eps_x, G_x the larger horizontal difference of its taps (likewise
y); with a fill, torchvision returns v*m + (1 - m)*fill, m the same interpolation of the in-image indicator, whose
slope is at most m G_x + |v - fill| M_x (M_x the indicator's difference, nonzero at the image edge only). The fp32
weights, the accumulation and the fill blend add a few roundings of magnitude <= 256. A bilinear pixel is ambiguous
when its exact value is within eps_v = G_x eps_x + G_y eps_y + 16 u 256 of a half-integer, where torch.round may go
either way.
"""
import math

import numpy as np

from torchvision.transforms.functional import _get_inverse_affine_matrix

f32 = np.float32
U = 2.0 ** -24


def gray(img: np.ndarray) -> np.ndarray:
    r, g, b = (c.astype(f32) for c in img)
    return ((f32(0.2989) * r + f32(0.587) * g) + f32(0.114) * b).astype(np.uint8)


def blend(img: np.ndarray, other, ratio: float) -> np.ndarray:
    v = f32(ratio) * img.astype(f32) + f32(1.0 - ratio) * np.asarray(other, dtype=f32)
    return np.clip(v, 0, 255).astype(f32).astype(np.uint8)


def _mean(values: np.ndarray, mean_mode: str) -> np.float32:
    """torch.mean of the fp32 values (exact integers): CPU divides the sum, CUDA multiplies by the fp32 1/N."""
    s, n = f32(int(values.astype(np.int64).sum())), values.size
    return s / f32(n) if mean_mode == "cpu" else s * (f32(1.0) / f32(n))


def _sharpness(img: np.ndarray, ratio: float) -> np.ndarray:
    C, H, W = img.shape
    if H <= 2 or W <= 2:
        return img.copy()
    v = img.astype(np.int64)
    s = 4 * v[:, 1:-1, 1:-1]
    for dy in range(3):
        for dx in range(3):
            s = s + v[:, dy:dy + H - 2, dx:dx + W - 2]
    blurred = img.copy()
    blurred[:, 1:-1, 1:-1] = (2 * s + 13) // 26  # round(s / 13): never a tie
    return blend(img, blurred, ratio)


def _autocontrast(img: np.ndarray) -> np.ndarray:
    out = np.empty_like(img)
    for c, ch in enumerate(img):
        mn, mx = f32(ch.min()), f32(ch.max())
        with np.errstate(divide="ignore"):
            scale = (f32(1) / (mx - mn)) * f32(255)  # torch's 255 / t is t.reciprocal() * 255
        if not np.isfinite(scale):
            mn, scale = f32(0), f32(1)
        out[c] = np.clip((ch.astype(f32) - mn) * scale, 0, 255).astype(np.uint8)
    return out


def _equalize(img: np.ndarray) -> np.ndarray:
    out = np.empty_like(img)
    for c, ch in enumerate(img):
        hist = np.bincount(ch.reshape(-1), minlength=256).astype(np.int64)
        nz = hist[hist != 0]
        step = int(nz[:-1].sum()) // 255
        if step == 0:
            out[c] = ch
            continue
        lut = (np.cumsum(hist) + step // 2) // step
        lut = np.clip(np.concatenate([[0], lut[:-1]]), 0, 255)
        out[c] = lut[ch].astype(np.uint8)
    return out


def affine_matrix(op: str, magnitude: float, H: int, W: int):
    """The inverse matrix torchvision's _apply_op builds through F.affine / F.rotate."""
    if op == "ShearX":
        return _get_inverse_affine_matrix([-0.5 * W, -0.5 * H], 0.0, [0.0, 0.0], 1.0,
                                          [math.degrees(math.atan(magnitude)), 0.0])
    if op == "ShearY":
        return _get_inverse_affine_matrix([-0.5 * W, -0.5 * H], 0.0, [0.0, 0.0], 1.0,
                                          [0.0, math.degrees(math.atan(magnitude))])
    if op == "TranslateX":
        return _get_inverse_affine_matrix([0.0, 0.0], 0.0, [1.0 * int(magnitude), 0.0], 1.0, [0.0, 0.0])
    if op == "TranslateY":
        return _get_inverse_affine_matrix([0.0, 0.0], 0.0, [0.0, 1.0 * int(magnitude)], 1.0, [0.0, 0.0])
    assert op == "Rotate"
    return _get_inverse_affine_matrix([0.0, 0.0], -magnitude, [0.0, 0.0], 1.0, [0.0, 0.0])


def _affine(img: np.ndarray, matrix, bilinear: bool, fill):
    C, H, W = img.shape
    m = np.array(matrix, dtype=f32)
    ca = (m[:3] / f32(0.5 * W)).astype(np.float64)
    cb = (m[3:] / f32(0.5 * H)).astype(np.float64)
    x = (np.arange(W) - W * 0.5 + 0.5)[None, :]
    y = (np.arange(H) - H * 0.5 + 0.5)[:, None]
    gx = x * ca[0] + y * ca[1] + ca[2]
    gy = x * cb[0] + y * cb[1] + cb[2]
    ix = ((gx + 1) * W - 1) / 2
    iy = ((gy + 1) * H - 1) / 2
    tx = np.abs(x * ca[0]) + np.abs(y * ca[1]) + abs(ca[2])
    ty = np.abs(x * cb[0]) + np.abs(y * cb[1]) + abs(cb[2])
    eps_x = 2 * U * (W / 2 * (2 * tx + np.abs(gx) + np.abs(gx + 1)) + 2 * np.abs(ix) + 1)
    eps_y = 2 * U * (H / 2 * (2 * ty + np.abs(gy) + np.abs(gy + 1)) + 2 * np.abs(iy) + 1)
    fillv = None if fill is None else np.broadcast_to(np.array(fill, dtype=np.float64), (C,))
    src = img.astype(np.float64)
    if not bilinear:
        xi, yi = np.rint(ix).astype(np.int64), np.rint(iy).astype(np.int64)
        inb = (xi >= 0) & (xi < W) & (yi >= 0) & (yi < H)
        val = src[:, np.clip(yi, 0, H - 1), np.clip(xi, 0, W - 1)]
        other = np.zeros(C) if fillv is None else np.rint(fillv)
        out = np.where(inb[None], val, other[:, None, None])
        amb = (np.abs(ix - np.floor(ix) - 0.5) < eps_x) | (np.abs(iy - np.floor(iy) - 0.5) < eps_y)
        return out.astype(np.uint8), amb
    x0, y0 = np.floor(ix).astype(np.int64), np.floor(iy).astype(np.int64)
    fx, fy = ix - x0, iy - y0
    taps, inside = {}, {}
    for dy in (0, 1):
        for dx in (0, 1):
            xx, yy = x0 + dx, y0 + dy
            inside[dy, dx] = ((xx >= 0) & (xx < W) & (yy >= 0) & (yy < H)).astype(np.float64)
            taps[dy, dx] = inside[dy, dx] * src[:, np.clip(yy, 0, H - 1), np.clip(xx, 0, W - 1)]

    def lerp(t):
        return (1 - fy) * ((1 - fx) * t[0, 0] + fx * t[0, 1]) + fy * ((1 - fx) * t[1, 0] + fx * t[1, 1])

    def slopes(t):
        return (np.maximum(np.abs(t[0, 1] - t[0, 0]), np.abs(t[1, 1] - t[1, 0])),
                np.maximum(np.abs(t[1, 0] - t[0, 0]), np.abs(t[1, 1] - t[0, 1])))

    val = lerp(taps)
    g_x, g_y = slopes(taps)
    if fillv is not None:
        mask = lerp(inside)
        m_x, m_y = slopes(inside)
        # v*m + (1 - m)*fill: its slope is at most m G + |v - fill| M per axis
        g_x = mask * g_x + np.abs(val - fillv[:, None, None]) * m_x
        g_y = mask * g_y + np.abs(val - fillv[:, None, None]) * m_y
        val = val * mask + (1 - mask) * fillv[:, None, None]
    eps_v = g_x * eps_x + g_y * eps_y + 16 * U * 256
    amb = (np.abs(val - np.floor(val) - 0.5) < eps_v).any(0)
    return np.clip(np.rint(val), 0, 255).astype(np.uint8), amb


def apply_op(img: np.ndarray, op: str, magnitude: float, bilinear: bool, fill, mean_mode: str = "cuda"):
    """(output uint8 [C, H, W], ambiguous bool [H, W]) of torchvision's _apply_op on the uint8 image [C, H, W]. ``fill``
    is None or a list of 1 or C values; ``mean_mode`` is the device whose torch.mean Contrast reproduces."""
    C, H, W = img.shape
    none = np.zeros((H, W), dtype=bool)
    if op in ("ShearX", "ShearY", "TranslateX", "TranslateY", "Rotate"):
        return _affine(img, affine_matrix(op, magnitude, H, W), bilinear, fill)
    r = 1.0 + magnitude
    if op == "Identity":
        out = img.copy()
    elif op == "Brightness":
        out = blend(img, 0.0, r)
    elif op == "Color":
        out = img.copy() if C == 1 else blend(img, gray(img)[None], r)
    elif op == "Contrast":
        out = blend(img, _mean(gray(img) if C == 3 else img, mean_mode), r)
    elif op == "Sharpness":
        out = _sharpness(img, r)
    elif op == "Posterize":
        out = img & np.uint8(-int(2 ** (8 - int(magnitude))) & 0xFF)
    elif op == "Solarize":
        out = np.where(img.astype(f32) >= f32(magnitude), 255 - img, img).astype(np.uint8)
    elif op == "AutoContrast":
        out = _autocontrast(img)
    elif op == "Equalize":
        out = _equalize(img)
    else:
        raise ValueError(op)
    return out, none
