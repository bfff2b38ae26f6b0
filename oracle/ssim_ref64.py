"""Float64 numpy statement of the SSIM loss term and its gradient for rgb (the specification of csrc/ssim.cu).

    loss = weight * (1 - mean_{c,i,j} S_c(i,j)),   x = gt * mask, y = rgb * mask
    S = l * cs,  l = (2 mu_x mu_y + C1) / (mu_x^2 + mu_y^2 + C1),  cs = (2 s_xy + C2) / (s_x + s_y + C2)

with mu, E[x^2], E[y^2], E[xy] the separable 11-tap Gaussian filter (sigma 1.5) of x, y, x^2, y^2, xy with valid padding
(the map is (H-10) x (W-10) per channel), s_x = E[x^2] - mu_x^2, s_y = E[y^2] - mu_y^2, s_xy = E[xy] - mu_x mu_y.

The gradient goes through the three maps a = dS/dmu_y, b = dS/dE[y^2], c = dS/dE[xy] (each with the other moments held
fixed) and the transposed (full) filter G^T:

    dL/drgb(q) = k [ (G^T a)(q) + 2 y(q) (G^T b)(q) + x(q) (G^T c)(q) ] mask(q),   k = -weight * g / (3 (H-10) (W-10))

Images are [H, W, 3] (rgb, gt in [0, 1]), the mask [H, W, 1] or None.  The default window is torch's fp32
``_gauss_window(11, 1.5)`` (what the kernels use), promoted to float64."""
from __future__ import annotations

import numpy as np

C1, C2 = 0.01 ** 2, 0.03 ** 2


# torch's float32 _gauss_window(11, 1.5) (exp, then division by the sum), bit for bit: the taps csrc/ssim.cu uses
TAPS_F32 = np.array([float.fromhex(h) for h in (
    "0x1.0d957p-10", "0x1.f1fe02p-8", "0x1.26eb18p-5", "0x1.bff0fep-4", "0x1.b43c3ep-3", "0x1.10656p-2",
    "0x1.b43c3ep-3", "0x1.bff0fep-4", "0x1.26eb18p-5", "0x1.f1fe02p-8", "0x1.0d957p-10")], dtype=np.float32)


def window(size: int = 11, sigma: float = 1.5) -> np.ndarray:
    """The same window evaluated in float64."""
    x = np.arange(size, dtype=np.float64) - size // 2
    g = np.exp(-(x ** 2) / (2 * sigma ** 2))
    return g / g.sum()


def _valid(a: np.ndarray, w: np.ndarray, axis: int) -> np.ndarray:
    n = a.shape[axis] - len(w) + 1
    out = np.zeros(a.shape[:axis] + (n,) + a.shape[axis + 1:])
    for t, wt in enumerate(w):
        out += wt * np.take(a, np.arange(t, t + n), axis=axis)
    return out


def _full_t(a: np.ndarray, w: np.ndarray, axis: int) -> np.ndarray:
    """Transpose of _valid: out[q] = sum_t w[t] a[q - t], zero outside a."""
    n = a.shape[axis] + len(w) - 1
    out = np.zeros(a.shape[:axis] + (n,) + a.shape[axis + 1:])
    for t, wt in enumerate(w):
        sl = [slice(None)] * a.ndim
        sl[axis] = slice(t, t + a.shape[axis])
        out[tuple(sl)] += wt * a
    return out


def filt(a: np.ndarray, w: np.ndarray) -> np.ndarray:
    return _valid(_valid(a, w, 0), w, 1)


def filt_t(a: np.ndarray, w: np.ndarray) -> np.ndarray:
    return _full_t(_full_t(a, w, 0), w, 1)


def ssim_loss(rgb, gt, mask=None, weight: float = 1.0, grad: float = 1.0, taps=None):
    """Returns (loss, d(grad * loss)/d rgb [H,W,3], maps) in float64; maps = dict(S, a, b, c), each [H-10, W-10, 3]."""
    w = np.asarray(TAPS_F32 if taps is None else taps, dtype=np.float64)
    y = np.asarray(rgb, dtype=np.float64)
    x = np.asarray(gt, dtype=np.float64)
    H, W, _ = y.shape
    if H < len(w) or W < len(w):
        raise ValueError(f"SSIM needs an image of at least {len(w)} x {len(w)} pixels, got {H} x {W}")
    m = np.ones((H, W, 1)) if mask is None else np.asarray(mask, dtype=np.float64).reshape(H, W, 1)
    x, y = x * m, y * m
    mu1, mu2 = filt(x, w), filt(y, w)
    e11, e22, e12 = filt(x * x, w), filt(y * y, w), filt(x * y, w)
    s1, s2, s12 = e11 - mu1 ** 2, e22 - mu2 ** 2, e12 - mu1 * mu2
    A, B = 2 * mu1 * mu2 + C1, mu1 ** 2 + mu2 ** 2 + C1
    Cn, D = 2 * s12 + C2, s1 + s2 + C2
    lum, cs = A / B, Cn / D
    S = lum * cs
    loss = weight * (1.0 - S.mean())
    a = (2 * mu1 / B - 2 * mu2 * A / B ** 2) * cs + lum * (-2 * mu1 / D + 2 * mu2 * Cn / D ** 2)
    b = -lum * Cn / D ** 2
    c = 2 * lum / D
    k = -weight * grad / S.size
    v = k * (filt_t(a, w) + 2 * y * filt_t(b, w) + x * filt_t(c, w)) * m
    return float(loss), v, dict(S=S, a=a, b=b, c=c)
