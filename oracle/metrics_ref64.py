"""Float64 statement of the per-step metrics (the reference's ``get_metrics_dict``, street_gaussians_ns/sgn_splatfacto.py:1015-1040,
and the psnr of ``get_image_metrics_and_images``, :1109-1187) from the same fp32 inputs the kernel reads (csrc/metrics.cu).

* psnr = 10 log10(1 / mean((gt*m - rgb*m)^2)) over H*W*3 (torchmetrics PeakSignalNoiseRatio, data_range 1); the products are
  rounded to fp32 as the kernel and torch round them, the rest is exact in float64.  +inf when the images are equal.
* scale_mean = mean(exp(scales)), log_scale_mean = mean(scales), sigmoid_opacity = mean(1 / (1 + exp(-x))) over the rows of
  the given sub-models (exact exp and sigmoid in float64; an exp beyond the fp32 range is inf, as the fp32 exp of the kernel
  and of torch gives), radii_mean = mean(radii).
* A mean over zero rows is NaN, as torch.mean of an empty tensor gives.
"""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np

NAMES = ("psnr", "scale_mean", "log_scale_mean", "sigmoid_opacity", "radii_mean")


def gt_float(gt: np.ndarray) -> np.ndarray:
    """The float image the reference compares against: uint8 / 255 rounded to fp32 (``image.float() / 255``)."""
    if gt.dtype == np.uint8:
        return (gt.astype(np.float32) / np.float32(255.0)).astype(np.float32)
    return gt.astype(np.float32)


def psnr(rgb: np.ndarray, gt: np.ndarray, mask: Optional[np.ndarray] = None) -> float:
    r = rgb.astype(np.float32)
    g = gt_float(gt)
    if mask is not None:
        m = mask.astype(np.float32).reshape(r.shape[0], r.shape[1], 1)
        g, r = (g * m).astype(np.float32), (r * m).astype(np.float32)
    d = g.astype(np.float64) - r.astype(np.float64)  # exact: the difference of two fp32 values rounded once to fp32 by torch
    d = d.astype(np.float32).astype(np.float64)
    sse = float(np.sum((d * d).astype(np.float32).astype(np.float64)))  # the kernel squares in fp32
    if sse == 0.0:
        return float("inf")
    return -10.0 * np.log10(sse / d.size)


def _mean(x: np.ndarray) -> float:
    return float(np.mean(x)) if x.size else float("nan")


def param_means(scales: Sequence[np.ndarray], opacities: Sequence[np.ndarray]):
    """(scale_mean, log_scale_mean, sigmoid_opacity) over the concatenated rows of the given sub-models."""
    s = np.concatenate([np.asarray(a, np.float64).reshape(-1, 3) for a in scales]) if scales else np.zeros((0, 3))
    o = np.concatenate([np.asarray(a, np.float64).reshape(-1) for a in opacities]) if opacities else np.zeros(0)
    with np.errstate(over="ignore"):
        e = np.exp(s)
        e[e.astype(np.float32) == np.inf] = np.inf  # each term is an fp32 value in the kernel and in torch: it overflows there
        sig = 1.0 / (1.0 + np.exp(-o))
    return _mean(e), _mean(s), _mean(sig)


def radii_mean(radii: np.ndarray) -> float:
    r = np.asarray(radii, np.int64)
    return float(r.sum()) / r.size if r.size else float("nan")


def metrics(rgb=None, gt=None, mask=None, scales=None, opacities=None, radii=None) -> np.ndarray:
    """The five values in the kernel's order, float64; a term without inputs is NaN."""
    out = np.full(5, np.nan)
    if rgb is not None:
        out[0] = psnr(rgb, gt, mask)
    if scales is not None:
        out[1:4] = param_means(scales, opacities)
    if radii is not None:
        out[4] = radii_mean(radii)
    return out
