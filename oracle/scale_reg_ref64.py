"""float64 statement of the scale regularisation (csrc/scale_reg.cu) and of its gradient.

nerfstudio 1.0's SplatfactoModel.get_loss_dict, with s = exp(scales) [N, 3]:

    scale_reg = 0.1 * mean(max(amax(s) / amin(s), max_ratio) - max_ratio)

The gradient is the one torch autograd gives that expression: torch.maximum hands half of the cotangent to each side when
the ratio equals max_ratio, and amax / amin split theirs evenly between the tied elements of a row.  An element that is
both the max and the min (all three equal) receives both shares.
"""
from __future__ import annotations

from typing import Tuple

import numpy as np


def scale_reg(scales: np.ndarray, max_ratio: float) -> float:
    """The term's value over the rows of ``scales`` [N, 3] (log scales); NaN for N = 0."""
    s = np.exp(np.asarray(scales, np.float64).reshape(-1, 3))
    if s.shape[0] == 0:
        return float("nan")
    r = s.max(axis=1) / s.min(axis=1)
    return float(0.1 * np.mean(np.maximum(r, max_ratio) - max_ratio))


def scale_reg_grad(scales: np.ndarray, max_ratio: float, v: float = 1.0) -> np.ndarray:
    """d scale_reg / d scales * v, [N, 3]; rows with ratio < max_ratio get exact zeros."""
    s = np.exp(np.asarray(scales, np.float64).reshape(-1, 3))
    n = s.shape[0]
    out = np.zeros_like(s)
    if n == 0:
        return out
    mx, mn = s.max(axis=1), s.min(axis=1)
    r = mx / mn
    g = np.where(r > max_ratio, 1.0, np.where(r == max_ratio, 0.5, 0.0)) * (0.1 * v / n)
    is_mx, is_mn = s == mx[:, None], s == mn[:, None]
    d = (is_mx * (g / mn / is_mx.sum(axis=1))[:, None]
         - is_mn * (g * r / mn / is_mn.sum(axis=1))[:, None])
    out[:] = d * s
    return out


def scale_reg_segments(segments, max_ratio: float, v: float = 1.0) -> Tuple[float, list]:
    """Value and per-segment gradients over several segments' scales, concatenated in order (a frame's visible rows)."""
    allrows = np.concatenate([np.asarray(x, np.float64).reshape(-1, 3) for x in segments]) if segments else np.zeros((0, 3))
    val = scale_reg(allrows, max_ratio)
    g = scale_reg_grad(allrows, max_ratio, v)
    out, o = [], 0
    for x in segments:
        k = np.asarray(x).reshape(-1, 3).shape[0]
        out.append(g[o:o + k])
        o += k
    return val, out
