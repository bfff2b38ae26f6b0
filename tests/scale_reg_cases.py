"""Inputs of the scale regularisation tests (oracle/scale_reg_ref64.py, csrc/scale_reg.cu): log-scale rows [n, 3] that put the
ratio amax(exp) / amin(exp) everywhere the gradient changes form."""
from __future__ import annotations

import math
from typing import Dict

import numpy as np


def exact_ratio_rows(max_ratio: float, n: int, dtype=np.float64, seed: int = 0) -> np.ndarray:
    """n rows [a, a, b] whose exp ratio is exactly ``max_ratio`` when exp and the division are computed in ``dtype`` by numpy
    (a search over a; the float64 ones hold for torch's float64 CPU exp as well)."""
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < n:
        a = dtype(rng.uniform(-6.0, 1.0))
        b0 = dtype(math.log(max_ratio) + float(a))
        for b in (b0, np.nextafter(b0, dtype(np.inf)), np.nextafter(b0, dtype(-np.inf))):
            if np.exp(b) / np.exp(a) == dtype(max_ratio):
                out.append((a, a, b))
                break
    return np.asarray(out, dtype)


def cases(max_ratio: float = 10.0, dtype=np.float64, seed: int = 0) -> Dict[str, np.ndarray]:
    """name -> log scales [n, 3] in ``dtype``."""
    rng = np.random.default_rng(seed)
    lr = math.log(max_ratio)
    a = rng.uniform(-6.0, 1.0, 64)
    c = {}
    c["random"] = (rng.standard_normal((1000, 3)) * 1.5 - 4.0)
    c["all_equal"] = np.repeat(a[:, None], 3, axis=1)
    c["max_tie_2"] = np.stack([a, a + lr + 0.7, a + lr + 0.7], 1)      # two elements share the max, ratio > max_ratio
    c["min_tie_2"] = np.stack([a, a, a + lr + 0.3], 1)                  # two elements share the min
    c["max_tie_2_perm"] = np.stack([a + lr + 1.1, a + 0.2, a + lr + 1.1], 1)
    c["min_tie_2_perm"] = np.stack([a + lr + 2.0, a, a], 1)
    c["distinct_above"] = np.stack([a, a + 0.5, a + lr + 0.5], 1)
    c["distinct_below"] = np.stack([a, a + 0.5, a + lr - 0.5], 1)
    c["just_below"] = np.stack([a, a, a + lr - 1e-6], 1)
    c["just_above"] = np.stack([a, a, a + lr + 1e-6], 1)
    c = {k: np.asarray(v, dtype) for k, v in c.items()}
    c["at_ratio"] = exact_ratio_rows(max_ratio, 16, dtype, seed)
    return c


def segments(rows: np.ndarray, sizes) -> list:
    """``rows`` cut into consecutive segments of the given sizes (the remainder goes to a last one)."""
    out, o = [], 0
    for n in sizes:
        out.append(rows[o:o + n])
        o += n
    if o < rows.shape[0]:
        out.append(rows[o:])
    return out
