"""Inputs of the bilateral-grid kernel tests (tests/test_gpu_bilagrid.py): grid shapes, image sizes and colour
distributions, all seeded.

The slice blocks are 64 columns x 32 rows of one grid cell; the sizes include images smaller than a block, sizes that are not
multiples of it, images with fewer pixels than grid cells, and the 1920 x 1280 of the Waymo rig.  The colour distribution puts
pixels on both clamp boundaries of the guidance: black (gray exactly 0), grays beyond 1 and below 0, and colours whose float32
gray is exactly 1."""
from __future__ import annotations

import numpy as np

from oracle.bilagrid_ref64 import IDENTITY

# (L, Hg, Wg, H, W)
SLICE_CASES = {
    "default_1x1": (8, 16, 16, 1, 1),
    "default_7x13": (8, 16, 16, 7, 13),
    "default_65x130": (8, 16, 16, 65, 130),
    "default_97x211": (8, 16, 16, 97, 211),
    "nonsquare_4x9x3": (3, 4, 9, 50, 77),
    "depth1": (1, 5, 6, 33, 40),
    "one_node_xy": (4, 1, 1, 20, 70),
    "deep": (32, 3, 4, 40, 60),
    "rig_1280x1920": (8, 16, 16, 1280, 1920),
}

TV_CASES = {  # (N, L, Hg, Wg)
    "one_default": (1, 8, 16, 16),
    "rig_425": (425, 8, 16, 16),
    "nonsquare": (3, 3, 4, 9),
    "depth1": (2, 1, 5, 6),
    "one_node_xy": (5, 4, 1, 1),
}


def identity(L: int, Hg: int, Wg: int) -> np.ndarray:
    return np.tile(np.asarray(IDENTITY, np.float32).reshape(12, 1, 1, 1), (1, L, Hg, Wg))


def random_grid(L: int, Hg: int, Wg: int, seed: int, scale: float = 0.25) -> np.ndarray:
    rng = np.random.default_rng(seed)
    return (identity(L, Hg, Wg) + scale * rng.standard_normal((12, L, Hg, Wg))).astype(np.float32)


def colours(H: int, W: int, seed: int) -> np.ndarray:
    """[H, W, 3] float32: mostly uniform in [0, 1], with 3 % black, 3 % above 1, 3 % below 0, 3 % of float32 gray exactly 1 and
    3 % in smooth patches (neighbouring pixels on the same grid level)."""
    rng = np.random.default_rng(seed)
    c = rng.uniform(0.0, 1.0, (H, W, 3)).astype(np.float32)
    u = rng.uniform(size=(H, W))
    c[u < 0.03] = 0.0
    c[(u >= 0.03) & (u < 0.06)] = rng.uniform(1.05, 1.5, (int(((u >= 0.03) & (u < 0.06)).sum()), 3)).astype(np.float32)
    c[(u >= 0.06) & (u < 0.09)] = rng.uniform(-0.5, -0.05, (int(((u >= 0.06) & (u < 0.09)).sum()), 3)).astype(np.float32)
    c[(u >= 0.09) & (u < 0.12)] = ones_gray()
    c[(u >= 0.12) & (u < 0.15)] = np.float32(0.42)
    return c


def ones_gray() -> np.ndarray:
    """A colour whose float32 gray, (0.299 r + 0.587 g) + 0.114 b with one rounding per operation, is exactly 1."""
    f = np.float32
    for b in (f(1.0), np.nextafter(f(1.0), f(2.0)), np.nextafter(f(1.0), f(0.0))):
        for r in (f(1.0), np.nextafter(f(1.0), f(2.0)), np.nextafter(f(1.0), f(0.0))):
            c = np.array([r, 1.0, b], np.float32)
            if (f(0.299) * c[0] + f(0.587) * c[1]) + f(0.114) * c[2] == f(1.0):
                return c
    raise AssertionError("no colour with float32 gray 1 near white")


def cotangent(H: int, W: int, seed: int) -> np.ndarray:
    return np.random.default_rng(seed).standard_normal((H, W, 3)).astype(np.float32)
