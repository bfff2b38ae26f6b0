"""Named, seeded inputs for the depth and semantic kernels (csrc/depth.cu, csrc/semantic.cu), and the fp32 error floors their
results are held to.  oracle/depth_ref64.py and tests/semantic_cases.py state what the kernels compute, edge values included.

  * SIZES: images from 1x1 to 1920x1280: P just under and just over one block (256), one pixel either side of the loss grid
    (1056 x 256 = 270336 threads), and two sizes above 2^21 that the grid does not divide;
  * depth_pixels: depth / target / mask images whose first pixels carry the rule edges (DEPTH_EDGES): targets that are negative,
    -0.0 or NaN, masks of -0.0, fractional or NaN, D == T, and ratios exactly at the metric thresholds and just inside them;
  * sem_inputs: logits, int64 labels (with label_edges: -1, C, 255, 2^31, -2^40) and masks (-0.0 and fractional), plain,
    "confident" (the label is the arg-max by a margin of 10 to 20, shifted by an offset) or "ties" (logits on a half-integer
    grid: many equal maxima);
  * CarryCase: hand-built refinement plans (flags, prefix sums, totals) for widths 1 .. 64 and 1 .. 16 split samples.

The floors are a few fp32 ulps (U = 2^-24) of each pixel's own terms, summed the way the kernel sums them."""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional

import numpy as np

U = 2.0 ** -24
f32 = np.float32
GRID = 1056 * 256  # DEPTH_BLOCKS / SEM_BLOCKS x 256 threads: one pass of the loss and metric kernels

SIZES = [(1, 1), (1, 255), (255, 1), (16, 16), (17, 15), (1, GRID - 1), (1, GRID + 1), (1280, 1920), (1447, 1451)]
assert (1447 * 1451) > 2 ** 21 and (1447 * 1451) % GRID and (1280 * 1920) % GRID


def size_id(hw) -> str:
    return f"{hw[0]}x{hw[1]}"


# ---- depth ----------------------------------------------------------------------------------------------------------------
_nx = np.nextafter
NAN = f32("nan")

# (D, T, mask): one pixel per rule (mask 1 where the rule is not about the mask)
DEPTH_EDGES = [
    (3.0, -2.0, 1.0), (3.0, -0.0, 1.0), (3.0, NAN, 1.0), (3.0, 0.0, 1.0),        # invalid targets
    (3.0, 2.0, -0.0), (3.0, 2.0, 0.0), (3.0, 2.0, 0.25), (3.0, 2.0, NAN),        # masks: -0.0 / 0 drop, 0.25 / NaN keep
    (7.5, 7.5, 1.0), (0.0, 0.0, 1.0),                                           # D == T: zero cotangent (T = 0 invalid)
    (5.0, 4.0, 1.0), (4.0, 5.0, 1.0), (25.0, 16.0, 1.0), (16.0, 25.0, 1.0),      # r = 1.25 and 1.5625 exactly
    (125.0, 64.0, 1.0), (64.0, 125.0, 1.0),                                     # r = 1.953125 exactly
    (float(_nx(f32(5.0), f32(0))), 4.0, 1.0), (float(_nx(f32(25.0), f32(0))), 16.0, 1.0),  # just inside each threshold
    (float(_nx(f32(125.0), f32(0))), 64.0, 1.0),
    (0.0, 2.0, 1.0), (-1.0, 2.0, 1.0), (1e-4, 2.0, 1.0),                        # clamped to 1e-3 in the metrics
]


def depth_pixels(H: int, W: int, seed: int, mask: Optional[str] = "frac", edges: bool = True):
    """(D, T, mask or None) float32 [H, W]: depths in (0.5, 30.5), a return on about a third of the pixels, the rule edges first."""
    rng = np.random.default_rng(seed)
    P = H * W
    D = (rng.random(P) * 30 + 0.5).astype(f32)
    T = np.where(rng.random(P) < 0.35, rng.random(P) * 30 + 0.5, 0.0).astype(f32)
    tie = rng.random(P) < 0.02
    D[tie] = T[tie]
    M = None
    if mask == "frac":
        M = rng.random(P).astype(f32)
        M[rng.random(P) < 0.2] = 0.0
        M[rng.random(P) < 0.05] = -0.0
        M[rng.random(P) < 0.3] = 1.0
    elif mask == "binary":
        M = (rng.random(P) > 0.3).astype(f32)
    if edges:
        k = min(len(DEPTH_EDGES), P)
        e = np.array(DEPTH_EDGES[:k], f32)
        D[:k], T[:k] = e[:, 0], e[:, 1]
        if M is not None:
            M[:k] = e[:, 2]
        else:  # without a mask, the mask rules do not apply: those pixels keep an ordinary valid target
            T[:k][np.array([m != 1.0 for m in e[:, 2]])] = 2.0
    return D.reshape(H, W), T.reshape(H, W), None if M is None else M.reshape(H, W)


def depth_loss_floor(D, T, ok, w: float) -> float:
    """|D - T| rounded once per pixel, summed in fp64, the mean rounded once to fp32: two ulps of each."""
    e = np.abs(D.astype(np.float64).reshape(-1)[ok] - T.astype(np.float64).reshape(-1)[ok])
    n = max(int(ok.sum()), 1)
    L = abs(w) * e.sum() / n
    return 2 * U * (abs(w) * e.sum() / n + L)


# ---- semantic -------------------------------------------------------------------------------------------------------------
def label_edges(C: int) -> List[int]:
    return [-1, C, 255, 2 ** 31, -2 ** 40]


SEM_CLASSES = [1, 2, 7, 8, 31, 32, 33, 63, 64]


def sem_inputs(H: int, W: int, C: int, seed: int, kind: str = "plain", offset: float = 0.0, mask: Optional[str] = "frac"):
    """(logits float32 [H, W, C], labels int64 [H, W], mask float32 [H, W] or None)."""
    rng = np.random.default_rng([seed, C, H, W])
    P = H * W
    lab = rng.integers(0, C, P).astype(np.int64)
    if kind == "ties":
        x = (np.round(rng.standard_normal((P, C)) * 2) / 2).astype(f32)
        x[: P // 8] = 0.5  # every class ties
    else:
        x = (rng.standard_normal((P, C)) * 3).astype(f32)
    if kind == "confident":  # the label wins by 10 .. 20 over the largest other logit
        x = rng.standard_normal((P, C)).astype(f32)
        x[np.arange(P), lab] = x.max(axis=1) + rng.uniform(10, 20, P).astype(f32)
        x = (x + f32(offset)).astype(f32)
    ign = rng.random(P) < 0.1
    ign[-1] = False  # the last pixel keeps an in-range label: an out-of-range label there would index past the buffers
    edges = np.array(label_edges(C), np.int64)
    lab[ign] = edges[rng.integers(0, len(edges), int(ign.sum()))]
    M = None
    if mask == "frac":
        M = rng.random(P).astype(f32)
        M[rng.random(P) < 0.15] = 0.0
        M[rng.random(P) < 0.05] = -0.0
        M[rng.random(P) < 0.3] = 1.0
    return x.reshape(H, W, C), lab.reshape(H, W), None if M is None else M.reshape(H, W)


def ce_floor(s, lab) -> np.ndarray:
    """Per-pixel floor of the kernel's CE = (m - S[l]) + log1p(z1), z1 = sum over the other classes of exp(S - m): two ulps of
    |m - S[l]| and of CE, and of z1's own terms (each exp argument rounded, C sequential adds) as they pass through log1p."""
    s = np.asarray(s, np.float64)
    n, C = s.shape
    r = np.arange(n)
    a = s.argmax(axis=1)
    m = s[r, a]
    t = np.exp(s - m[:, None])
    t[r, a] = 0.0
    z1 = t.sum(axis=1)
    d = np.abs(m - s[r, lab])
    ce = d + np.log1p(z1)
    return 2 * U * (d + ce + (t * (C + 4 + np.abs(s - m[:, None]))).sum(axis=1) / (1 + z1))


def grad_floor(s, lab, k: float) -> np.ndarray:
    """Per-element floor of the kernel's k (softmax - onehot), softmax = exp(S - m) / z with z summed sequentially over C
    classes (k = g w / n itself rounded twice)."""
    s = np.asarray(s, np.float64)
    n, C = s.shape
    m = s.max(axis=1, keepdims=True)
    e = np.exp(s - m)
    p = e / e.sum(axis=1, keepdims=True)
    sbar = (p * np.abs(s - m)).sum(axis=1, keepdims=True)
    one = np.zeros_like(p)
    one[np.arange(n), lab] = 1.0
    return 2 * U * abs(k) * ((C + 6 + np.abs(s - m) + sbar) * p + 2 * one) + abs(k) * 1e-38


# ---- refinement carry -------------------------------------------------------------------------------------------------------
RF_SPLIT, RF_DUP, RF_KEEP_ORIG, RF_KEEP_SPLIT, RF_KEEP_DUP = 0x01, 0x02, 0x04, 0x08, 0x10


@dataclass
class CarryCase:
    name: str
    n: int
    width: int
    n_split_samples: int
    moments: bool
    culled: bool = False  # every row culled: no output row
    seed: int = 0

    def plan(self):
        """(flags uint8 [n], scan int32 [4, n], totals [4]): rows culled, kept, split (its original removed, some of its
        samples culled with it), duplicated, and split rows whose samples are all culled (counted in totals[3] only)."""
        rng = np.random.default_rng(500 + self.seed)
        kind = rng.integers(0, 5, self.n)
        f = np.zeros(self.n, np.uint8)
        if not self.culled:
            f[kind == 1] = RF_KEEP_ORIG
            f[kind == 2] = RF_SPLIT | RF_KEEP_SPLIT
            f[kind == 3] = RF_DUP | RF_KEEP_ORIG | RF_KEEP_DUP
            f[kind == 4] = RF_SPLIT
        marks = np.stack([(f & b) != 0 for b in (RF_KEEP_ORIG, RF_KEEP_SPLIT, RF_KEEP_DUP, RF_SPLIT)]).astype(np.int32)
        scan = np.cumsum(marks, axis=1, dtype=np.int32)
        totals = [int(x) for x in scan[:, -1]] if self.n else [0, 0, 0, 0]
        return f, scan, totals

    def out_rows(self, totals) -> int:
        return totals[0] + self.n_split_samples * totals[1] + totals[2]


def _carry_cases() -> List[CarryCase]:
    out = []
    for w in (1, 2, 3, 63, 64):
        for s in (1, 2, 16):
            for mom in (False, True):
                out.append(CarryCase(f"w{w}_s{s}_{'m' if mom else 'nom'}", 3001, w, s, mom))
    out.append(CarryCase("n0", 0, 5, 2, True))
    out.append(CarryCase("all_culled_w64", 777, 64, 2, True, culled=True))
    out.append(CarryCase("all_culled_w1", 777, 1, 16, False, culled=True))
    for i, c in enumerate(out):
        c.seed = i
    return out


CARRY_CASES = _carry_cases()
