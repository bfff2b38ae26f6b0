"""Named, seeded inputs for the step kernels after the render (oracle/step_ref64.py states what they compute):

  * LOSS_CASES: images from 1x1 to 1920x1280 (3P odd, 3P = 2 mod 4, multiples of 4), float and uint8 ground truth,
    with and without a mask (binary and fractional), views offset by 1..3 floats / bytes, each term alone;
  * DENSIFY_CASES: segment tables (one segment, 33, 1024, empty segments first / in the middle / last, a first row0 > 0
    with gaps, mixed ``first`` flags) on images with H > W, W > H and max(H, W) not a power of two;
  * EXCHANGE_CASES: slice lists for the two-shot exchange (short and empty slices, 48 slices, row-skipping slices of
    widths 1 .. 45 with row0 > 0, padding and union patterns) at world sizes 1, 2, 3, 4, 8.

Every object_acc carries the entropy's edge values (OA_EDGES) in its first pixels, and about a tenth of the rgb values
tie with the ground truth as the kernel reads it (u8 / 255.f), so their gradient must be exactly 0."""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional, Tuple

import numpy as np

from oracle.step_ref64 import CLAMP_HI, CLAMP_LO, gt_f32

f32 = np.float32
_nx = np.nextafter
OA_EDGES = np.array([CLAMP_LO, CLAMP_HI, _nx(CLAMP_LO, f32(0)), _nx(CLAMP_LO, f32(1)), _nx(CLAMP_HI, f32(0)),
                     _nx(CLAMP_HI, f32(1)), 0.0, 1.0, 0.5, _nx(f32(0.5), f32(0)), _nx(f32(0.5), f32(1)), 0.5 + 2 ** -20,
                     0.5 - 2 ** -20, 0.4999, 0.5001], f32)


# ---- loss epilogue -------------------------------------------------------------------------------------------------------
@dataclass
class LossCase:
    name: str
    H: int
    W: int
    gt: str = "f32"                       # "f32" or "u8"
    mask: Optional[str] = None            # None, "binary" or "frac"
    off: Tuple[int, int, int] = (0, 0, 0)  # float offsets of the rgb, gt (float) and v_rgb views from 16-byte alignment
    u8_off: int = 0                       # byte offset of a uint8 ground truth
    terms: Tuple[str, ...] = ("l1", "sky", "ent")
    w: Tuple[float, float, float] = (0.8, 1.0, 0.001)
    seed: int = 0

    @property
    def P(self) -> int:
        return self.H * self.W


def loss_inputs(c: LossCase) -> dict:
    """Host arrays: rgb [H,W,3] f32, gt (f32 or u8) [H,W,3], mask [H,W,1] or None, accumulation, sky_mask (u8), object_acc."""
    rng = np.random.default_rng(1000 + c.seed)
    H, W = c.H, c.W
    if c.gt == "u8":
        gt = rng.integers(0, 256, (H, W, 3)).astype(np.uint8)
    else:
        gt = rng.random((H, W, 3), dtype=np.float32)
    rgb = rng.random((H, W, 3), dtype=np.float32)
    tie = rng.random((H, W, 3)) < 0.1
    rgb[tie] = gt_f32(gt)[tie]
    mask = None
    if c.mask == "binary":
        mask = (rng.random((H, W, 1)) > 0.3).astype(f32)
    elif c.mask == "frac":
        mask = rng.random((H, W, 1), dtype=np.float32)
        mask[rng.random((H, W, 1)) < 0.2] = 0.0
        mask[rng.random((H, W, 1)) < 0.2] = 1.0
    acc = rng.random((H, W, 1), dtype=np.float32)
    sky = (rng.random((H, W, 1)) < 0.3).astype(np.uint8)
    oa = rng.random((H, W, 1), dtype=np.float32)
    flat = oa.reshape(-1)
    k = min(len(OA_EDGES), flat.size)
    flat[:k] = OA_EDGES[:k]
    return dict(rgb=rgb if "l1" in c.terms else None, gt=gt if "l1" in c.terms else None, mask=mask if "l1" in c.terms else None,
                accumulation=acc if "sky" in c.terms else None, sky_mask=sky if "sky" in c.terms else None,
                object_acc=oa if "ent" in c.terms else None)


SHAPES = [(1, 1), (1, 3), (3, 5), (7, 1), (2, 1), (6, 3), (16, 16), (240, 320), (1280, 1920)]


def _loss_cases() -> List[LossCase]:
    out = []
    for H, W in SHAPES:
        big = H * W > 100_000
        variants = [dict(), dict(gt="u8"), dict(mask="binary"), dict(gt="u8", mask="frac"), dict(off=(1, 0, 0)),
                    dict(gt="u8", u8_off=3)]
        if not big:
            variants += [dict(mask="frac"), dict(off=(0, 2, 0)), dict(off=(0, 0, 3)), dict(off=(3, 3, 3), mask="binary"),
                         dict(gt="u8", u8_off=1), dict(gt="u8", u8_off=2, off=(2, 0, 1))]
        for i, v in enumerate(variants):
            tag = "_".join(f"{k}{'-'.join(map(str, x)) if isinstance(x, tuple) else x}" for k, x in v.items()) or "plain"
            out.append(LossCase(f"{H}x{W}_{tag}", H, W, seed=len(out), **v))
    # each term alone (the other inputs null), with its weight zero and non-zero
    for t in ("l1", "sky", "ent"):
        for wv in (0.0, 1.7):
            w = tuple(wv if x == t else 1.0 for x in ("l1", "sky", "ent"))
            out.append(LossCase(f"only_{t}_w{wv}", 16, 16, terms=(t,), w=w, seed=len(out)))
    out.append(LossCase("only_l1_u8_mask_w0.5", 6, 3, gt="u8", mask="binary", terms=("l1",), w=(0.5, 0.0, 0.0), seed=len(out)))
    return out


LOSS_CASES = _loss_cases()


# ---- densification statistics -------------------------------------------------------------------------------------------
@dataclass
class DensifyCase:
    name: str
    H: int
    W: int
    N: int
    segs: List[Tuple[int, int, int]]  # (row0, count, first)
    seed: int = 0

    def inputs(self, call: int):
        """v_records [N, 12] f32 (v_xy in columns 0, 1) and radii [N] i32 of call ``call``: zeros, negative and positive radii
        (radius 0 or below is invisible), exact-zero gradients, gradients from 1e-20 to 1e3."""
        rng = np.random.default_rng(7000 + 31 * self.seed + call)
        v = np.zeros((self.N, 12), f32)
        v[:] = rng.normal(size=(self.N, 12)).astype(f32) * 1e-3
        v[:, 0:2] *= (10.0 ** rng.uniform(-17, 6, (self.N, 1))).astype(f32)
        v[rng.random(self.N) < 0.05, 0:2] = 0.0
        radii = rng.integers(-3, 40, self.N).astype(np.int32)
        radii[rng.random(self.N) < 0.3] = 0
        radii[rng.random(self.N) < 0.02] = rng.integers(500, 3000, 1)[0]
        return v, radii

    def prior(self, count: int, s: int):
        """Statistics of a segment before a call with first = 0: what earlier calls left."""
        rng = np.random.default_rng(9000 + 31 * self.seed + s)
        return (rng.random(count, dtype=np.float32) * 1e-2, rng.integers(1, 50, count).astype(f32),
                rng.random(count, dtype=np.float32) * 0.1)


def _contiguous(counts, firsts, row0=0):
    segs, r = [], row0
    for c, f in zip(counts, firsts):
        segs.append((r, int(c), int(f)))
        r += int(c)
    return segs, r


def _densify_cases() -> List[DensifyCase]:
    rng = np.random.default_rng(123)
    out = [DensifyCase("one_first", 240, 320, 1000, [(0, 1000, 1)]),
           DensifyCase("one_later", 1280, 1920, 1000, [(0, 1000, 0)])]
    counts = rng.integers(1, 400, 33)
    segs, n = _contiguous(counts, rng.integers(0, 2, 33))
    out.append(DensifyCase("s33_mixed_first", 1920, 1280, n, segs))
    counts = rng.integers(0, 20, 1024)
    segs, n = _contiguous(counts, rng.integers(0, 2, 1024))
    out.append(DensifyCase("s1024_mixed_first", 333, 177, n, segs))
    segs, n = _contiguous([0, 0, 50, 0, 300, 0, 7, 0, 0], [1, 0, 1, 1, 0, 0, 1, 0, 1])
    out.append(DensifyCase("empty_first_middle_last", 177, 333, n, segs))
    # the background (rows 0 .. 300) left out: the table starts at the first actor; sub-models left out between actors too
    segs = [(300, 120, 0), (420, 64, 1), (600, 1, 0), (601, 255, 1), (1000, 0, 1), (1000, 33, 0)]
    out.append(DensifyCase("row0_gt0_with_gaps", 1080, 1920, 1100, segs))
    segs = [(5000, 2048, 1), (9000, 3000, 0), (12000, 0, 0)]
    out.append(DensifyCase("row0_5000_gaps_tail", 1280, 1919, 13000, segs))
    for i, c in enumerate(out):
        c.seed = i
    return out


DENSIFY_CASES = _densify_cases()


# ---- two-shot exchange ----------------------------------------------------------------------------------------------------
@dataclass
class ArSlice:
    off: int          # floats from the arena base (multiple of 4)
    length: int       # floats (multiple of 4)
    width: int = 0    # > 0: row skipping
    row0: int = 0
    nrows: int = 0


@dataclass
class ExchangeCase:
    name: str
    slices: List[ArSlice]
    arena: int                       # floats
    union_rows: int = 0              # entries of the visibility arrays (0: no row skipping)
    pattern: str = "random"          # union pattern: "random", "all", "none", "boundary", "one_rank"
    max_ctas: int = 0
    seed: int = 0
    worlds: Tuple[int, ...] = (1, 2, 3, 4, 8)


def _lay_out(lengths, widths=None, rows=None, gap=4, row_gap=1):
    """Slices back to back with ``gap`` floats between them (never touched) and, for row skipping, each slice's rows
    behind the previous slice's rows and one sentinel entry."""
    slices, off, r0 = [], 8, 3
    for i, n in enumerate(lengths):
        w = widths[i] if widths else 0
        nr = rows[i] if rows else 0
        slices.append(ArSlice(off, n, w, r0 if w else 0, nr))
        off += n + gap
        if w:
            r0 += nr + row_gap
    return slices, off + 8, r0 + 5


def _exchange_cases() -> List[ExchangeCase]:
    out = []
    s, a, _ = _lay_out([4 * k for k in range(9)] + [0, 4, 0])   # 0 .. 8 units: below world for every world size
    out.append(ExchangeCase("short_and_empty", s, a))
    rng = np.random.default_rng(5)
    s, a, _ = _lay_out([4 * int(x) for x in rng.integers(0, 300, 48)])
    out.append(ExchangeCase("slices48", s, a))
    s, a, _ = _lay_out([4 * 5000 + 4, 4 * 17])
    out.append(ExchangeCase("grid_stride_one_cta", s, a, max_ctas=1))
    widths = [1, 2, 3, 4, 5, 9, 45, 3, 6, 9]
    rows = [1001, 502, 337, 251, 203, 113, 23, 338, 170, 113]
    lengths = []
    for w, r in zip(widths, rows):
        n = w * r + int(rng.integers(0, 9))   # padding behind nrows * width
        lengths.append((n + 3) // 4 * 4)
    s, a, u = _lay_out(lengths, widths, rows)
    for pat in ("random", "all", "none", "boundary", "one_rank"):
        out.append(ExchangeCase(f"skip_{pat}", s, a, union_rows=u, pattern=pat))
    out.append(ExchangeCase("skip_random_one_cta", s, a, union_rows=u, pattern="random", max_ctas=1))
    for i, c in enumerate(out):
        c.seed = i
    return out


EXCHANGE_CASES = _exchange_cases()


def rank_flags(c: ExchangeCase, world: int) -> np.ndarray:
    """[world, union_rows] uint8: each rank's visibility (its radii > 0).  The entry just behind every slice's rows and every
    entry past the last slice's rows are set (by rank 0), so a read past a slice's rows changes what is exchanged."""
    rng = np.random.default_rng(300 + c.seed * 10 + world)
    R = c.union_rows
    f = np.zeros((world, R), np.uint8)
    if c.pattern == "random":
        f[:] = rng.random((world, R)) < 0.25 / world
    elif c.pattern == "all":
        f[0] = 1
    elif c.pattern == "boundary":
        # isolated seen rows at float4 unit boundaries: the rows holding float 4i (and 4i - 1) of each slice, every 7th unit
        for sl in c.slices:
            if sl.width:
                for i in range(0, sl.length // 4, 7):
                    for fl in (4 * i, 4 * i - 1):
                        if 0 <= fl // sl.width < sl.nrows:
                            f[rng.integers(0, world), sl.row0 + fl // sl.width] = 1
    elif c.pattern == "one_rank":
        f[world - 1] = rng.random(R) < 0.3
    for sl in c.slices:
        if sl.width:
            f[0, sl.row0 + sl.nrows] = 1
    last = max((sl.row0 + sl.nrows for sl in c.slices if sl.width), default=0)
    f[0, last:] = 1
    return f
