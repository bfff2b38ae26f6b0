"""Hand-built inputs of the blend kernels: records, per-tile lists and class sub-lists placed so that each case drives
chosen code paths of csrc/blend.cu (list lengths around the 8- and 32-entry batch edges and the strip splits, image
edges, where pixels stop, where the object entries sit, degenerate entries, one very large Gaussian).

No projection and no binning: a case goes straight into ``raster.blend_fwd`` / ``raster.blend_bwd``.  Each case is
named and seeded.  The builder keeps every skip / stop decision (and every post-op branch point) at least ``MARGIN``
away from its threshold, measured with the float64 reference (oracle/blend_ref64.py), by nudging the opacity of the
Gaussians that take part in a close call; so the kernels are compared with the reference on every pixel, unmasked.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from functools import lru_cache
from typing import Callable, Dict, List, Optional

import numpy as np

from oracle import blend_ref64 as ref

TILE = 16
MARGIN = 5e-5
OBJ_BIT = np.int64(1) << 31


@dataclass
class Case:
    name: str
    seed: int
    inp: ref.Inputs
    opts: ref.Opts
    # SGN_SPLIT_FWD_MAIN / _FWD_ACC / _BWD_MAIN / _BWD_ACC (0: the kernels' defaults)
    splits: Dict[str, int] = field(default_factory=dict)
    fwd: Optional[dict] = None  # the reference forward (filled by the builder)


class Builder:
    def __init__(self, width: int, height: int, seed: int):
        self.W, self.H = width, height
        self.rng = np.random.default_rng(seed)
        self.rows: List[np.ndarray] = []
        self.obj: List[bool] = []
        self.tx = (width + TILE - 1) // TILE
        self.tiles = self.tx * ((height + TILE - 1) // TILE)
        self.lists: List[List[int]] = [[] for _ in range(self.tiles)]
        self.fixed: set = set()  # Gaussians whose opacity is part of the design (never nudged)

    def gauss(self, x, y, sx, sy=None, rho=0.0, o=0.5, rgb=None, depth=None, obj=False, conic=None, fixed=False) -> int:
        sy = sx if sy is None else sy
        if conic is None:
            cov = np.array([[sx * sx, rho * sx * sy], [rho * sx * sy, sy * sy]])
            inv = np.linalg.inv(cov)
            conic = (inv[0, 0], inv[0, 1], inv[1, 1])
        r = np.zeros(12, np.float32)
        r[0:2] = (x, y)
        r[2:5] = conic
        r[5] = o
        r[6:9] = self.rng.uniform(0.0, 1.0, 3) if rgb is None else rgb
        r[9] = self.rng.uniform(0.5, 4.0) if depth is None else depth
        r[10] = np.int32((int(obj) << 3) | 16).view(np.float32)
        self.rows.append(r)
        self.obj.append(bool(obj))
        if fixed:
            self.fixed.add(len(self.rows) - 1)
        return len(self.rows) - 1

    def tile_origin(self, t):
        return (t % self.tx) * TILE, (t // self.tx) * TILE

    def random_in_tile(self, t, n, p_obj=0.4, sigma=(1.0, 5.0), o=(0.05, 0.6), rgb_hi=1.0, pad=4.0):
        x0, y0 = self.tile_origin(t)
        ids = []
        for _ in range(n):
            sx, sy = self.rng.uniform(*sigma, 2)
            ids.append(self.gauss(x0 + self.rng.uniform(-pad, TILE + pad), y0 + self.rng.uniform(-pad, TILE + pad), sx, sy,
                                  rho=self.rng.uniform(-0.6, 0.6), o=self.rng.uniform(*o),
                                  rgb=self.rng.uniform(0.0, rgb_hi, 3), obj=self.rng.random() < p_obj))
        self.lists[t] += ids
        return ids

    def flat(self, t, o, obj=False, n=1):
        """n entries of a Gaussian so wide that its alpha is o over the whole tile (to within 1e-4)."""
        x0, y0 = self.tile_origin(t)
        ids = [self.gauss(x0 + 8.0, y0 + 8.0, 2000.0, o=o, obj=obj, fixed=True) for _ in range(n)]
        self.lists[t] += ids
        return ids

    def inputs(self, sky=None) -> ref.Inputs:
        rec = np.stack(self.rows).astype(np.float32) if self.rows else np.zeros((1, 12), np.float32)
        payload = []
        tile_bins = np.zeros((self.tiles, 2), np.int32)
        for t, l in enumerate(self.lists):
            tile_bins[t] = (len(payload), len(payload) + len(l))
            payload += [int(g) | (int(OBJ_BIT) if self.obj[g] else 0) for g in l]
        M = len(payload)
        sorted_ids = np.array(payload, np.int64).astype(np.uint32).view(np.int32) if M else np.zeros(0, np.int32)
        cls_ids, cls_bins = partition(sorted_ids, tile_bins)  # stride = the list buffer's length
        return ref.Inputs(self.W, self.H, rec, sorted_ids, tile_bins, cls_ids, cls_bins, sky)


def _settle(b: Builder, opts: ref.Opts, sky=None, rounds: int = 60, margin: float = MARGIN):
    """Nudges the opacity of Gaussians in close calls until no decision is within ``margin`` of its threshold."""
    for _ in range(rounds):
        inp = b.inputs(sky)
        fw = ref.forward(inp, opts)
        bad = np.nonzero(fw["gauss_margin"] < margin)[0]
        bad = [g for g in bad if g not in b.fixed]
        if not bad and fw["margin"].min() >= margin:
            return inp, fw
        if not bad:  # a post-op branch point: nudge every Gaussian blended at the offending pixels
            ys, xs = np.nonzero(fw["margin"] < margin)
            for y, x in zip(ys, xs):
                l = b.lists[(y // TILE) * b.tx + x // TILE]
                bad += [g for g in l if g not in b.fixed]
            assert bad, "a designed decision is within the margin"
        for g in set(bad):
            b.rows[g][5] *= np.float32(1.0 + b.rng.uniform(-0.03, 0.03))
    raise AssertionError("could not move every decision away from its threshold")


def _case(name, seed, b: Builder, opts=None, splits=None, sky=None, margin=MARGIN):
    """sky: (lo, hi) of a uniform sky colour, or None for no sky."""
    opts = opts or ref.Opts()
    sk = None
    if sky is not None:
        opts.has_sky = True
        sk = b.rng.uniform(sky[0], sky[1], (b.H, b.W, 3)).astype(np.float32)
    splits = splits or {}
    if splits.get("SGN_SPLIT_FWD_MAIN"):
        opts.split_fwd_main = splits["SGN_SPLIT_FWD_MAIN"]
    inp, fw = _settle(b, opts, sk, margin=margin)
    return Case(name, seed, inp, opts, splits, fw)


def forced(n):
    return {k: n for k in ("SGN_SPLIT_FWD_MAIN", "SGN_SPLIT_FWD_ACC", "SGN_SPLIT_BWD_MAIN", "SGN_SPLIT_BWD_ACC")}


# ------------------------------------------------------------------------------------------------------------------
# the cases
# ------------------------------------------------------------------------------------------------------------------
LENGTHS = [0, 1, 7, 8, 9, 31, 32, 33, 63, 64, 65]


def lengths(seed=101):
    """One tile per list length around the 8-entry exit check and the 32-entry staging batches; objects interleaved."""
    b = Builder(TILE * len(LENGTHS), TILE, seed)
    for t, n in enumerate(LENGTHS):
        b.random_in_tile(t, n, o=(0.05, 0.9))
    return _case("lengths", seed, b)


def lengths_sky_eval(seed=102):
    """The same lengths with sky, the eval clamp and colours above 1 (the clamp at 1 zeroes their gradient); sky colours
    outside [0, 1] make the eval clamp zero the gradient of weakly covered pixels."""
    b = Builder(TILE * len(LENGTHS), TILE, seed)
    for t, n in enumerate(LENGTHS):
        b.random_in_tile(t, n, o=(0.05, 0.9), rgb_hi=3.0)
    return _case("lengths_sky_eval", seed, b, ref.Opts(eval_clamp=True), sky=(-0.3, 1.3))


def split_default(seed=103):
    """Lists at the default strip boundaries (768/769, 1536/1537, 3072/3073 entries, and one above 6144): 1, 2, 4 and 8
    strips forward; the backward splits on traversal depth (384), which the stopping pixels keep below the length."""
    lens = [768, 769, 1536, 1537, 3072, 3073, 6200, 100]
    b = Builder(TILE * 4, TILE * 2, seed)
    for t, n in enumerate(lens):
        b.random_in_tile(t, n, p_obj=0.3, sigma=(1.0, 4.0), o=(0.005, 0.05))
    return _case("split_default", seed, b)


def split_forced(seed=104):
    """Strip thresholds forced down to 16: tiles of 16, 17, 33, 65 and 200 entries run PPL 8/4/2/1/1 forward, and the
    low opacities keep the backward's depths (and the background pass's sub-lists) above the thresholds too."""
    lens = [16, 17, 33, 65, 200]
    b = Builder(TILE * len(lens), TILE, seed)
    for t, n in enumerate(lens):
        b.random_in_tile(t, n, p_obj=0.35, sigma=(1.0, 6.0), o=(0.02, 0.15))
    return _case("split_forced", seed, b, splits=forced(16))


def shape(w, h, lens, seed, split=4):
    """Images smaller than a tile or not a multiple of it: strips of every PPL have rows outside the image."""
    def make():
        b = Builder(w, h, seed)
        for t in range(b.tiles):
            b.random_in_tile(t, lens[t % len(lens)], o=(0.05, 0.7))
        return _case(f"shape_{w}x{h}", seed, b, splits=forced(split))
    return make


def termination(seed=105):
    """Where the main streams stop: every pixel inside a batch (entry 13 of 20), on the 8-entry exit check (entry 7),
    on the 32-entry batch edge (entry 31 of 64), never (40 weak entries), and a tile whose left half stops while its
    right half stays live.  Object entries ride along, so object streams stop inside the main traversal."""
    b = Builder(TILE * 5, TILE, seed)
    for k in range(20):
        b.flat(0, 0.5, obj=k % 3 == 0)             # T = 0.5^k: 0.5^14 <= 1e-4 < 0.5^13
    for k in range(24):
        b.flat(1, 0.71, obj=k % 2 == 1)            # 0.29^8 <= 1e-4 < 0.29^7
    for k in range(64):
        b.flat(2, 0.2535, obj=k % 5 == 0)          # 0.7465^32 <= 1e-4 < 0.7465^31
    b.random_in_tile(3, 40, o=(0.01, 0.05))
    x0, y0 = b.tile_origin(4)
    for k in range(12):
        b.lists[4].append(b.gauss(x0 + 1.0 + 0.3 * k, y0 + 8.0, 3.0, 20.0, o=0.95, obj=k % 4 == 0))
    b.random_in_tile(4, 30, o=(0.02, 0.3))
    return _case("termination", seed, b)


def objects(seed=106):
    """Object entries: none in a tile, only objects in a tile (empty background sub-list under BG_TODO pixels), object
    entries only behind the point where every main stream has stopped (the residual runs on the object sub-list and
    crosses a 32-entry batch), exactly one object entry behind it, and strong object entries that stop the object
    streams inside the main traversal."""
    b = Builder(TILE * 5, TILE, seed)
    b.random_in_tile(0, 40, p_obj=0.0)
    b.random_in_tile(1, 40, p_obj=1.0)
    b.random_in_tile(2, 3, p_obj=1.0, o=(0.05, 0.2))
    b.flat(2, 0.8, n=8)                           # every main stream stops at entry 3 + 5
    b.random_in_tile(2, 45, p_obj=1.0, o=(0.05, 0.3))
    b.random_in_tile(2, 10, p_obj=0.0)
    b.flat(3, 0.8, n=8)
    b.flat(3, 0.3, obj=True)                      # the one object entry behind the exit point
    b.random_in_tile(3, 5, p_obj=0.0)
    for k in range(10):
        b.flat(4, 0.7, obj=True)                  # object streams stop at their 8th entry
        b.random_in_tile(4, 2, p_obj=0.0, o=(0.02, 0.1))
    return _case("objects", seed, b)


def degenerate(seed=107):
    """Alpha clamped at 0.999 forward and 0.99 backward (opacity 1 at a pixel centre), opacity 0 / negative / NaN,
    a negative-definite conic (sigma < 0), a NaN conic, entries that reach no pixel of their tile, colours above 1;
    sky on, eval clamp on."""
    b = Builder(TILE * 2, TILE, seed)
    for t in range(2):
        x0, y0 = b.tile_origin(t)
        b.random_in_tile(t, 6, o=(0.05, 0.4))
        b.lists[t].append(b.gauss(x0 + 5.5, y0 + 6.5, 1.5, o=1.0, fixed=True))       # raw 1 at (5, 6): clamped
        b.lists[t].append(b.gauss(x0 + 9.5, y0 + 3.5, 2.0, o=0.0, fixed=True))
        b.lists[t].append(b.gauss(x0 + 9.5, y0 + 3.5, 2.0, o=-0.5, fixed=True))
        b.lists[t].append(b.gauss(x0 + 9.5, y0 + 3.5, 2.0, o=float("nan"), fixed=True))
        b.lists[t].append(b.gauss(x0 + 8.0, y0 + 8.0, 0, conic=(-0.2, 0.01, -0.3), o=0.8, fixed=True))
        b.lists[t].append(b.gauss(x0 + 8.0, y0 + 8.0, 0, conic=(float("nan"), 0.0, 0.5), o=0.8, fixed=True, obj=True))
        b.lists[t].append(b.gauss(x0 + 90.0, y0 - 60.0, 2.0, o=0.9, fixed=True))      # reaches no pixel
        b.lists[t].append(b.gauss(x0 + 12.0, y0 + 12.0, 3.0, o=0.9, rgb=(4.0, 0.2, 2.5), obj=True))
        b.random_in_tile(t, 6, o=(0.05, 0.4))
    return _case("degenerate", seed, b, ref.Opts(eval_clamp=True), sky=(0.0, 1.0))


def raw_mode(seed=108):
    """gsplat rasterize_gaussians semantics: no post-ops, a background colour (and depth), no class streams."""
    b = Builder(40, 24, seed)
    for t, n in enumerate([12, 33, 0, 70, 5, 9]):
        b.random_in_tile(t, n, p_obj=0.0, o=(0.05, 0.8))
    return _case("raw_mode", seed, b, ref.Opts(raw_mode=True, class_streams=False, background=(0.2, 0.4, 0.6, 5.0)))


def large(seed=109):
    """One Gaussian of sigma 250 px and opacity 0.9 over a 1920x1280 frame, with a sub-pixel one (sigma 0.3 px) in front
    of it in one tile.  The large one is listed in every tile it reaches, except the few tiles where its 1/255 contour
    passes within MARGIN of a pixel centre (that decision cannot be nudged away without moving thousands of others)."""
    b = Builder(1920, 1280, seed)
    big = b.gauss(960.3, 640.7, 250.0, o=0.9, rgb=(0.8, 0.5, 0.3), depth=20.0, fixed=True)
    small = b.gauss(301.2, 402.6, 0.3, o=0.8, rgb=(0.2, 0.9, 0.4), depth=3.0, obj=True, fixed=True)
    reach = 250.0 * np.sqrt(2 * np.log(255 * 0.9)) + 2.0
    for t in range(b.tiles):
        x0, y0 = b.tile_origin(t)
        cx, cy = np.clip(960.3, x0, x0 + TILE), np.clip(640.7, y0, y0 + TILE)
        if np.hypot(cx - 960.3, cy - 640.7) <= reach:
            b.lists[t].append(big)
    ts = (402 // TILE) * b.tx + 301 // TILE
    b.lists[ts].insert(0, small)
    opts = ref.Opts()
    fw = ref.forward(b.inputs(), opts)
    m = fw["margin"]
    for t in range(b.tiles):
        x0, y0 = b.tile_origin(t)
        if m[y0:y0 + TILE, x0:x0 + TILE].min() < MARGIN:
            b.lists[t].remove(big)
    return _case("large", seed, b, opts)


CASES: Dict[str, Callable[[], Case]] = {
    "lengths": lengths,
    "lengths_sky_eval": lengths_sky_eval,
    "split_default": split_default,
    "split_forced": split_forced,
    "shape_1x1": shape(1, 1, [5], 110, split=1),
    "shape_15x33": shape(15, 33, [3, 20, 70], 111),
    "shape_17x3": shape(17, 3, [9, 40], 112),
    "shape_16x80": shape(16, 80, [0, 5, 9, 17, 33], 113),
    "termination": termination,
    "objects": objects,
    "degenerate": degenerate,
    "raw_mode": raw_mode,
    "large": large,
}


def tiny(w, h, seed, sky=True, eval_clamp=False, n=6):
    """A few Gaussians per tile, opacities below the backward clamp (0.99) and every decision 1e-3 from its threshold:
    the float64 forward is differentiable there, and central differences check the backward."""
    b = Builder(w, h, seed)
    for t in range(b.tiles):
        b.random_in_tile(t, n, p_obj=0.5, sigma=(1.5, 4.0), o=(0.1, 0.8), rgb_hi=0.9)
    return _case(f"tiny_{w}x{h}", seed, b, ref.Opts(eval_clamp=eval_clamp), sky=(-0.2, 1.2) if sky else None, margin=1e-3)


def partition(sorted_ids: np.ndarray, tile_bins: np.ndarray):
    """cls_ids [2, max(M,1)], cls_bins [2, tiles, 2]: the stable partition of every tile's list by the object flag."""
    stride = max(len(sorted_ids), 1)
    tiles = tile_bins.shape[0]
    cls_ids = np.zeros((2, stride), np.int32)
    cls_bins = np.zeros((2, tiles, 2), np.int32)
    fill = [0, 0]
    for t in range(tiles):
        seg = sorted_ids[tile_bins[t, 0]:tile_bins[t, 1]]
        for c in (0, 1):
            part = seg[(seg < 0) == bool(c)]
            cls_bins[c, t] = (fill[c], fill[c] + len(part))
            cls_ids[c, fill[c]:fill[c] + len(part)] = part
            fill[c] += len(part)
    return cls_ids, cls_bins


@lru_cache(maxsize=None)
def get(name: str) -> Case:
    return CASES[name]()


def cotangents(case: Case, kind: str, seed: int = 7) -> Dict[str, np.ndarray]:
    """Seeded cotangents of the final outputs: U(-1, 1), or 1 everywhere for kind 'const'."""
    rng = np.random.default_rng(seed)
    H, W = case.inp.height, case.inp.width
    shapes = dict(rgb=(H, W, 3), accumulation=(H, W), depth=(H, W), object_acc=(H, W), background_acc=(H, W))
    if not case.opts.class_streams:
        shapes.pop("object_acc"), shapes.pop("background_acc")
    if kind == "const":
        return {k: np.ones(s, np.float32) for k, s in shapes.items()}
    return {k: rng.uniform(-1.0, 1.0, s).astype(np.float32) for k, s in shapes.items()}
