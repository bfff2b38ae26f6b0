"""Hand-built inputs of the binning kernels: named, seeded rows built directly as projection outputs (records, radii,
tile_bbox, tiles_touched, touch_mask), without the projection, so each case drives chosen paths of csrc/binning.cu and
csrc/binning_local.cu: every mask shape of the small-run decode, warp sums at the 32-entry edges, warp-path and CTA-path
runs (33 .. 1024 and 1025 .. whole-image AABBs at block widths 16 and 2), depth ties, invisible rows carrying garbage, M = 0
and M = 1, one-class and alternating-class tiles, long tile lists, and tile counts at the 16-bit key edges.

Rows of two kinds: "mask" rows carry a hand-set touch mask (AABBs of at most 32 tiles; the emit step trusts the mask, so
their geometry is a placeholder) and tiles_touched = popcount; "gaussian" rows carry a real conic and opacity, and their
tiles_touched / mask come from the touch test of oracle/bin_ref64.py.  The builder moves each gaussian row's opacity until
no tile of its AABB lies in the touch band, so that test is exact.  ``Case.paths()`` reports what a case drives.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from functools import lru_cache
from typing import Callable, Dict, List

import numpy as np

from oracle import bin_ref64 as ref

VISIBLE = 16


@dataclass
class Case:
    name: str
    width: int
    height: int
    bw: int
    records: np.ndarray
    radii: np.ndarray
    bbox: np.ndarray
    touched: np.ndarray
    mask: np.ndarray
    geometric: bool  # every visible row is a gaussian row (sgn_bin_count recomputes the same masks)
    notes: Dict[str, object] = field(default_factory=dict)

    @property
    def tiles_x(self):
        return (self.width + self.bw - 1) // self.bw

    @property
    def tiles(self):
        return self.tiles_x * ((self.height + self.bw - 1) // self.bw)

    @property
    def N(self):
        return len(self.radii)

    def h(self):
        return ref.rows(self.records, self.radii, self.bbox, self.touched, self.mask)

    def ref(self, cap=None):
        key = ("ref", cap)
        if key not in self.notes:
            self.notes[key] = ref.reference(self.h(), self.width, self.height, self.bw, cap)
        return self.notes[key]

    def paths(self) -> Dict[str, int]:
        """Runs of each emit path (entries > 0), tiles by class content, the longest list."""
        h = self.h()
        area = ref.areas(h)
        run = (h["radii"] > 0) & (h["touched"] > 0)
        r = self.ref()
        ids, bins = r["ids"][:r["M"]], r["bins"]
        tile_of = np.repeat(np.arange(self.tiles), bins[:, 1] - bins[:, 0])
        obj = np.bincount(tile_of[ids < 0], minlength=self.tiles)
        bg = np.bincount(tile_of[ids >= 0], minlength=self.tiles)
        return dict(small=int((run & (area <= ref.COOP_AREA)).sum()),
                    warp=int((run & (area > ref.COOP_AREA) & (area <= ref.HUGE_AREA)).sum()),
                    cta=int((run & (area > ref.HUGE_AREA)).sum()), M=r["M"], tiles=self.tiles,
                    bg_only=int(((bg > 0) & (obj == 0)).sum()), obj_only=int(((obj > 0) & (bg == 0)).sum()),
                    both=int(((obj > 0) & (bg > 0)).sum()), longest=int((bins[:, 1] - bins[:, 0]).max(initial=0)))


class Builder:
    def __init__(self, width, height, bw, seed):
        self.width, self.height, self.bw = width, height, bw
        self.tx, self.ty = (width + bw - 1) // bw, (height + bw - 1) // bw
        self.rng = np.random.default_rng(seed)
        self.rows: List[dict] = []

    def _rec(self, xy, conic, opac, depth, obj, visible=True):
        r = np.zeros(12, np.float32)
        r[0:2], r[2:5], r[5], r[9] = xy, conic, opac, depth
        r[6:9] = self.rng.uniform(0, 1, 3)
        r[10] = np.array([(ref.AUX_OBJECT if obj else 0) | (VISIBLE if visible else 0)], np.int32).view(np.float32)[0]
        return r

    def depth(self):
        return np.float32(self.rng.uniform(0.5, 60.0))

    def mask_row(self, bb, mask, depth=None, obj=None):
        """A row with a hand-set mask over the AABB bb = (x0, y0, x1, y1) of at most 32 tiles."""
        x0, y0, x1, y1 = bb
        area = (x1 - x0) * (y1 - y0)
        assert 0 < area <= ref.COOP_AREA and 0 <= x0 < x1 <= self.tx and 0 <= y0 < y1 <= self.ty, bb
        mask = int(mask)
        assert mask >> area == 0
        obj = bool(self.rng.integers(2)) if obj is None else obj
        xy = ((x0 + x1) * self.bw / 2, (y0 + y1) * self.bw / 2)
        self.rows.append(dict(kind="mask", rec=self._rec(xy, (1.0, 0.0, 1.0), 0.5, self.depth() if depth is None else depth, obj),
                              radii=1, bbox=bb, touched=bin(mask).count("1"), mask=mask))
        return len(self.rows) - 1

    def gaussian(self, xy, cov, opac, depth=None, obj=None, bb=None, conic=None, settle=True):
        """A row with a real conic (the inverse of the 2D covariance cov, or `conic` as given); bb defaults to the tile AABB
        of the 3-sigma radius."""
        cov = np.asarray(cov, np.float64)
        if conic is None:
            inv = np.linalg.inv(cov)
            conic = (inv[0, 0], inv[0, 1], inv[1, 1])
        if bb is None:
            r = 3.0 * np.sqrt(np.linalg.eigvalsh(cov).max())
            bb = (int(np.clip((xy[0] - r) // self.bw, 0, self.tx)), int(np.clip((xy[1] - r) // self.bw, 0, self.ty)),
                  int(np.clip((xy[0] + r) // self.bw + 1, 0, self.tx)), int(np.clip((xy[1] + r) // self.bw + 1, 0, self.ty)))
        assert bb[2] > bb[0] and bb[3] > bb[1], bb
        obj = bool(self.rng.integers(2)) if obj is None else obj
        self.rows.append(dict(kind="gauss", rec=self._rec(xy, conic, opac, self.depth() if depth is None else depth, obj),
                              radii=1, bbox=tuple(int(v) for v in bb), settle=settle))
        return len(self.rows) - 1

    def rotated_cov(self, sx, sy, ang):
        c, s = np.cos(ang), np.sin(ang)
        R = np.array([[c, -s], [s, c]])
        return R @ np.diag([sx * sx, sy * sy]) @ R.T

    def invisible(self, n=1, garbage=True):
        """Rows with radii <= 0 and tiles_touched 0; with `garbage`, random bbox / mask / depth bits / class bit."""
        for _ in range(n):
            r = self._rec((0, 0), (0, 0, 0), 0, 0, bool(self.rng.integers(2)), visible=False)
            bb, mask = (0, 0, 0, 0), 0
            if garbage:
                r[[0, 1, 2, 3, 4, 5, 9]] = self.rng.integers(0, 2 ** 32, 7, dtype=np.uint64).astype(np.uint32).view(np.float32)
                bb = tuple(int(v) for v in self.rng.integers(0, 65536, 4))
                mask = int(self.rng.integers(0, 2 ** 32))
            self.rows.append(dict(kind="inv", rec=r, radii=int(-self.rng.integers(0, 2)), bbox=bb, touched=0, mask=mask))

    def small_random(self, n, max_area=ref.COOP_AREA, tiles=None):
        """n mask rows with random shapes and non-empty random masks (at random places or on the given tiles)."""
        for _ in range(n):
            w = int(self.rng.integers(1, min(max_area, self.tx) + 1))
            hh = int(self.rng.integers(1, max(1, min(max_area // w, self.ty)) + 1))
            if tiles is not None:
                t = int(self.rng.choice(tiles))
                x0, y0 = min(t % self.tx, self.tx - w), min(t // self.tx, self.ty - hh)
            else:
                x0, y0 = int(self.rng.integers(0, self.tx - w + 1)), int(self.rng.integers(0, self.ty - hh + 1))
            m = 0
            while m == 0:
                m = int(self.rng.integers(0, 2 ** (w * hh)))
            self.mask_row((x0, y0, x0 + w, y0 + hh), m)

    def _settle(self, rec, bb):
        """Move the opacity until no AABB tile lies in the touch band; returns the must-keep flags of the AABB tiles."""
        for _ in range(400):
            tiles, must, may = ref.touch_row(rec, bb, self.width, self.height, self.bw)
            if np.array_equal(must, may):
                return must
            o = float(rec[5]) * np.exp(self.rng.uniform(-0.08, 0.08))
            rec[5] = np.float32(min(max(o, 1.0 / 254.0), 0.99))
        raise AssertionError("could not move every AABB tile out of the touch band")

    def case(self, name, notes=None) -> Case:
        N = len(self.rows)
        rec = np.zeros((N, 12), np.float32)
        radii = np.zeros(N, np.int32)
        bbox = np.zeros((N, 4), np.int64)
        touched = np.zeros(N, np.int64)
        mask = np.zeros(N, np.uint32)
        for g, r in enumerate(self.rows):
            rec[g], radii[g], bbox[g] = r["rec"], r["radii"], r["bbox"]
            if r["kind"] == "gauss":
                must = self._settle(rec[g], bbox[g]) if r["settle"] else \
                    ref.touch_row(rec[g], bbox[g], self.width, self.height, self.bw)[1]
                touched[g] = must.sum()
                if len(must) <= ref.COOP_AREA:
                    mask[g] = np.uint32(int((must.astype(np.int64) << np.arange(len(must))).sum()))
            else:
                touched[g], mask[g] = r["touched"], np.uint32(r["mask"])
        geometric = all(r["kind"] != "mask" for r in self.rows)
        return Case(name, self.width, self.height, self.bw, rec, radii, bbox, touched, mask, geometric, dict(notes or {}))


# ------------------------------------------------------------------------------------------------------------------
# the cases
# ------------------------------------------------------------------------------------------------------------------
SHAPES = [(w, h) for w in range(1, 33) for h in range(1, 33) if w * h <= ref.COOP_AREA]


def mask_shapes(seed=301):
    """Every AABB shape w x h with w h <= 32, each with a full, a first-bit, a last-bit and two random masks, placed at random,
    in the last (partial) tile column, in the last (partial) tile row and at that corner of a 1000 x 700 image (block
    width 16: 63 x 44 tiles, the last column 8 px wide and the last row 12 px high); invisible rows interleaved."""
    b = Builder(1000, 700, 16, seed)
    for k, (w, h) in enumerate(SHAPES):
        area = w * h
        rnd = [int(b.rng.integers(1, 2 ** area)) for _ in range(2)]
        places = [(int(b.rng.integers(0, b.tx - w + 1)), int(b.rng.integers(0, b.ty - h + 1))), (b.tx - w, int(b.rng.integers(0, b.ty - h + 1))),
                  (int(b.rng.integers(0, b.tx - w + 1)), b.ty - h), (b.tx - w, b.ty - h), (int(b.rng.integers(0, b.tx - w + 1)), 0)]
        for (x0, y0), m in zip(places, [2 ** area - 1, 1, 1 << (area - 1)] + rnd):
            b.mask_row((x0, y0, x0 + w, y0 + h), m)
        if k % 3 == 0:
            b.invisible()
    return b.case("mask_shapes")


def warp_sums(seed=302):
    """Depths rising with the row, so warp k of the emit kernel holds rows 32k .. 32k+31.  Flattened warp sequences of
    exactly 32 (one entry per row), 33, 1024 (32 full 32-tile masks), 0 + 32 (31 empty rows and one full mask), 1 and
    a random mix; then a partial last warp of 7 rows."""
    b = Builder(1000, 700, 16, seed)
    full_shapes = [(32, 1), (16, 2), (8, 4), (4, 8), (2, 16), (1, 32)]
    plan = []
    plan.append([(1, 1, 1)] * 32)
    plan.append([(1, 1, 1)] * 31 + [(2, 1, 3)])
    plan.append([(w, h, 2 ** 32 - 1) for w, h in (full_shapes * 6)[:32]])
    plan.append([(1, 1, 0)] * 31 + [(8, 4, 2 ** 32 - 1)])
    plan.append([(1, 1, 0)] * 17 + [(3, 5, 1 << 14)] + [(1, 1, 0)] * 14)
    sums = []
    row = 0
    for warp in plan:
        sums.append(sum(bin(m).count("1") for _, _, m in warp))
        for w, h, m in warp:
            x0, y0 = int(b.rng.integers(0, b.tx - w + 1)), int(b.rng.integers(0, b.ty - h + 1))
            if m == 0:  # a visible row that reaches no tile
                b.gaussian((x0 * 16 + 8, y0 * 16 + 8), np.eye(2), 1e-3, depth=np.float32(1.0 + 0.01 * row), bb=(x0, y0, x0 + 1, y0 + 1))
            else:
                b.mask_row((x0, y0, x0 + w, y0 + h), m, depth=np.float32(1.0 + 0.01 * row))
            row += 1
    for _ in range(32 + 7):
        w, h = SHAPES[int(b.rng.integers(len(SHAPES)))]
        x0, y0 = int(b.rng.integers(0, b.tx - w + 1)), int(b.rng.integers(0, b.ty - h + 1))
        b.mask_row((x0, y0, x0 + w, y0 + h), int(b.rng.integers(1, 2 ** (w * h))), depth=np.float32(1.0 + 0.01 * row))
        row += 1
    return b.case("warp_sums", notes={"warp_sums": sums})


def big_runs(width, height, bw, seed):
    """Gaussian rows only.  AABBs of 33 (33 x 1 and 11 x 3), 64, 1024 (32 x 32), 1025 (41 x 25) tiles and the whole image,
    each covered by a rotated ellipse of about its size (of at most 6 tiles of sigma); thin rotated ellipses (the reached set is sparse and not a
    rectangle); a degenerate conic on a 48-tile and a 6-tile AABB (every tile kept); an opacity below 1/255 on a 100-tile
    AABB (no tile although radii > 0); 150 random small Gaussians, depths random, so warps mix small and big runs."""
    def make():
        b = Builder(width, height, bw, seed)
        dims = [(33, 1), (11, 3), (8, 8), (32, 32), (41, 25), (b.tx, b.ty)]
        for w, h in dims * 2:
            x0, y0 = int(b.rng.integers(0, b.tx - w + 1)), int(b.rng.integers(0, b.ty - h + 1))
            cx, cy = (x0 + w / 2) * bw + b.rng.uniform(-2, 2), (y0 + h / 2) * bw + b.rng.uniform(-2, 2)
            # at most 6 tiles of sigma: a wider ellipse's rim crosses too many tiles to keep them all out of the touch band
            cov = b.rotated_cov(min(w, 30) * bw / 5.0, min(h, 30) * bw / 5.0, b.rng.uniform(0, np.pi))
            b.gaussian((cx, cy), cov, b.rng.uniform(0.2, 0.95), bb=(x0, y0, x0 + w, y0 + h))
        for _ in range(6):  # thin rotated ellipses
            L = b.rng.uniform(0.05, 0.15) * min(width, height)
            b.gaussian((b.rng.uniform(0.3, 0.7) * width, b.rng.uniform(0.3, 0.7) * height),
                       b.rotated_cov(L, b.rng.uniform(0.5, 1.5) * bw / 2, b.rng.uniform(0.2, 1.4)), b.rng.uniform(0.3, 0.9))
        b.gaussian((width / 2, height / 2), np.eye(2), 0.5, bb=(2, 1, 10, 7), conic=(1.0, 2.0, 1.0))
        b.gaussian((width / 3, height / 3), np.eye(2), 0.5, bb=(4, 4, 7, 6), conic=(1.0, 0.0, -1.0))
        x0, y0 = b.tx // 3, b.ty // 3
        b.gaussian(((x0 + 5) * bw, (y0 + 5) * bw), b.rotated_cov(3 * bw, 3 * bw, 0.3), 0.9 / 255, bb=(x0, y0, x0 + 10, y0 + 10),
                   settle=False)
        for _ in range(150):
            s = b.rng.uniform(0.2, 1.6) * bw
            b.gaussian((b.rng.uniform(0.0, 1.0) * width, b.rng.uniform(0.0, 1.0) * height),
                       b.rotated_cov(s, s * b.rng.uniform(0.1, 1.0), b.rng.uniform(0, np.pi)), b.rng.uniform(0.05, 0.95))
        b.invisible(40)
        order = b.rng.permutation(len(b.rows))
        b.rows = [b.rows[i] for i in order]
        return b.case(f"big_runs_{width}x{height}_bw{bw}")
    return make


def ties(seed=303):
    """200 mask rows and 8 gaussian rows of 40-tile AABBs all at depth 5.0 (identical bits) in both classes, 60 rows 1 ulp
    apart around it, invisible rows with garbage interleaved: the lists fall back on the row tie-break everywhere."""
    b = Builder(320, 240, 16, seed)
    d0 = np.float32(5.0)
    ulps = [np.float32(d0)]
    for k in range(1, 4):
        ulps.append(np.nextafter(ulps[-1], np.float32(np.inf)))
    lo = np.nextafter(d0, np.float32(0))
    ulps = [np.nextafter(lo, np.float32(0)), lo] + ulps
    for k in range(260):
        w, h = SHAPES[int(b.rng.integers(len(SHAPES)))]
        w, h = min(w, b.tx), min(h, b.ty)
        x0, y0 = int(b.rng.integers(0, b.tx - w + 1)), int(b.rng.integers(0, b.ty - h + 1))
        d = d0 if k < 200 else ulps[k % len(ulps)]
        b.mask_row((x0, y0, x0 + w, y0 + h), int(b.rng.integers(1, 2 ** (w * h))), depth=d, obj=bool(k % 2))
        if k % 4 == 0:
            b.invisible()
    for k in range(8):
        x0, y0 = int(b.rng.integers(0, b.tx - 8 + 1)), int(b.rng.integers(0, b.ty - 5 + 1))
        b.gaussian(((x0 + 4) * 16, (y0 + 2.5) * 16), b.rotated_cov(30, 20, 0.4 * k), 0.9, depth=d0, obj=bool(k % 2),
                   bb=(x0, y0, x0 + 8, y0 + 5))
    return b.case("ties")


def empty(seed=304):
    """M = 0: invisible rows with garbage and visible rows that reach no tile."""
    b = Builder(200, 120, 16, seed)
    b.invisible(30)
    for k in range(10):
        b.gaussian((20.0 + 15 * k, 60.0), np.eye(2) * 100, 0.5 / 255, bb=(k, 2, k + 2, 4), settle=False)
    b.invisible(5)
    return b.case("empty")


def single(seed=305):
    """One entry (the last tile of a 13 x 8 image at block width 4), between invisible rows."""
    b = Builder(50, 30, 4, seed)
    b.invisible(7)
    b.mask_row((b.tx - 2, b.ty - 1, b.tx, b.ty), 2, obj=True)
    b.invisible(9)
    return b.case("single")


def classes(seed=306):
    """256 x 232 at block width 2 (128 x 116 = 14848 tiles, 1856 look-back windows of 8 warps): a band of background-only
    tiles, a band of object-only tiles, a band of alternating classes, tiles listing 512, 513 and 600 entries (the class
    kernel's 32 x 16-entry step), and random rows everywhere else; most tiles are empty."""
    b = Builder(256, 232, 2, seed)
    T = b.tx
    for k in range(300):  # background-only band: rows 0..9
        x0 = int(b.rng.integers(0, T - 4))
        b.mask_row((x0, k % 10, x0 + 4, k % 10 + 1), int(b.rng.integers(1, 16)), obj=False)
    for k in range(300):  # object-only band: rows 20..29
        x0 = int(b.rng.integers(0, T - 4))
        b.mask_row((x0, 20 + k % 10, x0 + 4, 21 + k % 10), int(b.rng.integers(1, 16)), obj=True)
    for k in range(400):  # alternating: rows 40..49, classes alternate in depth order
        x0 = int(b.rng.integers(0, T - 2))
        b.mask_row((x0, 40 + k % 10, x0 + 2, 41 + k % 10), 3, depth=np.float32(1.0 + 0.001 * k), obj=bool(k % 2))
    for n, (tx, ty) in zip((512, 513, 600), ((5, 60), (6, 60), (100, 100))):
        for k in range(n):
            b.mask_row((tx, ty, tx + 1, ty + 1), 1, obj=bool(b.rng.integers(2)) if n != 600 else bool(k % 2),
                       depth=np.float32(2.0 + 0.0005 * k))
    b.small_random(1500)
    b.invisible(100)
    order = b.rng.permutation(len(b.rows))
    b.rows = [b.rows[i] for i in order]
    return b.case("classes_bw2")


def tile_count(tx, ty, bw, seed):
    """A tx x ty tile grid (images whose size is not a multiple of the block width), random small rows, the first and the
    last tile listed (the last one is the largest key below the capped form's padding sentinel)."""
    def make():
        b = Builder(tx * bw - bw // 2 if bw > 1 and tx > 1 else tx * bw, ty * bw - (1 if bw > 1 else 0), bw, seed)
        assert (b.tx, b.ty) == (tx, ty)
        b.small_random(min(400, 4 * tx * ty), max_area=min(ref.COOP_AREA, tx * ty))
        b.mask_row((0, 0, 1, 1), 1)
        b.mask_row((tx - 1, ty - 1, tx, ty), 1)
        b.invisible(20)
        return b.case(f"tiles_{tx * ty}")
    return make


def local_sizes(counts, seed):
    """One tile per entry of `counts` on a 16-px-high strip at block width 16, tile t listing counts[t] 1 x 1 rows
    (the local variant's size classes: up to 1024 entries, up to 8192, above)."""
    def make():
        b = Builder(16 * len(counts), 16, 16, seed)
        for t, n in enumerate(counts):
            for k in range(n):
                b.mask_row((t, 0, t + 1, 1), 1, depth=np.float32(b.rng.integers(1, 200) * 0.25))
        order = b.rng.permutation(len(b.rows))
        b.rows = [b.rows[i] for i in order]
        return b.case("local_" + "_".join(str(n) for n in counts))
    return make


CASES: Dict[str, Callable[[], Case]] = {
    "mask_shapes": mask_shapes,
    "warp_sums": warp_sums,
    "big_runs_1920x1280_bw16": big_runs(1920, 1280, 16, 310),
    "big_runs_400x300_bw2": big_runs(400, 300, 2, 311),
    "ties": ties,
    "empty": empty,
    "single": single,
    "classes_bw2": classes,
    "tiles_1": tile_count(1, 1, 16, 320),
    "tiles_15": tile_count(15, 1, 16, 321),
    "tiles_16": tile_count(4, 4, 16, 322),
    "tiles_17": tile_count(17, 1, 16, 323),
    "tiles_65535": tile_count(255, 257, 2, 324),
    "tiles_65536": tile_count(256, 256, 2, 325),
    "local_1024_1025_8192_1": local_sizes((1024, 1025, 8192, 1), 330),
    "local_8193": local_sizes((3, 8193), 331),
}
# the cases every binning path is compared on (the local variant's overflow case only through its fallback)
LIST_CASES = [n for n in CASES if n != "local_8193"]


@lru_cache(maxsize=None)
def get(name: str) -> Case:
    return CASES[name]()
