"""Hand-built inputs of the projection kernels: named, seeded frames whose Gaussians are placed so that each case drives
chosen paths of csrc/project.cu and sgn_touch.cuh (FOV clamps on every side, the near plane, needles and sub-pixel
Gaussians, image edges and block widths, segment layouts, visibility patterns inside the 128-row chunks, every SH degree
schedule, Fourier dims 1..8, tiles at the touch threshold).

Every camera has fx != fy and an off-centre principal point.  The builder keeps every decision the float64 reference
(oracle/project_ref64.py) reports -- near plane, FOV clamps, discriminant floor, radius ceil, the four AABB truncations,
each colour channel's pre-clamp value -- at least ``MARGIN`` (relative) from its threshold, by nudging scales, colours
and (for Gaussians that are not part of the design) means; so the kernels are compared with the reference unmasked.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from functools import lru_cache
from typing import Callable, Dict, List

import numpy as np
import torch

from oracle import project_ref64 as ref
from street_gaussians_ns_b200.scene import Camera, Frame, GaussianSet, Segment

MARGIN = 1e-4
CH = 128  # rows per chunk of the fused kernels


@dataclass
class Case:
    name: str
    frame: Frame
    st: ref.Settings
    fwd: dict
    notes: Dict[str, object] = field(default_factory=dict)


def _yaw(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, 0.0, s], [0.0, 1.0, 0.0], [-s, 0.0, c]])


class Builder:
    def __init__(self, width, height, fx, fy, cx, cy, seed, st: ref.Settings, c2w=None):
        c2w = np.concatenate([np.eye(3), np.zeros((3, 1))], 1) if c2w is None else c2w
        self.cam = Camera(c2w=c2w, fx=fx, fy=fy, cx=cx, cy=cy, width=width, height=height)
        self.rng = np.random.default_rng(seed)
        self.st = st
        self.K = (st.sh_degree + 1) ** 2
        self.segs: List[dict] = []
        vm = self.cam.viewmat().astype(np.float64)
        self.Rv, self.tv = vm[:, :3], vm[:, 3]
        self.limx, self.limy = self.cam.fov_limits()

    def segment(self, cls=0, pose=None, F=1):
        """pose: (yaw, centre) for an object segment; F: Fourier dim (a seeded basis in [-1, 1] when F > 1)."""
        idft = None if F == 1 else self.rng.uniform(-1.0, 1.0, F).astype(np.float32)
        self.segs.append(dict(cls=cls, pose=pose, F=F, idft=idft, rows=[], fixed=[]))
        return len(self.segs) - 1

    def world(self, px, py, z):
        """World point seen at pixel (px, py) and view depth z."""
        pv = np.array([(px - self.cam.cx) * z / self.cam.fx, (py - self.cam.cy) * z / self.cam.fy, z])
        return self.Rv.T @ (pv - self.tv)

    def add(self, s, px, py, z, scale, quat=None, logit=None, dc=None, fixed=False, u=None, v=None):
        """One Gaussian at pixel (px, py) / depth z (or at normalised view coordinates u = x/z, v = y/z); linear scale(s)."""
        if u is not None:
            px, py = u * self.cam.fx + self.cam.cx, v * self.cam.fy + self.cam.cy
        seg = self.segs[s]
        w = self.world(px, py, z)
        if seg["pose"] is not None:
            R = _yaw(seg["pose"][0]).astype(np.float32).astype(np.float64)
            t = np.asarray(seg["pose"][1], np.float64).astype(np.float32).astype(np.float64)
            w = R.T @ (w - t)
        sc = np.broadcast_to(np.asarray(scale, np.float64), (3,))
        q = self.rng.normal(size=4) if quat is None else np.asarray(quat, np.float64)
        F = seg["F"]
        row = dict(means=w, scales=np.log(sc), quats=q,
                   features_dc=self.rng.normal(0, 0.6, (F, 3)) if dc is None else np.broadcast_to(dc, (F, 3)).copy(),
                   features_rest=self.rng.normal(0, 0.15, (self.K - 1, 3)),
                   opacities=np.array([self.rng.normal(0.5, 2.0) if logit is None else logit]))
        seg["rows"].append(row)
        seg["fixed"].append(fixed)
        return s, len(seg["rows"]) - 1

    def scatter(self, s, n, px=None, py=None, z=(1.0, 20.0), scale=(0.01, 0.5)):
        W, H = self.cam.width, self.cam.height
        px = px or (-0.3 * W, 1.3 * W)
        py = py or (-0.3 * H, 1.3 * H)
        for _ in range(n):
            zz = self.rng.uniform(*z)
            self.add(s, self.rng.uniform(*px), self.rng.uniform(*py), zz,
                     np.exp(self.rng.uniform(np.log(scale[0]), np.log(scale[1]), 3)))

    def frame(self) -> Frame:
        segs = []
        for sg in self.segs:
            n = len(sg["rows"])
            def cat(k, shape):
                return torch.from_numpy(np.stack([r[k] for r in sg["rows"]]).astype(np.float32).reshape(n, *shape)
                                        if n else np.zeros((0, *shape), np.float32)).contiguous()
            gs = GaussianSet(cat("means", (3,)), cat("scales", (3,)), cat("quats", (4,)), cat("features_dc", (sg["F"], 3)),
                             cat("features_rest", (self.K - 1, 3)), cat("opacities", (1,)))
            if sg["pose"] is not None:
                segs.append(Segment(gs, sg["cls"], _yaw(sg["pose"][0]), np.asarray(sg["pose"][1], np.float64), sg["idft"]))
            else:
                segs.append(Segment(gs, sg["cls"], idft=sg["idft"]))
        return Frame(self.cam, segs)

    def settle(self, name, rounds=80, notes=None) -> Case:
        for _ in range(rounds):
            fr = self.frame()
            fw = ref.forward(fr, self.st)
            bad = np.nonzero(fw["margin"] < MARGIN)[0]
            if not len(bad):
                return Case(name, fr, self.st, fw, notes or {})
            where = [(s, i) for s, sg in enumerate(self.segs) for i in range(len(sg["rows"]))]
            mg = fw["margins"]
            for g in bad:
                s, i = where[g]
                row, fixed = self.segs[s]["rows"][i], self.segs[s]["fixed"][i]
                if mg["pre"][g] < MARGIN:
                    row["features_dc"] = row["features_dc"] + self.rng.uniform(-0.05, 0.05, row["features_dc"].shape)
                if min(mg[k][g] for k in ("disc", "ceil", "tmin_x", "tmin_y", "tmax_x", "tmax_y")) < MARGIN:
                    row["scales"] = row["scales"] + self.rng.uniform(-0.01, 0.01, 3)
                    row["means"] = row["means"] + self.rng.uniform(-1e-4, 1e-4, 3) * (np.abs(row["means"]).max() + 0.1)
                if min(mg[k][g] for k in ("near", "fovx", "fovy")) < MARGIN:
                    assert not fixed, f"{name}: a designed near-plane / FOV decision is within the margin"
                    row["means"] = row["means"] * (1 + self.rng.uniform(-1e-3, 1e-3, 3))
        raise AssertionError(f"{name}: could not move every decision away from its threshold")


def _cam(b_w, b_h, seed, st=None, fx=None, fy=None, c2w=None):
    st = st or ref.Settings()
    fx = fx or 0.9 * b_w
    fy = fy or 1.07 * fx
    return Builder(b_w, b_h, fx, fy, 0.47 * b_w + 0.3, 0.53 * b_h - 0.2, seed, st, c2w)


# ------------------------------------------------------------------------------------------------------------------
# the cases
# ------------------------------------------------------------------------------------------------------------------
def fov_clamp(seed=201):
    """Gaussians just inside (1 - 1e-3), just outside (1 + 1e-3) and far outside (1.6x) each FOV limit, on each side and
    at the four corners (both axes clamped), in an unposed and a posed segment, plus a random spread over 2x the FOV."""
    b = _cam(160, 96, seed)
    for s in (b.segment(0), b.segment(1, pose=(0.3, (0.5, -0.2, -4.0)), F=3)):
        for f in (1 - 1e-3, 1 + 1e-3, 1.6):
            for sx, sy in ((1, 0), (-1, 0), (0, 1), (0, -1), (1, 1), (-1, 1), (1, -1), (-1, -1)):
                z = b.rng.uniform(3.0, 8.0)
                u = sx * f * b.limx if sx else b.rng.uniform(-0.5, 0.5) * b.limx
                v = sy * f * b.limy if sy else b.rng.uniform(-0.5, 0.5) * b.limy
                b.add(s, 0, 0, z, np.exp(b.rng.uniform(np.log(0.8), np.log(3.0), 3)), u=u, v=v, fixed=True)
        for _ in range(60):
            b.add(s, 0, 0, b.rng.uniform(2.0, 15.0), np.exp(b.rng.uniform(np.log(0.05), np.log(2.5), 3)),
                  u=b.rng.uniform(-2, 2) * b.limx, v=b.rng.uniform(-2, 2) * b.limy)
    return b.settle("fov_clamp")


def near_plane(seed=202):
    """z just above and just below clip_thresh (1 +- 1e-3), z = 0, z < 0, and a Gaussian 2 cm in front of the camera whose
    radius is far larger than the image (its AABB is clamped on all four sides); random depths around the plane."""
    b = _cam(64, 48, seed)
    s = b.segment(0)
    clip = b.st.clip_thresh
    for z in (clip * (1 + 1e-3), clip * (1 - 1e-3), 0.0, -1.0, clip * 1.05):
        b.add(s, 30.0, 20.0, z, 0.0005, fixed=True)
    b.add(s, 33.0, 21.0, 0.02, 0.01, fixed=True)
    for _ in range(40):
        b.add(s, b.rng.uniform(-10, 74), b.rng.uniform(-10, 58), b.rng.uniform(0.003, 0.05),
              np.exp(b.rng.uniform(np.log(1e-4), np.log(5e-3), 3)))
    return b.settle("near_plane")


def shapes(seed=203):
    """Needles (scale ratio 1e4) at several rotations, sigma = 1e-5 (the 0.3 blur dominates), a Gaussian that covers the
    whole image, quaternions of norm 1e-3, 1 and 1e3 with both signs of w."""
    b = _cam(128, 96, seed)
    s = b.segment(0)
    for k in range(8):
        b.add(s, b.rng.uniform(10, 118), b.rng.uniform(10, 86), b.rng.uniform(3, 10), (0.5, 5e-5, 5e-5), fixed=True)
    for k in range(6):
        b.add(s, b.rng.uniform(0, 128), b.rng.uniform(0, 96), b.rng.uniform(1, 10), 1e-5, fixed=True)
    b.add(s, 60.0, 50.0, 3.0, (4.0, 3.0, 2.0), fixed=True)
    for norm in (1e-3, 1.0, 1e3):
        for sign in (1, -1):
            q = b.rng.normal(size=4)
            q[0] = sign * abs(q[0])
            b.add(s, b.rng.uniform(10, 118), b.rng.uniform(10, 86), b.rng.uniform(2, 8),
                  np.exp(b.rng.uniform(np.log(0.02), np.log(0.3), 3)), quat=norm * q / np.linalg.norm(q), fixed=True)
    b.scatter(s, 40)
    return b.settle("shapes")


def edges(w, h, bw, seed):
    """Centres off the image by less than their radius on every side and at the corners, on a w x h image at block width
    bw; a Gaussian to the right of the last, partial tile column (its clipped pixel rectangle is out of reach, the
    unclipped one is not)."""
    def make():
        b = _cam(w, h, seed, ref.Settings(block_width=bw))
        s = b.segment(0)
        for px, py in ((-2.5, h / 2), (w + 2.5, h / 2), (w / 2, -2.5), (w / 2, h + 2.5), (-1.5, -1.5), (w + 1.5, h + 1.5),
                       (-1.5, h + 1.5), (w + 1.5, -1.5)):
            z = b.rng.uniform(2, 6)
            b.add(s, px, py, z, 4.0 * z / b.cam.fx, fixed=True)
        if w % bw:
            z = 4.0
            b.add(s, w + 4.3, h / 2 + 0.2, z, 1.0 * z / b.cam.fx, logit=0.0, fixed=True)
        b.scatter(s, 30, z=(2.0, 30.0), scale=(0.005, 0.3))
        return b.settle(f"edges_{w}x{h}_bw{bw}")
    return make


def layout(seed=204):
    """Segments of 1, 127, 0, 128, 129, 255 and 0 rows (an empty segment in the middle and one at the end), posed and
    unposed, Fourier dims 1..5."""
    b = _cam(96, 64, seed)
    for k, n in enumerate((1, 127, 0, 128, 129, 255, 0)):
        s = b.segment(k % 2, pose=(0.1 * k, (0.2 * k, 0.0, -3.0)) if k % 2 else None, F=1 + k % 5)
        b.scatter(s, n)
    return b.settle("layout")


def posed40(seed=205):
    """40 posed segments with Fourier dims 1..8."""
    b = _cam(96, 64, seed)
    for k in range(40):
        s = b.segment(1, pose=(b.rng.uniform(-1, 1), b.rng.uniform(-2, 2, 3) + (0, 0, -8)), F=1 + k % 8)
        b.scatter(s, int(b.rng.integers(3, 40)))
    return b.settle("posed40")


def nseg1024(seed=206):
    """nseg = 1024 (the limit) with 0..3 rows each."""
    b = _cam(48, 32, seed)
    for k in range(1024):
        s = b.segment(k % 2, pose=(0.01 * (k % 50), (0.0, 0.0, -2.0)) if k % 2 else None, F=1 + k % 3)
        b.scatter(s, int(b.rng.integers(0, 4)), z=(1.0, 10.0))
    return b.settle("nseg1024")


def staged_mix(seed=207):
    """One segment of 3 chunks + a tail: chunk 0 alternates visible and invisible rows, chunk 1 has no visible row, chunk 2
    has exactly one visible row (lane 127), the tail chunk is random."""
    b = _cam(64, 48, seed)
    s = b.segment(0, F=2)
    for r in range(3 * CH):
        c, lane = divmod(r, CH)
        visible = (c == 0 and lane % 2 == 0) or (c == 2 and lane == CH - 1)
        z = b.rng.uniform(2, 10) if visible else -b.rng.uniform(1, 5)
        b.add(s, b.rng.uniform(5, 59), b.rng.uniform(5, 43), z, np.exp(b.rng.uniform(np.log(0.01), np.log(0.2), 3)),
              fixed=True)
    b.scatter(s, 50)
    return b.settle("staged_mix")


def colour(deg, use, seed):
    """sh_degree deg with sh_degree_to_use use: DC colours that put every channel's pre-clamp value on both sides of 0,
    opacity logits of +-15 and opacities just above 1/255 (tau near 0); an unposed and a posed segment (F = deg + 2)."""
    def make():
        b = _cam(64, 48, seed, ref.Settings(sh_degree=deg, sh_degree_to_use=use))
        segs = (b.segment(0), b.segment(1, pose=(0.4, (0.3, 0.2, -5.0)), F=deg + 2))
        for s in segs:
            for k in range(60):
                logit = (15.0, -15.0, float(np.log(1.06 / 254.0)), float(np.log(1.3 / 253.7)), None)[k % 5]
                dc = b.rng.uniform(-3.0, 1.5, 3) if deg > 0 else b.rng.uniform(-4, 4, 3)
                b.add(s, b.rng.uniform(0, 64), b.rng.uniform(0, 48), b.rng.uniform(1.0, 12.0),
                      np.exp(b.rng.uniform(np.log(0.02), np.log(0.4), 3)), logit=logit, dc=dc)
        return b.settle(f"colour_d{deg}_u{use}")
    return make


def touch(bw, seed):
    """Thin rotated Gaussians crossing tile corners, AABBs of 1 to 33 tiles and (block width 2) above 1024 tiles, and
    Gaussians whose opacity puts the nearest pixel centre of some AABB tile 5e-4 inside the touch threshold tau."""
    def make():
        b = _cam(333, 177, seed, ref.Settings(block_width=bw))
        s = b.segment(0)
        for k in range(24):
            tx, ty = b.rng.integers(1, 333 // bw), b.rng.integers(1, 177 // bw)
            ang = b.rng.uniform(0, np.pi)
            b.add(s, tx * bw + b.rng.uniform(-0.3, 0.3), ty * bw + b.rng.uniform(-0.3, 0.3), 5.0,
                  (b.rng.uniform(0.01, 0.05), 2e-4, 2e-4), quat=(np.cos(ang / 2), 0, 0, np.sin(ang / 2)))
        for r_px in (0.4, 1.0, 2.5, 5.0, 8.0, 10.0, 12.0, 20.0, 40.0, 80.0):
            for _ in range(3):
                z = b.rng.uniform(3, 8)
                b.add(s, b.rng.uniform(0, 333), b.rng.uniform(0, 177), z,
                      r_px * z / b.cam.fx * np.exp(b.rng.uniform(-0.2, 0.2, 3)))
        b.scatter(s, 30)
        case = b.settle(f"touch_bw{bw}")
        # opacities: tau = (min sigma of one AABB tile) + 5e-4 (geometry unchanged, so no other decision moves)
        fw = case.fwd
        rows = b.segs[s]["rows"]
        near_tau = []
        for g in np.nonzero(fw["vis"])[0][::2]:
            rec = fw["records"][g]
            _, _, d, _ = ref.touch_min_sigma(rec[0:2], rec[2:5], 0.5, fw["tmin"][g], fw["tmax"][g], 333, 177, bw)
            sig = d + np.log(255 * 0.5)
            cand = np.nonzero((sig > 0.3) & (sig < 5.0))[0]
            if len(cand):
                o = np.exp(sig[cand[0]] + 5e-4) / 255.0
                rows[g]["opacities"] = np.array([np.log(o / (1 - o))])
                near_tau.append(int(g))
        case = b.settle(f"touch_bw{bw}", notes={"near_tau": near_tau})
        return case
    return make


CASES: Dict[str, Callable[[], Case]] = {
    "fov_clamp": fov_clamp,
    "near_plane": near_plane,
    "shapes": shapes,
    **{f"edges_333x177_bw{bw}": edges(333, 177, bw, 210 + bw) for bw in (2, 3, 7, 8, 16)},
    "edges_1x1_bw16": edges(1, 1, 16, 230),
    "edges_17x3_bw16": edges(17, 3, 16, 231),
    "edges_17x3_bw2": edges(17, 3, 2, 232),
    "layout": layout,
    "posed40": posed40,
    "nseg1024": nseg1024,
    "staged_mix": staged_mix,
    **{f"colour_d{d}_u{u}": colour(d, u, 240 + 4 * d + u) for d in range(4) for u in range(d + 1)},
    "touch_bw16": touch(16, 260),
    "touch_bw2": touch(2, 261),
}


@lru_cache(maxsize=None)
def get(name: str) -> Case:
    return CASES[name]()


def v_records(case: Case, kind: str, seed: int = 11) -> np.ndarray:
    """[N,12] cotangents of the records: U(-1, 1) in the columns of ``kind`` (xy, conic, opacity, rgb, depth or all)."""
    cols = dict(xy=[0, 1], conic=[2, 3, 4], opacity=[5], rgb=[6, 7, 8], depth=[9], all=list(range(10)))[kind]
    N = case.fwd["records"].shape[0]
    v = np.zeros((N, 12), np.float32)
    v[:, cols] = np.random.default_rng(seed).uniform(-1.0, 1.0, (N, len(cols)))
    return v
