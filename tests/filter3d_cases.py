"""Inputs and float64 statements for the directed tests of the 3D-filtered projection (tests/test_gpu_filter3d_directed.py).

A filtered case is a hand-built frame of tests/project_cases.py (or tests/antialias_cases.py's comp_edges, or
``thin_discs`` below) with one filter size sigma per row, set by a family from the row's own scales s = exp(ls):
  zero       sigma = 0;
  faint      0.05 x min s: coef ~ 1;
  even       the median of s: both backward terms (through s' and through coef) count;
  dominant   20 x max s: coef is tiny and the row is essentially the filter's sphere;
  needle     sqrt(min s x max s): between a needle's thin and long axes;
  underflow  rows with a thin axis (one whose s^2 is 0 in float32, such as exp(-80)): 0.1 .. 0.5 x max s, so in float32
             r = 0 on that axis and coef = 0; other rows: even;
  identity   rows with a thin axis: 0, so s^2 + sigma^2 == 0 in float32 and the filter is the identity there (r = 1);
             other rows: faint;
  mixed      each row draws one of the seven families above (seeded).
On rows with a thin axis, min, median and max are taken over the other axes: the thin axis' s^2 is 0 in float32 and 3e-70
in float64, and a sigma near it would make the two disagree by far more than rounding.

Settling: a filtered decision (near plane, FOV clamp, discriminant floor, radius ceil, tile box, visibility) within
project_cases.MARGIN of its threshold re-draws that row's sigma -- scaled by U(1 - w, 1 + w) from the case's seed, with
w = 0.1 for the first 20 rounds and 0.1 wider for each 20 rounds after, up to 0.5, for every row still unsettled (a row
whose sigma hardly moves its radius, a thin axis' filter beside a long axis, needs the wider steps) -- and never the case's
parameters, so the designed near-plane and FOV rows stay where they are; every row must settle.  A row that is
off the margin with a radius above RADIUS_MAX px (a dominant filter on a Gaussian already metres wide) halves its sigma
instead: past 5000 px no radius is 1e-4 (relative) from an integer.

``v_pose_ref`` / ``v_view_ref``: float64 cotangents of the box poses and of the view for the filtered projection, in both
modes -- tests/pose_cases.py's, tests/camera_cases.py's and tests/antialias_cases.py's statements with the covariance
built from filter3d_ref64.filtered_scales and the opacity sigmoid(logit) x coef (x comp of the filtered covariance in the
antialiased mode); sigma is a constant.
"""
from __future__ import annotations

import zlib
from dataclasses import dataclass
from functools import lru_cache
from typing import List

import numpy as np
import torch

from oracle import filter3d_ref64 as f3
from oracle import project_aa_ref64 as aa
from oracle import project_ref64 as ref
from tests import antialias_cases as ac
from tests import camera_cases as cc
from tests import pose_cases as pz
from tests import project_cases as pc

F64 = torch.float64
FAMILIES = ("zero", "faint", "even", "dominant", "needle", "underflow", "identity")
PURE = ("zero", "faint", "even", "dominant", "needle")
ROUNDS = 200
RADIUS_MAX = 1000  # px: the radius ceil's margin (relative to r) cannot clear MARGIN once r nears 1 / (2 MARGIN)


@dataclass
class FCase:
    name: str
    base: pc.Case
    family: str
    sigmas: List[np.ndarray]  # float32, one array per segment
    fams: np.ndarray          # per row: the index in FAMILIES of the family that set its sigma
    thin: np.ndarray          # [N, 3]: the axes whose s^2 is 0 in float32
    fwd: dict                 # filter3d_ref64.forward, float64, classic mode

    @property
    def frame(self):
        return self.base.frame

    @property
    def st(self):
        return self.base.st

    def rows(self, family: str) -> np.ndarray:
        return self.fams == FAMILIES.index(family)


def thin_discs(seed=280):
    """Discs with one thin axis of exp(-80) (its s^2 is 0 in float32) and two axes a few pixels wide, the thin axis within
    30 degrees of the view axis: the screen covariance before the blur keeps full rank, so comp > 0 in the antialiased mode
    (comp_edges' thin rows are needles, whose comp is 0 with or without a filter); and a scatter."""
    b = pc._cam(128, 96, seed)
    for s in (b.segment(0), b.segment(1, pose=(0.2, (0.1, -0.1, -4.0)), F=2)):
        for k in range(10):
            z = b.rng.uniform(2, 8)
            ax = b.rng.normal(size=3)
            ax[2] = 0.0
            ang = b.rng.uniform(0.0, np.pi / 6)
            q = np.concatenate([[np.cos(ang / 2)], np.sin(ang / 2) * ax / np.linalg.norm(ax)])
            wide = b.rng.uniform(2.0, 8.0, 2) * z / b.cam.fx
            b.add(s, b.rng.uniform(15, 113), b.rng.uniform(15, 81), z, [wide[0], wide[1], ac.THIN], quat=q, fixed=True)
        b.scatter(s, 30)
    return b.settle("thin_discs")


def base_case(name: str) -> pc.Case:
    return _extra(name) if name in ("comp_edges", "thin_discs") else pc.get(name)


@lru_cache(maxsize=None)
def _extra(name: str) -> pc.Case:
    return ac.comp_edges() if name == "comp_edges" else thin_discs()


def thin_axes(ls: np.ndarray) -> np.ndarray:
    s = np.exp(np.asarray(ls, np.float32))
    with np.errstate(under="ignore"):
        return (s * s) == 0


def family_sigma(family: str, ls: np.ndarray, thin: np.ndarray, rng) -> np.ndarray:
    """float64 sigma of ``family`` for rows of log-scales ls [n, 3] (thin: their thin axes)."""
    s = np.exp(np.asarray(ls, np.float64))
    assert not thin.all(1).any(), "a row with three thin axes has no scale to set sigma from"
    st = np.where(thin, np.nan, s)
    lo, med, hi = np.nanmin(st, 1), np.nanmedian(st, 1), np.nanmax(st, 1)
    has_thin = thin.any(1)
    n = s.shape[0]
    if family == "zero":
        return np.zeros(n)
    if family == "faint":
        return 0.05 * lo
    if family == "even":
        return med
    if family == "dominant":
        return 20.0 * hi
    if family == "needle":
        return np.sqrt(s.min(1) * s.max(1))
    if family == "underflow":
        return np.where(has_thin, rng.uniform(0.1, 0.5, n) * hi, med)
    if family == "identity":
        return np.where(has_thin, 0.0, 0.05 * lo)
    raise ValueError(family)


def _split(frame, sig: np.ndarray) -> List[np.ndarray]:
    cuts = np.cumsum([s.params.num_points for s in frame.segments])[:-1]
    return [a.copy() for a in np.split(sig, cuts)]


def make(name: str) -> FCase:
    """``name`` = "<base case>/<family>"."""
    case_name, family = name.split("/")
    base = base_case(case_name)
    fr = base.frame
    ls = np.concatenate([s.params.scales.numpy() for s in fr.segments]) if fr.segments else np.zeros((0, 3), np.float32)
    N = ls.shape[0]
    thin = thin_axes(ls)
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    fams = rng.integers(0, len(FAMILIES), N) if family == "mixed" else np.full(N, FAMILIES.index(family))
    sig = np.zeros(N)
    for k, f in enumerate(FAMILIES):
        m = fams == k
        if m.any():
            sig[m] = family_sigma(f, ls[m], thin[m], rng)
    sig = sig.astype(np.float32)
    for k in range(ROUNDS):
        fw = f3.forward(fr, base.st, _split(fr, sig))
        bad = np.nonzero(fw["margin"] < pc.MARGIN)[0]
        if not len(bad):
            return FCase(name, base, family, _split(fr, sig), fams, thin, fw)
        assert np.all(sig[bad] > 0), f"{name}: a row without a filter is within the margin (its base case is settled)"
        w = min(0.5, 0.1 * (1 + k // 20))
        f = np.where(fw["radii"][bad] > RADIUS_MAX, 0.5, rng.uniform(1 - w, 1 + w, len(bad)))
        sig[bad] = (sig[bad] * f).astype(np.float32)
    raise AssertionError(f"{name}: could not move every filtered decision away from its threshold")


CONFIGS = ([f"{n}/mixed" for n in pc.CASES] + [f"{n}/{f}" for n in ("shapes", "posed40", "layout") for f in PURE]
           + [f"comp_edges/{f}" for f in ("needle", "underflow", "identity")]
           + [f"thin_discs/{f}" for f in ("underflow", "identity")])


@lru_cache(maxsize=None)
def get(name: str) -> FCase:
    return make(name)


def zero_filter(case: pc.Case) -> List[np.ndarray]:
    return [np.zeros(s.params.num_points, np.float32) for s in case.frame.segments]


# ------------------------------------------------------------------------------------------------------------------
# pose and view cotangents of the filtered projection
# ------------------------------------------------------------------------------------------------------------------
def _sigma(sigmas) -> torch.Tensor:
    return torch.tensor(np.concatenate([np.asarray(s, np.float64) for s in sigmas]) if len(sigmas) else np.zeros(0), dtype=F64)


def _opacity(cat, sigma, a, b, c, vt, antialiased):
    o = torch.sigmoid(cat["opacities"][:, 0]) * f3.coef(cat["scales"], sigma)
    if antialiased:
        o = o * aa.compensation(a, b, c)
    return o * vt


def pose_loss(frame, st: ref.Settings, sigmas, v_records: np.ndarray, pose: torch.Tensor, antialiased: bool = False):
    """sum(records * v_records) over the columns a pose moves (xy, conic, depth, and the opacity through comp) of the
    filtered projection of the frame composed from ``pose`` [n_posed, 16]."""
    _, cat = pz.compose(frame, pose)
    sigma = _sigma(sigmas)
    pr = ref.project_core(cat["means"], cat["quats"], f3.filtered_scales(cat["scales"], sigma), frame.camera, st.block_width,
                          st.clip_thresh, F64)
    vt = torch.from_numpy(pr["vis"])
    v = torch.tensor(np.asarray(v_records, np.float64), dtype=F64)
    opac = _opacity(cat, sigma, pr["a"], pr["b"], pr["c"], vt, antialiased)
    return ((pr["xy"] * v[:, 0:2]).sum(1) + ((pr["conic"] * v[:, 2:5]).sum(1) + pr["z"] * v[:, 9]) * vt + opac * v[:, 5]).sum()


def v_pose_ref(frame, st: ref.Settings, sigmas, v_records: np.ndarray, antialiased: bool = False) -> np.ndarray:
    """[n_posed, 16] float64 cotangents of the poses of the filtered projection."""
    leaf = pz.pose_leaves(pz.frame_poses(frame))
    if leaf.shape[0] == 0:
        return np.zeros((0, 16))
    loss = pose_loss(frame, st, sigmas, v_records, leaf, antialiased)
    return torch.autograd.grad(loss, leaf)[0].numpy() if loss.requires_grad else np.zeros(tuple(leaf.shape))


def view_loss(frame, st: ref.Settings, sigmas, v_records: np.ndarray, view: torch.Tensor, antialiased: bool = False):
    """(sum(records * v_records) over xy, conic, depth and opacity of the filtered projection with W | c = view[:12], the rows
    visible with the camera's own view): camera_cases.record_loss_view with the filtered scales and opacity."""
    sigma = _sigma(sigmas)
    return cc.record_loss_view(frame, st, v_records, view, scales=lambda cat: f3.filtered_scales(cat["scales"], sigma),
                               opacity=lambda cat, a, b, c: _opacity(cat, sigma, a, b, c, 1.0, antialiased))


def v_view_ref(frame, st: ref.Settings, sigmas, v_records: np.ndarray, antialiased: bool = False) -> np.ndarray:
    """[12] float64 cotangent of the camera's own viewmat for the filtered projection."""
    leaf = torch.tensor(np.asarray(frame.camera.viewmat(), np.float64).reshape(-1), dtype=F64).requires_grad_(True)
    loss, vis = view_loss(frame, st, sigmas, v_records, leaf, antialiased)
    if not vis.any():
        return np.zeros(12)
    return torch.autograd.grad(loss, leaf)[0].numpy()
