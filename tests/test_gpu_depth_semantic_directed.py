"""The depth and semantic kernels -- sgn_lidar_depth_map, sgn_depth_loss_fwd / _bwd, sgn_depth_metrics, sgn_semantic_loss_fwd /
_bwd, sgn_semantic_metrics and sgn_refine_carry -- on hand-built inputs (tests/depth_semantic_cases.py) against the float64
statements of oracle/depth_ref64.py and tests/semantic_cases.py, through the C entry points of libsgn_raster.so.

  * Sizes: every loss, metric and map entry point at P = 1x1, 1x255, 255x1, 16x16, 17x15, one pixel either side of the
    1056 x 256 grid of one pass, 1920x1280 and 1447x1451 (above 2^21, not a multiple of the grid).
  * Map: a 2.5 M-point sweep (the scatter's grid-stride loop runs three times) in its own, reversed and shuffled order (the
    same bits), M = 1 and 257, z at clip_thresh and one float above, clip_thresh 0 with z = +-0, u and v at 0, -0.0, W (H) and
    the float below, two points on one pixel at equal depth, NaN and infinite coordinates, a depth that overflows to +inf in
    fp32, and a to_world 1e4 m from the origin.  The hit set is exact; a depth is within 4 ulps of its point's terms.  Random
    sweeps leave out the points within 1e-3 px of a pixel edge, or within 8 fp32 ulps of the coordinate's terms on images
    wider than 2^13 px (fp32 and fp64 may floor those differently); hand-placed points are all kept.  A canary behind every output shows a write past its end.
  * Depth loss and metrics: targets negative, -0.0 or NaN; masks -0.0, fractional or NaN; D == T; a NaN depth; no and one
    valid pixel; ratios exactly at 1.25, 1.5625, 1.953125; incoming gradient null or not; weight 0; every required pointer
    null; a short scratch.
  * Semantic loss and metrics: C in {1, 2, 7, 8, 31, 32, 33, 63, 64} (0 and 65 refused), int64 labels -1, C, 255, 2^31 and
    -2^40, masks -0.0 and fractional, confident logits (margin 10-20, offsets 0, 30 and 1000), logits of +-1e4, -inf among
    finite logits, all -inf, NaN, arg-max ties up to C = 64 (the full 64x64 shared histogram).  Every result repeats bit for bit.
  * Carry: widths 1, 2, 3, 63, 64 x n_split_samples 1, 2, 16 x with and without moments, n = 0, every row culled: bit-identical
    to the features_dc rows sgn_refine_apply writes from the same plan, and to the float64 row map.

Bars, as tests/test_gpu_ssim.py: a value or cotangent is within max(2 e_t, floor) of float64, where e_t is torch fp32's own
error on the same case (F.cross_entropy over the valid pixels; the depth L1 of depth.depth_loss_torch) and the floor is a few
fp32 ulps of each pixel's own terms (depth_semantic_cases: depth_loss_floor, ce_floor, grad_floor).  n_valid, the metric
counts, the confusion matrix and the map's hit set are compared exactly.

Observed on an H100 80GB HBM3 (700 W power limit): 172 tests in 66 s.  On the confident cases (256x391 pixels, mean CE 3.2e-6
at C = 2, 2.1e-5 at C = 19, 4.8e-5 at C = 64) the kernel's loss is within 2e-12 of float64 and torch fp32's within 4e-9,
1.7e-8 and 2.2e-8.  The earlier form (max + logf(z)) - S[label] was off by 6.6e-8 .. 1.9e-6 at C = 2 and 1.2e-7 .. 2.1e-6 at
C = 19 (offsets 0 .. 1000): it fails all nine.  (max - S[label]) + logf(z), z summed over every class, was off by 4.0e-8 at
C = 19 and 1.3e-7 at C = 64 at every offset (2.3x and 5.9x torch's error): the small terms round into the max's own 1, so it
fails the six cases with C = 19 and 64; the kernel sums them apart and takes log1pf.

Mutants of depth.cu and semantic.cu, and how many tests of this file each fails: `p.target[i] > 0.f` as `>=` in depth_valid
(33), the scatter's `u < (float)p.width` as `<=` (2: u at W, and at W on the last row, whose write lands in the canary),
`!(z > p.clip_thresh)` as `>=` (1), `v >= 0.f` as `v > 0.f` (2), `l >= p.C` as `l > p.C` in sem_label (38; run without the
two C = 64 metric cases, where the mutant would index past the 64x64 shared histogram), `x[c] > best` as `>=` in the arg-max
(17), and the two cross-entropy forms above (9 and 6).
"""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import depth_ref64 as dref
from street_gaussians_ns_b200 import _lib
from street_gaussians_ns_b200.depth import depth_loss_torch
from tests import depth_semantic_cases as dc
from tests import semantic_cases as sref

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
ERR_INVALID, ERR_WORKSPACE = -1, -3
f32 = np.float32
CANARY = np.int32(0x7FBADBAD)  # a NaN payload no kernel writes
TAIL = 64  # canary elements behind every buffer


def L():
    return _lib.load()


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def dev_in(arr):
    """A device copy of ``arr`` with TAIL zero elements behind it (reads one element past the end stay inside the buffer)."""
    if arr is None:
        return None
    flat = torch.from_numpy(np.ascontiguousarray(arr).reshape(-1).copy())
    buf = torch.zeros(flat.numel() + TAIL, dtype=flat.dtype, device=DEV)
    buf[:flat.numel()].copy_(flat)
    return buf[:flat.numel()]


class Out:
    """An output of ``n`` elements inside a buffer filled with the canary, TAIL elements longer."""

    def __init__(self, n, dtype=torch.float32):
        words = (torch.tensor([], dtype=dtype).element_size() * (n + TAIL) + 3) // 4
        self.raw = torch.full((words,), int(CANARY), dtype=torch.int32, device=DEV)
        self.buf = self.raw.view(dtype)
        self.n = n
        self.t = self.buf[:n]

    def host(self):
        torch.cuda.synchronize()
        tail = self.raw.cpu().numpy()
        nb = self.t.element_size() * self.n
        assert np.all(tail[(nb + 3) // 4:] == CANARY), "a write past the end of the output"
        return self.t.cpu().numpy()


def bits(a):
    return np.ascontiguousarray(a, dtype=f32).view(np.int32)


def within(got, want, bound):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    err = np.abs(got - want)
    ok = err <= bound
    return bool(np.all(ok)), (float(np.max(err - bound)) if err.size else 0.0)


# ---- lidar depth map ------------------------------------------------------------------------------------------------------
def camera(W, H, f=None, cx=None, cy=None, clip=0.01, viewmat=None):
    cs = _lib.CameraStruct()
    vm = np.eye(3, 4) if viewmat is None else np.asarray(viewmat, np.float64)
    for i, v in enumerate(vm.reshape(-1)):
        cs.viewmat[i] = float(v)
    f = 0.8 * max(W, H) if f is None else f
    cs.fx = cs.fy = f
    cs.cx = W / 2 if cx is None else cx
    cs.cy = H / 2 if cy is None else cy
    cs.width, cs.height, cs.clip_thresh, cs.block_width = W, H, clip, 16
    return cs


def lidar_map(points, cs, to_world=None):
    pts = np.ascontiguousarray(points, f32).reshape(-1, 3)
    M = pts.shape[0]
    d = dev_in(pts) if M else None
    tw = None
    if to_world is not None:  # a host array: the entry point composes it with the viewmat on the host
        tw = (C.c_float * 12)(*np.asarray(to_world, f32).reshape(-1).tolist())
    out = Out(cs.width * cs.height)
    _lib.check(L().sgn_lidar_depth_map(_p(d), M, C.byref(cs), None if tw is None else C.cast(tw, C.c_void_p), _p(out.t), None),
               "sgn_lidar_depth_map")
    return out.host().reshape(cs.height, cs.width)


def composed(cs, to_world=None):
    V = np.array(list(cs.viewmat), f32).astype(np.float64).reshape(3, 4)
    A = dref.compose(V, None if to_world is None else np.asarray(to_world, f32).astype(np.float64))
    return A.astype(f32).astype(np.float64)  # the kernel rounds the composed matrix once (the viewmat alone is fp32 already)


def map_ref(points, cs, to_world=None):
    A = composed(cs, to_world)
    pts = np.asarray(points, f32).astype(np.float64).reshape(-1, 3)
    want, pix = dref.lidar_depth_map_ref64(pts, A, cs.fx, cs.fy, cs.cx, cs.cy, cs.width, cs.height, cs.clip_thresh)
    # the depth's own terms, for the bound: 4 ulps of |A20 x| + |A21 y| + |A22 z| + |A23| of the largest point on the pixel
    with np.errstate(invalid="ignore", over="ignore"):
        terms = np.abs(pts * A[2, :3]).sum(axis=1) + abs(A[2, 3])
    bound = np.zeros(cs.width * cs.height)
    hit = pix >= 0
    np.maximum.at(bound, pix[hit], 4 * dc.U * terms[hit])
    return want, pix, bound.reshape(want.shape)


def check_map(got, want, bound):
    assert np.array_equal(got > 0, want > 0), int(((got > 0) != (want > 0)).sum())
    assert not np.any((got != 0) & ~(got > 0))  # no NaN, no negative, no empty marker left behind
    hit = want > 0
    ok, worst = within(got[hit], want[hit], bound[hit])
    assert ok, worst


def off_edges(pu, pv, cs, margin=1e-3):
    """The points whose pixel coordinates lie more than ``margin`` px, and more than 8 fp32 ulps of the coordinate's terms
    (u and u - cx, v and v - cy), from an integer: on images wider than 2^13 px an ulp of those terms is above 1e-3 px, so
    there the kernel's fp32 u can floor differently at 1e-3."""
    def far(c, c0):
        with np.errstate(invalid="ignore"):
            big = np.maximum(np.abs(c), np.abs(c - c0)).astype(f32)
            return np.abs(c - np.round(c)) > np.maximum(margin, 8 * np.spacing(big).astype(np.float64))
    return far(pu, cs.cx) & far(pv, cs.cy)


def random_sweep(W, H, M, seed, f=None):
    """Points whose pixels cover the image and 5 % around it, at depths 1 .. 60, with the points near a pixel edge
    (off_edges) left out."""
    rng = np.random.default_rng(seed)
    cs = camera(W, H, f)
    u = rng.uniform(-0.05 * W - 0.5, 1.05 * W + 0.5, M)
    v = rng.uniform(-0.05 * H - 0.5, 1.05 * H + 0.5, M)
    z = rng.uniform(1.0, 60.0, M)
    pts = np.stack([(u - cs.cx) * z / cs.fx, (v - cs.cy) * z / cs.fy, z], axis=1).astype(f32)
    _, pu, pv = dref.project_points_ref64(pts.astype(np.float64), composed(cs), cs.fx, cs.fy, cs.cx, cs.cy)
    return cs, pts[off_edges(pu, pv, cs)]


@pytest.mark.parametrize("hw", dc.SIZES, ids=dc.size_id)
def test_map_sizes(hw):
    H, W = hw
    cs, pts = random_sweep(W, H, min(3 * H * W + 50, 400_000), seed=H * 7 + W)
    got = lidar_map(pts, cs)
    want, pix, bound = map_ref(pts, cs)
    assert (pix >= 0).sum() > 0
    check_map(got, want, bound)


def test_map_sweep_that_loops():
    """2.5 M points against a 4224-block grid of 256 threads: every thread takes three points."""
    cs, pts = random_sweep(1920, 1280, 2_500_000, seed=11, f=1600.0)
    assert pts.shape[0] > 2 * 4 * 1056 * 256
    got = lidar_map(pts, cs)
    want, pix, bound = map_ref(pts, cs)
    assert (pix >= 0).sum() > 2_000_000
    check_map(got, want, bound)
    assert np.array_equal(bits(lidar_map(pts[::-1], cs)), bits(got))
    perm = np.random.default_rng(3).permutation(pts.shape[0])
    assert np.array_equal(bits(lidar_map(pts[perm], cs)), bits(got))
    assert np.array_equal(bits(lidar_map(pts, cs)), bits(got))


@pytest.mark.parametrize("M", [1, 257])
def test_map_small_sweeps(M):
    cs, pts = random_sweep(64, 48, 4 * M, seed=M)
    pts = pts[:M]
    assert pts.shape[0] == M
    got = lidar_map(pts, cs)
    want, _, bound = map_ref(pts, cs)
    check_map(got, want, bound)


W8, H6 = 8, 6
_nx = np.nextafter
CLIP = f32(0.01)


def _hand_cases():
    """name -> (points, camera kwargs, viewmat or None).  Points at x = y = 0 land exactly on (cx, cy)."""
    big = f32(3e38)
    return {
        "z_at_clip": ([[0, 0, CLIP]], {}, None),
        "z_one_float_above_clip": ([[0, 0, _nx(CLIP, f32(1))]], {}, None),
        "clip0_z_pos_and_neg_zero": ([[0, 0, 0.0], [0, 0, -0.0]], {"clip": 0.0}, None),
        "clip0_tiny_z": ([[0, 0, f32(1e-30)]], {"clip": 0.0}, None),
        "u_at_0": ([[0, 0, 2.0]], {"cx": 0.0}, None),
        "u_at_neg0": ([[-0.0, -0.0, 2.0]], {"cx": -0.0}, [[1, 0, -0.0, -0.0], [0, 1, 0, 0], [0, 0, 1, 0]]),
        "u_at_W": ([[0, 0, 2.0]], {"cx": float(W8)}, None),
        "u_below_W": ([[0, 0, 2.0]], {"cx": float(_nx(f32(W8), f32(0)))}, None),
        "v_at_0": ([[0, 0, 2.0]], {"cy": 0.0}, None),
        "v_at_neg0": ([[-0.0, -0.0, 2.0]], {"cy": -0.0}, [[1, 0, 0, 0], [0, 1, -0.0, -0.0], [0, 0, 1, 0]]),
        "v_at_H": ([[0, 0, 2.0]], {"cy": float(H6)}, None),
        "v_below_H": ([[0, 0, 2.0]], {"cy": float(_nx(f32(H6), f32(0)))}, None),
        "u_at_W_last_row": ([[0, 0, 2.0]], {"cx": float(W8), "cy": float(_nx(f32(H6), f32(0)))}, None),
        "two_equal_depths": ([[0.25, 0.25, 5.0], [0.26, 0.24, 5.0]], {}, None),
        "two_equal_and_nearer": ([[0.25, 0.25, 5.0], [0.26, 0.24, 5.0], [0.1, 0.1, 2.0]], {}, None),
        "nan_coords": ([[np.nan, 0, 3.0], [0, np.nan, 3.0], [0, 0, np.nan], [0.1, 0.1, 2.0]], {}, None),
        "inf_coords": ([[np.inf, 0, 3.0], [-np.inf, 0, 3.0], [0, np.inf, 3.0], [0, 0, np.inf], [0, 0, -np.inf], [0.1, 0.1, 2.0]],
                       {}, None),
        # pv.z = 2 * 3e38 overflows to +inf in fp32 while u, v stay at (cx, cy): its bits are the empty marker
        "z_overflows_to_inf": ([[0, 0, big]], {}, [[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 2, 0]]),
        "z_overflow_beside_a_return": ([[0, 0, big], [1.0, 0.5, 3.0]], {}, [[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 2, 0]]),
    }


HAND = _hand_cases()


@pytest.mark.parametrize("case", list(HAND))
def test_map_hand_placed(case):
    pts, kw, vm = HAND[case]
    kw = dict(kw)
    cs = camera(W8, H6, f=10.0, clip=kw.pop("clip", CLIP), viewmat=vm, **kw)
    pts = np.asarray(pts, f32)
    with np.errstate(invalid="ignore", over="ignore"):
        got = lidar_map(pts, cs)
        want, pix, bound = map_ref(pts, cs)
    check_map(got, want, bound)
    expect_hits = {"z_at_clip": 0, "z_one_float_above_clip": 1, "clip0_z_pos_and_neg_zero": 0, "clip0_tiny_z": 1, "u_at_0": 1,
                   "u_at_neg0": 1, "u_at_W": 0, "u_below_W": 1, "v_at_0": 1, "v_at_neg0": 1, "v_at_H": 0, "v_below_H": 1,
                   "u_at_W_last_row": 0, "two_equal_depths": 1, "two_equal_and_nearer": 1, "nan_coords": 1, "inf_coords": 1,
                   "z_overflows_to_inf": 0, "z_overflow_beside_a_return": 1}[case]
    assert int((got > 0).sum()) == expect_hits
    col = {"u_at_0": 0, "u_at_neg0": 0, "u_below_W": W8 - 1}.get(case)
    if col is not None:
        assert got[H6 // 2, col] == 2.0
    row = {"v_at_0": 0, "v_at_neg0": 0, "v_below_H": H6 - 1}.get(case)
    if row is not None:
        assert got[row, W8 // 2] == 2.0
    if case == "two_equal_depths":
        assert got[3, 4] == 5.0  # u = 10 * 0.25 / 5 + 4 = 4.5
    if case in ("z_overflows_to_inf", "z_overflow_beside_a_return"):
        assert got[H6 // 2, W8 // 2] == 0.0  # +inf (0x7f800000) is the empty marker: no return
    if case == "z_overflow_beside_a_return":
        assert got[3, 5] == 6.0


def test_map_to_world_far_from_origin():
    """A camera and a lidar 1e4 m from the world origin: the sweep is in the lidar's frame (small coordinates), the composed
    camera-from-lidar matrix is computed in fp64 and rounded once, so no 1e4 m term reaches the fp32 arithmetic."""
    a = 0.3
    R = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
    t = np.array([1.0e4, 2.5, -1.0e4 + 7.0])
    tw = np.concatenate([R, t[:, None]], axis=1).astype(f32)
    cam_pos = np.array([1.0e4 - 3.0, 1.0, -1.0e4], np.float64)
    vm = np.concatenate([np.eye(3), -cam_pos[:, None]], axis=1)  # world -> camera: x - cam_pos
    W, H = 640, 480
    cs = camera(W, H, f=500.0, viewmat=vm)
    rng = np.random.default_rng(9)
    cam_pts = np.stack([rng.uniform(-20, 20, 200_000), rng.uniform(-15, 15, 200_000), rng.uniform(1, 40, 200_000)], axis=1)
    world = cam_pts + cam_pos
    lidar = ((world - t) @ R).astype(f32)  # to_world @ lidar = world
    A = composed(cs, tw)
    assert np.abs(A[:, 3]).max() < 100  # the 1e4 m translations cancel in the composition
    _, pu, pv = dref.project_points_ref64(lidar.astype(np.float64), A, cs.fx, cs.fy, cs.cx, cs.cy)
    lidar = lidar[off_edges(pu, pv, cs)]
    got = lidar_map(lidar, cs, to_world=tw)
    want, pix, bound = map_ref(lidar, cs, tw)
    assert (pix >= 0).sum() > 50_000
    check_map(got, want, bound)


def test_map_argument_errors():
    cs = camera(8, 6)
    pts = dev_in(np.zeros((4, 3), f32))
    out = Out(48)
    assert L().sgn_lidar_depth_map(_p(pts), 4, None, None, _p(out.t), None) == ERR_INVALID
    assert L().sgn_lidar_depth_map(_p(pts), 4, C.byref(cs), None, None, None) == ERR_INVALID
    assert L().sgn_lidar_depth_map(None, 4, C.byref(cs), None, _p(out.t), None) == ERR_INVALID
    assert L().sgn_lidar_depth_map(_p(pts), -1, C.byref(cs), None, _p(out.t), None) == ERR_INVALID
    neg = camera(8, 6, clip=-1e-3)
    assert L().sgn_lidar_depth_map(_p(pts), 4, C.byref(neg), None, _p(out.t), None) == ERR_INVALID
    empty = camera(8, 6)
    empty.width = 0
    assert L().sgn_lidar_depth_map(_p(pts), 4, C.byref(empty), None, _p(out.t), None) == ERR_INVALID
    assert np.all(bits(out.host()) == CANARY)  # a refused call writes nothing
    assert L().sgn_lidar_depth_map(None, 0, C.byref(cs), None, _p(out.t), None) == 0  # an empty sweep: an empty map
    assert not out.host().any()


# ---- depth loss and metrics -----------------------------------------------------------------------------------------------
def depth_loss(D, T, M, w, g):
    H, W = D.shape
    d, t, m = dev_in(D), dev_in(T), dev_in(M)
    sb = L().sgn_depth_scratch_bytes()
    scratch = torch.full((sb,), 0xFF, dtype=torch.uint8, device=DEV)
    loss, nv = Out(1), Out(1, torch.int32)
    _lib.check(L().sgn_depth_loss_fwd(H, W, _p(d), _p(t), _p(m), w, _p(loss.t), _p(nv.t), _p(scratch), sb, None), "sgn_depth_loss_fwd")
    v = Out(H * W)
    gd = None if g is None else torch.tensor([g], dtype=torch.float32, device=DEV)
    _lib.check(L().sgn_depth_loss_bwd(H, W, _p(d), _p(t), _p(m), w, _p(nv.t), _p(gd), _p(v.t), None), "sgn_depth_loss_bwd")
    return loss.host()[0], int(nv.host()[0]), v.host().reshape(H, W)


def depth_torch(D, T, M, w, g):
    d = torch.from_numpy(D).to(DEV).requires_grad_(True)
    lt = depth_loss_torch(d, torch.from_numpy(T).to(DEV), None if M is None else torch.from_numpy(M).to(DEV), w)
    (lt * (1.0 if g is None else g)).backward()
    return float(lt.detach()), d.grad.cpu().numpy().astype(np.float64)


def check_depth_loss(D, T, M, w, g):
    got_l, got_n, got_v = depth_loss(D, T, M, w, g)
    want_l, n = dref.depth_loss_ref64(D, T, M, w)
    want_v = dref.depth_loss_grad_ref64(D, T, M, w, 1.0 if g is None else g)
    assert got_n == n
    if n == 0:
        assert got_l == 0.0 and np.all(bits(got_v) == 0)
        return got_l, got_v
    ok = dref.valid_ref64(T, M)
    t_l, t_v = depth_torch(D, T, M, w, g)
    e_t = abs(t_l - want_l)
    floor = dc.depth_loss_floor(D, T, ok, w)
    assert abs(float(got_l) - want_l) <= max(2 * e_t, floor), (float(got_l), want_l, e_t, floor)
    bound = np.maximum(2 * np.abs(t_v - want_v), 4 * dc.U * np.abs(want_v))
    good, worst = within(got_v, want_v, bound)
    assert good, worst
    assert np.array_equal(got_v == 0, want_v == 0)
    again = depth_loss(D, T, M, w, g)  # the same bits on a second run
    assert bits(again[0]) == bits(got_l) and again[1] == got_n and np.array_equal(bits(again[2]), bits(got_v))
    return got_l, got_v


@pytest.mark.parametrize("hw", dc.SIZES, ids=dc.size_id)
@pytest.mark.parametrize("mask", [None, "frac"])
def test_depth_loss_sizes(hw, mask):
    D, T, M = dc.depth_pixels(*hw, seed=hw[0] * 31 + hw[1], mask=mask)
    check_depth_loss(D, T, M, 0.25, None if hw[0] % 2 else -1.75)


def test_depth_loss_edges_each_rule():
    D, T, M = dc.depth_pixels(4, 8, seed=1, mask="frac")
    _, v = check_depth_loss(D, T, M, 0.5, 2.0)
    k = len(dc.DEPTH_EDGES)
    v = v.reshape(-1)[:k]
    assert np.all(v[:4] == 0) and v[4] == 0 and v[5] == 0  # invalid target; mask -0.0 and 0
    assert v[6] > 0 and v[7] > 0                            # mask 0.25 and NaN keep the pixel (D > T)
    assert v[8] == 0.0                                      # D == T: sign 0


@pytest.mark.parametrize("w", [0.0, 1.0])
@pytest.mark.parametrize("g", [None, 0.5])
def test_depth_loss_weight_and_gradient(w, g):
    D, T, M = dc.depth_pixels(17, 15, seed=4, mask="binary")
    got_l, got_v = check_depth_loss(D, T, M, w, g)
    if w == 0.0:
        assert got_l == 0.0 and not got_v.any()


def test_depth_loss_none_and_one_valid():
    D, T, _ = dc.depth_pixels(16, 16, seed=2, mask=None, edges=False)
    check_depth_loss(D, np.zeros_like(T), None, 1.0, 3.0)
    check_depth_loss(D, T, np.zeros_like(T), 1.0, 3.0)
    one = np.zeros_like(T)
    one[7, 9] = 4.0
    got_l, got_v = check_depth_loss(D, one, None, 0.3, None)
    e = abs(D[7, 9] - f32(4.0))  # rounded once in fp32, then w * e / 1 in fp64 and rounded once more
    assert got_l == f32(float(f32(0.3)) * float(e)) and np.count_nonzero(got_v) == 1


def test_depth_loss_nan_depth():
    """A NaN depth on a valid pixel: the loss is NaN, its cotangent 0 (sign(NaN) is taken as 0), the others are unchanged."""
    D, T, M = dc.depth_pixels(4, 8, seed=6, mask="binary", edges=False)
    T[0, 0], M[0, 0], D[0, 0] = 2.0, 1.0, np.nan
    got_l, got_n, got_v = depth_loss(D, T, M, 0.5, None)
    want_l, n = dref.depth_loss_ref64(D, T, M, 0.5)
    want_v = dref.depth_loss_grad_ref64(D, T, M, 0.5)
    assert np.isnan(got_l) and np.isnan(want_l) and got_n == n
    assert got_v[0, 0] == 0.0 and want_v[0, 0] == 0.0
    assert np.all(np.abs(got_v - want_v) <= 4 * dc.U * np.abs(want_v))


def depth_metrics(D, T, M):
    H, W = D.shape
    d, t, m = dev_in(D), dev_in(T), dev_in(M)
    sb = L().sgn_depth_scratch_bytes()
    scratch = torch.full((sb,), 0xFF, dtype=torch.uint8, device=DEV)
    out = Out(8)
    _lib.check(L().sgn_depth_metrics(H, W, _p(d), _p(t), _p(m), _p(out.t), _p(scratch), sb, None), "sgn_depth_metrics")
    return out.host()


def check_depth_metrics(D, T, M):
    got = depth_metrics(D, T, M).astype(np.float64)
    want = dref.depth_metrics_ref64(D, T, M)
    n = int(want[7])
    assert got[7] == n
    if n == 0:
        assert np.all(np.isnan(got[:7]))
        return got
    for i in range(4):
        assert abs(got[i] - want[i]) <= 2 * dc.U * abs(want[i]) + 1e-300, (dref.METRIC_NAMES[i], got[i], want[i])
    assert np.array_equal(np.rint(got[4:7] * n), np.rint(want[4:7] * n)), (got[4:7] * n, want[4:7] * n)
    assert np.array_equal(bits(depth_metrics(D, T, M)), bits(got))
    return got


@pytest.mark.parametrize("hw", dc.SIZES, ids=dc.size_id)
def test_depth_metrics_sizes(hw):
    D, T, M = dc.depth_pixels(*hw, seed=hw[0] * 13 + hw[1], mask="frac")
    check_depth_metrics(D, T, M)
    check_depth_metrics(D, T, None)


def test_depth_metrics_thresholds_and_edges():
    """Only the edge pixels: each ratio exactly at 1.25, 1.5625, 1.953125 is outside its threshold, the float below is inside."""
    e = np.array(dc.DEPTH_EDGES, f32)
    D, T, M = e[:, 0].reshape(1, -1).copy(), e[:, 1].reshape(1, -1).copy(), e[:, 2].reshape(1, -1).copy()
    got = check_depth_metrics(D, T, M)
    ok = dref.valid_ref64(T, M)
    d = np.fmax(D.reshape(-1)[ok], f32(1e-3)).astype(np.float64)
    t = T.reshape(-1)[ok].astype(np.float64)
    r = np.maximum(d / t, t / d)
    assert {1.25, 1.5625, 1.953125} <= set(r.tolist())
    n = int(ok.sum())
    assert got[7] == n == 15
    assert [round(x * n) for x in got[4:7]] == [int((r < 1.25).sum()), int((r < 1.5625).sum()), int((r < 1.953125).sum())]


def test_depth_metrics_nan_depth_counts_as_1e_3():
    D, T, M = dc.depth_pixels(3, 5, seed=8, mask=None, edges=False)
    T[:] = 2.0
    D[1, 2] = np.nan
    got = check_depth_metrics(D, T, M)
    clamped = D.copy()
    clamped[1, 2] = f32(1e-3)
    assert np.array_equal(bits(got), bits(depth_metrics(clamped, T, M)))
    assert np.all(np.isfinite(got))


def test_depth_metrics_none_and_one_valid():
    D, T, _ = dc.depth_pixels(16, 16, seed=3, mask=None, edges=False)
    check_depth_metrics(D, np.zeros_like(T), None)
    one = np.zeros_like(T)
    one[3, 3] = 5.0
    got = check_depth_metrics(D, one, None)
    assert got[7] == 1


def test_depth_argument_errors():
    D, T, M = dc.depth_pixels(4, 4, seed=0)
    d, t, m = dev_in(D), dev_in(T), dev_in(M)
    sb = L().sgn_depth_scratch_bytes()
    assert sb == 8 * 8 * 1056
    sc = torch.zeros(sb, dtype=torch.uint8, device=DEV)
    loss, nv, out, v = Out(1), Out(1, torch.int32), Out(8), Out(16)
    fwd = [4, 4, _p(d), _p(t), _p(m), 1.0, _p(loss.t), _p(nv.t), _p(sc), sb, None]
    for i in (0, 1):
        for bad in (0, -1):
            a = list(fwd)
            a[i] = bad
            assert L().sgn_depth_loss_fwd(*a) == ERR_INVALID
    for i in (2, 3, 6, 7, 8):  # depth, target, loss, n_valid, scratch
        a = list(fwd)
        a[i] = None
        assert L().sgn_depth_loss_fwd(*a) == ERR_INVALID, i
    a = list(fwd)
    a[9] = sb - 1
    assert L().sgn_depth_loss_fwd(*a) == ERR_WORKSPACE and b"scratch" in L().sgn_last_error()
    assert np.all(bits(loss.host()) == CANARY) and np.all(nv.host().view(np.int32) == CANARY)
    _lib.check(L().sgn_depth_loss_fwd(*fwd), "sgn_depth_loss_fwd")
    bwd = [4, 4, _p(d), _p(t), _p(m), 1.0, _p(nv.t), None, _p(v.t), None]
    for i in (2, 3, 6, 8):  # depth, target, n_valid, v_depth
        a = list(bwd)
        a[i] = None
        assert L().sgn_depth_loss_bwd(*a) == ERR_INVALID, i
    a = list(bwd)
    a[0] = 0
    assert L().sgn_depth_loss_bwd(*a) == ERR_INVALID
    assert np.all(bits(v.host()) == CANARY)
    met = [4, 4, _p(d), _p(t), _p(m), _p(out.t), _p(sc), sb, None]
    for i in (2, 3, 5, 6):  # depth, target, out, scratch
        a = list(met)
        a[i] = None
        assert L().sgn_depth_metrics(*a) == ERR_INVALID, i
    a = list(met)
    a[7] = sb - 8
    assert L().sgn_depth_metrics(*a) == ERR_WORKSPACE
    a = list(met)
    a[1] = -3
    assert L().sgn_depth_metrics(*a) == ERR_INVALID
    assert np.all(bits(out.host()) == CANARY)


# ---- semantic loss and metrics --------------------------------------------------------------------------------------------
def sem_loss(x, lab, M, w, g, C_arg=None):
    H, W, Cn = x.shape
    xd, ld, md = dev_in(x), dev_in(np.asarray(lab, np.int64)), dev_in(M)
    sb = L().sgn_semantic_scratch_bytes()
    scratch = torch.full((sb,), 0xFF, dtype=torch.uint8, device=DEV)
    loss, nv = Out(1), Out(1, torch.int32)
    _lib.check(L().sgn_semantic_loss_fwd(H, W, Cn, _p(xd), _p(ld), _p(md), w, _p(loss.t), _p(nv.t), _p(scratch), sb, None),
               "sgn_semantic_loss_fwd")
    v = Out(H * W * Cn)
    gd = None if g is None else torch.tensor([g], dtype=torch.float32, device=DEV)
    _lib.check(L().sgn_semantic_loss_bwd(H, W, Cn, _p(xd), _p(ld), _p(md), w, _p(nv.t), _p(gd), _p(v.t), None), "sgn_semantic_loss_bwd")
    return loss.host()[0], int(nv.host()[0]), v.host().reshape(H * W, Cn)


def sem_torch(x, lab, ok, w, g):
    """torch fp32: F.cross_entropy summed over the valid pixels, over their count, and its autograd cotangent."""
    Cn = x.shape[-1]
    xt = torch.from_numpy(x.reshape(-1, Cn)).to(DEV).requires_grad_(True)
    sel = torch.from_numpy(np.flatnonzero(ok)).to(DEV)
    lt = F.cross_entropy(xt[sel], torch.from_numpy(np.asarray(lab).reshape(-1)[ok]).to(DEV), reduction="sum") * w / int(ok.sum())
    (lt * (1.0 if g is None else g)).backward()
    return float(lt.detach()), xt.grad.cpu().numpy().astype(np.float64)


def check_sem_loss(x, lab, M, w=0.7, g=None, tag=None):
    Cn = x.shape[-1]
    got_l, got_n, got_v = sem_loss(x, lab, M, w, g)
    ok = sref.valid_ref(lab, Cn, M)
    n = int(ok.sum())
    want_l, n_ref = sref.loss_ref64(x, lab, M, w)
    want_v = sref.grad_ref64(x, lab, M, w, 1.0 if g is None else g).reshape(-1, Cn)
    assert got_n == n == n_ref
    if n == 0:
        assert got_l == 0.0 and np.all(bits(got_v) == 0)
        return
    s = x.reshape(-1, Cn)[ok]
    l_ok = np.asarray(lab).reshape(-1)[ok]
    t_l, t_v = sem_torch(x, lab, ok, w, g)
    e_t = abs(t_l - want_l)
    floor = abs(w) / n * float(dc.ce_floor(s, l_ok).sum()) + dc.U * abs(want_l)
    err = abs(float(got_l) - want_l)
    if tag:
        print(f"{tag}: loss {want_l:.6e} |kernel - fp64| {err:.3e} |torch - fp64| {e_t:.3e} floor {floor:.3e}")
    assert err <= max(2 * e_t, floor), (float(got_l), want_l, err, e_t, floor)
    k = (1.0 if g is None else g) * w / n
    bound = np.zeros_like(want_v)
    bound[ok] = np.maximum(2 * np.abs(t_v[ok] - want_v[ok]), dc.grad_floor(s, l_ok, k))
    good, worst = within(got_v, want_v, bound)
    assert good, worst
    assert np.all(bits(got_v[~ok]) == 0)
    again = sem_loss(x, lab, M, w, g)
    assert bits(again[0]) == bits(got_l) and again[1] == got_n and np.array_equal(bits(again[2]), bits(got_v))


@pytest.mark.parametrize("hw", dc.SIZES, ids=dc.size_id)
def test_semantic_loss_sizes(hw):
    x, lab, M = dc.sem_inputs(*hw, 19, seed=1)
    check_sem_loss(x, lab, M, g=None if hw[1] % 2 else 1.5)


@pytest.mark.parametrize("C", dc.SEM_CLASSES)
@pytest.mark.parametrize("hw", [(17, 15), (1, dc.GRID + 1)], ids=dc.size_id)
def test_semantic_loss_classes(C, hw):
    x, lab, M = dc.sem_inputs(*hw, C, seed=2, mask="frac" if C % 2 else None)
    check_sem_loss(x, lab, M, w=0.3, g=-2.0)


@pytest.mark.parametrize("offset", [0.0, 30.0, 1000.0])
@pytest.mark.parametrize("C", [2, 19, 64])
def test_semantic_loss_confident(C, offset):
    """The label is the arg-max by 10 .. 20: CE is about C e^-margin, far below ulp(max) once the logits are large."""
    x, lab, M = dc.sem_inputs(256, 391, C, seed=3, kind="confident", offset=offset)
    check_sem_loss(x, lab, M, w=1.0, tag=f"confident C={C} offset={offset:g}")


def test_semantic_loss_large_logits():
    x, lab, M = dc.sem_inputs(16, 16, 7, seed=4)
    rng = np.random.default_rng(4)
    x = (np.sign(x) * 1e4 * (rng.random(x.shape) < 0.5) + x).astype(f32)
    x[0, 0] = 1e4
    x[0, 1] = -1e4
    x[0, 1, 3] = 1e4
    check_sem_loss(x, lab, M, w=0.9)


def _special(kind, C=5):
    """A 1 x 6 image: pixel 2 holds the special logits, the others are ordinary; every label is in range."""
    rng = np.random.default_rng(C)
    x = rng.standard_normal((1, 6, C)).astype(f32)
    lab = np.array([[0, 1, 2, 3, 4, 0]], np.int64) % C
    if kind == "neg_inf_off_label":
        x[0, 2, 0] = -np.inf  # the label is 2
    elif kind == "neg_inf_on_label":
        x[0, 2, 2] = -np.inf
    elif kind == "all_neg_inf":
        x[0, 2, :] = -np.inf
    elif kind == "nan_one":
        x[0, 2, 3] = np.nan
    elif kind == "nan_first":
        x[0, 2, 0] = np.nan
    elif kind == "nan_all":
        x[0, 2, :] = np.nan
    return x, lab


@pytest.mark.parametrize("kind", ["neg_inf_off_label", "neg_inf_on_label", "all_neg_inf", "nan_one", "nan_first", "nan_all"])
def test_semantic_non_finite_logits(kind):
    """The rules of tests/semantic_cases.py: a -inf off the label is a zero softmax entry (finite loss); on the label CE = +inf
    with the label's cotangent exactly -k; all -inf or any NaN makes CE, so the loss, NaN and the pixel's cotangent row NaN.
    The arg-max takes the first NaN, else the first maximum (all -inf: class 0).  Ordinary pixels are unaffected."""
    x, lab = _special(kind)
    w = 0.5
    got_l, got_n, got_v = sem_loss(x, lab, None, w, None)
    want_l, n = sref.loss_ref64(x, lab, None, w)
    want_v = sref.grad_ref64(x, lab, None, w).reshape(-1, 5)
    assert got_n == n == 6
    k = w / n
    if kind == "neg_inf_off_label":
        assert np.isfinite(got_l) and abs(float(got_l) - want_l) <= 1e-6 * abs(want_l)
        assert got_v[2, 0] == 0.0 and want_v[2, 0] == 0.0
    elif kind == "neg_inf_on_label":
        assert got_l == np.inf and want_l == np.inf
        assert got_v[2, 2] == f32(-k) and want_v[2, 2] == -k
    else:
        assert np.isnan(got_l) and np.isnan(want_l)
        assert np.all(np.isnan(got_v[2])) and np.all(np.isnan(want_v[2]))
    fin = np.isfinite(want_v)
    good, worst = within(got_v[fin], want_v[fin], 1e-6 * np.abs(want_v[fin]) + 1e-7 * k)
    assert good, worst
    assert np.array_equal(np.isfinite(got_v), fin)
    conf = semantic_confusion(x, lab, None)
    want_c = sref.confusion_ref64(x, lab, None)
    assert np.array_equal(conf, want_c)
    expect = {"all_neg_inf": 0, "nan_one": 3, "nan_first": 0, "nan_all": 0}.get(kind)
    if expect is not None:
        assert conf[lab[0, 2], expect] >= 1 and want_c[lab[0, 2], expect] >= 1


@pytest.mark.parametrize("C", [1, 5, 64])
def test_semantic_labels_and_masks(C):
    """Every out-of-range int64 label and the -0.0 mask leave the pixel out; a fractional mask keeps it with weight 1."""
    rng = np.random.default_rng(C)
    n = 40
    x = rng.standard_normal((1, n, C)).astype(f32)
    lab = rng.integers(0, C, (1, n)).astype(np.int64)
    edges = dc.label_edges(C)
    lab[0, :len(edges)] = edges
    M = np.ones((1, n), f32)
    M[0, 10], M[0, 11], M[0, 12], M[0, 13] = -0.0, 0.0, 0.375, 1e-30
    check_sem_loss(x, lab, M, w=1.25, g=0.5)
    _, nv, _ = sem_loss(x, lab, M, 1.0, None)
    assert nv == n - len(edges) - 2
    assert np.array_equal(semantic_confusion(x, lab, M), sref.confusion_ref64(x, lab, M))


def test_semantic_no_and_one_valid_pixel():
    x, lab, _ = dc.sem_inputs(16, 16, 3, seed=5, mask=None)
    check_sem_loss(x, np.full_like(lab, 255), None)
    check_sem_loss(x, lab, np.zeros((16, 16), f32))
    one = np.full_like(lab, -1)
    one[5, 5] = 2
    check_sem_loss(x, one, None, w=2.0, g=3.0)


def semantic_confusion(x, lab, M):
    H, W, Cn = x.shape
    xd, ld, md = dev_in(x), dev_in(np.asarray(lab, np.int64)), dev_in(M)
    out = Out(Cn * Cn, torch.int64)
    _lib.check(L().sgn_semantic_metrics(H, W, Cn, _p(xd), _p(ld), _p(md), _p(out.t), None), "sgn_semantic_metrics")
    return out.host().reshape(Cn, Cn)


@pytest.mark.parametrize("hw", dc.SIZES, ids=dc.size_id)
def test_semantic_metrics_sizes(hw):
    x, lab, M = dc.sem_inputs(*hw, 19, seed=6, kind="ties")
    got = semantic_confusion(x, lab, M)
    assert np.array_equal(got, sref.confusion_ref64(x, lab, M))
    assert np.array_equal(semantic_confusion(x, lab, M), got)


@pytest.mark.parametrize("C", dc.SEM_CLASSES)
def test_semantic_metrics_classes_with_ties(C):
    """Half-integer logits (an eighth of the pixels tie in every class); at C = 64 all 64 x 64 cells of the shared histogram
    are reached."""
    x, lab, M = dc.sem_inputs(300, 347, C, seed=7, kind="ties")
    got = semantic_confusion(x, lab, M)
    want = sref.confusion_ref64(x, lab, M)
    assert np.array_equal(got, want)
    if C == 64:
        assert np.count_nonzero(want) == 64 * 64
    ties = x.reshape(-1, C)[: x.shape[0] * x.shape[1] // 8]
    assert np.all(ties == 0.5)


def test_semantic_argument_errors():
    x, lab, M = dc.sem_inputs(4, 4, 3, seed=0)
    xd, ld, md = dev_in(x), dev_in(lab), dev_in(M)
    sb = L().sgn_semantic_scratch_bytes()
    assert sb == 16 * 1056
    sc = torch.zeros(sb, dtype=torch.uint8, device=DEV)
    loss, nv, v, conf = Out(1), Out(1, torch.int32), Out(48), Out(65 * 65, torch.int64)
    fwd = [4, 4, 3, _p(xd), _p(ld), _p(md), 1.0, _p(loss.t), _p(nv.t), _p(sc), sb, None]
    for C_bad in (0, 65, -1):
        a = list(fwd)
        a[2] = C_bad
        assert L().sgn_semantic_loss_fwd(*a) == ERR_INVALID
    for i, bad in ((0, 0), (1, -2)):
        a = list(fwd)
        a[i] = bad
        assert L().sgn_semantic_loss_fwd(*a) == ERR_INVALID
    for i in (3, 4, 7, 8, 9):  # logits, labels, loss, n_valid, scratch
        a = list(fwd)
        a[i] = None
        assert L().sgn_semantic_loss_fwd(*a) == ERR_INVALID, i
    a = list(fwd)
    a[10] = sb - 1
    assert L().sgn_semantic_loss_fwd(*a) == ERR_WORKSPACE and b"scratch" in L().sgn_last_error()
    assert np.all(bits(loss.host()) == CANARY)
    _lib.check(L().sgn_semantic_loss_fwd(*fwd), "sgn_semantic_loss_fwd")
    bwd = [4, 4, 3, _p(xd), _p(ld), _p(md), 1.0, _p(nv.t), None, _p(v.t), None]
    for i in (3, 4, 7, 9):
        a = list(bwd)
        a[i] = None
        assert L().sgn_semantic_loss_bwd(*a) == ERR_INVALID, i
    for C_bad in (0, 65):
        a = list(bwd)
        a[2] = C_bad
        assert L().sgn_semantic_loss_bwd(*a) == ERR_INVALID
    assert np.all(bits(v.host()) == CANARY)
    met = [4, 4, 3, _p(xd), _p(ld), _p(md), _p(conf.t), None]
    for i in (3, 4, 6):
        a = list(met)
        a[i] = None
        assert L().sgn_semantic_metrics(*a) == ERR_INVALID, i
    for C_bad in (0, 65):
        a = list(met)
        a[2] = C_bad
        assert L().sgn_semantic_metrics(*a) == ERR_INVALID
    assert np.all(conf.host().view(np.int64) == np.int64(0x7FBADBAD7FBADBAD))


# ---- refinement carry -----------------------------------------------------------------------------------------------------
def refine_config(nss):
    cfg = _lib.RefineConfig()
    cfg.densify, cfg.n_split_samples = 1, nss
    cfg.max_size, cfg.inv_size_fac = 320.0, float(f32(1) / f32(1.6))
    return cfg


@pytest.mark.parametrize("case", dc.CARRY_CASES, ids=lambda c: c.name)
def test_carry_matches_refine_apply(case):
    n, w, nss = case.n, case.width, case.n_split_samples
    flags, scan, totals = case.plan()
    rows = case.out_rows(totals)
    rng = np.random.default_rng(case.seed)
    src = rng.standard_normal((n, w)).astype(f32)
    sm, sv = rng.standard_normal((n, w)).astype(f32), rng.random((n, w)).astype(f32)
    cfg = refine_config(nss)
    fl, scd = dev_in(flags), dev_in(scan)
    tot = (C.c_int32 * 4)(*totals)
    s_d, sm_d, sv_d = dev_in(src), dev_in(sm), dev_in(sv)
    dst, dm, dv = Out(rows * w), Out(rows * w), Out(rows * w)
    mom = [_p(sm_d), _p(sv_d), _p(dm.t), _p(dv.t)] if case.moments else [None] * 4
    _lib.check(L().sgn_refine_carry(n, C.byref(cfg), _p(fl), _p(scd), tot, _p(s_d), _p(dst.t), w, *mom, None), "sgn_refine_carry")
    got = dst.host().reshape(rows, w)
    got_m = (dm.host().reshape(rows, w), dv.host().reshape(rows, w)) if case.moments else None
    want, want_m = sref.carry_ref(src, flags, nss, (sm, sv) if case.moments else None)
    assert np.array_equal(bits(got), bits(want))
    if case.moments:
        assert np.array_equal(bits(got_m[0]), bits(want_m[0])) and np.array_equal(bits(got_m[1]), bits(want_m[1]))
    if rows == 0:
        return
    # the same plan through sgn_refine_apply, features_dc at this width (the other tensors at their fixed widths)
    widths = [3, 3, 4, w, 0, 1]
    srcs = [dev_in(rng.standard_normal((n, k)).astype(f32)) if k else None for k in widths]
    srcs[3] = s_d
    dsts = [Out(rows * k) if k else None for k in widths]
    t = _lib.RefineTensors()
    for k in range(6):
        t.width[k] = widths[k]
        if widths[k]:
            t.src[k], t.dst[k] = srcs[k].data_ptr(), dsts[k].t.data_ptr()
    keep = {}
    if case.moments:
        for k in range(6):
            if widths[k]:
                a = sm_d if k == 3 else dev_in(rng.standard_normal((n, widths[k])).astype(f32))
                b = sv_d if k == 3 else dev_in(rng.random((n, widths[k])).astype(f32))
                keep[k] = (a, b, Out(rows * widths[k]), Out(rows * widths[k]))
                t.src_m[k], t.src_v[k], t.dst_m[k], t.dst_v[k] = a.data_ptr(), b.data_ptr(), keep[k][2].t.data_ptr(), keep[k][3].t.data_ptr()
    samples = dev_in(rng.standard_normal((max(nss * totals[3], 1), 3)).astype(f32))
    _lib.check(L().sgn_refine_apply(n, C.byref(cfg), C.byref(t), _p(fl), _p(scd), tot, _p(samples), None), "sgn_refine_apply")
    assert np.array_equal(bits(dsts[3].host().reshape(rows, w)), bits(got))
    if case.moments:
        assert np.array_equal(bits(keep[3][2].host().reshape(rows, w)), bits(got_m[0]))
        assert np.array_equal(bits(keep[3][3].host().reshape(rows, w)), bits(got_m[1]))


def test_carry_writes_nothing_without_rows():
    cfg = refine_config(2)
    tot = (C.c_int32 * 4)(0, 0, 0, 0)
    dst = Out(16)
    assert L().sgn_refine_carry(0, C.byref(cfg), None, None, tot, None, None, 4, None, None, None, None, None) == 0
    flags = dev_in(np.zeros(5, np.uint8))
    scan = dev_in(np.zeros((4, 5), np.int32))
    src = dev_in(np.ones((5, 4), f32))
    assert L().sgn_refine_carry(5, C.byref(cfg), _p(flags), _p(scan), tot, _p(src), _p(dst.t), 4, None, None, None, None, None) == 0
    assert np.all(bits(dst.host()) == CANARY)


def test_carry_argument_errors():
    flags = dev_in(np.full(5, dc.RF_KEEP_ORIG, np.uint8))
    scan = dev_in(np.cumsum(np.ones((4, 5), np.int32), axis=1).astype(np.int32))
    src, dst = dev_in(np.ones((5, 4), f32)), Out(20)
    tot = (C.c_int32 * 4)(5, 0, 0, 0)
    cfg = refine_config(2)
    base = [5, C.byref(cfg), _p(flags), _p(scan), tot, _p(src), _p(dst.t), 4, None, None, None, None, None]
    for i, bad in ((0, -1), (7, 0), (7, 65)):
        a = list(base)
        a[i] = bad
        assert L().sgn_refine_carry(*a) == ERR_INVALID, (i, bad)
    for i in (1, 2, 3, 4, 5, 6):
        a = list(base)
        a[i] = None
        assert L().sgn_refine_carry(*a) == ERR_INVALID, i
    for nss in (0, 17):
        bad_cfg = refine_config(nss)
        a = list(base)
        a[1] = C.byref(bad_cfg)
        assert L().sgn_refine_carry(*a) == ERR_INVALID, nss
    a = list(base)
    a[8] = _p(src)  # exp_avg without exp_avg_sq
    assert L().sgn_refine_carry(*a) == ERR_INVALID
    assert np.all(bits(dst.host()) == CANARY)
