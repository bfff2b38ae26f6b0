"""CPU checks of the float64 statement of the lidar depth supervision (oracle/depth_ref64.py) on hand-built cases: the map's
nearest-return rule, pixel edges and the drop rules, the loss and its cotangent (with n_valid = 0 and a mask that removes every
return), and the metrics."""
import numpy as np
import pytest

from oracle.depth_ref64 import (compose, depth_loss_grad_ref64, depth_loss_ref64, depth_metrics_ref64, lidar_depth_map_ref64,
                                project_points_ref64)

W, H, F, CX, CY, CLIP = 8, 6, 10.0, 4.0, 3.0, 0.01
EYE = np.concatenate([np.eye(3), np.zeros((3, 1))], axis=1)


def dmap(points, A=EYE):
    return lidar_depth_map_ref64(np.asarray(points, np.float64), A, F, F, CX, CY, W, H, CLIP)


def test_nearer_return_wins():
    # both on pixel (4, 3): u = 10 x / z + 4, v = 10 y / z + 3
    m, pix = dmap([[0.25, 0.25, 5.0], [0.1, 0.1, 2.0], [0.25, 0.25, 5.0]])
    assert pix[0] == pix[1] == pix[2] == 3 * W + 4
    assert m[3, 4] == 2.0
    assert np.count_nonzero(m) == 1
    m2, _ = dmap([[0.1, 0.1, 2.0], [0.25, 0.25, 5.0]])  # order does not matter
    assert np.array_equal(m, m2)


def test_pixel_edges():
    # u exactly 4 (x = 0): the pixel to the right of the edge; u exactly 0 is inside, u exactly W is off the image
    m, pix = dmap([[0.0, 0.0, 3.0]])
    assert pix[0] == 3 * W + 4 and m[3, 4] == 3.0
    z = 4.0
    x0 = -CX * (z + 1e-6) / F  # u = 0
    _, pix = dmap([[x0, 0.0, z]])
    _, u, _ = project_points_ref64([[x0, 0.0, z]], EYE, F, F, CX, CY)
    assert u[0] == pytest.approx(0.0, abs=1e-12)
    assert pix[0] in (-1, 3 * W + 0)  # the float64 rounding of u decides; never another pixel
    xw = (W - CX) * (z + 1e-6) / F  # u = W
    _, u, _ = project_points_ref64([[xw, 0.0, z]], EYE, F, F, CX, CY)
    _, pix = dmap([[xw, 0.0, z]])
    assert pix[0] == (-1 if u[0] >= W else 3 * W + W - 1)


def test_dropped_points():
    pts = [[0.0, 0.0, -2.0],        # behind the camera
           [5.0, 0.0, 1.0],         # off the image (u = 54)
           [0.0, 0.0, CLIP],        # z == clip_thresh is dropped
           [0.0, -1.0, 2.0],        # v = -2: above the image
           [0.0, 0.0, CLIP * 1.5]]  # just past the near plane: kept
    m, pix = dmap(pts)
    assert list(pix[:4]) == [-1, -1, -1, -1]
    assert pix[4] == 3 * W + 4 and m[3, 4] == CLIP * 1.5
    assert np.count_nonzero(m) == 1


def test_empty_sweep_and_to_world():
    m, pix = dmap(np.zeros((0, 3)))
    assert m.shape == (H, W) and not m.any() and pix.shape == (0,)
    # a sweep in its own frame, shifted by to_world: the same map as the world-frame points
    tw = np.concatenate([np.eye(3), np.array([[0.5], [-0.25], [1.0]])], axis=1)
    pts = np.array([[0.1, 0.2, 3.0], [-0.3, 0.1, 6.0], [0.0, 0.0, 2.5]])
    a, _ = dmap(pts, compose(EYE, tw))
    b, _ = dmap(pts + tw[:, 3])
    assert np.allclose(a, b, rtol=1e-12, atol=0)


def _case(seed=0, n=(5, 7)):
    rng = np.random.default_rng(seed)
    D = rng.uniform(0.5, 20.0, n)
    T = np.where(rng.random(n) < 0.4, rng.uniform(0.5, 20.0, n), 0.0)
    return D, T


def test_loss_and_cotangent():
    D, T = _case()
    ok = T > 0
    n = int(ok.sum())
    L, nv = depth_loss_ref64(D, T, weight=0.3)
    assert nv == n and L == pytest.approx(0.3 * np.abs(D - T)[ok].sum() / n, rel=1e-15)
    g = depth_loss_grad_ref64(D, T, weight=0.3, g=2.0)
    assert np.all(g[~ok] == 0)
    eps = 1e-7  # central differences on the valid pixels (|D - T| is smooth away from D == T)
    for i, j in zip(*np.nonzero(ok)):
        Dp, Dm = D.copy(), D.copy()
        Dp[i, j] += eps
        Dm[i, j] -= eps
        fd = (depth_loss_ref64(Dp, T, weight=0.3)[0] - depth_loss_ref64(Dm, T, weight=0.3)[0]) / (2 * eps) * 2.0
        assert g[i, j] == pytest.approx(fd, rel=1e-6)
    # a tie D == T has a zero cotangent
    D2 = D.copy()
    D2[ok] = T[ok]
    assert np.all(depth_loss_grad_ref64(D2, T) == 0) and depth_loss_ref64(D2, T)[0] == 0.0


def test_no_valid_pixel():
    D, _ = _case()
    T = np.zeros_like(D)
    assert depth_loss_ref64(D, T, weight=5.0) == (0.0, 0)
    assert not depth_loss_grad_ref64(D, T, weight=5.0).any()
    m = depth_metrics_ref64(D, T)
    assert np.isnan(m[:7]).all() and m[7] == 0


def test_mask_removes_every_return():
    D, T = _case(1)
    mask = (T == 0).astype(np.float64)  # keeps exactly the pixels without a return
    assert depth_loss_ref64(D, T, mask, weight=1.0) == (0.0, 0)
    assert not depth_loss_grad_ref64(D, T, mask).any()
    half = np.ones_like(D)
    half[:, :3] = 0
    L, n = depth_loss_ref64(D, T, half)
    ok = (T > 0) & (half != 0)
    assert n == int(ok.sum()) and L == pytest.approx(np.abs(D - T)[ok].mean(), rel=1e-15)


def test_metrics():
    T = np.array([[2.0, 4.0, 0.0], [10.0, 1.0, 5.0]])
    D = np.array([[2.0, 5.0, 7.0], [0.0, 1.3, 9.0]], np.float32)  # D = 0 is clamped to 1e-3
    m = depth_metrics_ref64(D, T)
    d = np.array([2.0, 5.0, np.float32(1e-3), np.float32(1.3), 9.0], np.float64)
    t = np.array([2.0, 4.0, 10.0, 1.0, 5.0])
    r = np.maximum(d / t, t / d)
    assert m[7] == 5
    assert m[0] == pytest.approx(np.mean(np.abs(d - t) / t))
    assert m[2] == pytest.approx(np.sqrt(np.mean((d - t) ** 2)))
    assert m[3] == pytest.approx(np.sqrt(np.mean(np.log(d / t) ** 2)))
    assert list(m[4:7]) == [1 / 5, 3 / 5, 4 / 5]  # ratios 1, 1.25 (not < 1.25), 1e4, 1.3, 1.8
    assert r[1] == 1.25


def test_non_finite_and_edge_rules():
    """The rules oracle/depth_ref64.py states for targets, masks and depths that are not ordinary numbers."""
    D = np.array([3.0, 3.0, 3.0, 3.0, 3.0, 3.0, 3.0, 7.5], np.float32)
    T = np.array([-2.0, -0.0, np.nan, 2.0, 2.0, 2.0, 2.0, 7.5], np.float32)
    M = np.array([1.0, 1.0, 1.0, -0.0, 0.25, np.nan, 1.0, 1.0], np.float32)
    ok = [False, False, False, False, True, True, True, True]
    from oracle.depth_ref64 import valid_ref64
    assert valid_ref64(T, M).tolist() == ok
    L, n = depth_loss_ref64(D, T, M, weight=2.0)
    assert n == 4 and L == pytest.approx(2.0 * 3 / 4)
    g = depth_loss_grad_ref64(D, T, M, weight=2.0, g=1.0)
    assert g.tolist() == [0, 0, 0, 0, 0.5, 0.5, 0.5, 0.0]  # D == T: sign 0
    Dn = D.copy()
    Dn[4] = np.nan  # a NaN depth: the loss is NaN, its cotangent 0
    assert np.isnan(depth_loss_ref64(Dn, T, M)[0])
    gn = depth_loss_grad_ref64(Dn, T, M)
    assert gn[4] == 0.0 and np.isfinite(gn).all()
    # the metrics take fmax(D, 1e-3): a NaN depth counts as 1e-3
    assert np.array_equal(depth_metrics_ref64(Dn, T, M), depth_metrics_ref64(np.where(np.isnan(Dn), np.float32(1e-3), Dn), T, M))


def test_metric_thresholds_are_exclusive():
    T = np.array([4.0, 5.0, 16.0, 25.0, 64.0, 125.0], np.float32)
    D = np.array([5.0, 4.0, 25.0, 16.0, 125.0, 64.0], np.float32)  # r = 1.25, 1.25, 1.5625, 1.5625, 1.953125, 1.953125
    m = depth_metrics_ref64(D, T)
    assert list(m[4:8]) == [0.0, 2 / 6, 4 / 6, 6.0]
    below = np.nextafter(D, np.float32(0)).astype(np.float32)
    below[1::2] = D[1::2]
    assert list(depth_metrics_ref64(below, T)[4:7] * 6) == [1.0, 3.0, 5.0]


def test_map_clip_and_overflow_rules():
    m, pix = dmap([[0, 0, CLIP], [0, 0, np.nextafter(np.float32(CLIP), np.float32(1))]])
    assert pix[0] == -1 and pix[1] == 3 * W + 4
    zero, pix = lidar_depth_map_ref64(np.array([[0, 0, 0.0], [0, 0, -0.0]]), EYE, F, F, CX, CY, W, H, 0.0)
    assert (pix == -1).all() and not zero.any()
    # NaN and infinite coordinates drop the point
    _, pix = dmap([[np.nan, 0, 3.0], [0, 0, np.nan], [np.inf, 0, 3.0], [0, 0, np.inf], [0, 0, -np.inf]])
    assert (pix == -1).all()
    # a depth that overflows float32 (6e38) is no return, like the map's +inf empty marker
    A = EYE.copy()
    A[2, 2] = 2.0
    m, pix = dmap([[0, 0, 3e38], [1.0, 0.5, 3.0]], A)
    assert pix[0] == -1 and m[3, 4] == 0.0 and m[3, 5] == 6.0
