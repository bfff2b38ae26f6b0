"""Float64 statement of the lidar depth supervision in numpy: the checker of csrc/depth.cu (sgn_lidar_depth_map,
sgn_depth_loss_fwd / _bwd, sgn_depth_metrics) and of depth.py.

Map: a point p goes through the camera-from-point 3x4 ``A`` (the viewmat, or the viewmat times the sweep's to_world):
pv = A [p; 1], z = pv.z, rw = 1 / (z + 1e-6), u = pv.x rw fx + cx, v = pv.y rw fy + cy.  It is dropped when z <= clip_thresh
or when (u, v) lies outside [0, W) x [0, H); otherwise it lands on pixel (floor(u), floor(v)), where the smallest z wins.
Pixels without a return are 0.  Edges: z == clip_thresh is dropped (so are z = +-0 with clip_thresh = 0); u == 0 or -0.0 is
column 0 and u == W is off the image (the same for v and H); a NaN z, u or v (a NaN or infinite coordinate) drops the point;
a return whose depth is +inf in float32 (it overflows there) is no return, since it equals the map's empty marker.

Loss over the valid pixels (target > 0 and mask != 0): L = w sum |D - T| / n_valid, 0 when n_valid = 0; its cotangent is
g w sign(D - T) / n_valid on the valid pixels and 0 elsewhere.  A target that is <= 0, -0.0 or NaN makes the pixel invalid; a
mask of -0.0 removes it, a fractional or NaN mask keeps it (NaN != 0).  D == T has a zero cotangent (sign 0).  A NaN depth on a
valid pixel makes the loss NaN, and its cotangent is 0: sign(NaN) is taken as 0, neither above nor below the target.

Metrics over the same pixels with d = fmax(D, float32(1e-3)), t = T: abs_rel, sq_rel, rmse, rmse_log, a1, a2, a3 (the fraction
with max(d/t, t/d) < 1.25^k: a ratio of exactly 1.25, 1.5625 or 1.953125 is outside) and n_valid; the means are NaN when
n_valid = 0.  fmax ignores a NaN, so a NaN depth counts as 1e-3, like a pixel that rendered no depth: eval scores it as a miss
instead of turning every metric of the image into NaN."""
from __future__ import annotations

import numpy as np

METRIC_NAMES = ("abs_rel", "sq_rel", "rmse", "rmse_log", "a1", "a2", "a3", "n_valid")


def compose(viewmat, to_world=None) -> np.ndarray:
    """The camera-from-point 3x4 in float64: ``viewmat`` [3,4] (or [4,4]) times [to_world; 0 0 0 1]."""
    V = np.asarray(viewmat, np.float64)[:3, :4]
    if to_world is None:
        return V.copy()
    T = np.eye(4)
    T[:3, :4] = np.asarray(to_world, np.float64)[:3, :4]
    return V @ T


def project_points_ref64(points, A, fx, fy, cx, cy):
    """(z, u, v) float64 [M] of every point."""
    P = np.asarray(points, np.float64).reshape(-1, 3)
    A = np.asarray(A, np.float64)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        pv = P @ A[:, :3].T + A[:, 3]
        z = pv[:, 2]
        rw = 1.0 / (z + 1e-6)
        u = pv[:, 0] * rw * fx + cx
        v = pv[:, 1] * rw * fy + cy
    return z, u, v


def lidar_depth_map_ref64(points, A, fx, fy, cx, cy, width: int, height: int, clip_thresh: float):
    """Returns (map float64 [H, W], pixel int64 [M]: the flat pixel each point lands on, -1 when it is dropped)."""
    z, u, v = project_points_ref64(points, A, fx, fy, cx, cy)
    with np.errstate(invalid="ignore", over="ignore"):
        keep = (z > clip_thresh) & (u >= 0) & (u < width) & (v >= 0) & (v < height) & np.isfinite(z.astype(np.float32))
    pix = np.full(z.shape[0], -1, np.int64)
    pix[keep] = np.floor(v[keep]).astype(np.int64) * width + np.floor(u[keep]).astype(np.int64)
    flat = np.full(height * width, np.inf)
    np.minimum.at(flat, pix[keep], z[keep])
    flat[np.isinf(flat)] = 0.0
    return flat.reshape(height, width), pix


def valid_ref64(target, mask=None) -> np.ndarray:
    T = np.asarray(target, np.float64).reshape(-1)
    with np.errstate(invalid="ignore"):
        ok = T > 0
        if mask is not None:
            ok &= np.asarray(mask, np.float64).reshape(-1) != 0
    return ok


def depth_loss_ref64(depth, target, mask=None, weight: float = 1.0):
    """(L, n_valid)."""
    D, T = np.asarray(depth, np.float64).reshape(-1), np.asarray(target, np.float64).reshape(-1)
    ok = valid_ref64(target, mask)
    n = int(ok.sum())
    if n == 0:
        return 0.0, 0
    return float(weight) * float(np.abs(D[ok] - T[ok]).sum()) / n, n


def depth_loss_grad_ref64(depth, target, mask=None, weight: float = 1.0, g: float = 1.0) -> np.ndarray:
    """dL/dD (times g), float64 with the shape of ``depth``."""
    D, T = np.asarray(depth, np.float64), np.asarray(target, np.float64)
    ok = valid_ref64(target, mask).reshape(D.shape)
    n = int(ok.sum())
    out = np.zeros(D.shape)
    if n:
        e = D[ok] - T[ok]
        out[ok] = g * weight * np.where(np.isnan(e), 0.0, np.sign(e)) / n
    return out


def depth_metrics_ref64(depth, target, mask=None) -> np.ndarray:
    """float64 [8] in METRIC_NAMES order."""
    D, T = np.asarray(depth, np.float32).reshape(-1), np.asarray(target, np.float64).reshape(-1)
    ok = valid_ref64(target, mask)
    n = int(ok.sum())
    if n == 0:
        return np.array([np.nan] * 7 + [0.0])
    d = np.fmax(D[ok], np.float32(1e-3)).astype(np.float64)
    t = T[ok]
    e = d - t
    r = np.maximum(d / t, t / d)
    return np.array([np.mean(np.abs(e) / t), np.mean(e * e / t), np.sqrt(np.mean(e * e)),
                     np.sqrt(np.mean((np.log(d) - np.log(t)) ** 2)),
                     np.mean(r < 1.25), np.mean(r < 1.25 ** 2), np.mean(r < 1.25 ** 3), float(n)])
