"""Float64 statement of the sky lookup's gradient for its direction, and of that gradient reduced to the view's rotation
(the specification of csrc/sky.cu's cube_dir_grad and sgn_sky_bwd_view_rot), on top of oracle/sky_ref64.py.

Not autograd: the lookup's floor, clamp and face choice are piecewise, and nvdiffrast's gradient (texture.cu:1005-1046 with
indexCubeMapGrad, :123-148) is the derivative of the bilinear interpolation with the taps held fixed and the [0,1] clamp
of s, t passed straight through.  So, per lookup, with the taps a as the forward reads them (wrapped, and at a cube corner
the missing one THIRD times the sum of the other three):

    g_s = sum_ch v ((a10 - a00) + fv (a11 + a00 - a10 - a01)) R,   g_t = sum_ch v ((a01 - a00) + fu (a11 + a00 - a10 - a01)) R
    dL/dl = (m/2) (g_s U + g_t V) - sigma (m^2/2) (g_s <l,U> + g_t <l,V>) N_axis,   m = 1/|c|

(N_axis the unit vector of the major axis, sigma the sign of its component c) on the raw direction; an invalid lookup, a
zero cotangent or a non-finite value gives 0.

Camera form (EnvLight.forward, sgn_splatfacto.py:140-147): l = TO_OPENGL (R_c2w u), u the normalised jittered camera-space
direction, so v_d = TO_OPENGL^T v_l = (v_l.x, -v_l.z, v_l.y), v_R[i][j] = sum v_d[i] u[j], and in the view's layout
(viewmat[:3,:3] = (R_c2w diag(1,-1,-1))^T) v_view[4j+i] = s_j v_R[i][j], s = (1, -1, -1); the translation entries are 0."""
from __future__ import annotations

import numpy as np

from oracle import sky_ref64 as ref

EPS = 2.0 ** -24
SIGNS = np.array([1.0, -1.0, -1.0])


def _taps(tex: np.ndarray, lk: dict, R: int):
    """a [..., 4, 3] float64: the four taps with the corner rule (invalid lookups: zeros)."""
    idx = ref.taps(lk, R)
    flat = np.asarray(tex, np.float64).reshape(-1, 3)
    miss = idx < 0
    a = flat[np.maximum(idx, 0)] * (~miss)[..., None]
    avg = a.sum(-2, keepdims=True) * ref.THIRD
    return np.where(miss[..., None], avg, a), idx


def face_grad(tex, l, v, R: int):
    """(g_s, g_t) [...] per lookup, float64 (0 for an invalid lookup)."""
    lk = ref.lookup(l, R)
    a, _ = _taps(tex, lk, R)
    v = np.asarray(v, np.float64)
    ad = a[..., 3, :] + a[..., 0, :] - a[..., 1, :] - a[..., 2, :]
    gs = (v * ((a[..., 1, :] - a[..., 0, :]) + lk["fv"][..., None] * ad)).sum(-1) * R
    gt = (v * ((a[..., 2, :] - a[..., 0, :]) + lk["fu"][..., None] * ad)).sum(-1) * R
    gs, gt = np.where(lk["valid"], gs, 0.0), np.where(lk["valid"], gt, 0.0)
    return gs, gt, lk


def _chain(l, gs, gt, lk):
    """dL/dl from the face-coordinate gradient, on the raw direction; non-finite -> 0."""
    l = np.asarray(l, np.float64)
    B = ref.BASIS[lk["face"]].astype(np.float64)  # [..., 3, 3]
    N, U, V = B[..., 0, :], B[..., 1, :], B[..., 2, :]
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        c = (l * N).sum(-1)  # |c| (N points along the major component's sign)
        m = 1.0 / c
        lu, lv = (l * U).sum(-1), (l * V).sum(-1)
        g = 0.5 * m[..., None] * (gs[..., None] * U + gt[..., None] * V) \
            - (0.5 * m * m * (gs * lu + gt * lv))[..., None] * N
    ok = lk["valid"][..., None] & np.isfinite(g).all(-1, keepdims=True)
    return np.where(ok, g, 0.0)


def grad_uv(tex, l, v, R: int) -> np.ndarray:
    """d <lookup(tex, l), v> / d l [..., 3] in float64 (the contract above)."""
    l = np.asarray(l, np.float64)
    gs, gt, lk = face_grad(tex, l, v, R)
    zero = (np.asarray(v) == 0).all(-1)
    return np.where(zero[..., None], 0.0, _chain(l, gs, gt, lk))


def grad_uv_bound(tex, l, v, R: int) -> np.ndarray:
    """Per-element fp32 bound of grad_uv evaluated in fp32 on the same direction: 2^-24 times 16 (the length of the rounding
    chain) times the gradient of |terms| (|v|, |a| and |l| throughout), plus the texel-coordinate noise -- fu, fv computed
    from an fp32 s R - 1/2, 4 R 2^-24 texel -- times |v| |a11 + a00 - a10 - a01| R through the chain, plus 1e-30."""
    l = np.asarray(l, np.float64)
    lk = ref.lookup(l, R)
    a, _ = _taps(tex, lk, R)
    av = np.abs(np.asarray(v, np.float64))
    aa = np.abs(a)
    ad = aa[..., 3, :] + aa[..., 0, :] + aa[..., 1, :] + aa[..., 2, :]
    gs = (av * ((aa[..., 1, :] + aa[..., 0, :]) + lk["fv"][..., None] * ad)).sum(-1) * R
    gt = (av * ((aa[..., 2, :] + aa[..., 0, :]) + lk["fu"][..., None] * ad)).sum(-1) * R
    noise = (av * np.abs(a[..., 3, :] + a[..., 0, :] - a[..., 1, :] - a[..., 2, :])).sum(-1) * R * 4 * R * EPS
    gs, gt = np.where(lk["valid"], gs, 0.0), np.where(lk["valid"], gt, 0.0)
    B = ref.BASIS[lk["face"]].astype(np.float64)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        m = 1.0 / np.abs((l * B[..., 0, :]).sum(-1))
        lu, lv = np.abs((l * B[..., 1, :]).sum(-1)), np.abs((l * B[..., 2, :]).sum(-1))
        scale = 0.5 * m * (1 + m * (lu + lv))
        b = (16 * EPS * (gs + gt) + 2 * noise) * scale
    b = np.where(lk["valid"] & np.isfinite(b), b, 0.0)
    return np.broadcast_to(b[..., None], l.shape) + 1e-30


def camera_rays(fx, fy, cx, cy, W: int, H: int, ju=None, jv=None) -> np.ndarray:
    """u [H, W, 3]: the normalised camera-space directions of sky_ref64.directions, before the rotation."""
    return ref.directions(np.eye(3), fx, fy, cx, cy, W, H, ju, jv) @ ref.TO_OPENGL


def view_from_rot(v_R: np.ndarray) -> np.ndarray:
    """v_view [12] (viewmat 3x4 row-major) from the cotangent of c2w[:3,:3]: v_view[4j+i] = s_j v_R[i][j]."""
    out = np.zeros(12)
    for i in range(3):
        for j in range(3):
            out[4 * j + i] = SIGNS[j] * v_R[i, j]
    return out


def grad_view(viewmat, camera_params, tex, v, R: int, ju=None, jv=None, l=None, parts: bool = False):
    """v_view [12] in float64 for the sky of a camera with world->camera ``viewmat`` (3x4) and ``camera_params`` (fx, fy, cx,
    cy, W, H), cotangent v [H, W, 3].  ``l``: look up these directions in place of the float64 ones (e.g. a kernel's own
    fp32 directions, so that both take the same face and texel decisions); the rotation chain still uses the float64 u.
    ``parts``: also return the per-entry sums of |terms| sum |v_d[i]| |u[j]| and the summed per-lookup bound of v_d."""
    fx, fy, cx, cy, W, H = camera_params
    c2w = ref.c2w_from_viewmat(np.asarray(viewmat, np.float64))
    u = camera_rays(fx, fy, cx, cy, W, H, ju, jv)
    if l is None:
        l = ref.directions(c2w, fx, fy, cx, cy, W, H, ju, jv)
    gl = grad_uv(tex, l, v, R)
    vd = np.stack([gl[..., 0], -gl[..., 2], gl[..., 1]], -1)
    out = view_from_rot(np.einsum("hwi,hwj->ij", vd, u))
    if not parts:
        return out
    b = grad_uv_bound(tex, l, v, R)
    terms = view_from_rot(np.abs(np.einsum("hwi,hwj->ij", np.abs(vd), np.abs(u))))
    noise = view_from_rot(np.abs(np.einsum("hwi,hwj->ij", b, np.abs(u))))
    return out, np.abs(terms), np.abs(noise)
