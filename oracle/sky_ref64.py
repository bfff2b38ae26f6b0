"""Float64 statement of the sky cube map lookup (the specification of csrc/sky.cu).

Directions (EnvLight.get_world_directions / forward, sgn_splatfacto.py:118-147): pixel (x = column, y = row),
    d = normalize(((x - cx + ju) / fx, (y - cy + jv) / fy, 1)),  d = c2w[:3,:3] @ d,  l = (d.x, d.z, -d.y)
with ju = jv = 0.5 in eval.  c2w[:3,:3] is the transpose of viewmat[:3,:3] with columns 1 and 2 negated.

Lookup (dr.texture(tex[None], l, filter_mode='linear', boundary_mode='cube')): the major axis picks the face; with the
face basis (N, U, V) of ``BASIS`` a direction on face f has face coordinates s = <l,U> / (2|<l,N>|) + 1/2,
t = <l,V> / (2|<l,N>|) + 1/2, clamped to [0,1]; texel space u = s R - 1/2, v = t R - 1/2, taps (floor u + {0,1},
floor v + {0,1}), bilinear weights from the fractions.  A tap off the face is carried onto the adjacent face (``wrap``, and
its independent geometric statement ``wrap_geometric``); a tap off both axes (a cube corner) takes K * (sum of the other
three), K = fp32 0.33333333.  Non-finite face coordinates sample 0.

The backward is torch float64 autograd of the same gather (``grad``), not a hand-written transpose."""
from __future__ import annotations

import numpy as np

# faces 0..5 = +x, -x, +y, -y, +z, -z; rows N, U, V: direction = N + a U + b V with a = 2s - 1, b = 2t - 1
BASIS = np.array([
    [[1, 0, 0], [0, 0, -1], [0, -1, 0]],
    [[-1, 0, 0], [0, 0, 1], [0, -1, 0]],
    [[0, 1, 0], [1, 0, 0], [0, 0, 1]],
    [[0, -1, 0], [1, 0, 0], [0, 0, -1]],
    [[0, 0, 1], [1, 0, 0], [0, -1, 0]],
    [[0, 0, -1], [-1, 0, 0], [0, -1, 0]],
], dtype=np.int64)
THIRD = float(np.float32(0.33333333))
TO_OPENGL = np.array([[1, 0, 0], [0, 0, 1], [0, -1, 0]], dtype=np.float64)


def c2w_from_viewmat(viewmat: np.ndarray) -> np.ndarray:
    """c2w[:3,:3] from the camera's world->camera 3x4 (Camera._viewmat only transposes and flips signs): exact."""
    R = np.asarray(viewmat)[:3, :3].T.copy()
    R[:, 1:] = -R[:, 1:]
    return R


def directions(c2w: np.ndarray, fx, fy, cx, cy, W: int, H: int, ju=None, jv=None) -> np.ndarray:
    """l [H, W, 3] in float64; ju / jv [H, W] (None = eval, 0.5)."""
    v, u = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    ju = 0.5 if ju is None else np.asarray(ju, np.float64)
    jv = 0.5 if jv is None else np.asarray(jv, np.float64)
    d = np.stack([(u - cx + ju) / fx, (v - cy + jv) / fy, np.ones_like(u)], -1)
    d = d / np.maximum(np.linalg.norm(d, axis=-1, keepdims=True), 1e-12)
    d = d @ np.asarray(c2w, np.float64)[:3, :3].T
    return d @ TO_OPENGL.T


def lookup(l: np.ndarray, R: int) -> dict:
    """Face decision and texel coordinates of directions l [..., 3] (evaluated in float64 on the given values), with the
    distance of every decision from its threshold: ``tie`` (major axis, relative to |c|), ``floor`` (texel space distance
    of u and v to the nearest integer) and ``clamp`` (texel space distance of s and t to 0 or 1)."""
    l = np.asarray(l, np.float64)
    x, y, z = l[..., 0], l[..., 1], l[..., 2]
    ax, ay, az = np.abs(x), np.abs(y), np.abs(z)
    with np.errstate(invalid="ignore", divide="ignore"):
        zmaj = az > np.fmax(ax, ay)
        ymaj = ~zmaj & (ay > ax)
        axis = np.where(zmaj, 2, np.where(ymaj, 1, 0))
        c = np.take_along_axis(l, axis[..., None], -1)[..., 0]
        face = 2 * axis + (c < 0)
        B = BASIS[face]
        ac = np.abs(c)
        m = 0.5 / ac  # U and V have one non-zero component each: <l,U> is that component of l, signed (no 0 * inf terms)
        comp = [(np.take_along_axis(l, np.argmax(np.abs(B[..., k, :]), -1)[..., None], -1)[..., 0]
                 * B[..., k, :].sum(-1)) for k in (1, 2)]
        s_raw = comp[0] * m + 0.5
        t_raw = comp[1] * m + 0.5
        valid = np.isfinite(s_raw) & np.isfinite(t_raw)
        s, t = np.clip(np.where(valid, s_raw, 0.5), 0, 1), np.clip(np.where(valid, t_raw, 0.5), 0, 1)
        u, v = s * R - 0.5, t * R - 0.5
        tie_z = np.abs(az - np.maximum(ax, ay))
        tie = np.where(zmaj, tie_z, np.minimum(tie_z, np.abs(ay - ax))) / ac
        fl = np.minimum(np.abs(u - np.round(u)), np.abs(v - np.round(v)))
        sr, tr = np.where(valid, s_raw, 0.5), np.where(valid, t_raw, 0.5)
        cl = R * np.minimum(np.minimum(np.abs(sr), np.abs(sr - 1)), np.minimum(np.abs(tr), np.abs(tr - 1)))
    i0, j0 = np.floor(u).astype(np.int64), np.floor(v).astype(np.int64)
    # 1 / (2|c|) outside the normal fp32 range: fp32 evaluation loses precision (subnormal) or saturates
    extreme = valid & ((ac < 2.0 ** -126) | (m < 2.0 ** -126))
    return dict(face=face, valid=valid, s=s, t=t, u=u, v=v, i0=i0, j0=j0, fu=u - i0, fv=v - j0, tie=tie, floor=fl, clamp=cl,
                extreme=extreme, fragile=valid & ((fl < 1e-4) | extreme))


def wrap(face, i, j, R: int):
    """Texel index (face * R + j') * R + i' reached by the off-face texel (i, j) of ``face`` (exactly one of i, j outside
    [0, R)): the neighbouring face g has N_g = the outward axis; on g the coordinate along an axis parallel to N_f is pinned
    to R - 1 / 0, the other follows the along-edge index.  The rule csrc/sky.cu evaluates."""
    face, i, j = np.broadcast_arrays(np.asarray(face, np.int64), np.asarray(i, np.int64), np.asarray(j, np.int64))
    off_i = (i < 0) | (i >= R)
    B = BASIS[face]
    e = np.where(off_i[..., None], B[..., 1, :], B[..., 2, :])
    a = np.where(off_i[..., None], B[..., 2, :], B[..., 1, :])
    sgn = np.where((i < 0) | (j < 0), -1, 1)
    out = sgn[..., None] * e
    k = np.where(off_i, j, i)
    axis = np.argmax(np.abs(out), -1)
    g = 2 * axis + (np.take_along_axis(out, axis[..., None], -1)[..., 0] < 0)
    N = B[..., 0, :]
    coord = []
    for c in (1, 2):
        Bg = BASIS[g][..., c, :]
        dn = (N * Bg).sum(-1)
        da = (a * Bg).sum(-1)
        coord.append(np.where(dn > 0, R - 1, np.where(dn < 0, 0, np.where(da > 0, k, R - 1 - k))))
    return (g * R + coord[1]) * R + coord[0]


def wrap_geometric(face, i, j, R: int):
    """The same as ``wrap`` by geometry alone: the off-face texel centre's direction, looked up again (float64), and the
    texel whose centre is nearest on the face it lands on."""
    face, i, j = np.broadcast_arrays(np.asarray(face, np.int64), np.asarray(i, np.int64), np.asarray(j, np.int64))
    a = 2 * (i + 0.5) / R - 1
    b = 2 * (j + 0.5) / R - 1
    B = BASIS[face].astype(np.float64)
    d = B[..., 0, :] + a[..., None] * B[..., 1, :] + b[..., None] * B[..., 2, :]
    lk = lookup(d, R)
    ii = np.clip(np.floor(lk["s"] * R), 0, R - 1).astype(np.int64)
    jj = np.clip(np.floor(lk["t"] * R), 0, R - 1).astype(np.int64)
    return (lk["face"] * R + jj) * R + ii


def taps(lk: dict, R: int):
    """idx [..., 4] texel indices of the taps (i,j), (i+1,j), (i,j+1), (i+1,j+1) (-1: missing corner tap; all -1: invalid)."""
    face, i0, j0 = lk["face"], lk["i0"], lk["j0"]
    out = []
    for di, dj in ((0, 0), (1, 0), (0, 1), (1, 1)):
        i, j = i0 + di, j0 + dj
        oi, oj = (i < 0) | (i >= R), (j < 0) | (j >= R)
        inside = (face * R + np.clip(j, 0, R - 1)) * R + np.clip(i, 0, R - 1)
        w = wrap(face, np.where(oi & oj, 0, i), np.where(oi & oj, 0, j), R) if (oi ^ oj).any() else inside
        out.append(np.where(~oi & ~oj, inside, np.where(oi & oj, -1, w)))
    idx = np.stack(out, -1)
    return np.where(lk["valid"][..., None], idx, -1)


def sample_torch(tex, l: np.ndarray, R: int, dtype=None):
    """out [..., 3] as a torch gather of tex [6, R, R, 3] (differentiable in tex); float64 unless ``dtype`` is given."""
    import torch
    lk = lookup(l, R)
    idx = taps(lk, R)
    dtype = dtype or tex.dtype
    flat = tex.reshape(-1, 3).to(dtype)
    miss = torch.from_numpy(idx < 0)
    a = flat[torch.from_numpy(np.maximum(idx, 0))] * (~miss)[..., None].to(dtype)  # [..., 4, 3]
    avg = a.sum(-2, keepdim=True) * THIRD
    a = torch.where(miss[..., None], avg, a)
    fu = torch.from_numpy(lk["fu"]).to(dtype)[..., None]
    fv = torch.from_numpy(lk["fv"]).to(dtype)[..., None]
    top = a[..., 0, :] + fu * (a[..., 1, :] - a[..., 0, :])
    bot = a[..., 2, :] + fu * (a[..., 3, :] - a[..., 2, :])
    return top + fv * (bot - top), lk, idx


def sample(tex: np.ndarray, l: np.ndarray, R: int) -> np.ndarray:
    import torch
    return sample_torch(torch.from_numpy(np.asarray(tex, np.float64)), l, R)[0].numpy()


def grad(tex_shape, l: np.ndarray, v: np.ndarray, R: int) -> np.ndarray:
    """d <sample(tex, l), v> / d tex (float64 autograd; independent of tex: the lookup is linear in it)."""
    import torch
    tex = torch.zeros(tex_shape, dtype=torch.float64, requires_grad=True)
    out = sample_torch(tex, l, R)[0]
    (out * torch.from_numpy(np.asarray(v, np.float64))).sum().backward()
    return tex.grad.numpy()


def grad_bound(l: np.ndarray, v: np.ndarray, R: int, parts: bool = False):
    """Per texel fp32 summation bound of the gradient: 2^-24 (n + 8) sum |w v| + 4 R 2^-24 sum |v| over the n contributions
    it receives (reordered fp32 sums, plus weights computed from a texel coordinate rounded in fp32).  ``parts``: also return
    the second term alone (the texel-coordinate noise)."""
    import torch
    tex = torch.zeros((6, R, R, 3), dtype=torch.float64, requires_grad=True)
    out = sample_torch(tex, l, R)[0]
    (out * torch.from_numpy(np.abs(np.asarray(v, np.float64)))).sum().backward()
    swv = np.abs(tex.grad.numpy())
    lk = lookup(l, R)
    idx = taps(lk, R)
    n = np.zeros(6 * R * R, np.float64)
    sv = np.zeros(6 * R * R, np.float64)
    vv = np.abs(np.asarray(v, np.float64)).reshape(-1, 3).max(-1)
    flat = idx.reshape(-1, 4)
    for k in range(4):
        ok = flat[:, k] >= 0
        n += np.bincount(flat[ok, k], minlength=n.size)
        sv += np.bincount(flat[ok, k], weights=vv[ok], minlength=n.size)
    eps = 2.0 ** -24
    coord = np.broadcast_to(4 * R * eps * sv[:, None], swv.reshape(-1, 3).shape)
    bound = eps * (n[:, None] + 8) * swv.reshape(-1, 3) + coord + 1e-12
    return (bound, coord) if parts else bound
