"""Host statements, in numpy, of the four kernels a training step runs after the render (the specification of
csrc/loss.cu, csrc/densify.cu, csrc/adam.cu and the peer-load path of csrc/collective.cu).

  * Loss epilogue.  ``loss_fwd64``: the three weighted means in float64 (L1 of gt*m - rgb*m over 3P values, the gt of a
    uint8 image being u8 / 255; sky * accumulation over P; the entropy -(oa log oa + (1-oa) log(1-oa)) of
    oa = clamp(object_acc, fp32(1e-5), fp32(1 - 1e-5)) over P).  ``loss_fwd_bound``: how far the kernel's fp32 sums may
    be from it.  ``loss_bwd_f32``: the cotangents replayed in float32 in the kernel's order (k = g * w / n, then
    -k * sgn(gt*m - rgb*m) * m; the entropy's closed-interval pass-through), ``loss_bwd64`` the same in float64.
  * Densification statistics.  ``densify_f32``: the update of sgn_densify_stats for one segment, replayed in float32
    with separately rounded operations (densify.cu is built with --fmad=false).
  * Adam.  ``adam_f32``: torch.optim.Adam's recurrence for one tensor in float32, separately rounded (adam.cu is built
    with --fmad=false; its sqrtf and division are IEEE), from the fp32 fields of an sgn_adam_tensor row;
    ``adam64``: the same recurrence in float64.
  * Two-shot exchange.  ``my_part``: rank r's part of a slice; ``skipped_units``: the float4 units of a row-skipping
    slice that nobody saw; ``exchange_f32``: the rank-order fp32 sum times ``scale``.
"""
from __future__ import annotations

import numpy as np

f32 = np.float32
U = 2.0 ** -24                      # unit roundoff of float32
CLAMP_LO = f32(1e-5)                # torch.clamp(min=1e-5) on a float32 tensor
CLAMP_HI = f32(1.0) - f32(1e-5)     # 1.f - 1e-5f in the kernel; equals fp32(1 - 1e-5) (pinned by the CPU test)
LOSS_THREADS, LOSS_BLOCKS = 256, 1056


# ---- loss epilogue -----------------------------------------------------------------------------------------------------
def gt_float(gt: np.ndarray) -> np.ndarray:
    """The ground truth as float64: u8 / 255, or the float image."""
    return gt.astype(np.float64) / 255.0 if gt.dtype == np.uint8 else gt.astype(np.float64)


def _l1_terms(rgb, gt, mask):
    g = gt_float(gt).reshape(-1, 3)
    r = rgb.astype(np.float64).reshape(-1, 3)
    m = np.ones((g.shape[0], 1)) if mask is None else mask.astype(np.float64).reshape(-1, 1)
    return np.abs(g * m - r * m), (np.abs(g) + np.abs(r)) * np.abs(m)


def _entropy_terms(oa32):
    oa = np.clip(oa32.astype(np.float32), CLAMP_LO, CLAMP_HI).astype(np.float64).reshape(-1)
    a, b = -oa * np.log(oa), -(1.0 - oa) * np.log1p(-oa)
    return a + b, a, b


def loss_fwd64(P, rgb=None, gt=None, mask=None, accumulation=None, sky_mask=None, object_acc=None, w=(1.0, 1.0, 1.0)):
    """[L1, sky, entropy], each weight * mean in float64; a term whose inputs are missing is 0."""
    wl, ws, we = (float(f32(x)) for x in w)
    l1 = wl * _l1_terms(rgb, gt, mask)[0].sum() / (3 * P) if rgb is not None else 0.0
    sky = 0.0
    if accumulation is not None and sky_mask is not None:
        sky = ws * np.where(sky_mask.reshape(-1) != 0, accumulation.astype(np.float64).reshape(-1), 0.0).sum() / P
    ent = we * _entropy_terms(object_acc)[0].sum() / P if object_acc is not None else 0.0
    return np.array([l1, sky, ent])


def sum_depth(n: int) -> int:
    """Additions a single term passes through in the forward: the per-thread strided sum (at most ceil(n / (1056 * 256))
    steps, plus 3 for the terms of a float4 unit that the aligned path adds first), the 5 + 3 levels of the block tree, the
    at most ceil(1056 / 256) = 5 partials each thread of the finish kernel adds, and its 5 + 3 tree levels."""
    return -(-n // (LOSS_BLOCKS * LOSS_THREADS)) + 3 + 8 + -(-LOSS_BLOCKS // LOSS_THREADS) + 8


def loss_fwd_bound(P, rgb=None, gt=None, mask=None, accumulation=None, sky_mask=None, object_acc=None, w=(1.0, 1.0, 1.0)):
    """Absolute error bound of the kernel's three terms against loss_fwd64, to first order in U and doubled:

        |got - ref| <= 2 w (d U S + E) / n + 2 U |ref|

    S is the sum of the terms' magnitudes (all terms are non-negative), d = sum_depth(n): each addition rounds the running
    sum once, and a term is in at most d of them.  E sums each term's own error: for L1, gt = u8 / 255 (1 rounding), the
    two products with the mask and the difference bound it by 3 U (|gt| + |rgb|) |m|; for the entropy, logf within 1 ulp (2 U relative) and two more roundings in each half,
    4 U (|a| + |b|), plus U for the rounding of 1 - oa (an absolute error of at most 2^-25 in 1 - oa changes
    (1 - oa) log(1 - oa) by at most 2^-25 (1 + |log(1 - oa)|) <= U).  The last term is the division by n and the weight."""
    wl, ws, we = (float(f32(x)) for x in w)
    ref = loss_fwd64(P, rgb, gt, mask, accumulation, sky_mask, object_acc, w)
    bound = np.zeros(3)
    if rgb is not None:
        t, mag = _l1_terms(rgb, gt, mask)
        d = sum_depth(3 * P)
        bound[0] = 2 * abs(wl) * (d * U * t.sum() + 3 * U * mag.sum()) / (3 * P)
    if accumulation is not None and sky_mask is not None:
        t = np.abs(np.where(sky_mask.reshape(-1) != 0, accumulation.astype(np.float64).reshape(-1), 0.0))
        bound[1] = 2 * abs(ws) * sum_depth(P) * U * t.sum() / P
    if object_acc is not None:
        t, a, b = _entropy_terms(object_acc)
        bound[2] = 2 * abs(we) * (sum_depth(P) * U * t.sum() + (4 * U * (a + b) + U).sum()) / P
    return bound + 2 * U * np.abs(ref)


def gt_f32(gt: np.ndarray) -> np.ndarray:
    """The ground truth as the kernel reads it: fp32(u8) / 255.f (IEEE division), or the float image."""
    return gt.astype(f32) / f32(255.0) if gt.dtype == np.uint8 else gt.astype(f32)


def _l1_sign(rgb, gt, mask):
    """sgn(fp32(gt*m) - fp32(rgb*m)): the products are rounded separately (the sign of a rounded difference is the sign of
    the exact one)."""
    g = gt_f32(gt).reshape(-1, 3)
    r = rgb.astype(f32).reshape(-1, 3)
    m = np.ones((g.shape[0], 1), f32) if mask is None else mask.astype(f32).reshape(-1, 1)
    return np.sign((g * m).astype(np.float64) - (r * m).astype(np.float64))


def loss_bwd_f32(P, rgb=None, gt=None, mask=None, sky_mask=None, object_acc=None, w=(1.0, 1.0, 1.0), g=(1.0, 1.0, 1.0)):
    """(v_rgb [P*3], v_acc [P], v_obj [P]) in float32, in the kernel's order.  v_rgb and v_acc are exact replays; v_obj
    uses float64 logs of the fp32 oa (compare it with a bound, see ent_bwd_bound)."""
    wl, ws, we = (f32(x) for x in w)
    g0, g1, g2 = (f32(x) for x in g)
    v_rgb = v_acc = v_obj = None
    if rgb is not None:
        k = (g0 * wl) / f32(3 * P)
        s = _l1_sign(rgb, gt, mask).astype(f32)
        m = np.ones((P, 1), f32) if mask is None else mask.astype(f32).reshape(-1, 1)
        v_rgb = ((-k * s) * m).astype(f32).reshape(-1)
    k1 = (g1 * ws) / f32(P)
    v_acc = np.where(sky_mask.reshape(-1) != 0, k1, f32(0)).astype(f32) if sky_mask is not None else np.zeros(P, f32)
    if object_acc is not None:
        v_obj = ent_bwd64(P, object_acc, we, g2).astype(f32)
    return v_rgb, v_acc, v_obj


def ent_k(P, w, g) -> np.float32:
    return (f32(g) * f32(w)) / f32(P)


def ent_bwd64(P, object_acc, w, g):
    """k * (log(1 - oa) - log(oa)) in float64 with the kernel's fp32 k, 0 outside the closed interval."""
    x = object_acc.astype(f32).reshape(-1)
    inside = (x >= CLAMP_LO) & (x <= CLAMP_HI)
    oa = np.clip(x, CLAMP_LO, CLAMP_HI).astype(np.float64)
    return np.where(inside, float(ent_k(P, w, g)) * (np.log1p(-oa) - np.log(oa)), 0.0)


def ent_bwd_bound(P, object_acc, w, g):
    """4 U |k| (|log oa| + |log(1 - oa)|): logf within 1 ulp for each log (2 U relative), the subtraction and the
    product with k one rounding each (k itself is the kernel's fp32 value in ent_bwd64)."""
    oa = np.clip(object_acc.astype(f32).reshape(-1), CLAMP_LO, CLAMP_HI).astype(np.float64)
    return 4 * U * abs(float(ent_k(P, w, g))) * (np.abs(np.log(oa)) + np.abs(np.log1p(-oa)))


def loss_bwd64(P, rgb=None, gt=None, mask=None, sky_mask=None, object_acc=None, w=(1.0, 1.0, 1.0), g=(1.0, 1.0, 1.0)):
    """The cotangents in float64 (torch's: d|x| = sgn(x), clamp passes the gradient on its closed interval)."""
    wl, ws, we = (float(f32(x)) for x in w)
    g0, g1, g2 = (float(x) for x in g)
    v_rgb = v_acc = v_obj = None
    if rgb is not None:
        gf, r = gt_float(gt).reshape(-1, 3), rgb.astype(np.float64).reshape(-1, 3)
        m = np.ones((P, 1)) if mask is None else mask.astype(np.float64).reshape(-1, 1)
        v_rgb = (-g0 * wl / (3 * P) * np.sign(gf * m - r * m) * m).reshape(-1)
    if sky_mask is not None:
        v_acc = np.where(sky_mask.reshape(-1) != 0, g1 * ws / P, 0.0)
    if object_acc is not None:
        x = object_acc.astype(f32).reshape(-1)
        inside = (x >= CLAMP_LO) & (x <= CLAMP_HI)
        oa = np.clip(x, CLAMP_LO, CLAMP_HI).astype(np.float64)
        v_obj = np.where(inside, g2 * we / P * (np.log1p(-oa) - np.log(oa)), 0.0)
    return v_rgb, v_acc, v_obj


# ---- densification statistics ------------------------------------------------------------------------------------------
def inv_max_size(height: int, width: int) -> np.float32:
    return f32(1.0) / f32(max(height, width))


def densify_f32(v_xy: np.ndarray, radii: np.ndarray, first: bool, prev, height: int, width: int):
    """One segment's (xys_grad_norm, vis_counts, max_2Dsize) after one call, from its rows' v_records[:, 0:2] and radii.
    ``prev``: the three arrays before the call (ignored when ``first``)."""
    x, y = v_xy[:, 0].astype(f32), v_xy[:, 1].astype(f32)
    gn = np.sqrt((x * x) + (y * y)).astype(f32)
    r = radii.astype(np.int64)
    vis = r > 0
    ratio = (r.astype(f32) * inv_max_size(height, width)).astype(f32)
    if first:
        return gn, np.ones_like(gn), np.where(vis, np.maximum(f32(0), ratio), f32(0)).astype(f32)
    g0, c0, m0 = (a.astype(f32) for a in prev)
    return (np.where(vis, gn + g0, g0).astype(f32), np.where(vis, c0 + f32(1), c0).astype(f32),
            np.where(vis, np.maximum(m0, ratio), m0).astype(f32))


# ---- Adam ----------------------------------------------------------------------------------------------------------------
def adam_f32(p, g, m, v, row):
    """One step of one tensor from its sgn_adam_tensor row (optim.ADAM_DTYPE): (p, m, v) in float32.

        m = m + (1 - beta1) (g - m)                      exp_avg.lerp_(grad, 1 - beta1)
        v = v beta2 + (1 - beta2) g g                    exp_avg_sq.mul_(beta2).addcmul_(grad, grad, value=1 - beta2)
        p = p - step_size (m / (sqrt(v) / sqrt_bc2 + eps))
    """
    w1, w2, b2 = f32(row["one_minus_beta1"]), f32(row["one_minus_beta2"]), f32(row["beta2"])
    ss, bc, eps = f32(row["step_size"]), f32(row["sqrt_bc2"]), f32(row["eps"])
    p, g, m, v = (a.astype(f32) for a in (p, g, m, v))
    m = m + w1 * (g - m)
    v = v * b2 + (w2 * g) * g
    p = p - ss * (m / (np.sqrt(v) / bc + eps))
    return p.astype(f32), m.astype(f32), v.astype(f32)


def adam64(p, g, m, v, lr, step, betas=(0.9, 0.999), eps=1e-15):
    """torch.optim.Adam's step ``step`` (1-based) in float64."""
    b1, b2 = betas
    p, g, m, v = (a.astype(np.float64) for a in (p, g, m, v))
    m = b1 * m + (1 - b1) * g
    v = b2 * v + (1 - b2) * g * g
    p = p - lr / (1 - b1 ** step) * m / (np.sqrt(v) / np.sqrt(1 - b2 ** step) + eps)
    return p, m, v


# ---- two-shot exchange ---------------------------------------------------------------------------------------------------
def my_part(len4: int, rank: int, world: int):
    """Rank ``rank``'s float4 units [b, e) of a slice of ``len4`` units: parts of ceil(len4 / world), the last ones short
    or empty."""
    per = (len4 + world - 1) // world
    b = min(len4, per * rank)
    return b, min(len4, b + per)


def skipped_units(len4: int, width: int, nrows: int, vis_rows: np.ndarray) -> np.ndarray:
    """Bool [len4]: units of a row-skipping slice that are neither pulled nor pushed.  Unit i covers floats 4i .. 4i+3,
    i.e. rows 4i // width .. (4i + 3) // width; only rows < nrows count (floats behind nrows * width are padding).  A
    unit is skipped when none of its rows was seen (``vis_rows``: the slice's own rows of the union)."""
    i = np.arange(len4, dtype=np.int64)
    ra, rb = 4 * i // width, np.minimum((4 * i + 3) // width, nrows - 1)
    skip = np.ones(len4, bool)
    live = ra < nrows
    seen = np.zeros(len4, bool)
    span = int((rb - ra)[live].max()) + 1 if live.any() else 0
    for d in range(span):
        r = ra + d
        ok = live & (r <= rb)
        seen[ok] |= vis_rows[r[ok]] != 0
    skip[live] = ~seen[live]
    return skip


def exchange_f32(replicas, scale: float) -> np.ndarray:
    """The rank-order fp32 sum of the replicas (starting from +0, as the kernel does) times ``scale``."""
    acc = np.zeros_like(replicas[0], dtype=f32)
    for x in replicas:
        acc = (acc + x.astype(f32)).astype(f32)
    return (acc * f32(scale)).astype(f32)
