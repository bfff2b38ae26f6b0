"""Float64 reference of the absolute screen-space gradient (AbsGS, Ye et al. 2024; gsplat's absgrad) that
``sgn_blend_bwd_absgrad`` accumulates.  TEST INFRASTRUCTURE -- never imported by the product package.

For every row k:  absgrad[k] = (sum_p |g_x(k,p)|, sum_p |g_y(k,p)|), where g(k,p) is the gradient of pixel p's MAIN-stream
outputs (rgb, accumulation, depth) with respect to row k's screen-space mean -- the per-pixel term whose sum over p is
v_records[k, 0:2]:  g = vs (a dx + b dy, b dx + c dy),  vs = d/d sigma = -o exp(-sigma) v_alpha  (blend_ref64's notation).
The objects-only and background-only streams and the extra channels add nothing.

Built on blend_ref64's traversal (``_run`` / ``_Stream``); the prologue that turns the final outputs' cotangents into those
of the raw blend is restated here for the main stream (blend_ref64.backward, which it mirrors, sums over pixels at once).
"""
from __future__ import annotations

from typing import Dict, Optional

import numpy as np

from oracle import blend_ref64 as ref


def _main_cotangents(inp: ref.Inputs, opts: ref.Opts, o, cot):
    """(vch [P,4], voa [P]): the cotangents of the main stream's blended channels (rgb, depth) and of 1 - T_final."""
    P = inp.height * inp.width
    get = lambda k: None if cot.get(k) is None else np.asarray(cot[k], np.float64).reshape(P, -1)
    v_rgb, v_acc, v_dep = (get(k) for k in ("rgb", "accumulation", "depth"))
    raw = o["raw"]
    alpha = 1.0 - o["final_T"][0]
    vch = np.zeros((P, 4))
    voa = np.zeros(P) if v_acc is None else v_acc[:, 0].copy()
    if opts.raw_mode:
        bg = np.asarray(opts.background, np.float64)
        if v_rgb is not None:
            vch[:, :3] = v_rgb
            voa -= v_rgb @ bg[:3]
        if v_dep is not None:
            vch[:, 3] = v_dep[:, 0]
            voa -= bg[3] * v_dep[:, 0]
        return vch, voa
    if v_rgb is not None:
        v = v_rgb.copy()
        cl = np.minimum(raw[:, :3], 1.0)
        fin = cl
        if opts.has_sky:
            sky = np.asarray(inp.sky, np.float64).reshape(P, 3)
            fin = cl * alpha[:, None] + sky * (1.0 - alpha[:, None])
        if opts.eval_clamp:
            v = np.where((fin < 0.0) | (fin > 1.0), 0.0, v)
        if opts.has_sky:
            voa += (v * (cl - sky)).sum(1)
            vch[:, :3] = np.where(raw[:, :3] <= 1.0, v * alpha[:, None], 0.0)
        else:
            vch[:, :3] = np.where(raw[:, :3] <= 1.0, v, 0.0)
    if v_dep is not None:
        ok = alpha > 1e-3
        a_ = np.where(ok, alpha, 1.0)
        vch[:, 3] = np.where(ok, v_dep[:, 0] / a_, 0.0)
        voa += np.where(ok, -v_dep[:, 0] * raw[:, 3] / (a_ * a_), 0.0)
    return vch, voa


def absgrad(inp: ref.Inputs, opts: ref.Opts, cot: Dict[str, Optional[np.ndarray]]):
    """(absgrad [N,2], bound [N,2], signed [N,2]) for the cotangents ``cot`` (keys rgb [H,W,3], accumulation, depth [H,W];
    other keys are ignored: their streams do not contribute).  ``bound`` is the per-element sum of the absolute values of
    the factors of each term, |vs| (|a dx| + |b dy|) with |vs| from the absolute values of v_alpha's terms, as
    blend_ref64.backward's out_abs: the scale of an fp32 evaluation's rounding.  ``signed`` is the sum of the same terms
    with their signs, i.e. blend_ref64.backward's v_records[:, 0:2] for main-stream cotangents."""
    rec, streams, o = ref._run(inp, opts)
    N = rec.shape[0] - 1
    vch, voa = _main_cotangents(inp, opts, o, cot)
    values = rec[:, ref.COL_RGBD]
    out = np.zeros((N + 1, 2))
    out_abs = np.zeros((N + 1, 2))
    signed = np.zeros((N + 1, 2))
    for e in streams:
        pid, inside = e["pid"], e["inside"]
        m = e["main"]
        v_ch = np.where(inside[:, :, None], vch[pid], 0.0)
        tfv = np.where(inside, voa[pid], 0.0)
        B = m.blended
        with np.errstate(all="ignore"):
            ab = np.minimum(opts.clamp_bwd, m.raw)
            ra = np.where(B, 1.0 / (1.0 - ab), 1.0)
            Tp = m.T_final[:, :, None] * np.cumprod(ra[:, :, ::-1], axis=2)[:, :, ::-1]  # T before entry k
            fac = np.where(B, ab * Tp, 0.0)
            colors = values[m.gid]
            cv = np.einsum("glc,gpc->gpl", colors, v_ch)
            cva = np.einsum("glc,gpc->gpl", np.abs(colors), np.abs(v_ch))
            x, xa = fac * cv, fac * cva
            behind = np.cumsum(x[:, :, ::-1], axis=2)[:, :, ::-1] - x
            behind_a = np.cumsum(xa[:, :, ::-1], axis=2)[:, :, ::-1] - xa
            v_alpha = m.T_final[:, :, None] * ra * tfv[:, :, None] + Tp * cv - ra * behind
            v_abs = np.abs(m.T_final[:, :, None] * ra * tfv[:, :, None]) + Tp * cva + ra * behind_a
            vs = np.where(B, -m.raw * v_alpha, 0.0)
            vsa = np.where(B, np.abs(m.raw) * v_abs, 0.0)
            dx, dy, a, b, c = m.dx, m.dy, m.a, m.b, m.c
            gx, gy = vs * (a * dx + b * dy), vs * (b * dx + c * dy)
            bx, by = vsa * (np.abs(a * dx) + np.abs(b * dy)), vsa * (np.abs(b * dx) + np.abs(c * dy))
        for col, (g, bnd) in enumerate(((gx, bx), (gy, by))):
            g = np.where(B, g, 0.0)
            np.add.at(out[:, col], m.gid, np.abs(g).sum(1))
            np.add.at(signed[:, col], m.gid, g.sum(1))
            np.add.at(out_abs[:, col], m.gid, np.where(B, bnd, 0.0).sum(1))
    return out[:N], out_abs[:N], signed[:N]
