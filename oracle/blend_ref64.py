"""Float64 reference of the tile blend, forward and backward, written from its specification (SURVEY.md Appendix A.6,
the post-ops of DESIGN.md §1).  TEST INFRASTRUCTURE -- never imported by the product package.

It takes what ``sgn_blend_fwd`` / ``sgn_blend_bwd`` take: records[N,12] (include/sgn_raster.h), the per-tile lists
(``sorted_ids`` with the object flag in bit 31, ``tile_bins``) and the class sub-lists (``cls_ids``, ``cls_bins``).

Forward, per pixel, front to back over its tile's list (gsplat rasterize_forward):
    sigma = a dx^2 / 2 + b dx dy + c dy^2 / 2,  (dx, dy) = Gaussian centre - pixel centre (j + 0.5, i + 0.5)
    alpha = min(clamp_fwd, o exp(-sigma));  skip when sigma < 0, o exp(-sigma) < 1/255 or either is NaN
    stop BEFORE blending an entry whose new transmittance would be <= 1e-4.
The objects-only and background-only accumulations run the same rule on the class-filtered lists; their last-entry
index is a position in the class sub-list.  The background slot of ``final_idx`` holds -2 (BG_SAME_AS_MAIN) for a
pixel whose main stream met no valid object entry while it was live (the stopping entry included), -3 (BG_TODO)
is never left: the background pass overwrites it with its own index.

Backward (gsplat rasterize_backward): back to front from the saved T_final with alpha = min(clamp_bwd, o exp(-sigma)),
T_k = T_{k+1} / (1 - alpha_k), a straight-through clamp (d alpha / d sigma = -o exp(-sigma) even where clamped).
Everything is accumulated in float64.

Every skip / stop decision (and the post-ops' branch points) records its relative distance from its threshold:
``forward(...)["margin"]`` is the per-pixel minimum, which test cases keep far from zero so that fp32 kernels and
this reference take the same branches.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, Optional

import numpy as np

TILE = 16
ALPHA_MIN = 1.0 / 255.0
T_STOP = 1e-4
ID_MASK = 0x7FFFFFFF
BG_SAME_AS_MAIN = -2
BG_TODO = -3
RECORD_FLOATS = 12
# record columns: x y | conic a b c | opacity | r g b | depth
COL_X, COL_Y, COL_A, COL_B, COL_C, COL_O = 0, 1, 2, 3, 4, 5
COL_RGBD = [6, 7, 8, 9]


@dataclass
class Opts:
    clamp_fwd: float = 0.999
    clamp_bwd: float = 0.99
    class_streams: bool = True
    has_sky: bool = False
    eval_clamp: bool = False
    raw_mode: bool = False
    background: tuple = (0.0, 0.0, 0.0, 0.0)
    split_fwd_main: int = 768  # list length up to which a tile is one strip (the kernel's default): tile_depth[1] depends on it


@dataclass
class Inputs:
    width: int
    height: int
    records: np.ndarray      # [N,12] float32 (float64 accepted: finite differences)
    sorted_ids: np.ndarray   # [M] int32 payloads, bit 31 = object
    tile_bins: np.ndarray    # [tiles,2] int32
    cls_ids: Optional[np.ndarray] = None   # [2, stride] int32: [0] background sub-lists, [1] object sub-lists
    cls_bins: Optional[np.ndarray] = None  # [2, tiles, 2] int32
    sky: Optional[np.ndarray] = None       # [H,W,3]

    @property
    def tiles_x(self) -> int:
        return (self.width + TILE - 1) // TILE

    @property
    def tiles(self) -> int:
        return self.tiles_x * ((self.height + TILE - 1) // TILE)


def strips_for(n: int, split: int) -> int:
    return 1 if n <= split else 2 if n <= 2 * split else 4 if n <= 4 * split else 8


def _tile_pixels(inp: Inputs, tiles: np.ndarray):
    """[G,256] pixel centres, flat pixel index (0 outside) and inside mask of each tile, rows in tile order."""
    tx, ty = tiles % inp.tiles_x, tiles // inp.tiles_x
    r, c = np.divmod(np.arange(TILE * TILE), TILE)
    i = ty[:, None] * TILE + r[None, :]
    j = tx[:, None] * TILE + c[None, :]
    inside = (i < inp.height) & (j < inp.width)
    pid = np.where(inside, i * inp.width + j, 0)
    return j + 0.5, i + 0.5, pid, inside, r


class _Stream:
    """One front-to-back stream over padded lists gid[G,L] (row N = a never-valid dummy) for pixels [G,P]."""

    def __init__(self, rec, gid, px, py, inside, clamp, gm=None):
        self.gid = gid
        r = rec[gid]  # [G,L,12]
        gx, gy, a, b, c, o = (r[:, None, :, k] for k in range(6))
        self.a, self.b, self.c = a, b, c
        self.dx = gx - px[:, :, None]
        self.dy = gy - py[:, :, None]
        L = gid.shape[1]
        with np.errstate(all="ignore"):
            qa, qb, qc = 0.5 * a * self.dx * self.dx, b * self.dx * self.dy, 0.5 * c * self.dy * self.dy
            sigma = qa + qb + qc
            self.vis = np.exp(-sigma)
            self.raw = o * self.vis
            s_ok = sigma >= 0
            a_ok = self.raw >= ALPHA_MIN
            self.valid = s_ok & a_ok & inside[:, :, None]
            alpha = np.where(self.valid, np.minimum(clamp, self.raw), 0.0)
            scale = np.abs(qa) + np.abs(qb) + np.abs(qc)
            m_sigma = np.where(a_ok & (scale > 0), np.abs(sigma) / np.where(scale > 0, scale, 1.0), np.inf)
            m_alpha = np.where(s_ok & np.isfinite(self.raw), np.abs(self.raw * 255.0 - 1.0), np.inf)
            m_valid = np.fmin(np.nan_to_num(m_sigma, nan=np.inf), np.nan_to_num(m_alpha, nan=np.inf))
        Tc = np.cumprod(1.0 - alpha, axis=2)  # transmittance after entry k (invalid entries: factor 1)
        k = np.arange(L)
        Tprev = np.concatenate([np.ones_like(Tc[:, :, :1]), Tc[:, :, :-1]], axis=2)
        if L:
            stopm = self.valid & (Tc <= T_STOP)
            self.ks = np.where(stopm.any(2), stopm.argmax(2), L)  # index of the stopping entry (L: never)
            self.blended = self.valid & (k[None, None, :] < self.ks[:, :, None])
            T_stop = np.take_along_axis(Tprev, np.minimum(self.ks, L - 1)[:, :, None], 2)[:, :, 0]
            self.T_final = np.where(self.ks >= L, Tc[:, :, -1], T_stop)
            self.last = np.where(self.blended.any(2), L - 1 - self.blended[:, :, ::-1].argmax(2), -1)
        else:
            self.ks = np.zeros(px.shape, np.int64)
            self.blended = self.valid
            self.T_final = np.ones(px.shape)
            self.last = np.full(px.shape, -1, np.int64)
        reached = k[None, None, :] <= self.ks[:, :, None]
        self.w = np.where(self.blended, alpha * Tprev, 0.0)
        self.n_blended = self.blended.sum(2)
        m_stop = np.where(self.valid & reached, np.abs(Tc / T_STOP - 1.0), np.inf)
        # fp32 transmittance drifts with the number of products: the stop margin is scaled down accordingly
        m_stop = m_stop.min(2, initial=np.inf) / np.maximum(1.0, self.n_blended / 250.0)
        m_valid = np.where(reached & inside[:, :, None], m_valid, np.inf)
        self.margin = np.minimum(m_valid.min(2, initial=np.inf), m_stop)
        self.margin = np.where(inside, self.margin, np.inf)
        # per-Gaussian: the closest call among the decisions it takes part in (a stop is charged to the stopping entry
        # and to the last one blended)
        if gm is not None and L:
            np.minimum.at(gm, gid, m_valid.min(1))
            G = np.arange(gid.shape[0])[:, None].repeat(px.shape[1], 1)
            for kk in (np.minimum(self.ks, L - 1), np.maximum(self.last, 0)):
                np.minimum.at(gm, gid[G, kk], np.where(inside, m_stop, np.inf))

    def backward(self, values, v_ch, tfv_acc, T_final, clamp, out, out_abs, v_val=None, v_val_abs=None):
        """Adds this stream's per-Gaussian geometry gradients to out[N+1, 0:6] and its channel gradients to v_val[N+1,C],
        and to out_abs / v_val_abs the same sums taken over the absolute values of their terms (what bounds the rounding
        error of an fp32 evaluation: these sums cancel, e.g. the depth cotangent's terms of a Gaussian that alone makes up
        a pixel's depth).  values [N+1,C] the blended channels (None: none), v_ch [G,P,C] their cotangents, tfv_acc [G,P]
        the cotangent of 1 - T_final, T_final [G,P]."""
        B = self.blended
        with np.errstate(all="ignore"):
            ab = np.minimum(clamp, self.raw)
            ra = np.where(B, 1.0 / (1.0 - ab), 1.0)
            Tp = T_final[:, :, None] * np.cumprod(ra[:, :, ::-1], axis=2)[:, :, ::-1]  # T before entry k
            fac = np.where(B, ab * Tp, 0.0)
            v_alpha = T_final[:, :, None] * ra * tfv_acc[:, :, None]
            v_abs = np.abs(v_alpha)
            if values is not None and values.shape[1]:
                colors = values[self.gid]  # [G,L,C]
                cv = np.einsum("glc,gpc->gpl", colors, v_ch)
                cva = np.einsum("glc,gpc->gpl", np.abs(colors), np.abs(v_ch))
                x, xa = fac * cv, fac * cva
                behind = np.cumsum(x[:, :, ::-1], axis=2)[:, :, ::-1] - x  # sum over later blended entries
                behind_a = np.cumsum(xa[:, :, ::-1], axis=2)[:, :, ::-1] - xa
                v_alpha = v_alpha + Tp * cv - ra * behind
                v_abs = v_abs + Tp * cva + ra * behind_a
                vc = np.einsum("gpl,gpc->glc", fac, v_ch)
                vca = np.einsum("gpl,gpc->glc", fac, np.abs(v_ch))
                np.add.at(v_val, self.gid, vc)
                np.add.at(v_val_abs, self.gid, vca)
            v_alpha = np.where(B, v_alpha, 0.0)
            vs = np.where(B, -self.raw * v_alpha, 0.0)  # d/d sigma
            vsa = np.where(B, np.abs(self.raw) * v_abs, 0.0)
            dx, dy, a, b, c = self.dx, self.dy, self.a, self.b, self.c
            terms = {
                COL_X: (vs * (a * dx + b * dy), vsa * (np.abs(a * dx) + np.abs(b * dy))),
                COL_Y: (vs * (b * dx + c * dy), vsa * (np.abs(b * dx) + np.abs(c * dy))),
                COL_A: (vs * 0.5 * dx * dx, vsa * 0.5 * dx * dx), COL_B: (vs * dx * dy, vsa * np.abs(dx * dy)),
                COL_C: (vs * 0.5 * dy * dy, vsa * 0.5 * dy * dy),
                COL_O: (self.vis * v_alpha, self.vis * v_abs),
            }
            for col, (t, ta) in terms.items():
                np.add.at(out[:, col], self.gid, np.where(B, t, 0.0).sum(1))
                np.add.at(out_abs[:, col], self.gid, np.where(B, ta, 0.0).sum(1))


def _padded(rows_per_tile, dummy):
    L = max((len(r) for r in rows_per_tile), default=0)
    g = np.full((len(rows_per_tile), L), dummy, np.int64)
    for n, r in enumerate(rows_per_tile):
        g[n, :len(r)] = r
    return g


def _groups(inp: Inputs):
    """Tiles grouped by list length (one vectorised pass per group)."""
    tb = np.asarray(inp.tile_bins, np.int64)
    lens = tb[:, 1] - tb[:, 0]
    for L in np.unique(lens):
        yield np.nonzero(lens == L)[0]


def _run(inp: Inputs, opts: Opts):
    rec = np.asarray(inp.records, np.float64)
    N = rec.shape[0]
    rec = np.concatenate([rec, np.zeros((1, RECORD_FLOATS))], 0)  # row N: opacity 0, valid for no pixel
    H, W = inp.height, inp.width
    P = H * W
    ids = np.asarray(inp.sorted_ids, np.int64)
    tb = np.asarray(inp.tile_bins, np.int64)
    cls = opts.class_streams
    S = 3 if cls else 1
    o = dict(raw=np.zeros((P, 4)), final_T=np.ones((S, P)), final_idx=np.full((S, P), -1, np.int64),
             tile_depth=np.zeros((3, inp.tiles), np.int64), margin=np.full(P, np.inf), hit=np.zeros(P, bool),
             gauss_margin=np.full(N + 1, np.inf))
    gm = o["gauss_margin"]
    streams = []
    for tiles in _groups(inp):
        px, py, pid, inside, prow = _tile_pixels(inp, tiles)
        lists = [ids[tb[t, 0]:tb[t, 1]] for t in tiles]
        main_rows = _padded([(l & ID_MASK) for l in lists], N)
        m = _Stream(rec, main_rows, px, py, inside, opts.clamp_fwd, gm)
        pos0 = tb[tiles, 0]
        o["raw"][pid[inside]] = np.einsum("gpl,glc->gpc", m.w, rec[main_rows][:, :, COL_RGBD])[inside]
        o["final_T"][0, pid[inside]] = m.T_final[inside]
        o["final_idx"][0, pid[inside]] = np.where(m.last >= 0, pos0[:, None] + m.last, -1)[inside]
        np.minimum.at(o["margin"], pid[inside], m.margin[inside])
        o["tile_depth"][0, tiles] = np.where(m.last >= 0, m.last + 1, 0).max(1)
        entry = dict(tiles=tiles, pid=pid, inside=inside, main=m)
        if cls:
            objm = [(l < 0) for l in lists]
            sub = []
            for c in (0, 1):
                rows = []
                for n, t in enumerate(tiles):
                    want = lists[n][objm[n] == bool(c)] & ID_MASK
                    s0, s1 = inp.cls_bins[c][t]
                    have = np.asarray(inp.cls_ids[c][s0:s1], np.int64) & ID_MASK
                    assert np.array_equal(want, have), f"tile {t}: class {c} sub-list is not the stable partition of the list"
                    rows.append(want)
                st = _Stream(rec, _padded(rows, N), px, py, inside, opts.clamp_fwd, gm)
                np.minimum.at(o["margin"], pid[inside], st.margin[inside])
                start = np.asarray(inp.cls_bins[c], np.int64)[tiles, 0]
                sub.append((st, start))
            (bst, bstart), (ost, ostart) = sub
            Lm = main_rows.shape[1]
            isobj = _padded([om.astype(np.int64) for om in objm], 0).astype(bool)
            # hit: a valid object entry met while the main stream was live (the stopping entry included)
            reached = np.arange(Lm)[None, None, :] <= m.ks[:, :, None]
            hit = (m.valid & reached & isobj[:, None, :]).any(2) if Lm else np.zeros(px.shape, bool)
            o["hit"][pid[inside]] = hit[inside]
            o["final_T"][1, pid[inside]] = ost.T_final[inside]
            o["final_idx"][1, pid[inside]] = np.where(ost.last >= 0, ostart[:, None] + ost.last, -1)[inside]
            o["final_T"][2, pid[inside]] = np.where(hit, bst.T_final, m.T_final)[inside]
            o["final_idx"][2, pid[inside]] = np.where(hit, np.where(bst.last >= 0, bstart[:, None] + bst.last, -1),
                                                      BG_SAME_AS_MAIN)[inside]
            o["tile_depth"][2, tiles] = np.where(hit & (bst.last >= 0), bst.last + 1, 0).max(1)
            # tile_depth[1]: how far the object streams ran past the main traversal, strip by strip.  A strip leaves the
            # list at the first 8-entry boundary (counted from the tile's first entry) at which all its main streams
            # have ended; the object streams still live there continue on the object sub-list.
            nobj_before = np.concatenate([np.zeros((len(tiles), 1), np.int64), np.cumsum(isobj, 1)], 1)
            n_obj = isobj.sum(1)
            for n, t in enumerate(tiles):
                Wn = strips_for(Lm, opts.split_fwd_main)
                rows_per = TILE // Wn
                for s in range(Wn):
                    sel = (prow // rows_per == s) & inside[n]
                    if not sel.any():
                        continue
                    ks = m.ks[n][sel]
                    e = Lm if (ks >= Lm).any() else min(Lm, 8 * -(-(int(ks.max()) + 1) // 8))
                    passed = int(nobj_before[n, e])
                    live = (ost.ks[n][sel] >= passed).any()
                    if live and passed < n_obj[n]:
                        kdeep = int(ost.last[n][sel].max())
                        if kdeep >= passed:
                            o["tile_depth"][1, t] = max(o["tile_depth"][1, t], kdeep + 1 - passed)
            entry.update(obj=ost, bg=bst, hit=hit)
        streams.append(entry)
    return rec, streams, o


def _post(inp: Inputs, opts: Opts, o):
    H, W = inp.height, inp.width
    raw = o["raw"]
    T = o["final_T"][0]
    alpha = 1.0 - T
    res = {}
    if opts.raw_mode:
        bg = np.asarray(opts.background, np.float64)
        res["rgb"] = raw[:, :3] + T[:, None] * bg[None, :3]
        res["depth"] = raw[:, 3] + T * bg[3]
    else:
        cl = np.minimum(raw[:, :3], 1.0)
        fin = cl
        if opts.has_sky:
            sky = np.asarray(inp.sky, np.float64).reshape(-1, 3)
            fin = cl * alpha[:, None] + sky * (1.0 - alpha[:, None])
        with np.errstate(all="ignore"):
            # the post-ops' branch points are met by fp32 sums and 1 - T, whose errors are absolute: their margins are
            # absolute distances, in units of 0.2 (5e-5 <-> 1e-5) for the sums and 0.02 for the final colour (one product)
            m = np.where(raw[:, :3] != 1.0, np.abs(raw[:, :3] - 1.0), np.inf).min(1) / 0.2  # clamp(max=1): gradient switch
            if opts.eval_clamp:
                m = np.minimum(m, np.where(fin != 0.0, np.abs(fin), np.inf).min(1) / 0.02)
                m = np.minimum(m, np.where(fin != 1.0, np.abs(fin - 1.0), np.inf).min(1) / 0.02)
                fin = np.clip(fin, 0.0, 1.0)
            m = np.minimum(m, np.abs(alpha - 1e-3) / 0.2)  # depth: alpha > 1e-3
            res["depth"] = np.where(alpha > 1e-3, raw[:, 3] / np.where(alpha > 1e-3, alpha, 1.0), 10.0)
        o["margin"] = np.minimum(o["margin"], m)
        res["rgb"] = fin
    res["accumulation"] = alpha
    if opts.class_streams:
        res["object_acc"] = 1.0 - o["final_T"][1]
        res["background_acc"] = 1.0 - o["final_T"][2]
    out = {k: v.reshape(H, W, -1) if v.ndim == 2 else v.reshape(H, W) for k, v in res.items()}
    out["raw"] = raw.reshape(H, W, 4)
    S = o["final_T"].shape[0]
    out["final_T"] = o["final_T"].reshape(S, H, W)
    out["final_idx"] = o["final_idx"].reshape(S, H, W)
    out["tile_depth"] = o["tile_depth"]
    out["margin"] = o["margin"].reshape(H, W)
    out["hit"] = o["hit"].reshape(H, W)
    out["gauss_margin"] = o["gauss_margin"][:-1]
    return out


def forward(inp: Inputs, opts: Opts) -> Dict[str, np.ndarray]:
    """rgb [H,W,3], accumulation / depth / object_acc / background_acc [H,W], raw [H,W,4], final_T / final_idx [S,H,W],
    tile_depth [3,tiles], margin [H,W] (smallest relative distance of any decision from its threshold), gauss_margin [N]
    (the same per Gaussian, skip / stop decisions only)."""
    _, _, o = _run(inp, opts)
    return _post(inp, opts, o)


def backward(inp: Inputs, opts: Opts, cot: Dict[str, Optional[np.ndarray]]):
    """(v_records [N,12] in record layout (float64), v_sky [H,W,3] or None, the forward, and [N,12] sums of the absolute
    values of each gradient's terms) for the cotangents ``cot`` of the final outputs (keys rgb [H,W,3], accumulation,
    depth, object_acc, background_acc [H,W]; None or missing = no cotangent)."""
    rec, streams, o = _run(inp, opts)
    fw = _post(inp, opts, dict(o))
    H, W = inp.height, inp.width
    P = H * W
    N = rec.shape[0] - 1
    get = lambda k: None if cot.get(k) is None else np.asarray(cot[k], np.float64).reshape(P, -1)
    v_rgb, v_acc, v_dep, v_obj, v_bg = (get(k) for k in ("rgb", "accumulation", "depth", "object_acc", "background_acc"))
    raw = o["raw"]
    T = o["final_T"][0]
    alpha = 1.0 - T
    vch = np.zeros((P, 4))
    voa = np.zeros(P) if v_acc is None else v_acc[:, 0].copy()
    v_sky = None
    if opts.raw_mode:  # out_c = blended_c + T_final * bg_c
        bg = np.asarray(opts.background, np.float64)
        if v_rgb is not None:
            vch[:, :3] = v_rgb
            voa -= v_rgb @ bg[:3]
        if v_dep is not None:
            vch[:, 3] = v_dep[:, 0]
            voa -= bg[3] * v_dep[:, 0]
    else:
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
                v_sky = (v * (1.0 - alpha[:, None])).reshape(H, W, 3)
                vch[:, :3] = np.where(raw[:, :3] <= 1.0, v * alpha[:, None], 0.0)
            else:
                vch[:, :3] = np.where(raw[:, :3] <= 1.0, v, 0.0)
        if v_dep is not None:
            ok = alpha > 1e-3
            a_ = np.where(ok, alpha, 1.0)
            vch[:, 3] = np.where(ok, v_dep[:, 0] / a_, 0.0)
            voa += np.where(ok, -v_dep[:, 0] * raw[:, 3] / (a_ * a_), 0.0)
    out = np.zeros((N + 1, RECORD_FLOATS))
    out_abs = np.zeros((N + 1, RECORD_FLOATS))
    for e in streams:
        pid, inside = e["pid"], e["inside"]

        def tile_view(x):  # [P] or [P,C] -> [G,256] or [G,256,C], zero outside the image
            g = x[pid]
            return np.where(inside.reshape(inside.shape + (1,) * (g.ndim - 2)), g, 0.0)

        m = e["main"]
        m.backward(rec[:, COL_RGBD], tile_view(vch), tile_view(voa), m.T_final, opts.clamp_bwd, out, out_abs,
                   out[:, 6:10], out_abs[:, 6:10])
        if v_obj is not None:
            e["obj"].backward(None, None, tile_view(v_obj[:, 0]), e["obj"].T_final, opts.clamp_bwd, out, out_abs)
        if v_bg is not None:
            e["bg"].backward(None, None, tile_view(v_bg[:, 0]), e["bg"].T_final, opts.clamp_bwd, out, out_abs)
    if opts.has_sky and v_sky is None and v_rgb is None:
        v_sky = np.zeros((H, W, 3))
    return out[:N], v_sky, fw, out_abs[:N]


# ------------------------------------------------------------------------------------------------------------------
# generic channels: the main stream (slot 0) compositing values[N,C] -- sgn_blend_extra_fwd / _bwd, and the Level-1
# rasterize_gaussians (out = blended + T_final * background, alpha = 1 - T_final)
# ------------------------------------------------------------------------------------------------------------------
def _channels(values, N):
    v = np.asarray(values, np.float64).reshape(N, -1)
    return np.concatenate([v, np.zeros((1, v.shape[1]))], 0)  # row N: the padding dummy


def forward_channels(inp: Inputs, opts: Opts, values, background=None) -> Dict[str, np.ndarray]:
    """out [H,W,C] = sum_k values[k,c] alpha_k T_k (+ T_final background[c]), abs [H,W,C] the same sum over |terms|,
    final_T / final_idx [H,W] of the main stream, margin [H,W] and gauss_margin [N] as in ``forward``."""
    rec, streams, o = _run(inp, opts)
    N = rec.shape[0] - 1
    vals = _channels(values, N)
    H, W, Cn = inp.height, inp.width, vals.shape[1]
    out = np.zeros((H * W, Cn))
    out_abs = np.zeros((H * W, Cn))
    for e in streams:
        pid, inside, m = e["pid"], e["inside"], e["main"]
        out[pid[inside]] = np.einsum("gpl,glc->gpc", m.w, vals[m.gid])[inside]
        out_abs[pid[inside]] = np.einsum("gpl,glc->gpc", m.w, np.abs(vals[m.gid]))[inside]
    T = o["final_T"][0]
    if background is not None:
        bg = np.asarray(background, np.float64).reshape(Cn)
        out += T[:, None] * bg[None, :]
        out_abs += T[:, None] * np.abs(bg)[None, :]
    return dict(out=out.reshape(H, W, Cn), abs=out_abs.reshape(H, W, Cn), final_T=T.reshape(H, W),
                final_idx=o["final_idx"][0].reshape(H, W), margin=o["margin"].reshape(H, W), gauss_margin=o["gauss_margin"][:-1])


def backward_channels(inp: Inputs, opts: Opts, values, v_out, v_alpha=None, background=None):
    """(v_values [N,C], v_records [N,12] with the geometry in columns 0..5 (the rest 0), and the sums of the absolute
    values of each gradient's terms in the same two layouts) for the cotangents v_out [H,W,C] of ``forward_channels``'s out
    and v_alpha [H,W] of 1 - T_final."""
    rec, streams, o = _run(inp, opts)
    N = rec.shape[0] - 1
    vals = _channels(values, N)
    H, W, Cn = inp.height, inp.width, vals.shape[1]
    P = H * W
    vch = np.asarray(v_out, np.float64).reshape(P, Cn)
    voa = np.zeros(P) if v_alpha is None else np.asarray(v_alpha, np.float64).reshape(P).copy()
    if background is not None:  # out_c = blended_c + T_final bg_c: T_final = 1 - alpha
        voa -= vch @ np.asarray(background, np.float64).reshape(Cn)
    out = np.zeros((N + 1, RECORD_FLOATS))
    out_abs = np.zeros((N + 1, RECORD_FLOATS))
    v_val = np.zeros((N + 1, Cn))
    v_val_abs = np.zeros((N + 1, Cn))
    for e in streams:
        pid, inside, m = e["pid"], e["inside"], e["main"]

        def tile_view(x):
            g = x[pid]
            return np.where(inside.reshape(inside.shape + (1,) * (g.ndim - 2)), g, 0.0)

        m.backward(vals, tile_view(vch), tile_view(voa), m.T_final, opts.clamp_bwd, out, out_abs, v_val, v_val_abs)
    return v_val[:N], out[:N], v_val_abs[:N], out_abs[:N]
