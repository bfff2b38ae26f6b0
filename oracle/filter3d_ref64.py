"""Float64 statement of Mip-Splatting's 3D smoothing filter: the filter sweep and the filtered projection.  TEST
INFRASTRUCTURE -- never imported by the product.

Written from the specification (Mip-Splatting, Yu et al. 2024, eq. 7 and its compute_3D_filter / get_scaling_with_3D_filter /
get_opacity_with_3D_filter), on top of oracle/project_ref64.py and oracle/project_aa_ref64.py, whose statements it reuses:

Sweep.  For row i of sub-model m with mean mu, over the views v in which m is present, p = A_vm mu + b_vm (camera space);
view v samples the row when z > near and u = fx x / z + cx in [-0.15 W, 1.15 W], w = fy y / z + cy in [-0.15 H, 1.15 H]
(inclusive).  nu_i = max over sampling views of max(fx, fy) / z; sigma_i = sqrt(variance) / nu_i.  Rows no view samples
take the lowest nu of all sampled rows (of all sub-models); with no row sampled every sigma is 0.

Projection.  With s = exp(scales): s' = sqrt(s^2 + sigma^2) replaces s in the covariance, and the opacity of a visible row
is sigmoid(logit) * coef (* comp in the antialiased mode, comp from the filtered covariance), coef = prod_k sqrt(s_k^2 /
(s_k^2 + sigma^2)).  sigma is a constant.  ``forward`` / ``backward`` mirror project_ref64's (the VJP by torch autograd).
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from oracle import project_aa_ref64 as aa
from oracle import project_ref64 as ref
from oracle.oracle_torch import expf_spec


def sweep(means: Sequence[np.ndarray], views: Sequence[dict], M: np.ndarray, present: np.ndarray, variance: float = 0.2,
          near: float = 0.2) -> Dict:
    """means[m] [n_m, 3]; views[v] = dict(fx, fy, cx, cy, width, height); M [V, S, 3, 4] object->camera; present [V, S].
    Returns sigma (list of [n_m]), nu (list, 0 = unsampled), sampled (list of bool masks), margin (list: per row, the
    smallest relative distance of any present view's z / u / w from its sampling boundary), fill (the unsampled rows' sigma)
    and n_sampled.  Every expression is evaluated in float64 in the order csrc/filter3d.cu writes it."""
    nus, margins = [], []
    for m, mu in enumerate(means):
        mu = np.asarray(mu, np.float64).reshape(-1, 3)
        nu = np.zeros(mu.shape[0])
        mg = np.full(mu.shape[0], np.inf)
        for v, vw in enumerate(views):
            if not present[v, m]:
                continue
            A = np.asarray(M[v, m], np.float64)
            z = ((A[2, 0] * mu[:, 0] + A[2, 1] * mu[:, 1]) + A[2, 2] * mu[:, 2]) + A[2, 3]
            x = ((A[0, 0] * mu[:, 0] + A[0, 1] * mu[:, 1]) + A[0, 2] * mu[:, 2]) + A[0, 3]
            y = ((A[1, 0] * mu[:, 0] + A[1, 1] * mu[:, 1]) + A[1, 2] * mu[:, 2]) + A[1, 3]
            fx, fy, cx, cy = (float(np.float32(vw[k])) for k in ("fx", "fy", "cx", "cy"))
            W, H = int(vw["width"]), int(vw["height"])
            front = z > near
            zs = np.where(front, z, 1.0)
            u = fx * x / zs + cx
            w = fy * y / zs + cy
            lo_u, hi_u, lo_w, hi_w = -0.15 * W, 1.15 * W, -0.15 * H, 1.15 * H
            inside = front & (u >= lo_u) & (u <= hi_u) & (w >= lo_w) & (w <= hi_w)
            nu = np.where(inside, np.maximum(nu, max(fx, fy) / zs), nu)
            mz = np.abs(z - near) / max(near, 1e-30)
            mu_ = np.minimum(np.abs(u - lo_u), np.abs(u - hi_u)) / max(W, 1)
            mw = np.minimum(np.abs(w - lo_w), np.abs(w - hi_w)) / max(H, 1)
            mg = np.minimum(mg, np.where(front, np.minimum.reduce([mz, mu_, mw]), mz))
        nus.append(nu)
        margins.append(mg)
    sampled = [nu > 0 for nu in nus]
    n_sampled = int(sum(s.sum() for s in sampled))
    sq = np.sqrt(variance)
    fill = 0.0
    if n_sampled:
        fill = sq / min(nu[s].min() for nu, s in zip(nus, sampled) if s.any())
    sigma = [np.where(s, sq / np.where(s, nu, 1.0), fill) for nu, s in zip(nus, sampled)]
    return dict(sigma=sigma, nu=nus, sampled=sampled, margin=margins, fill=fill, n_sampled=n_sampled)


def _axes(ls, sigma):
    """Per axis (r, v): v = s^2 + sigma^2 and r = s^2 / v, with r = 1 where v == 0 (sigma 0 and s^2 below the dtype's
    smallest number: the filter is the identity there).  In float64 v is never 0 for the scales the tests use; in float32 a
    thin axis of exp(-80) reaches v == 0 (sigma 0) or r == 0 (sigma > 0), as the kernels' float32 arithmetic does."""
    s = expf_spec(ls) if ls.dtype == torch.float32 else torch.exp(ls)  # float32: the kernels' exp sequence
    s2 = s * s
    v = s2 + (sigma * sigma)[:, None]
    pos = v > 0
    return torch.where(pos, s2 / torch.where(pos, v, torch.ones_like(v)), torch.ones_like(v)), v


def _sqrt0(x):
    """sqrt(x) for x >= 0 whose gradient at 0 is 0 rather than inf * 0 = nan (only float32 evaluations reach 0 here)."""
    pos = x > 0
    return torch.where(pos, torch.sqrt(torch.where(pos, x, torch.ones_like(x))), torch.zeros_like(x))


def coef(ls, sigma):
    """prod_k sqrt(s_k^2 / (s_k^2 + sigma^2)), s = exp(ls) (torch, differentiable in ls)."""
    return _sqrt0(_axes(ls, sigma)[0]).prod(-1)


def filtered_scales(ls, sigma):
    """s' = sqrt(exp(ls)^2 + sigma^2) (torch, differentiable in ls)."""
    return _sqrt0(_axes(ls, sigma)[1])


def forward(frame, st: ref.Settings, sigmas: Sequence, antialiased: bool = False, dtype=torch.float64,
            grad: bool = False) -> Dict:
    """The filtered fused projection of every segment of ``frame`` (sigmas[k]: segment k's filter sizes [n_k]).  Returns what
    project_ref64.forward returns (records, rec, leaves, radii, tmin, tmax, vis, margin, ...) plus ``coef`` (numpy, every row)."""
    cam = frame.camera
    leaves, mws, qrs, lss, fdcs, rests, opl, cls, sgs = [], [], [], [], [], [], [], [], []
    for sg, sig in zip(frame.segments, sigmas):
        lf = ref._leaves(sg, dtype, grad)
        leaves.append(lf)
        F = lf["features_dc"].shape[1]
        idft = torch.tensor(sg.idft_f32()[:F].astype(np.float64), dtype=dtype)
        fdcs.append((lf["features_dc"] * idft[None, :, None]).sum(1))
        if sg.has_pose:
            R, t, q = (torch.tensor(x.astype(np.float64), dtype=dtype) for x in sg.pose_f32())
            mws.append(lf["means"] @ R.reshape(3, 3).T + t)
            bw_, bx, by, bz = lf["quats"].unbind(-1)
            aw, ax, ay, az = q
            qrs.append(torch.stack([aw * bw_ - ax * bx - ay * by - az * bz, aw * bx + ax * bw_ + ay * bz - az * by,
                                    aw * by - ax * bz + ay * bw_ + az * bx, aw * bz + ax * by - ay * bx + az * bw_], -1))
        else:
            mws.append(lf["means"])
            qrs.append(lf["quats"])
        lss.append(lf["scales"])
        rests.append(lf["features_rest"])
        opl.append(lf["opacities"][:, 0])
        cls.append(np.full(sg.params.num_points, sg.cls, np.int64))
        sgs.append(torch.as_tensor(np.asarray(sig.detach().cpu() if torch.is_tensor(sig) else sig, np.float64), dtype=dtype))
    mw, qr, ls = torch.cat(mws), torch.cat(qrs), torch.cat(lss)
    fdc, rest, logit, sigma = torch.cat(fdcs), torch.cat(rests), torch.cat(opl), torch.cat(sgs)
    cls = np.concatenate(cls)
    N = mw.shape[0]
    pr = ref.project_core(mw, qr, filtered_scales(ls, sigma), cam, st.block_width, st.clip_thresh, dtype)
    vis = pr["vis"]
    vt = torch.from_numpy(vis)
    aux = np.where(cls == 1, ref.AUX_OBJECT, 0) | np.where(vis, ref.AUX_VISIBLE, 0)
    if st.sh_degree > 0:
        cp = torch.tensor(cam.cam_pos().astype(np.float64), dtype=dtype)
        d = mw.detach() - cp
        d = torch.where(vt[:, None], d, torch.ones_like(d))
        d = d / torch.sqrt((d * d).sum(-1, keepdim=True))
        Y = ref.sh_basis(st.deg_use, d)
        Kuse = (st.deg_use + 1) ** 2
        terms = Y[:, :1, None] * fdc[:, None, :]
        if Kuse > 1:
            terms = torch.cat([terms, Y[:, 1:Kuse, None] * rest[:, :Kuse - 1]], 1)
        pre = terms.sum(1) + 0.5
        pass_ = pre.detach().double().numpy() >= 0
        rgb = torch.where(torch.from_numpy(pass_), pre, torch.zeros_like(pre))
        aux = aux | np.where(vis, (pass_ * np.array([1, 2, 4])).sum(1), 0)
    else:
        rgb = torch.sigmoid(fdc)
        aux = aux | np.where(vis, 7, 0)
    cf = coef(ls, sigma)
    opac = torch.sigmoid(logit) * cf
    comp = None
    if antialiased:
        comp = aa.compensation(pr["a"], pr["b"], pr["c"]) * vt
        opac = opac * comp
    rec = torch.cat([pr["xy"], pr["conic"] * vt[:, None], (opac * vt)[:, None], rgb * vt[:, None], (pr["z"] * vt)[:, None]], 1)
    recn = np.zeros((N, 12))
    recn[:, :10] = rec.detach().double().numpy()
    recn[:, 2:5] = pr["conic"].detach().double().numpy()
    if comp is not None:
        recn[:, 11] = comp.detach().double().numpy()
    mg = pr["margins"]
    mg["pre"] = np.full(N, np.inf)
    margin = np.minimum.reduce([mg[k] for k in ref.MARGIN_NAMES]) if N else np.zeros(0)
    return dict(leaves=leaves, rec=rec, records=recn, radii=pr["radius"], tmin=pr["tmin"], tmax=pr["tmax"], vis=vis, aux=aux,
                num_tiles_hit=np.where(vis, (pr["tmax"][:, 0] - pr["tmin"][:, 0]) * (pr["tmax"][:, 1] - pr["tmin"][:, 1]), 0),
                margin=margin, coef=cf.detach().double().numpy())


def backward(frame, st: ref.Settings, sigmas: Sequence, v_records: np.ndarray, antialiased: bool = False,
             dtype=torch.float64) -> List[Dict[str, np.ndarray]]:
    """Gradients of sum(records[:, :10] * v_records[:, :10]) of the filtered projection w.r.t. the six parameter tensors of
    every segment (sigma held constant)."""
    fw = forward(frame, st, sigmas, antialiased, dtype, grad=True)
    v = torch.tensor(np.asarray(v_records, np.float64)[:, :10], dtype=dtype)
    return aa._grads(fw["leaves"], (fw["rec"] * v).sum())


def bake(ls: np.ndarray, logit: np.ndarray, sigma: np.ndarray):
    """Mip-Splatting's fused export in float64: (log s', logit(sigmoid(o) * coef))."""
    ls = np.asarray(ls, np.float64)
    s2 = np.exp(2.0 * ls)
    sig2 = np.asarray(sigma, np.float64).reshape(-1, 1) ** 2
    c = np.sqrt(s2 / (s2 + sig2)).prod(1, keepdims=True)
    o = 1.0 / (1.0 + np.exp(-np.asarray(logit, np.float64).reshape(-1, 1))) * c
    return 0.5 * np.log(s2 + sig2), np.log(o) - np.log1p(-o)
