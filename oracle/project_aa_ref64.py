"""Float64 statement of the projection in the antialiased rasterize mode.  TEST INFRASTRUCTURE -- never imported by the product.

Written from the specification (gsplat's antialiased mode; the reference's rasterize_mode, sgn_splatfacto.py:214-223, with
the multiply that its :946-949 leaves commented out), on top of oracle/project_ref64.py, whose statements it reuses unchanged:
  * comp = sqrt(max(0, det(cov2d) / det(cov2d + 0.3 I))), cov2d the screen covariance before the 0.3 px^2 blur;
  * the opacity of a visible row is sigmoid(logit) * comp, and comp is NOT detached: its gradient reaches means, scales and
    quats through cov2d (and the box poses / the view through the composition and the projection);
  * record [11] holds comp for visible rows (0 elsewhere); every other record field is the classic mode's.

``forward`` / ``backward`` mirror project_ref64's with that opacity.  ``comp_param_grads`` is the gradient of
sum(comp * v_comp) alone, ``l1_project_bwd`` project_ref64.l1_project_bwd with a cotangent of ``compensation`` too.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import numpy as np
import torch

from oracle import project_ref64 as ref
from oracle.oracle_torch import expf_spec


def compensation(a, b, c):
    """comp from the BLURRED cov2d entries (torch, differentiable).  Where the clamp holds (det_orig / det_blur <= 0) comp
    is 0 with a zero gradient: sqrt is only evaluated on the positive ratios."""
    det_orig = (a - 0.3) * (c - 0.3) - b * b
    det_blur = a * c - b * b
    safe = torch.where(det_blur != 0, det_blur, torch.ones_like(det_blur))
    r = det_orig / safe
    pos = r > 0
    return torch.where(pos, torch.sqrt(torch.where(pos, r, torch.ones_like(r))), torch.zeros_like(r))


def _geometry(frame, leaves: List[Dict[str, torch.Tensor]], st: ref.Settings, dtype) -> Dict:
    """project_ref64.project_core on the world means / quaternions composed from ``leaves`` (project_ref64.forward's compose)."""
    mws, qrs, lss = [], [], []
    for sg, lf in zip(frame.segments, leaves):
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
    ls = torch.cat(lss)
    s = expf_spec(ls) if dtype == torch.float32 else torch.exp(ls)
    return ref.project_core(torch.cat(mws), torch.cat(qrs), s, frame.camera, st.block_width, st.clip_thresh, dtype)


def forward(frame, st: ref.Settings, dtype=torch.float64, grad: bool = False) -> Dict:
    """project_ref64.forward with record [5] = sigmoid(logit) * comp and record [11] = comp (visible rows).  Adds ``comp``
    (numpy, 0 for invisible rows), ``comp_t`` (torch, differentiable) and ``comp_all`` (numpy, every row, unmasked)."""
    fw = ref.forward(frame, st, dtype, grad=grad)
    pr = _geometry(frame, fw["leaves"], st, dtype)
    vt = torch.from_numpy(pr["vis"])
    comp_all = compensation(pr["a"], pr["b"], pr["c"])
    comp = comp_all * vt
    rec = fw["rec"]
    rec = torch.cat([rec[:, :5], rec[:, 5:6] * comp[:, None], rec[:, 6:]], 1)
    records = fw["records"].copy()
    records[:, 5] = rec[:, 5].detach().double().numpy()
    records[:, 11] = comp.detach().double().numpy()
    return dict(fw, rec=rec, records=records, comp=records[:, 11].copy(), comp_t=comp,
                comp_all=comp_all.detach().double().numpy())


def _grads(leaves, loss) -> List[Dict[str, np.ndarray]]:
    flat = [t for lf in leaves for t in lf.values()]
    gs = torch.autograd.grad(loss, flat, allow_unused=True) if flat and loss.requires_grad else [None] * len(flat)
    out, k = [], 0
    for lf in leaves:
        d = {}
        for name, t in lf.items():
            d[name] = np.zeros(t.shape) if gs[k] is None else gs[k].double().numpy()
            k += 1
        out.append(d)
    return out


def backward(frame, st: ref.Settings, v_records: np.ndarray, dtype=torch.float64) -> List[Dict[str, np.ndarray]]:
    """Gradients of sum(records[:, :10] * v_records[:, :10]) w.r.t. the six parameter tensors of every segment."""
    fw = forward(frame, st, dtype, grad=True)
    v = torch.tensor(np.asarray(v_records, np.float64)[:, :10], dtype=dtype)
    return _grads(fw["leaves"], (fw["rec"] * v).sum())


def comp_param_grads(frame, st: ref.Settings, v_comp: np.ndarray, dtype=torch.float64) -> List[Dict[str, np.ndarray]]:
    """Gradients of sum(comp * v_comp) over every row w.r.t. means, scales and quats of every segment (comp unmasked: the
    caller decides which rows are visible by setting v_comp)."""
    leaves = [{k: getattr(sg.params, k).detach().cpu().double().to(dtype).clone().requires_grad_(True)
               for k in ("means", "scales", "quats")} for sg in frame.segments]
    pr = _geometry(frame, leaves, st, dtype)
    comp = compensation(pr["a"], pr["b"], pr["c"])
    return _grads(leaves, (comp * torch.tensor(np.asarray(v_comp, np.float64), dtype=dtype)).sum())


def l1_project_bwd(means, scales, glob_scale, quats, cam, v_xys, v_depths, v_conics, v_comp, bw=16, clip=0.01,
                   dtype=torch.float64):
    """(v_means, v_scales, v_quats) of sum(xys v_xys + depths v_depths + conics v_conics + compensation v_comp), the outputs
    of project_ref64.l1_project with compensation not detached; None cotangent = zeros."""
    m, s, q = (torch.tensor(np.asarray(x, np.float64), dtype=dtype).requires_grad_(True) for x in (means, scales, quats))
    pr = ref.project_core(m, q, s * glob_scale, cam, bw, clip, dtype)
    vt = torch.from_numpy(pr["vis"])
    outs = (pr["xy"], pr["z"] * vt, pr["conic"], compensation(pr["a"], pr["b"], pr["c"]) * vt)
    loss = 0.0
    for out, v in zip(outs, (v_xys, v_depths, v_conics, v_comp)):
        if v is not None:
            loss = loss + (out * torch.tensor(np.asarray(v, np.float64).reshape(out.shape), dtype=dtype)).sum()
    if not torch.is_tensor(loss):
        return tuple(np.zeros(np.shape(x)) for x in (means, scales, quats))
    gs = torch.autograd.grad(loss, (m, s, q), allow_unused=True)
    return tuple(np.zeros(np.shape(x)) if g is None else g.double().numpy() for g, x in zip(gs, (means, scales, quats)))
