"""Inputs and float64 statements for the antialiased rasterize mode (tests/test_gpu_project_antialiased.py).

``comp_edges`` is a hand-built frame (tests/project_cases.py's Builder) for the compensation's own edges: needles whose
screen covariance before the blur is exactly rank one in float32 -- along the camera's x or y axis, thin axes of scale
exp(-80) whose squares underflow -- so det(cov2d) is 0 and comp = 0; sub-pixel Gaussians (comp ~ 0.01 .. 0.5); Gaussians
many pixels wide (comp ~ 1); and a scatter.

``v_pose_ref`` / ``v_view_ref`` restate tests/pose_cases.py's and tests/camera_cases.py's float64 cotangents of the box poses
and of the view with the antialiased opacity, sigmoid(logit) * comp (comp not detached), in the loss as well.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle import project_aa_ref64 as aa
from oracle import project_ref64 as ref
from tests import camera_cases as cc
from tests import pose_cases as pz
from tests import project_cases as pc

F64 = torch.float64
THIN = float(np.exp(-80.0))  # a scale whose square underflows in float32


def comp_edges(seed=270):
    b = pc._cam(128, 96, seed)
    s = b.segment(0)
    needles = []
    for k in range(6):  # identity camera: the view axes are the world's (y, z flipped); quaternion (1, 0, 0, 0)
        long_axis = k % 2
        sc = [THIN, THIN, THIN]
        sc[long_axis] = b.rng.uniform(0.05, 0.4)
        needles.append(b.add(s, b.rng.uniform(15, 113), b.rng.uniform(15, 81), b.rng.uniform(2, 8), sc, quat=(1.0, 0, 0, 0),
                             logit=2.0, fixed=True)[1])
    for k in range(12):  # sub-pixel
        z = b.rng.uniform(2, 10)
        b.add(s, b.rng.uniform(5, 123), b.rng.uniform(5, 91), z, b.rng.uniform(0.02, 0.6) * z / b.cam.fx, fixed=True)
    for k in range(4):  # many pixels wide
        z = b.rng.uniform(3, 6)
        b.add(s, b.rng.uniform(20, 108), b.rng.uniform(20, 76), z, b.rng.uniform(8, 20) * z / b.cam.fx * np.ones(3), fixed=True)
    b.scatter(s, 60)
    return b.settle("comp_edges", notes={"needles": needles})


def _aa_opacity(opacities, a, b, c, vt):
    return torch.sigmoid(opacities[:, 0]) * aa.compensation(a, b, c) * vt


def v_pose_ref(frame, st: ref.Settings, v_records: np.ndarray) -> np.ndarray:
    """[n_posed, 16] float64 cotangents of the poses, antialiased mode (pose_cases.v_pose_ref plus the opacity column)."""
    leaf = pz.pose_leaves(pz.frame_poses(frame))
    if leaf.shape[0] == 0:
        return np.zeros((0, 16))
    _, cat = pz.compose(frame, leaf)
    pr = ref.project_core(cat["means"], cat["quats"], torch.exp(cat["scales"]), frame.camera, st.block_width, st.clip_thresh, F64)
    vt = torch.from_numpy(pr["vis"])
    v = torch.tensor(np.asarray(v_records, np.float64), dtype=F64)
    opac = _aa_opacity(cat["opacities"], pr["a"], pr["b"], pr["c"], vt)
    loss = ((pr["xy"] * v[:, 0:2]).sum(1) + ((pr["conic"] * v[:, 2:5]).sum(1) + pr["z"] * v[:, 9]) * vt + opac * v[:, 5]).sum()
    return torch.autograd.grad(loss, leaf)[0].numpy() if loss.requires_grad else np.zeros(tuple(leaf.shape))


def v_view_ref(frame, st: ref.Settings, v_records: np.ndarray) -> np.ndarray:
    """[12] float64 cotangent of the camera's own viewmat, antialiased mode (camera_cases.v_view_ref plus the opacity)."""
    view = torch.tensor(np.asarray(frame.camera.viewmat(), np.float64).reshape(-1), dtype=F64).requires_grad_(True)
    loss, vis = cc.record_loss_view(frame, st, v_records, view)
    if not vis.any():
        return np.zeros(12)
    _, cat = pz.compose(frame, pz.pose_leaves(pz.frame_poses(frame)))
    cat = {k: t.detach() for k, t in cat.items()}
    W = view[:12].reshape(3, 4)
    # the covariance part of record_loss_view again, with W the leaf: cov2d = J W S W^T J^T at the FOV-clamped point
    cam = frame.camera
    p = cat["means"] @ W[:, :3].T + W[:, 3]
    vt = torch.from_numpy(vis)
    zs = torch.where(vt, p[:, 2], torch.ones_like(p[:, 2]))
    qn = cat["quats"] / torch.sqrt((cat["quats"] ** 2).sum(-1, keepdim=True))
    M = ref._rotmat(qn) * torch.exp(cat["scales"])[:, None, :]
    limx, limy = cam.fov_limits()
    tx, ty = zs * torch.clamp(p[:, 0] / zs, -limx, limx), zs * torch.clamp(p[:, 1] / zs, -limy, limy)
    zero = torch.zeros_like(zs)
    J = torch.stack([cam.fx / zs, zero, -cam.fx * tx / (zs * zs), zero, cam.fy / zs, -cam.fy * ty / (zs * zs)], -1).reshape(-1, 2, 3)
    T = J @ W[:, :3]
    cov = T @ (M @ M.transpose(1, 2)) @ T.transpose(1, 2)
    opac = _aa_opacity(cat["opacities"], cov[:, 0, 0] + 0.3, cov[:, 0, 1], cov[:, 1, 1] + 0.3, vt)
    v = torch.tensor(np.asarray(v_records, np.float64), dtype=F64)
    return torch.autograd.grad(loss + (opac * v[:, 5]).sum(), view)[0].numpy()


EPS32 = float(np.finfo(np.float32).eps)
COND_K = 256.0


def comp_condition(records64: np.ndarray) -> np.ndarray:
    """Per row, kappa = c00 c11 / det(cov2d) of the un-blurred screen covariance (float64 records: the conic is the blurred
    inverse), 0 where comp is 0.  comp's gradient reaches the parameters through cov2d, whose cotangent is kappa times
    larger than what survives its contraction with d cov2d / d(means, scales, quats): an fp32 chain -- the kernel's, gsplat's
    -- carries a rounding error of a few eps32 kappa times the row's gradient scale (a needle's kappa is its squared aspect
    ratio on the screen).  COND_K: the few, as the H100 build of the kernel needs it (90 on the directed needles, whose kappa
    reaches 1e7: there an fp32 gradient through comp has no significant digit, and only its finiteness is checked).  comp
    itself, the square root of det(cov2d) / det(cov2d + 0.3 I), carries about eps32 kappa of relative error in float32 (the
    forward's noise term)."""
    X0, X1, X2 = records64[:, 2], records64[:, 3], records64[:, 4]
    dX = X0 * X2 - X1 * X1
    ok = (dX > 0) & (records64[:, 11] > 0)
    det = np.where(ok, 1.0 / np.where(ok, dX, 1.0), 0.0)
    c00, c11, b = X2 * det - 0.3, X0 * det - 0.3, -X1 * det
    det_o = c00 * c11 - b * b
    return np.where(ok & (det_o > 0), c00 * c11 / np.where(det_o > 0, det_o, 1.0), 0.0)
