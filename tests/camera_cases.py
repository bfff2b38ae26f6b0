"""Float64 reference of the camera pose correction and of the view cotangent (tests/test_camera_pose.py,
tests/test_gpu_camera_grad.py).

``exp_map_so3xr3`` .. ``view_of`` restate nerfstudio 1.x's CameraOptimizer in mode "SO3xR3" (cameras/lie_groups.py
exp_map_SO3xR3, CameraOptimizer.apply_to_camera) and ``scene.Camera._viewmat`` as float64 torch ops, from the specification
in street_gaussians_ns_b200/camera_pose.py (nerfstudio is not a dependency: no vectors of its own code back this).

``v_view_ref`` is the cotangent of viewmat[12] for given record cotangents: the geometry part of the projection (xy, conic,
depth; oracle/project_ref64.py ``project_core``) restated with the view as an autograd leaf, over the rows project_core finds
visible with the camera's own view.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle import project_ref64 as ref
from tests import pose_cases as pz

F64 = torch.float64


def skew(w: torch.Tensor) -> torch.Tensor:
    z = torch.zeros_like(w[..., 0])
    return torch.stack([z, -w[..., 2], w[..., 1], w[..., 2], z, -w[..., 0], -w[..., 1], w[..., 0], z], -1).reshape(*w.shape[:-1], 3, 3)


def exp_map_so3xr3(x: torch.Tensor) -> torch.Tensor:
    """[..., 6] -> [..., 3, 4] (R_a | t_a)."""
    w = x[..., 3:]
    theta = torch.clamp((w * w).sum(-1), min=1e-4).sqrt()
    f1 = torch.sin(theta) / theta
    f2 = (1.0 - torch.cos(theta)) / (theta * theta)
    K = skew(w)
    R = f1[..., None, None] * K + f2[..., None, None] * (K @ K) + torch.eye(3, dtype=x.dtype)
    return torch.cat([R, x[..., :3, None]], -1)


def adjusted_c2w(c2w: torch.Tensor, x: torch.Tensor) -> torch.Tensor:
    """c2w [3,4] @ [R_a t_a; 0 1]."""
    A = exp_map_so3xr3(x)
    return torch.cat([c2w[:, :3] @ A[:, :3], (c2w[:, :3] @ A[:, 3] + c2w[:, 3])[:, None]], 1)


def viewmat_of(c2w: torch.Tensor) -> torch.Tensor:
    """Camera._viewmat: R = c2w[:3,:3] diag(1,-1,-1), W = R^T, c = -W t -> [3, 4]."""
    R = c2w[:, :3] * torch.tensor([1.0, -1.0, -1.0], dtype=c2w.dtype)
    W = R.T
    return torch.cat([W, (-W @ c2w[:, 3])[:, None]], 1)


def view_of(c2w, x) -> torch.Tensor:
    """The 15-float device view: viewmat of the corrected c2w, then its position."""
    c = adjusted_c2w(torch.as_tensor(np.asarray(c2w, np.float64)) if not torch.is_tensor(c2w) else c2w, x)
    return torch.cat([viewmat_of(c).reshape(-1), c[:, 3]])


def regularizer(x: torch.Tensor) -> torch.Tensor:
    return x[:, :3].norm(dim=-1).mean() * 1e-2 + x[:, 3:].norm(dim=-1).mean() * 1e-3


def metrics(x: torch.Tensor):
    return {"camera_opt_translation": x[:, :3].norm(), "camera_opt_rotation": x[:, 3:].norm()}


def record_loss_view(frame, st: ref.Settings, v_records: np.ndarray, view: torch.Tensor, scales=None, opacity=None):
    """sum(records * v_records) over the geometry columns of the visible rows, with W | c = view[:12] (float64 leaf).
    ``scales(cat)``: the linear scales of the composed rows in place of exp(log-scales); ``opacity(cat, a, b, c)``: a
    per-row opacity from the blurred cov2d entries, whose column 5 term then joins the loss (visible rows)."""
    _, cat = pz.compose(frame, pz.pose_leaves(pz.frame_poses(frame)))
    cat = {k: v.detach() for k, v in cat.items()}
    s = torch.exp(cat["scales"]) if scales is None else scales(cat)
    vis = ref.project_core(cat["means"], cat["quats"], s, frame.camera, st.block_width, st.clip_thresh, F64)["vis"]
    cam = frame.camera
    W = view[:12].reshape(3, 4)
    p = cat["means"] @ W[:, :3].T + W[:, 3]
    z = p[:, 2]
    vt = torch.from_numpy(vis)
    zs = torch.where(vt, z, torch.ones_like(z))
    qr = cat["quats"]
    qn = qr / torch.sqrt((qr * qr).sum(-1, keepdim=True))
    M = ref._rotmat(qn) * s[:, None, :]
    S = M @ M.transpose(1, 2)
    limx, limy = cam.fov_limits()
    ux, uy = p[:, 0] / zs, p[:, 1] / zs
    cx_ = torch.clamp(ux, -limx, limx)
    cy_ = torch.clamp(uy, -limy, limy)
    tx, ty = zs * cx_, zs * cy_
    fx, fy = cam.fx, cam.fy
    zero = torch.zeros_like(zs)
    J = torch.stack([fx / zs, zero, -fx * tx / (zs * zs), zero, fy / zs, -fy * ty / (zs * zs)], -1).reshape(-1, 2, 3)
    T = J @ W[:, :3]
    cov = T @ S @ T.transpose(1, 2)
    a, b, c = cov[:, 0, 0] + 0.3, cov[:, 0, 1], cov[:, 1, 1] + 0.3
    det = torch.where(vt, a * c - b * b, torch.ones_like(a))
    conic = torch.stack([c / det, -b / det, a / det], -1)
    rw = 1.0 / (zs + 1e-6)
    xy = torch.stack([p[:, 0] * rw * fx + cam.cx, p[:, 1] * rw * fy + cam.cy], -1)
    v = torch.tensor(np.asarray(v_records, np.float64), dtype=F64)
    loss = (((xy * v[:, 0:2]).sum(1) + (conic * v[:, 2:5]).sum(1) + z * v[:, 9]) * vt).sum()
    if opacity is not None:
        loss = loss + (opacity(cat, a, b, c) * vt * v[:, 5]).sum()
    return loss, vis


def v_view_ref(frame, st: ref.Settings, v_records: np.ndarray) -> np.ndarray:
    """[12] float64: the cotangent of the camera's own viewmat for the record cotangents ``v_records`` [N, 12]."""
    leaf = torch.tensor(np.asarray(frame.camera.viewmat(), np.float64).reshape(-1), dtype=F64).requires_grad_(True)
    loss, vis = record_loss_view(frame, st, v_records, leaf)
    if not vis.any():
        return np.zeros(12)
    return torch.autograd.grad(loss, leaf)[0].numpy()
