"""Trainable camera poses: nerfstudio's ``CameraOptimizer`` in mode ``"SO3xR3"`` on this library's kernels.

The reference's method config carries a ``CameraOptimizerConfig`` and a ``camera_opt`` Adam group (street_gaussians_ns/
sgn_config.py:44,76-79, with ``gradient_accumulation_steps={"camera_opt": 100}``, :30), but its ``get_outputs`` renders
with ``camera.camera_to_worlds`` (sgn_splatfacto.py:810) and never applies the module.  Here it is applied:

    model = SceneGraphRasterModel(..., camera_optimizer=CameraPoseOptimizer(num_cameras))
    opt = FusedAdam(model.optimizer_params(), extra={"camera_opt.pose_adjustment": (model.camera_optimizer.pose_adjustment, 1e-3)})
    step = TrainStep(model, opt, gradient_accumulation_steps={"camera_opt.pose_adjustment": 100})

What it restates (nerfstudio 1.x ``cameras/camera_optimizers.py`` and ``cameras/lie_groups.py``, as the splatfacto models use
them; nerfstudio is not a dependency, so these are restated from that specification and no vectors of nerfstudio's own code
back them -- tests/camera_cases.py holds the float64 restatement the kernels are checked against):

    pose_adjustment [num_cameras, 6], zero-initialised: translation 0:3, rotation (axis times angle) 3:6 -- the name of
                  nerfstudio's parameter, so a checkpoint entry ``camera_optimizer.pose_adjustment`` loads
    exp_map_SO3xR3: w = x[3:], theta = sqrt(clamp(|w|^2, min=1e-4)),
                    R_a = I + sin(theta)/theta K + (1 - cos(theta))/theta^2 K^2 (K = skew(w)), t_a = x[0:3]
                    (below 0.01 rad the two factors are constants: w reaches R_a through K and K^2 only)
    apply_to_camera: c2w' = c2w [R_a t_a; 0 0 0 1]; the view is built from c2w' as ``Camera._viewmat`` builds it, and the SH
                    view directions use c2w'[:3, 3] (without a gradient, as the reference detaches the camera there)
    get_loss_dict:  camera_opt_regularizer = mean_rows |x[:, 0:3]| * 1e-2 + mean_rows |x[:, 3:6]| * 1e-3
    get_metrics_dict: camera_opt_translation = |x[:, 0:3]|, camera_opt_rotation = |x[:, 3:6]| (Frobenius norms)

``terms(camera)`` is ONE launch forward (sgn_camera_adjust_fwd: pose_adjustment + the camera's c2w -> the 15-float device view
that raster.render_frame(view=...) and sky.CubeMapSky take, the regulariser and the two metrics' norms) and one backward
(sgn_camera_adjust_bwd: the view's and the regulariser's cotangents -> every row of the gradient).  Everything stays on the
device: no read-back per step.

The sky is sampled with the corrected rotation.  By default it gives the camera no gradient; with
``CubeMapSky(view_grad=True)`` it adds its share of the rotation cotangent (the reference's ``EnvLight`` looks up
``c2w[:3,:3] @ d`` with a ``c2w`` that is not detached), which autograd sums with the projection's before
sgn_camera_adjust_bwd runs.

Not provided: the ``SE3`` mode (NotImplementedError), ``non_trainable_camera_indices``, intrinsics, the SH colour's view
direction gradient (the reference detaches the camera there), and a data-parallel exchange of the camera gradient (a
data-parallel TrainStep refuses it).
"""
from __future__ import annotations

import ctypes as C
from typing import Dict

import numpy as np
import torch

from . import _lib
from .raster import VIEW_LEN, _ptr, _stream
from .scene import Camera

TRANS_L2_PENALTY = 1e-2  # CameraOptimizerConfig.trans_l2_penalty
ROT_L2_PENALTY = 1e-3    # CameraOptimizerConfig.rot_l2_penalty


def _c2w_floats(camera: Camera):
    return (C.c_float * 12)(*np.asarray(camera.c2w, np.float32).reshape(-1).tolist())


class _CameraAdjust(torch.autograd.Function):
    """(view [15] -- or an empty tensor when index == -1 --, regulariser 0-d, norms [2] without gradient) of
    ``pose_adjustment`` in one launch forward (sgn_camera_adjust_fwd) and one backward (sgn_camera_adjust_bwd, which writes every
    row of the gradient)."""

    @staticmethod
    def forward(ctx, pose_adjustment: torch.Tensor, index: int, c2w):
        ctx.set_materialize_grads(False)
        pa = pose_adjustment.detach()
        view = torch.empty(VIEW_LEN if index >= 0 else 0, device=pa.device, dtype=torch.float32)
        reg = torch.empty((), device=pa.device, dtype=torch.float32)
        norms = torch.empty(2, device=pa.device, dtype=torch.float32)
        _lib.check(_lib.load().sgn_camera_adjust_fwd(_ptr(pa), pa.shape[0], index, c2w, TRANS_L2_PENALTY, ROT_L2_PENALTY,
                                                     _ptr(view) if index >= 0 else None, _ptr(reg), _ptr(norms), _stream()),
                   "sgn_camera_adjust_fwd")
        ctx.save_for_backward(pose_adjustment)  # autograd's version check: an in-place change before backward is an error
        ctx.index, ctx.c2w = index, c2w
        ctx.mark_non_differentiable(norms)
        return view, reg, norms

    @staticmethod
    def backward(ctx, v_view, v_reg, _v_norms):
        if not ctx.needs_input_grad[0] or ((v_view is None or ctx.index < 0) and v_reg is None):
            return None, None, None
        (pa,) = ctx.saved_tensors
        grad = torch.empty_like(pa)  # every row is written
        v = v_view[:_lib.VIEW_FLOATS].contiguous() if (v_view is not None and ctx.index >= 0) else None
        g = v_reg.reshape(1).contiguous() if v_reg is not None else None
        _lib.check(_lib.load().sgn_camera_adjust_bwd(_ptr(pa), pa.shape[0], ctx.index, ctx.c2w, TRANS_L2_PENALTY, ROT_L2_PENALTY,
                                                     _ptr(v), _ptr(g), _ptr(grad), _stream()), "sgn_camera_adjust_bwd")
        return grad, None, None


class CameraPoseOptimizer(torch.nn.Module):
    """nerfstudio's ``CameraOptimizer`` (see the module docstring).  ``mode``: "SO3xR3" or "off" (no parameters)."""

    def __init__(self, num_cameras: int, mode: str = "SO3xR3"):
        super().__init__()
        if mode == "SE3":
            raise NotImplementedError("CameraPoseOptimizer mode 'SE3' is not provided (only 'SO3xR3' and 'off')")
        if mode not in ("SO3xR3", "off"):
            raise ValueError(f"CameraPoseOptimizer mode must be 'SO3xR3' or 'off' (got {mode!r})")
        self.mode = mode
        self.num_cameras = int(num_cameras)
        if mode != "off":
            self.pose_adjustment = torch.nn.Parameter(torch.zeros(self.num_cameras, 6))

    @property
    def active(self) -> bool:
        return self.mode != "off"

    def check_index(self, camera: Camera) -> int:
        idx = camera.index
        if idx is None or not 0 <= int(idx) < self.num_cameras:
            raise IndexError(f"camera index {idx} outside [0, {self.num_cameras})")
        return int(idx)

    def _checked(self) -> torch.Tensor:
        if not self.active:
            raise RuntimeError("CameraPoseOptimizer in mode 'off' has no pose_adjustment")
        pa = self.pose_adjustment
        if not (pa.is_cuda and pa.dtype == torch.float32 and pa.is_contiguous() and tuple(pa.shape) == (self.num_cameras, 6)):
            raise _lib.SgnError(f"pose_adjustment must be a contiguous float32 [{self.num_cameras}, 6] CUDA tensor; got {pa.dtype} "
                                f"{tuple(pa.shape)} on {pa.device} (move the module with .to('cuda'))")
        return pa

    def terms(self, camera: Camera = None):
        """(view, regulariser, norms) in ONE launch: the corrected view of ``camera`` (float32 [15] on the device -- viewmat 3x4
        row-major, then cam_pos; None without a camera), ``camera_opt_regularizer`` (0-d) and the two metrics' norms ([2], no
        gradient).  View and regulariser are differentiable in ``pose_adjustment``; their backward is one launch too."""
        idx = -1 if camera is None else self.check_index(camera)
        pa = self._checked()
        view, reg, norms = _CameraAdjust.apply(pa, idx, None if camera is None else _c2w_floats(camera))
        return (None if camera is None else view), reg, norms

    def view(self, camera: Camera) -> torch.Tensor:
        """The corrected view of ``camera`` (its ``index`` row of ``pose_adjustment``), differentiable."""
        return self.terms(camera)[0]

    def regularizer(self) -> torch.Tensor:
        """``camera_opt_regularizer`` of CameraOptimizer.get_loss_dict (0-d, differentiable)."""
        return self.terms()[1]

    @staticmethod
    def metrics_of(norms: torch.Tensor) -> Dict[str, torch.Tensor]:
        return {"camera_opt_translation": norms[0], "camera_opt_rotation": norms[1]}

    def metrics(self) -> Dict[str, torch.Tensor]:
        """CameraOptimizer.get_metrics_dict: 0-d device tensors."""
        with torch.no_grad():
            return self.metrics_of(self.terms()[2])
