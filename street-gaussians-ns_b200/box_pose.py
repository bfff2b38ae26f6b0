"""Trainable corrections of the tracked actor boxes: the reference's ``BBoxOptimizer`` in the mode its method config
uses (``BBoxOptimizerConfig(mode="simple")``, street_gaussians_ns/sgn_config.py:45; data/utils/bbox_optimizers.py:54-166).

Two parameters, zero-initialised, with the reference's names and shapes -- a reference checkpoint's
``bbox_optimizer.delta_center`` / ``bbox_optimizer.delta_yaw`` load --

    delta_center [num_frames, num_bboxes, 3]      delta_yaw [num_frames, num_bboxes]

indexed by the annotated frame of a box (``frame_idx_map[Box.frame_id]``, scene graph :101-105) and by the position of
its track in the list of tracks (``bbox_list.index(trackId)``).  In the reference the corrected box leaves torch through
``.detach().numpy()`` (bbox_optimizers.py:158,164), so the parameters never receive a gradient; here ``poses`` is
differentiable torch arithmetic on the device and the render takes its result as an input
(``raster.render_frame(pose=...)``), whose cotangent the projection backward reduces.

What ``poses`` restates, in float64 like the reference's numpy path, cast to float32 at the end as ``object2world_gs``
casts (scene graph :410-413):

    center = center0 + delta_center
    q      = q(rot0) (x) (cos d, 0, 0, sin d)         d = delta_yaw -- cos d / sin d, not the half angle: the box turns
                                                      by 2 d about its own z axis, and so it does here
    R      = quaternion_matrix(q)
    q_out  = q / |q| with w >= 0                      what quaternion_from_matrix(R) returns, without the
                                                      eigen-decomposition, so that autograd goes through it

Like the reference in this mode, a zero correction still sends rot0 through R -> q -> R: a render with zero deltas
equals the uncorrected render to the float32 rounding of R, not bit for bit.  ``mode="off"`` has no parameters and hands
the annotated pose on unchanged.  Boxes without an annotated frame (interpolated between two timestamps, ``Box.frame ==
-1``; scene graph :340-341 skips them) pass through unmodified in either mode.

Not restated: ``center_noise`` / ``rot_noise`` (off in the reference's config), the ``SO3xR3`` / ``SE3`` modes, and the
regulariser / metrics of ``BBoxOptimizer`` (they read a ``pose_adjustment`` this mode does not have).
"""
from __future__ import annotations

from typing import Dict, Mapping, Sequence

import numpy as np
import torch

from .scene import quaternions_from_matrices


def _quat_mul(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """Hamilton product, real part first."""
    aw, ax, ay, az = a.unbind(-1)
    bw, bx, by, bz = b.unbind(-1)
    return torch.stack([aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
                        aw * by - ax * bz + ay * bw + az * bx, aw * bz + ax * by - ay * bx + az * bw], -1)


def _quat_matrix(q: torch.Tensor) -> torch.Tensor:
    """Rotation matrices [A,3,3] of quaternions [A,4] of any non-zero length (transformations.py quaternion_matrix)."""
    q = q * torch.sqrt(2.0 / (q * q).sum(-1, keepdim=True))
    o = q[:, :, None] * q[:, None, :]
    return torch.stack([1.0 - o[:, 2, 2] - o[:, 3, 3], o[:, 1, 2] - o[:, 3, 0], o[:, 1, 3] + o[:, 2, 0],
                        o[:, 1, 2] + o[:, 3, 0], 1.0 - o[:, 1, 1] - o[:, 3, 3], o[:, 2, 3] - o[:, 1, 0],
                        o[:, 1, 3] - o[:, 2, 0], o[:, 2, 3] + o[:, 1, 0], 1.0 - o[:, 1, 1] - o[:, 2, 2]], -1).reshape(-1, 3, 3)


class BoxPoseOptimizer(torch.nn.Module):
    def __init__(self, num_frames: int, track_ids: Sequence[str], frame_idx_map: Mapping[int, int], mode: str = "off"):
        """``track_ids``: every track of the sequence, in the order that numbers the boxes (the reference's
        ``object_annos.objects_meta.keys()``); ``frame_idx_map``: integer timestamp of an annotated frame -> its index
        (``build_frame_idx_map``, scene graph :101-105)."""
        super().__init__()
        if mode not in ("simple", "off"):
            raise ValueError(f"BoxPoseOptimizer mode must be 'simple' or 'off' (got {mode!r}); the SO3xR3 / SE3 modes are not provided")
        self.mode = mode
        self.num_frames, self.num_bboxes = int(num_frames), len(track_ids)
        self.bbox_list = list(track_ids)
        self._box_index = {t: i for i, t in enumerate(self.bbox_list)}
        self.frame_idx_map = {int(k): int(v) for k, v in frame_idx_map.items()}
        if mode == "simple":
            self.delta_center = torch.nn.Parameter(torch.zeros(self.num_frames, self.num_bboxes, 3))
            self.delta_yaw = torch.nn.Parameter(torch.zeros(self.num_frames, self.num_bboxes))

    def indices(self, boxes) -> tuple:
        """(frame_ids, box_ids) of ``ActorPose`` records: the rows of the parameters that correct them; -1 for a box that
        is not corrected (no annotated frame: ``frame == -1`` or ``frame_id`` None, or a timestamp / track the tables
        do not know)."""
        fi, bi = [], []
        for b in boxes:
            f = -1
            if b.frame != -1 and getattr(b, "frame_id", None) is not None:
                f = self.frame_idx_map.get(int(b.frame_id), -1)
            k = self._box_index.get(b.track_id, -1)
            if f < 0 or k < 0:
                f = k = -1
            fi.append(f)
            bi.append(k)
        return fi, bi

    def stage(self, frame_ids, box_ids, rot0, center0, device=None) -> Dict[str, torch.Tensor]:
        """The constants of ``poses`` for one set of boxes, on the device: index tensors, rot0 / center0 and the quaternions
        of rot0 (one batched eigen-decomposition on the host, ``scene.quaternions_from_matrices``).  They do not change
        while the annotation does not: stage once per timestamp, call ``forward`` every step."""
        if device is None:
            device = self.delta_center.device if self.mode == "simple" else torch.device("cpu")
        rot0 = np.asarray(rot0, np.float64).reshape(-1, 3, 3)
        center0 = np.asarray(center0, np.float64).reshape(-1, 3)
        fi = np.asarray(frame_ids, np.int64).reshape(-1)
        bi = np.asarray(box_ids, np.int64).reshape(-1)
        assert rot0.shape[0] == center0.shape[0] == fi.shape[0] == bi.shape[0]
        assert fi.max(initial=-1) < self.num_frames and bi.max(initial=-1) < self.num_bboxes, "frame / box index out of range"
        live = (fi >= 0) & (bi >= 0)
        q0 = quaternions_from_matrices(rot0) if rot0.shape[0] else np.zeros((0, 4))
        host = dict(frame=np.where(live, fi, 0), box=np.where(live, bi, 0), live=live, rot0=rot0, center0=center0, q0=q0)
        return {k: torch.from_numpy(np.ascontiguousarray(v)).to(device) for k, v in host.items()}

    def forward(self, staged: Dict[str, torch.Tensor]) -> torch.Tensor:
        """[A, 16] float32 rows (R 9 row-major, t 3, q 4) for ``raster.render_frame(pose=...)``."""
        return self.poses_f64(staged).float()

    def poses_f64(self, staged: Dict[str, torch.Tensor]) -> torch.Tensor:
        """``forward`` before its cast: the corrected poses in float64."""
        rot0, center0, q0 = staged["rot0"], staged["center0"], staged["q0"]
        A = rot0.shape[0]
        if self.mode == "off":
            return torch.cat([rot0.reshape(A, 9), center0, q0], 1)
        live = staged["live"][:, None]
        dc = self.delta_center[staged["frame"], staged["box"]].double()
        dy = self.delta_yaw[staged["frame"], staged["box"]]
        c, sn = torch.cos(dy).double(), torch.sin(dy).double()  # evaluated in the parameter's precision, as the reference does
        zero = torch.zeros_like(c)
        q = _quat_mul(q0, torch.stack([c, zero, zero, sn], -1))
        R = _quat_matrix(q).reshape(A, 9)
        qn = q / torch.sqrt((q * q).sum(-1, keepdim=True))
        qn = torch.where(qn[:, :1] < 0, -qn, qn)
        return torch.cat([torch.where(live, R, rot0.reshape(A, 9)), torch.where(live, center0 + dc, center0),
                          torch.where(live, qn, q0)], 1)

    def poses(self, frame_ids, box_ids, rot0, center0) -> torch.Tensor:
        """``forward(stage(...))``: frame_ids / box_ids [A] (-1: pass the box through), rot0 [A,3,3], center0 [A,3] float64."""
        return self.forward(self.stage(frame_ids, box_ids, rot0, center0))
