"""Per-timestamp actor poses for the scene-graph path (SURVEY.md 8f rank 4): the part of the reference's
``InterpolatedAnnotation`` / ``Box`` (street_gaussians_ns/data/utils/dynamic_annotation.py:75-171, 212-344) that
``SplatfactoSceneGraphModel.get_outputs`` consumes (sgn_splatfacto_scene_graph.py:323-345): the boxes annotated at a
timestamp, or -- between two annotated timestamps -- boxes interpolated for the tracks present in both
(centre lerp, rotation slerp).  ``PoseTable.poses_at`` plugs into ``SceneGraphRasterModel(poses_at=...)``.

No open3d / lidar I/O here: whether a track has seed points is a callback (the reference skips tracks without an
aggregated lidar ply or with fewer than 10 000 points, dynamic_annotation.py:320-325, 352-361).

The quaternion helpers restate nerfstudio.cameras.camera_utils (Gohlke's transformations.py, public algorithm;
nerfstudio is not in this image): real-first quaternions, float64.
"""
from __future__ import annotations

import bisect
import json
import math
from dataclasses import dataclass
from typing import Callable, Dict, List, Optional, Sequence

import numpy as np

from .scene import quaternion_from_matrix

_EPS = np.finfo(float).eps * 4.0
FILTER_LABEL = ["car"]                  # dynamic_annotation.py:19
EXP_RATE = np.array([1.3, 1.3, 1.1])    # dynamic_annotation.py:22: box sizes are inflated


def parse_timestamp(timestamp, l: int = 16) -> str:
    """dynamic_annotation.py:91-97: timestamps are normalised to l-digit integer strings."""
    if isinstance(timestamp, str):
        timestamp = float(timestamp)
    timestamp_str = str(int(timestamp))
    timestamp *= np.power(10, l - len(timestamp_str))
    return str(int(timestamp))


def quaternion_matrix(q: Sequence[float]) -> np.ndarray:
    """Homogeneous rotation matrix of a (w, x, y, z) quaternion (transformations.py quaternion_matrix)."""
    q = np.array(q, dtype=np.float64, copy=True)
    n = float(np.dot(q, q))
    if n < _EPS:
        return np.identity(4)
    q *= math.sqrt(2.0 / n)
    q = np.outer(q, q)
    return np.array([
        [1.0 - q[2, 2] - q[3, 3], q[1, 2] - q[3, 0], q[1, 3] + q[2, 0], 0.0],
        [q[1, 2] + q[3, 0], 1.0 - q[1, 1] - q[3, 3], q[2, 3] - q[1, 0], 0.0],
        [q[1, 3] - q[2, 0], q[2, 3] + q[1, 0], 1.0 - q[1, 1] - q[2, 2], 0.0],
        [0.0, 0.0, 0.0, 1.0]])


def quaternion_slerp(quat0, quat1, fraction: float, spin: int = 0, shortestpath: bool = True) -> np.ndarray:
    """Spherical linear interpolation (transformations.py quaternion_slerp)."""
    q0 = np.array(quat0[:4], dtype=np.float64, copy=True)
    q1 = np.array(quat1[:4], dtype=np.float64, copy=True)
    q0 /= math.sqrt(float(np.dot(q0, q0)))
    q1 /= math.sqrt(float(np.dot(q1, q1)))
    if fraction == 0.0:
        return q0
    if fraction == 1.0:
        return q1
    d = float(np.dot(q0, q1))
    if abs(abs(d) - 1.0) < _EPS:
        return q0
    if shortestpath and d < 0.0:
        d = -d
        np.negative(q1, q1)
    angle = math.acos(d) + spin * math.pi
    if abs(angle) < _EPS:
        return q0
    isin = 1.0 / math.sin(angle)
    q0 *= math.sin((1.0 - fraction) * angle) * isin
    q1 *= math.sin(fraction * angle) * isin
    q0 += q1
    return q0


@dataclass
class TrackBox:
    """The fields of the reference ``Box`` the path reads (dynamic_annotation.py:100-122)."""

    track_id: str
    center: np.ndarray   # [3] float64, world frame (after the dataparser transform and scale)
    rot: np.ndarray      # [3,3] float64 object -> world
    size: np.ndarray
    label: str
    frame_id: int        # the timestamp (integer form)
    frame: int = -1      # index of the annotated frame; -1 for interpolated boxes (Box default, :101)

    def transform(self, translation, rotation) -> None:  # :194-199
        self.center = np.dot(rotation, self.center) + translation
        self.rot = np.dot(rotation, self.rot)

    def scale(self, scale_factor) -> None:  # :201-204
        self.center = self.center * scale_factor
        self.size = self.size * scale_factor

    @staticmethod
    def interpolate(box1: "TrackBox", box2: "TrackBox", frame_id) -> "TrackBox":
        """``Box.interploate`` (:157-171): lerp of the centres, slerp of the rotations; size / label / track of box1."""
        frame_id = int(frame_id)
        t = (frame_id - box1.frame_id) / (box2.frame_id - box1.frame_id)
        center = box1.center * (1 - t) + box2.center * t
        quat = quaternion_slerp(quaternion_from_matrix(box1.rot), quaternion_from_matrix(box2.rot), t)
        return TrackBox(box1.track_id, center, quaternion_matrix(quat)[:3, :3], box1.size, box1.label, frame_id)


def frame_interpolation(frame_1: List[TrackBox], frame_2: List[TrackBox], frame_id) -> List[TrackBox]:
    """dynamic_annotation.py:75-88: only tracks present in BOTH neighbouring frames are interpolated."""
    a = {b.track_id: b for b in frame_1}
    b = {b.track_id: b for b in frame_2}
    return [TrackBox.interpolate(a[k], b[k], frame_id) for k in a if k in b]


class PoseTable:
    """``InterpolatedAnnotation`` without the lidar side (dynamic_annotation.py:212-290, 306-344)."""

    def __init__(self, frames: Sequence[dict], self_car_label=None, transform_matrix: Optional[np.ndarray] = None,
                 scale_factor: float = 1.0, has_points: Optional[Callable[[str], bool]] = None,
                 filter_label: Optional[List[str]] = FILTER_LABEL, ignore_static: bool = True):
        frames = sorted(frames, key=lambda x: x["timestamp"])
        self.transform_matrix = np.eye(4) if transform_matrix is None else np.asarray(transform_matrix, dtype=np.float64)
        self.scale_factor = scale_factor
        self.self_car_label = self_car_label
        self.has_points = has_points or (lambda gid: True)
        self.annos: Dict[str, List[TrackBox]] = {}
        self.objects_meta: Dict[str, TrackBox] = {}
        self.objects_frames: Dict[str, List[int]] = {}
        for i, item in enumerate(frames):
            ts = parse_timestamp(item["timestamp"])
            self.annos[str(ts)] = self._load_frame(item["objects"], ts, i, filter_label, ignore_static)
        self.all_names = list(self.annos.keys())
        self._all_ints = [int(i) for i in self.all_names]
        self.unique_track_ids = list(self.objects_meta.keys())

    @classmethod
    def from_json(cls, path, **kw) -> "PoseTable":
        with open(path) as f:
            return cls(json.load(f)["frames"], **kw)

    def _load_frame(self, obj_list, timestamp, frame, filter_label, ignore_static) -> List[TrackBox]:
        boxes = []
        for obj in obj_list:
            if filter_label is not None and obj["type"] not in filter_label and not obj["type"].endswith("Car"):
                continue
            if ignore_static and not obj["is_moving"]:
                continue
            if self.self_car_label is not None and obj["gid"] == self.self_car_label:
                continue
            gid = obj["gid"]
            if not self.has_points(gid):
                continue
            box = TrackBox(gid, np.array(obj["translation"], dtype=np.float64), quaternion_matrix(obj["rotation"])[:3, :3],
                           EXP_RATE * np.array(obj["size"], dtype=np.float64), obj["type"], int(timestamp), frame)
            box.transform(self.transform_matrix[:3, 3], self.transform_matrix[:3, :3])
            box.scale(self.scale_factor)
            boxes.append(box)
            if gid not in self.objects_meta:  # "use first box as meta"
                self.objects_meta[gid] = box
                self.objects_frames[gid] = []
            self.objects_frames[gid].append(frame)
        return boxes

    def __len__(self) -> int:
        return len(self.all_names)

    def __getitem__(self, frame_id) -> List[TrackBox]:
        """dynamic_annotation.py:250-290."""
        if not len(self):
            return []
        if isinstance(frame_id, (int, float)):
            if isinstance(frame_id, float) and 0 <= frame_id <= 1:
                # "assume it is a portion of the whole sequence rather than a timestamp"
                frame_id = self.all_names[min(round(frame_id * len(self.all_names)), len(self.all_names) - 1)]
            else:
                frame_id = parse_timestamp(frame_id)
        elif isinstance(frame_id, str):
            frame_id = parse_timestamp(frame_id)
        else:
            raise ValueError("frame_id should be int or str")
        if frame_id in self.annos:
            return self.annos[frame_id]
        if frame_id < self.all_names[0] or frame_id > self.all_names[-1]:  # (string comparison, as in the reference)
            return []
        k = bisect.bisect(self._all_ints, int(frame_id))
        return frame_interpolation(self.annos[self.all_names[k - 1]], self.annos[self.all_names[k]], frame_id)

    def poses_at(self, time) -> list:
        """Boxes at a camera time as the ``ActorPose`` records SceneGraphRasterModel consumes.  ``frame`` is the box's
        annotated-frame index (-1 for interpolated boxes, which is what the reference's Fourier time then uses,
        sgn_splatfacto_scene_graph.py:239-245), ``frame_list`` the track's annotated frames and ``frame_id`` the annotated
        frame's timestamp (None for interpolated boxes: the box corrections skip them, :340-341)."""
        from .model import ActorPose
        return [ActorPose(b.track_id, b.rot, b.center, b.frame, self.objects_frames[b.track_id],
                          frame_id=b.frame_id if b.frame != -1 else None) for b in self[time]]

    def frame_idx_map(self) -> Dict[int, int]:
        """Integer timestamp of every annotated frame -> its index (``build_frame_idx_map``, scene graph :101-105): what
        ``box_pose.BoxPoseOptimizer(len(table), table.unique_track_ids, table.frame_idx_map())`` indexes its rows by."""
        return {int(ts): i for i, ts in enumerate(self.all_names)}
