"""Generates tests/golden/reference_bbox.npz: what THE REFERENCE'S OWN ``BBoxOptimizer.apply_to_bbox`` in mode "simple"
(street_gaussians_ns/data/utils/bbox_optimizers.py:140-166) makes of a handful of boxes with non-zero ``delta_center`` /
``delta_yaw``, followed by the quaternion ``object2world_gs`` derives from the corrected rotation
(sgn_splatfacto_scene_graph.py:413), on the CPU.

The reference's module cannot be imported as shipped (nerfstudio, pytorch3d and open3d are absent): the packages it names
are replaced by stand-ins (tests/golden/reference_loader.py explains the approach).  What is NOT the reference's code here:
  * ``quaternion_from_matrix`` / ``quaternion_matrix`` (nerfstudio.cameras.camera_utils): this library's restatements
    (``scene.quaternion_from_matrix``, ``pose_table.quaternion_matrix``);
  * ``pytorch3d.transforms.quaternion_multiply``: restated below (Hamilton product, then the real part made non-negative).
The arithmetic between them -- indexing by ``frame_idx_map[frame_id]`` and ``bbox_list.index(trackId)``, centre + delta,
cos / sin of the yaw (not of half of it), the product's order -- is the reference's.

Arrays: ``rot0`` [A,3,3], ``center0`` [A,3] (float64 inputs), ``frame_ids`` / ``box_ids`` [A] (-1: the box has no annotated
frame and the reference does not call apply_to_bbox on it, scene graph :340-341), ``delta_center`` [F,B,3] and ``delta_yaw``
[F,B] (float32 parameters), and the results ``center`` [A,3], ``rot`` [A,3,3], ``q`` [A,4] (float64).

    SGN_REFERENCE_ROOT=<checkout of street-gaussians-ns> python tests/golden/make_golden_reference_bbox.py
"""
import dataclasses
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import reference_loader as rl  # noqa: E402

from street_gaussians_ns_b200.pose_table import quaternion_matrix  # noqa: E402
from street_gaussians_ns_b200.scene import quaternion_from_matrix  # noqa: E402

OUT = os.path.join(HERE, "reference_bbox.npz")
NUM_FRAMES, TRACKS = 4, ["t0", "t1", "t2"]
TIMESTAMPS = [1000, 1100, 1200, 1300]


def quaternion_multiply(a, b):
    aw, ax, ay, az = torch.unbind(a, -1)
    bw, bx, by, bz = torch.unbind(b, -1)
    ab = torch.stack((aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
                      aw * by - ax * bz + ay * bw + az * bx, aw * bz + ax * by - ay * bx + az * bw), -1)
    return torch.where(ab[..., 0:1] < 0, -ab, ab)


@dataclasses.dataclass
class _InstantiateConfig:
    pass


def load_reference():
    assert rl.available(), "SGN_REFERENCE_ROOT does not name a street-gaussians-ns checkout"
    pkg = rl._module("street_gaussians_ns")
    pkg.__path__ = [os.path.join(rl.REFERENCE_ROOT, "street_gaussians_ns")]
    for sub in ("data", "data.utils"):
        rl._module("street_gaussians_ns." + sub).__path__ = [os.path.join(rl.REFERENCE_ROOT, "street_gaussians_ns", *sub.split("."))]
    no = rl._unavailable
    rl._module("nerfstudio.cameras.lie_groups", exp_map_SE3=no("exp_map_SE3"), exp_map_SO3xR3=no("exp_map_SO3xR3"))
    rl._module("nerfstudio.configs.base_config", InstantiateConfig=_InstantiateConfig)
    rl._module("nerfstudio.utils.poses")
    rl._module("nerfstudio.engine.optimizers", OptimizerConfig=object)
    rl._module("nerfstudio.engine.schedulers", SchedulerConfig=object)
    rl._module("nerfstudio.cameras.camera_utils", quaternion_from_matrix=quaternion_from_matrix, quaternion_matrix=quaternion_matrix)
    rl._module("pytorch3d.transforms", quaternion_multiply=quaternion_multiply)
    rl._module("street_gaussians_ns.data.utils.dynamic_annotation", InterpolatedAnnotation=object, Box=object)
    return rl._load("street_gaussians_ns.data.utils.bbox_optimizers", "street_gaussians_ns/data/utils/bbox_optimizers.py")


def build():
    mod = load_reference()
    rng = np.random.default_rng(41)
    frame_idx_map = {ts: torch.tensor(i, dtype=torch.int) for i, ts in enumerate(TIMESTAMPS)}
    opt = mod.BBoxOptimizer(mod.BBoxOptimizerConfig(mode="simple"), NUM_FRAMES, len(TRACKS), frame_idx_map, "cpu", bbox_list=TRACKS)
    with torch.no_grad():
        opt.delta_center.copy_(torch.from_numpy(rng.uniform(-0.3, 0.3, (NUM_FRAMES, len(TRACKS), 3)).astype(np.float32)))
        opt.delta_yaw.copy_(torch.from_numpy(rng.uniform(-0.8, 0.8, (NUM_FRAMES, len(TRACKS))).astype(np.float32)))
        opt.delta_yaw[1, 2] = 2.0   # cos < 0: the product's real part changes sign
        opt.delta_yaw[2, 0] = 0.0   # a zero correction still goes rot -> quaternion -> rot
        opt.delta_center[2, 0] = 0.0
    picks = [(0, 0), (1, 2), (2, 0), (3, 1), (0, 2), (-1, 1), (2, 1)]  # (frame, box); frame -1: an interpolated box
    rot0, center0, center, rot, quat = [], [], [], [], []
    for k, (f, b) in enumerate(picks):
        q = rng.normal(size=4)
        if k == 3:
            q = np.array([0.05, 0.2, -0.1, 0.97])  # a rotation by almost pi
        R = quaternion_matrix(q)[:3, :3]
        c = rng.uniform(-30, 30, 3)
        rot0.append(R)
        center0.append(c)
        box = types.SimpleNamespace(center=c.copy(), rot=R.copy(), frame_id=TIMESTAMPS[max(f, 0)], trackId=TRACKS[b])
        if f >= 0:
            opt.apply_to_bbox(box)
        center.append(np.asarray(box.center, np.float64))
        rot.append(np.asarray(box.rot, np.float64))
        quat.append(quaternion_from_matrix(box.rot))
    return dict(rot0=np.stack(rot0), center0=np.stack(center0), frame_ids=np.array([f for f, _ in picks], np.int64),
                box_ids=np.array([b for _, b in picks], np.int64), delta_center=opt.delta_center.detach().numpy(),
                delta_yaw=opt.delta_yaw.detach().numpy(), center=np.stack(center), rot=np.stack(rot), q=np.stack(quat),
                timestamps=np.array(TIMESTAMPS, np.int64), tracks=np.array(TRACKS))


if __name__ == "__main__":
    d = build()
    np.savez_compressed(OUT, **d)
    print(OUT, os.path.getsize(OUT), "bytes")
    print(d["q"])
