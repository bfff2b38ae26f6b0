"""Float64 reference of the pose cotangents and hand-built frames for them (tests/test_box_pose.py, tests/test_gpu_pose_grad.py).

The composition of a posed segment -- means_w = R m + t, q_w = q_box (x) q (Hamilton, w first, q un-normalised) -- is
restated here with R, t and q_box as float64 autograd LEAVES instead of constants; everything behind it is the existing
float64 statement of the pipeline (oracle/project_ref64.py: ``project_core``; oracle/oracle_torch.py: ``project`` /
``colours`` / ``blend``), so autograd yields the reference answer for v_R [3,3], v_t [3], v_q [4].  Colour contributes nothing:
the SH view direction is taken from detached means (sgn_splatfacto.py:934), here as there.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import numpy as np
import torch

from oracle import oracle_torch
from oracle import project_ref64 as ref
from tests import project_cases as pc

PARAMS = ("means", "scales", "quats", "features_dc", "features_rest", "opacities")


def frame_poses(frame) -> np.ndarray:
    """[n_posed, 16] float32: the poses the segment table carries (R 9 row-major, t 3, q 4), in segment order."""
    rows = [np.concatenate(s.pose_f32()) for s in frame.segments if s.has_pose]
    return np.stack(rows).astype(np.float32) if rows else np.zeros((0, 16), np.float32)


def pose_leaves(pose: np.ndarray, dtype=torch.float64):
    return torch.tensor(np.asarray(pose, np.float64), dtype=dtype).requires_grad_(True)


def compose(frame, pose: torch.Tensor, dtype=torch.float64, grad_params: bool = False):
    """(leaves per segment, concatenated world-space tensors) with the posed segments composed from ``pose`` [n_posed, 16]."""
    leaves, mws, qws, dcs, rests, scales, opacs, cls = [], [], [], [], [], [], [], []
    k = 0
    for s in frame.segments:
        lf = {n: getattr(s.params, n).detach().cpu().to(dtype).clone().requires_grad_(grad_params) for n in PARAMS}
        leaves.append(lf)
        F = lf["features_dc"].shape[1]
        idft = torch.tensor(s.idft_f32()[:F].astype(np.float64), dtype=dtype)
        dcs.append((lf["features_dc"] * idft[None, :, None]).sum(1, keepdim=True))
        if s.has_pose:
            R, t, a = pose[k, 0:9].reshape(3, 3), pose[k, 9:12], pose[k, 12:16]
            k += 1
            mws.append(lf["means"] @ R.T + t)
            qws.append(oracle_torch.quat_mul(a[None, :].expand_as(lf["quats"]), lf["quats"]))
        else:
            mws.append(lf["means"])
            qws.append(lf["quats"])
        rests.append(lf["features_rest"])
        scales.append(lf["scales"])
        opacs.append(lf["opacities"])
        cls.append(torch.full((s.params.num_points,), s.cls, dtype=torch.int32))
    cat = dict(means=torch.cat(mws), quats=torch.cat(qws), features_dc=torch.cat(dcs), features_rest=torch.cat(rests),
               scales=torch.cat(scales), opacities=torch.cat(opacs), cls=torch.cat(cls))
    return leaves, cat


def record_loss(frame, st: ref.Settings, v_records: np.ndarray, pose: torch.Tensor, dtype=torch.float64):
    """sum(records * v_records) over the geometry columns (xy, conic, depth) of the visible rows: all of the record a pose moves."""
    _, cat = compose(frame, pose, dtype)
    s = torch.exp(cat["scales"]) if dtype == torch.float64 else oracle_torch.expf_spec(cat["scales"])
    pr = ref.project_core(cat["means"], cat["quats"], s, frame.camera, st.block_width, st.clip_thresh, dtype)
    vt = torch.from_numpy(pr["vis"])
    v = torch.tensor(np.asarray(v_records, np.float64), dtype=dtype)
    return ((pr["xy"] * v[:, 0:2]).sum(1) + ((pr["conic"] * v[:, 2:5]).sum(1) + pr["z"] * v[:, 9]) * vt).sum(), pr["vis"]


def v_pose_ref(frame, st: ref.Settings, v_records: np.ndarray, pose: Optional[np.ndarray] = None, dtype=torch.float64) -> np.ndarray:
    """[n_posed, 16] float64: the cotangents of the poses for the record cotangents ``v_records`` [N, 12]."""
    leaf = pose_leaves(frame_poses(frame) if pose is None else pose, dtype)
    if leaf.shape[0] == 0:
        return np.zeros((0, 16))
    loss, _ = record_loss(frame, st, v_records, leaf, dtype)
    if not loss.requires_grad:
        return np.zeros(tuple(leaf.shape))
    return torch.autograd.grad(loss, leaf)[0].double().numpy()


def render_loss(frame, pose: torch.Tensor, sorted_ids, tile_bins, w_img, w_alpha, w_obj, sh_degree=3, block_width=16):
    """The float64 render (oracle_torch) of the frame composed from ``pose``, contracted with image-space weights
    (rgb + depth [H,W,4], accumulation [H,W], object_acc [H,W])."""
    _, cat = compose(frame, pose)
    pr = oracle_torch.project(cat, frame.camera, block_width, use_spec_exp=False)
    rgbs, opac = oracle_torch.colours(cat, frame.camera, sh_degree, sh_degree)
    col = torch.cat([rgbs, pr["depths"][:, None]], 1)
    img, alpha = oracle_torch.blend(frame.camera, sorted_ids, tile_bins, pr["xys"], pr["conics"], col, opac, block_width)
    empty = torch.zeros(cat["means"].shape[0], 0, dtype=torch.float64)
    _, obj = oracle_torch.blend(frame.camera, sorted_ids, tile_bins, pr["xys"], pr["conics"], empty, opac, block_width, 0.999, cat["cls"], 1)
    return (img * w_img).sum() + (alpha * w_alpha).sum() + (obj * w_obj).sum()


# ------------------------------------------------------------------------------------------------------------------
# hand-built frames: every decision of the projection is >= project_cases.MARGIN from its threshold
# ------------------------------------------------------------------------------------------------------------------
def _on_screen(b, s, n, z=(2.0, 12.0)):
    W, H = b.cam.width, b.cam.height
    b.scatter(s, n, px=(0.05 * W, 0.95 * W), py=(0.05 * H, 0.95 * H), z=z, scale=(0.02, 0.25))


def one_actor(seed=301):
    """One actor of 200 rows (a full chunk and a tail), no background."""
    b = pc._cam(160, 96, seed)
    _on_screen(b, b.segment(1, pose=(0.4, (0.3, -0.1, -6.0)), F=3), 200)
    return b.settle("one_actor")


def actors_and_background(seed=302):
    """A background of 300 rows, then actors of 300 (not a multiple of 128), 50 (less than a chunk), 128 and 0 rows."""
    b = pc._cam(160, 96, seed)
    _on_screen(b, b.segment(0), 300)
    for k, n in enumerate((300, 50, 128, 0)):
        s = b.segment(1, pose=(-0.5 + 0.35 * k, (0.4 * k - 0.5, 0.1 * k, -5.0 - k)), F=1 + k)
        _on_screen(b, s, n)
    return b.settle("actors_and_background")


def off_screen(seed=303):
    """A background, an actor in view and an actor whose 140 rows all project far outside the image: its cotangent is zero."""
    b = pc._cam(160, 96, seed)
    _on_screen(b, b.segment(0), 100)
    _on_screen(b, b.segment(1, pose=(0.2, (0.0, 0.0, -4.0)), F=2), 90)
    s = b.segment(1, pose=(-0.3, (1.0, 0.0, -5.0)), F=2)
    b.scatter(s, 140, px=(30.0 * b.cam.width, 40.0 * b.cam.width), py=(0.0, 96.0), z=(2.0, 6.0), scale=(0.01, 0.05))
    return b.settle("off_screen")


def clip_plane(seed=304):
    """An actor that straddles the near plane: half of its 260 rows lie behind clip_thresh, half in front."""
    b = pc._cam(160, 96, seed)
    s = b.segment(1, pose=(0.7, (0.0, 0.1, -0.5)), F=1)
    _on_screen(b, s, 130, z=(0.3, 6.0))
    _on_screen(b, s, 130, z=(-3.0, 0.005))
    return b.settle("clip_plane")


CASES = {"one_actor": one_actor, "actors_and_background": actors_and_background, "off_screen": off_screen, "clip_plane": clip_plane}
_BUILT: Dict[str, pc.Case] = {}


def get(name: str) -> pc.Case:
    if name not in _BUILT:
        _BUILT[name] = CASES[name]()
    return _BUILT[name]


def groups(v: np.ndarray) -> List[np.ndarray]:
    """(v_R, v_t, v_q) of [n, 16] rows."""
    return [v[:, 0:9], v[:, 9:12], v[:, 12:16]]


def rel_l2(a: np.ndarray, b: np.ndarray) -> float:
    d = float(np.linalg.norm(np.asarray(b, np.float64)))
    return float(np.linalg.norm(np.asarray(a, np.float64) - np.asarray(b, np.float64))) / d if d > 0 else float(np.abs(a).max(initial=0.0))
