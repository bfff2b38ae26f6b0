"""Host-side scene-graph bookkeeping: Gaussian sets, actor poses, the IDFT basis, the camera.

This is the small amount of per-frame host logic the reference runs in Python before it reaches
the rasterizer (street_gaussians_ns/sgn_splatfacto_scene_graph.py:305-360, :404-433 and
street_gaussians_ns/sgn_splatfacto.py:822-841).  It produces the *segment table* the fused CUDA
compose+project kernel consumes: one row per visible sub-model, in the reference's concatenation
order (background first, then actors in annotation order).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import List, Optional, Sequence

import numpy as np
import torch

MAX_FOURIER = 8

CLS_BACKGROUND = 0
CLS_OBJECT = 1

PARAM_NAMES = ("means", "scales", "quats", "features_dc", "features_rest", "opacities")


@dataclass
class GaussianSet:
    """One sub-model's ``gauss_params`` (street_gaussians_ns/sgn_splatfacto.py:291-300).

    means[n,3]; scales[n,3] (log); quats[n,4] (wxyz, un-normalised); features_dc[n,F,3];
    features_rest[n,K-1,3]; opacities[n,1] (logit).  All float32, contiguous.
    """

    means: torch.Tensor
    scales: torch.Tensor
    quats: torch.Tensor
    features_dc: torch.Tensor
    features_rest: torch.Tensor
    opacities: torch.Tensor

    @property
    def num_points(self) -> int:
        return int(self.means.shape[0])

    @property
    def fourier_dim(self) -> int:
        return int(self.features_dc.shape[1])

    def tensors(self):
        return [getattr(self, k) for k in PARAM_NAMES]

    def to(self, device) -> "GaussianSet":
        return GaussianSet(*[t.to(device).contiguous() for t in self.tensors()])

    def requires_grad_(self, flag: bool = True) -> "GaussianSet":
        for t in self.tensors():
            t.requires_grad_(flag)
        return self

    def detach_clone(self) -> "GaussianSet":
        return GaussianSet(*[t.detach().clone() for t in self.tensors()])

    def validate(self, sh_degree: int) -> None:
        n = self.num_points
        K = (sh_degree + 1) ** 2
        assert self.means.shape == (n, 3), f"means must be [n,3], got {tuple(self.means.shape)}"
        assert self.scales.shape == (n, 3), "scales must be [n,3]"
        assert self.quats.shape == (n, 4), "quats must be [n,4]"
        assert self.features_dc.dim() == 3 and self.features_dc.shape[0] == n and self.features_dc.shape[2] == 3
        assert 1 <= self.features_dc.shape[1] <= MAX_FOURIER, "fourier_features_dim must be in [1, 8]"
        assert self.features_rest.shape == (n, K - 1, 3), (
            f"features_rest must be [n,{K - 1},3], got {tuple(self.features_rest.shape)}"
        )
        assert self.opacities.shape == (n, 1), "opacities must be [n,1]"
        for t in self.tensors():
            assert t.dtype == torch.float32, "gauss_params must be float32"


def idft_basis(time: float, dim: int) -> np.ndarray:
    """Cached front of :func:`_idft_basis` (all actors of a frame share the same few time values)."""
    key = (float(time), int(dim))
    hit = _IDFT_CACHE.get(key)
    if hit is None:
        if len(_IDFT_CACHE) > 4096:
            _IDFT_CACHE.clear()
        hit = _IDFT_CACHE[key] = _idft_basis(*key)
    return hit


_IDFT_CACHE: dict = {}
_POSE_CACHE: dict = {}


def _idft_basis(time: float, dim: int) -> np.ndarray:
    """The reference's ``IDFT`` (street_gaussians_ns/sgn_splatfacto_scene_graph.py:420-433).

    basis[k] = cos(2*pi*t*k/dim) for even k, sin(2*pi*t*(k+1)/dim) for odd k, evaluated in float32
    with the reference's operation order (torch CPU ops) so the product and the reference see the
    same bits.  Returns float32 [dim].
    """
    t = torch.tensor(float(time)).view(-1, 1)
    idft = torch.zeros(t.shape[0], dim, dtype=t.dtype)
    indices = torch.arange(dim, dtype=torch.int)
    even_indices = indices[::2]
    odd_indices = indices[1::2]
    idft[:, even_indices] = torch.cos(t * even_indices * 2 * math.pi / dim)
    idft[:, odd_indices] = torch.sin(t * (odd_indices + 1) * 2 * math.pi / dim)
    return idft[0].numpy().astype(np.float32)


def fourier_time(frame: int, frame_list: Sequence[int], scale: float = 1.0) -> float:
    """Normalised actor time (street_gaussians_ns/sgn_splatfacto_scene_graph.py:239-245)."""
    if len(frame_list) == 1:
        normalized = 1.0
    else:
        normalized = (frame - frame_list[0]) / (frame_list[-1] - frame_list[0])
    return normalized * scale


def quaternion_from_matrix(matrix: np.ndarray) -> np.ndarray:
    """Rotation matrix -> quaternion (w,x,y,z), w >= 0.

    Restates ``nerfstudio.cameras.camera_utils.quaternion_from_matrix`` (isprecise=False), which
    the reference calls on the CPU in float64 (sgn_splatfacto_scene_graph.py:413): the quaternion
    is the eigenvector of the symmetric 4x4 K matrix with the largest eigenvalue.
    """
    M = np.asarray(matrix, dtype=np.float64)
    m00, m01, m02 = M[0, 0], M[0, 1], M[0, 2]
    m10, m11, m12 = M[1, 0], M[1, 1], M[1, 2]
    m20, m21, m22 = M[2, 0], M[2, 1], M[2, 2]
    K = np.array(
        [
            [m00 - m11 - m22, 0.0, 0.0, 0.0],
            [m01 + m10, m11 - m00 - m22, 0.0, 0.0],
            [m02 + m20, m12 + m21, m22 - m00 - m11, 0.0],
            [m21 - m12, m02 - m20, m10 - m01, m00 + m11 + m22],
        ]
    )
    K /= 3.0
    w, V = np.linalg.eigh(K)
    q = V[np.array([3, 0, 1, 2]), np.argmax(w)]
    if q[0] < 0.0:
        q = -q
    return q


def quaternions_from_matrices(mats: np.ndarray) -> np.ndarray:
    """Batched :func:`quaternion_from_matrix` over ``mats[n,3,3]``: one ``np.linalg.eigh`` call for all boxes of a frame
    (the same LAPACK routine per matrix, so the same bits as the one-by-one form; tests/test_scene_host.py checks it)."""
    M = np.asarray(mats, dtype=np.float64).reshape(-1, 3, 3)
    n = M.shape[0]
    K = np.zeros((n, 4, 4))
    K[:, 0, 0] = M[:, 0, 0] - M[:, 1, 1] - M[:, 2, 2]
    K[:, 1, 0] = M[:, 0, 1] + M[:, 1, 0]
    K[:, 1, 1] = M[:, 1, 1] - M[:, 0, 0] - M[:, 2, 2]
    K[:, 2, 0] = M[:, 0, 2] + M[:, 2, 0]
    K[:, 2, 1] = M[:, 1, 2] + M[:, 2, 1]
    K[:, 2, 2] = M[:, 2, 2] - M[:, 0, 0] - M[:, 1, 1]
    K[:, 3, 0] = M[:, 2, 1] - M[:, 1, 2]
    K[:, 3, 1] = M[:, 0, 2] - M[:, 2, 0]
    K[:, 3, 2] = M[:, 1, 0] - M[:, 0, 1]
    K[:, 3, 3] = M[:, 0, 0] + M[:, 1, 1] + M[:, 2, 2]
    K /= 3.0
    w, V = np.linalg.eigh(K)
    q = V[np.arange(n), :, np.argmax(w, axis=1)][:, [3, 0, 1, 2]]
    q[q[:, 0] < 0.0] *= -1.0
    return q


@dataclass
class Segment:
    """One visible sub-model for one frame: parameters + (for actors) the object->world pose."""

    params: GaussianSet
    cls: int = CLS_BACKGROUND
    rot: Optional[np.ndarray] = None  # [3,3] object->world (Box.rot)
    center: Optional[np.ndarray] = None  # [3] (Box.center)
    idft: Optional[np.ndarray] = None  # [F] float32; None -> [1, 0, ...]
    name: str = ""
    # per-row 3D smoothing filter sizes sigma [count] (float32, on the parameters' device; model.compute_filter_3d): the
    # projection renders every row with scales sqrt(s^2 + sigma^2) and its opacity times coef (include/sgn_raster.h,
    # sgn_camera.filter_3d).  None: no filter.  A frame's segments carry one all together or none at all
    filter_3d: Optional[torch.Tensor] = None

    @property
    def has_pose(self) -> bool:
        return self.rot is not None

    def pose_f32(self):
        """(R[9], t[3], q[4]) as float32, the casts ``object2world_gs`` applies (:410-416)."""
        if not self.has_pose:
            return (
                np.eye(3, dtype=np.float32).reshape(-1),
                np.zeros(3, dtype=np.float32),
                np.array([1, 0, 0, 0], dtype=np.float32),
            )
        R = np.asarray(self.rot, dtype=np.float64)
        # box rotations are static per (frame, actor): cache the eigen-decomposition based quaternion
        key = R.tobytes()
        hit = _POSE_CACHE.get(key)
        if hit is None:
            if len(_POSE_CACHE) > 65536:
                _POSE_CACHE.clear()
            hit = _POSE_CACHE[key] = (R.astype(np.float32).reshape(-1), quaternion_from_matrix(R).astype(np.float32))
        return (hit[0], np.asarray(self.center, dtype=np.float64).astype(np.float32), hit[1])

    def idft_f32(self) -> np.ndarray:
        F = self.params.fourier_dim
        out = np.zeros(MAX_FOURIER, dtype=np.float32)
        if self.idft is None:
            out[0] = 1.0
            assert F == 1, "a segment with fourier_features_dim > 1 needs an IDFT basis"
        else:
            assert len(self.idft) == F, f"idft has {len(self.idft)} terms, features_dc has {F}"
            out[:F] = np.asarray(self.idft, dtype=np.float32)
        return out


@dataclass
class Camera:
    """The fields of a nerfstudio ``Cameras[1]`` the path reads (SURVEY.md 8b)."""

    c2w: np.ndarray  # [3,4] OpenGL camera_to_worlds
    fx: float
    fy: float
    cx: float
    cy: float
    width: int
    height: int
    time: float = 0.0
    # the camera's row of a camera pose optimiser (nerfstudio: camera.metadata["cam_idx"]); None: rendered as given
    index: Optional[int] = None

    def __post_init__(self):
        self.c2w = np.asarray(self.c2w, dtype=np.float32).reshape(3, 4)
        # nerfstudio stores intrinsics as float32 tensors and the reference reads them with .item()
        self.fx = float(np.float32(self.fx))
        self.fy = float(np.float32(self.fy))
        self.cx = float(np.float32(self.cx))
        self.cy = float(np.float32(self.cy))
        self.width = int(self.width)
        self.height = int(self.height)

    def viewmat(self) -> np.ndarray:
        """World->camera 3x4, float32 (street_gaussians_ns/sgn_splatfacto.py:825-836)."""
        key = self.c2w.tobytes()
        cached = getattr(self, "_vm_cache", None)
        if cached is not None and cached[0] == key:
            return cached[1]
        vm = self._viewmat()
        self._vm_cache = (key, vm)
        return vm

    def _viewmat(self) -> np.ndarray:
        c2w = torch.from_numpy(self.c2w)
        R = c2w[:3, :3]
        T = c2w[:3, 3:4]
        R_edit = torch.diag(torch.tensor([1, -1, -1], dtype=R.dtype))
        R = R @ R_edit
        R_inv = R.T
        T_inv = -R_inv @ T
        viewmat = torch.eye(4, dtype=R.dtype)
        viewmat[:3, :3] = R_inv
        viewmat[:3, 3:4] = T_inv
        return viewmat[:3, :].contiguous().numpy().astype(np.float32)

    def cam_pos(self) -> np.ndarray:
        return self.c2w[:3, 3].astype(np.float32).copy()

    def fov_limits(self):
        """1.3 * tan(fov/2) as gsplat's project_cov3d_ewa computes it (double 0.5*W/fx -> float)."""
        tan_x = np.float32(0.5 * self.width / self.fx)
        tan_y = np.float32(0.5 * self.height / self.fy)
        return float(np.float32(1.3) * tan_x), float(np.float32(1.3) * tan_y)


@dataclass
class Frame:
    """Everything one ``get_outputs(camera)`` call needs: the camera and the visible segments."""

    camera: Camera
    segments: List[Segment] = field(default_factory=list)

    @property
    def num_points(self) -> int:
        return sum(s.params.num_points for s in self.segments)

    def row_offsets(self) -> List[int]:
        off, out = 0, []
        for s in self.segments:
            out.append(off)
            off += s.params.num_points
        return out
