"""Seeded synthetic scenes for BASELINE.json's configs (SURVEY.md 8d).

All tensors are generated on the CPU with ``torch.Generator().manual_seed(S)`` so every box
(this container, the GPU box) sees identical inputs; callers move them to the device.
"""
from __future__ import annotations

import math
from typing import List, Optional, Tuple

import numpy as np
import torch

from .scene import CLS_BACKGROUND, CLS_OBJECT, Camera, Frame, GaussianSet, Segment, fourier_time, idft_basis


def random_quats(n: int, gen: torch.Generator) -> torch.Tensor:
    """Uniform random rotations, the law of ``random_quat_tensor`` (sgn_splatfacto.py:39-54)."""
    u = torch.rand(n, generator=gen)
    v = torch.rand(n, generator=gen)
    w = torch.rand(n, generator=gen)
    return torch.stack(
        [
            torch.sqrt(1 - u) * torch.sin(2 * math.pi * v),
            torch.sqrt(1 - u) * torch.cos(2 * math.pi * v),
            torch.sqrt(u) * torch.sin(2 * math.pi * w),
            torch.sqrt(u) * torch.cos(2 * math.pi * w),
        ],
        dim=-1,
    )


def make_background(n: int, seed: int = 0, sh_degree: int = 3,
                    box=((-40.0, 40.0), (-6.0, 14.0), (-90.0, -1.5)),
                    scale_mu: float = 0.08) -> GaussianSet:
    g = torch.Generator().manual_seed(seed)
    K = (sh_degree + 1) ** 2
    u = torch.rand(n, 3, generator=g)
    lo = torch.tensor([b[0] for b in box])
    hi = torch.tensor([b[1] for b in box])
    means = lo + u * (hi - lo)
    scales = (math.log(scale_mu) + 0.6 * torch.randn(n, 3, generator=g)).clamp(math.log(0.005), math.log(2.0))
    quats = random_quats(n, g)
    opac = 0.5 + 2.0 * torch.randn(n, 1, generator=g)
    dc = 0.6 * torch.randn(n, 1, 3, generator=g)
    rest = 0.08 * torch.randn(n, K - 1, 3, generator=g)
    return GaussianSet(means.contiguous(), scales.contiguous(), quats.contiguous(), dc.contiguous(),
                       rest.contiguous(), opac.contiguous())


ACTOR_EXTENT = (1.9, 1.7, 4.6)  # object-frame box: x width, y height, z length (metres)


def make_actor(n: int, seed: int, sh_degree: int = 3, fourier_dim: int = 5) -> GaussianSet:
    g = torch.Generator().manual_seed(seed)
    K = (sh_degree + 1) ** 2
    ext = torch.tensor(ACTOR_EXTENT)
    means = (torch.rand(n, 3, generator=g) - 0.5) * ext
    scales = math.log(0.03) + 0.4 * torch.randn(n, 3, generator=g)
    quats = random_quats(n, g)
    opac = 0.5 + 2.0 * torch.randn(n, 1, generator=g)
    dc = 0.3 * torch.randn(n, fourier_dim, 3, generator=g)
    rest = 0.08 * torch.randn(n, K - 1, 3, generator=g)
    return GaussianSet(means.contiguous(), scales.contiguous(), quats.contiguous(), dc.contiguous(),
                       rest.contiguous(), opac.contiguous())


def actor_pose(index: int, seed: int = 1000) -> Tuple[np.ndarray, np.ndarray]:
    """Box pose of actor ``index`` on the 4-lane x 8-row grid of SURVEY.md 8d (rot, center)."""
    lanes = (-5.25, -1.75, 1.75, 5.25)
    lane, row = index % 4, index // 4
    rng = np.random.RandomState(seed + index)
    yaw = rng.uniform(-0.2, 0.2)
    c, s = math.cos(yaw), math.sin(yaw)
    rot = np.array([[c, 0.0, s], [0.0, 1.0, 0.0], [-s, 0.0, c]], dtype=np.float64)  # about the up (y) axis
    center = np.array([lanes[lane], -1.2, -(6.0 + 7.0 * row)], dtype=np.float64)
    return rot, center


def street_points(n: int, seed: int = 0, box=((-40.0, 40.0), (-6.0, 14.0), (-90.0, -1.5)), n_outliers: int = 8) -> torch.Tensor:
    """A street-like seed cloud [n, 3] float32 over config 3's box: 70 % a thin ground slab, 30 % sparse volume, and
    ``n_outliers`` points 1-5 km away (lidar returns off buildings and the sky) -- the non-uniform density initialisation sees."""
    g = torch.Generator().manual_seed(seed)
    lo = torch.tensor([b[0] for b in box])
    hi = torch.tensor([b[1] for b in box])
    n_ground = int(0.7 * n)
    n_vol = n - n_ground - n_outliers
    ground = lo + torch.rand(n_ground, 3, generator=g) * (hi - lo)
    ground[:, 1] = -1.6 + 0.05 * torch.randn(n_ground, generator=g)
    vol = lo + torch.rand(n_vol, 3, generator=g) * (hi - lo)
    far = torch.randn(n_outliers, 3, generator=g)
    far = far / far.norm(dim=1, keepdim=True) * (1000.0 + 4000.0 * torch.rand(n_outliers, 1, generator=g))
    pts = torch.cat([ground, vol, far])
    return pts[torch.randperm(n, generator=g)].contiguous()


def actor_points(n: int, seed: int = 0) -> torch.Tensor:
    """An aggregated lidar cloud [n, 3] of one actor: points on the faces of the ACTOR_EXTENT box."""
    g = torch.Generator().manual_seed(seed)
    ext = torch.tensor(ACTOR_EXTENT)
    p = (torch.rand(n, 3, generator=g) - 0.5) * ext
    axis = torch.randint(0, 3, (n,), generator=g)
    side = torch.where(torch.rand(n, generator=g) < 0.5, -0.5, 0.5)
    p[torch.arange(n), axis] = side * ext[axis]
    return p.contiguous()


def make_camera(width: int = 1920, height: int = 1280, c2w: Optional[np.ndarray] = None, time: float = 0.0) -> Camera:
    if c2w is None:
        c2w = np.concatenate([np.eye(3), np.zeros((3, 1))], axis=1)
    f = 2055.0 * (width / 1920.0)
    return Camera(c2w=c2w, fx=f, fy=f, cx=width / 2.0, cy=height / 2.0, width=width, height=height, time=time)


def make_frame(n_background: int, n_actors: int = 0, n_per_actor: int = 10000, width: int = 1920,
               height: int = 1280, sh_degree: int = 3, fourier_dim: int = 5, frame: int = 21,
               num_frames: int = 85, seed: int = 0, c2w: Optional[np.ndarray] = None,
               background: Optional[GaussianSet] = None, actors: Optional[List[GaussianSet]] = None,
               actor_shift: Optional[np.ndarray] = None) -> Frame:
    """Background + ``n_actors`` actors at frame index ``frame`` of an ``num_frames`` track."""
    cam = make_camera(width, height, c2w=c2w, time=float(frame))
    bg = background if background is not None else make_background(n_background, seed=seed, sh_degree=sh_degree)
    segs = [Segment(params=bg, cls=CLS_BACKGROUND, name="background")]
    t = fourier_time(frame, list(range(num_frames)), 1.0)
    basis = idft_basis(t, fourier_dim)
    for a in range(n_actors):
        ps = actors[a] if actors is not None else make_actor(n_per_actor, seed=seed + 1 + a, sh_degree=sh_degree,
                                                             fourier_dim=fourier_dim)
        rot, center = actor_pose(a)
        if actor_shift is not None:
            center = center + actor_shift
        segs.append(Segment(params=ps, cls=CLS_OBJECT, rot=rot, center=center, idft=basis, name=f"object_{a}"))
    return Frame(camera=cam, segments=segs)


def config_frame(cfg: int, scale: float = 1.0, seed: int = 0) -> Frame:
    """BASELINE.json configs 1-3.  ``scale`` < 1 shrinks Gaussian counts AND the image for quick tests."""
    if cfg == 1:
        return make_frame(int(50_000 * scale), 0, width=640, height=480, seed=seed)
    if cfg == 2:
        return make_frame(int(1_000_000 * scale), 0, seed=seed)
    if cfg == 3:
        return make_frame(int(1_000_000 * scale), 32, n_per_actor=max(1, int(10_000 * scale)), seed=seed)
    raise ValueError(f"unknown config {cfg}")


def waymo_rig(num_frames: int = 85) -> List[np.ndarray]:
    """cfg 4/5 camera rig: 5 cameras (yaw 0, +-50, +-100 deg) x ``num_frames`` poses, 0.5 m/frame along -z."""
    poses = []
    for f in range(num_frames):
        for yaw_deg in (0.0, 50.0, -50.0, 100.0, -100.0):
            y = math.radians(yaw_deg)
            c, s = math.cos(y), math.sin(y)
            R = np.array([[c, 0.0, s], [0.0, 1.0, 0.0], [-s, 0.0, c]])
            t = np.array([[0.0], [0.0], [-0.5 * f]])
            poses.append(np.concatenate([R, t], axis=1))
    return poses


def cotangents(height: int, width: int, seed: int = 7):
    """The fixed linear loss of cfg 2/3: sum(w*rgb) + sum(v*alpha), w,v ~ U(0,1)."""
    g = torch.Generator().manual_seed(seed)
    w = torch.rand(height, width, 3, generator=g)
    v = torch.rand(height, width, generator=g)
    return w, v


class WaymoScene:
    """BASELINE.json configs 4 / 5: Waymo-shape synthetic -- 5 cameras x ``num_frames`` frames, 1.68 M background + 32 x
    10 k actor Gaussians (2 M).  Actors are boxes parked on the road grid of SURVEY.md 8d; an actor has a box in a frame
    only while the ego vehicle is within ``actor_range`` metres of it, so the sub-models in view change per frame
    (as the reference's per-timestamp annotations do, data/utils/dynamic_annotation.py:252-286)."""

    def __init__(self, scale: float = 1.0, num_frames: int = 85, actor_range: float = 45.0, n_actors: int = 32):
        self.num_frames, self.actor_range = num_frames, actor_range
        self.n_bg = int(1_680_000 * scale)
        self.n_act = max(1, int(10_000 * scale))
        self.width = max(64, int(1920 * scale) // 16 * 16)
        self.height = max(48, int(1280 * scale) // 16 * 16)
        self.background = make_background(self.n_bg, seed=0, box=((-40.0, 40.0), (-6.0, 14.0), (-135.0, 45.0)))
        self.actors = {str(a): make_actor(self.n_act, seed=1 + a) for a in range(n_actors)}
        self.boxes = [actor_pose(a) for a in range(n_actors)]
        rig = waymo_rig(num_frames)  # index = frame * 5 + camera
        self.cameras = [make_camera(self.width, self.height, c2w=rig[i], time=float(i // 5)) for i in range(len(rig))]

    def boxes_at(self, frame: int):
        """[(actor index, rot, center)] of the actors that have a box in ``frame``."""
        ego_z = -0.5 * frame
        return [(a, rot, center) for a, (rot, center) in enumerate(self.boxes) if abs(center[2] - ego_z) <= self.actor_range]

    def frame(self, camera_index: int, fourier_dim: int = 5) -> Frame:
        """The rasterizer-level Frame (CPU tensors) of camera ``camera_index`` (= frame * 5 + rig camera)."""
        cam = self.cameras[camera_index]
        f = int(cam.time)
        segs = [Segment(params=self.background, cls=CLS_BACKGROUND, name="background")]
        basis = idft_basis(fourier_time(f, list(range(self.num_frames)), 1.0), fourier_dim)
        for a, rot, center in self.boxes_at(f):
            segs.append(Segment(params=self.actors[str(a)], cls=CLS_OBJECT, rot=rot, center=center, idft=basis, name=f"object_{a}"))
        return Frame(camera=cam, segments=segs)
