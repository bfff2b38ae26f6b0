"""A sub-model's initial Gaussians from seed points: ``SplatfactoModel.populate_modules`` (street_gaussians_ns/sgn_splatfacto.py:
253-300) for one sub-model, with its nearest-neighbour scales from the GPU search of knn.py instead of sklearn on the CPU.

Random draws come from ``generator`` -- by default torch's default CPU generator -- in the reference's order, on the CPU, so
that under equal seeds every tensor equals a seeded reference run's (the scales up to the fp32 rounding of the distances).
"""
from __future__ import annotations

from typing import Optional, Union

import torch

from .knn import knn_log_scales
from .scene import GaussianSet
from .synthetic import random_quats

C0 = 0.28209479177387814  # RGB2SH (sgn_splatfacto.py:57-62)

Device = Union[str, torch.device, None]


def _device(device: Device) -> torch.device:
    return torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())


def _geometry(means: torch.Tensor, generator, device):
    """means on the device, their kNN scales, then the quaternion draws and the opacities (sgn_splatfacto.py:255-267)."""
    means = means.to(device=device, dtype=torch.float32).contiguous()
    n = means.shape[0]
    scales = knn_log_scales(means, 3)
    quats = random_quats(n, generator).to(device)
    opacities = torch.logit(0.1 * torch.ones(n, 1)).to(device)
    return means, scales, quats, opacities


def gaussians_from_points(xyz: torch.Tensor, rgb: torch.Tensor, sh_degree: int = 3, fourier_dim: int = 5,
                          generator: Optional[torch.Generator] = None, device: Device = None) -> GaussianSet:
    """The seed-point branch of ``populate_modules`` (``seed_points = (xyz, rgb)``, ``random_init`` off).

    ``xyz`` [N, 3] positions; ``rgb`` [N, 3] colours in 0..255, uint8 (COLMAP ``points3D``) or float (an actor's lidar cloud).
    means = xyz; scales = log(mean distance to the 3 nearest other points), repeated x3 -- -inf for a point with three or more
    exact duplicates (the mean is 0), as the reference computes it; quats uniform random (three ``torch.rand(N)`` draws of
    ``random_quat_tensor``); opacities = logit(0.1); features_dc [N, fourier_dim, 3] zeros with ``[:, 0] = RGB2SH(rgb / 255)``,
    or ``logit(rgb / 255, eps=1e-10)`` when ``sh_degree == 0``; features_rest [N, (sh_degree + 1)^2 - 1, 3] zeros.  N >= 4.
    The tensors are returned on ``device`` (default: the current CUDA device).
    """
    device = _device(device)
    xyz, rgb = torch.as_tensor(xyz), torch.as_tensor(rgb)
    if xyz.dim() != 2 or xyz.shape[1] != 3 or rgb.shape != xyz.shape:
        raise ValueError(f"xyz and rgb must both be [N, 3], got {tuple(xyz.shape)} and {tuple(rgb.shape)}")
    n = xyz.shape[0]
    dim_sh = (sh_degree + 1) ** 2
    shs = torch.zeros((n, dim_sh, 3), device=rgb.device).float()
    if sh_degree > 0:
        shs[:, 0, :3] = (rgb / 255 - 0.5) / C0
    else:
        shs[:, 0, :3] = torch.logit(rgb / 255, eps=1e-10)
    features_dc = torch.zeros(n, fourier_dim, 3, device=rgb.device)
    features_dc[:, 0, :3] = shs[:, 0, :3]
    means, scales, quats, opacities = _geometry(xyz, generator, device)
    return GaussianSet(means, scales, quats, features_dc.to(device).contiguous(), shs[:, 1:, :].to(device).contiguous(), opacities)


def random_gaussians(num_random: int = 50000, random_scale: float = 10.0, sh_degree: int = 3, fourier_dim: int = 5,
                     generator: Optional[torch.Generator] = None, device: Device = None) -> GaussianSet:
    """The random branch of ``populate_modules`` (no seed points, or ``random_init``).

    means = (rand(N, 3) - 0.5) * random_scale; scales, quats and opacities as in ``gaussians_from_points``; then
    features_dc [N, fourier_dim, 3] zeros with ``[:, 0] = rand(N, 3)`` -- raw values, not SH-converted, as the reference
    does -- and features_rest zeros.
    """
    device = _device(device)
    means = (torch.rand((num_random, 3), generator=generator) - 0.5) * random_scale
    means, scales, quats, opacities = _geometry(means, generator, device)  # the quaternion draws come before the colours'
    features_dc = torch.zeros(num_random, fourier_dim, 3)
    features_dc[:, 0, :3] = torch.rand(num_random, 3, generator=generator)
    features_rest = torch.zeros((num_random, (sh_degree + 1) ** 2 - 1, 3), device=device)
    return GaussianSet(means, scales, quats, features_dc.to(device).contiguous(), features_rest, opacities)


def replay_scene_graph_init(generator: Optional[torch.Generator] = None, num_random: int = 50000) -> None:
    """Consume the draws of the scene graph's own random initialisation, which the reference makes and then discards before
    it builds the background (sgn_splatfacto_scene_graph.py:50-52 runs the random branch of populate_modules for the
    wrapper model): rand(num_random, 3) for the means, three rand(num_random) for the quaternions, rand(num_random, 3) for the
    colours.  Nothing is computed from them."""
    torch.rand(num_random, 3, generator=generator)
    for _ in range(3):
        torch.rand(num_random, generator=generator)
    torch.rand(num_random, 3, generator=generator)


