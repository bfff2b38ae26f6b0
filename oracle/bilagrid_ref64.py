"""float64 statement of the bilateral-grid slice and total variation (csrc/bilagrid.cu, bilagrid.py).

Slice of an H x W image ``rgb`` [H, W, 3] with one grid [12, L, Hg, Wg] (a 3x4 affine per node, row-major by output channel):

    gx = (j + 0.5) / W * (Wg - 1),  gy = (i + 0.5) / H * (Hg - 1),  gz = clamp(0.299 r + 0.587 g + 0.114 b, 0, 1) * (L - 1)
    M  = trilinear interpolation of the grid at (gx, gy, gz), corners clamped to the grid;  out = M[:, :3] c + M[:, 3]

as an explicit 8-corner gather (``slice_ref64``), which equals ``F.grid_sample(grid[None], 2 [x, y, gray] - 1,
align_corners=True, padding_mode="border")`` followed by the affine (``slice_grid_sample``).  The gradient through gz passes
only where the gray is strictly inside (0, 1): grid_sample's border clip treats the border itself as outside.

``slice_grads_ref64`` states the gradients in closed form: d grid is the trilinear scatter of d_out (x) (c, 1);
d c = A^T d_out + (d_out . dM/dgz (c, 1)) (L - 1) (0.299, 0.587, 0.114), with dM/dgz = M(z0 + 1) - M(z0) at the floor z0
(one-sided at a node, as grid_sample's floor makes it).

Total variation over grids [N, 12, L, Hg, Wg]: (1 / N) sum over the axes L, Hg, Wg of mean((forward difference)^2), each
mean over all images and coefficients.  An axis of size 1 has no differences and adds 0 (torch's mean of an empty tensor would
be NaN).

``guide`` (optional: gz [H, W] and the strictly-inside mask [H, W]) replaces the computed guidance: the GPU tests pass the
kernel's float32 rounding of both (``guide_f32``), so that the one-sided derivative at a node and the clamp take the same
branch as the kernel.
"""
from __future__ import annotations

from typing import Tuple

import numpy as np
import torch
import torch.nn.functional as F

GRAY = (0.299, 0.587, 0.114)
IDENTITY = (1.0, 0.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 0.0, 1.0, 0.0)


def identity_grids(n: int, L: int = 8, Hg: int = 16, Wg: int = 16, dtype=torch.float32) -> torch.Tensor:
    """[n, 12, L, Hg, Wg] with every node the identity affine."""
    return torch.tensor(IDENTITY, dtype=dtype).reshape(1, 12, 1, 1, 1).repeat(n, 1, L, Hg, Wg)


def gray_of(rgb: torch.Tensor) -> torch.Tensor:
    return GRAY[0] * rgb[..., 0] + GRAY[1] * rgb[..., 1] + GRAY[2] * rgb[..., 2]


def _coords(H: int, W: int, Hg: int, Wg: int, dtype=torch.float64, device=None) -> Tuple[torch.Tensor, torch.Tensor]:
    gx = (torch.arange(W, dtype=dtype, device=device) + 0.5) / W * (Wg - 1)
    gy = (torch.arange(H, dtype=dtype, device=device) + 0.5) / H * (Hg - 1)
    return gx[None, :].expand(H, W), gy[:, None].expand(H, W)


def _lower(c: torch.Tensor, g: int) -> torch.Tensor:
    return torch.clamp(torch.floor(c), max=max(g - 2, 0)).long()


def _gz(rgb: torch.Tensor, L: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """(gz with its gradient where gray is strictly inside (0, 1), gray)."""
    gray = gray_of(rgb)
    inside = (gray > 0) & (gray < 1)
    gz = torch.where(inside, gray, gray.detach().clamp(0, 1)) * (L - 1)
    return gz, gray


def _corners(grid: torch.Tensor, gx, gy, gz):
    """The 8 corner indices and weights of the trilinear gather; gz may carry a gradient."""
    L, Hg, Wg = grid.shape[1:]
    x0, y0, z0 = _lower(gx, Wg), _lower(gy, Hg), _lower(gz.detach(), L)
    fx, fy, fz = gx - x0, gy - y0, gz - z0
    x1, y1, z1 = torch.clamp(x0 + 1, max=Wg - 1), torch.clamp(y0 + 1, max=Hg - 1), torch.clamp(z0 + 1, max=L - 1)
    out = []
    for dz, zi, wz in ((0, z0, 1 - fz), (1, z1, fz)):
        for dy, yi, wy in ((0, y0, 1 - fy), (1, y1, fy)):
            for dx, xi, wx in ((0, x0, 1 - fx), (1, x1, fx)):
                out.append((zi, yi, xi, wx * wy * wz))
    return out


def guide_f32(rgb: np.ndarray, L: int) -> Tuple[np.ndarray, np.ndarray]:
    """(gz, strictly inside) as the kernel rounds them: the gray and gz in float32, one rounding per operation."""
    c = np.asarray(rgb, np.float32)
    f = np.float32
    gray = (f(0.299) * c[..., 0] + f(0.587) * c[..., 1]) + f(0.114) * c[..., 2]
    gz = np.clip(gray, f(0), f(1)) * f(L - 1)
    return gz.astype(np.float64), (gray > 0) & (gray < 1)


def slice_ref64(grid: torch.Tensor, rgb: torch.Tensor, guide=None) -> torch.Tensor:
    """The slice as an explicit gather: grid [12, L, Hg, Wg], rgb [H, W, 3] -> [H, W, 3], differentiable in both (in float64
    when given float64).  ``guide``: see the module docstring (the value depends on gz only)."""
    L, Hg, Wg = grid.shape[1:]
    H, W = rgb.shape[:2]
    gx, gy = _coords(H, W, Hg, Wg, rgb.dtype, rgb.device)
    if guide is None:
        gz, _ = _gz(rgb, L)
    else:
        gz = torch.as_tensor(guide[0], dtype=rgb.dtype, device=rgb.device)
    M = 0
    for zi, yi, xi, w in _corners(grid, gx, gy, gz):
        M = M + w[..., None] * grid[:, zi, yi, xi].permute(1, 2, 0)
    M = M.reshape(H, W, 3, 4)
    return (M[..., :3] * rgb[:, :, None, :]).sum(-1) + M[..., 3]


def slice_grid_sample(grid: torch.Tensor, rgb: torch.Tensor) -> torch.Tensor:
    """The same through F.grid_sample (the published implementation's form)."""
    H, W = rgb.shape[:2]
    xs = (torch.arange(W, dtype=rgb.dtype) + 0.5) / W
    ys = (torch.arange(H, dtype=rgb.dtype) + 0.5) / H
    x, y = xs[None, :].expand(H, W), ys[:, None].expand(H, W)
    xyz = torch.stack([x, y, gray_of(rgb)], -1)
    M = F.grid_sample(grid[None], (2.0 * xyz - 1.0)[None, None], mode="bilinear", padding_mode="border", align_corners=True)
    M = M[0, :, 0].permute(1, 2, 0).reshape(H, W, 3, 4)
    return (M[..., :3] * rgb[:, :, None, :]).sum(-1) + M[..., 3]


def slice_grads_ref64(grid, rgb, d_out, guide=None) -> Tuple[np.ndarray, np.ndarray]:
    """(d_rgb [H, W, 3], d_grid [12, L, Hg, Wg]) in closed form, float64 numpy.  The inputs are numpy arrays or tensors; with
    CUDA tensors the statement is evaluated on that device (in float64)."""
    g = torch.as_tensor(grid).to(torch.float64)
    dev = g.device
    c = torch.as_tensor(rgb).to(dev, torch.float64)
    d = torch.as_tensor(d_out).to(dev, torch.float64)
    L, Hg, Wg = g.shape[1:]
    H, W = c.shape[:2]
    gx, gy = _coords(H, W, Hg, Wg, device=dev)
    if guide is None:
        gray = gray_of(c)
        inside, z = (gray > 0) & (gray < 1), gray.clamp(0, 1) * (L - 1)
    else:
        z, inside = torch.as_tensor(guide[0]).to(dev, torch.float64), torch.as_tensor(guide[1]).to(dev, torch.bool)
    cin = torch.cat([c, torch.ones(H, W, 1, dtype=torch.float64, device=dev)], -1)
    gvec = (d[..., :, None] * cin[..., None, :]).reshape(H, W, 12)
    d_grid = torch.zeros(12, L, Hg, Wg, dtype=torch.float64, device=dev)
    M = torch.zeros(H, W, 12, dtype=torch.float64, device=dev)
    corners = _corners(g, gx, gy, z)
    for zi, yi, xi, w in corners:
        M += w[..., None] * g[:, zi, yi, xi].permute(1, 2, 0)
        flat = ((zi * Hg + yi) * Wg + xi).reshape(-1)
        contrib = (w[..., None] * gvec).reshape(-1, 12)
        d_grid.view(12, -1).index_add_(1, flat, contrib.t())
    z0 = _lower(z, L)
    z1 = torch.clamp(z0 + 1, max=L - 1)
    x0, y0 = _lower(gx, Wg), _lower(gy, Hg)
    fx, fy = gx - x0, gy - y0
    x1, y1 = torch.clamp(x0 + 1, max=Wg - 1), torch.clamp(y0 + 1, max=Hg - 1)

    def plane(zi):
        return sum(w[..., None] * g[:, zi, yi, xi].permute(1, 2, 0)
                   for yi, xi, w in ((y0, x0, (1 - fy) * (1 - fx)), (y0, x1, (1 - fy) * fx), (y1, x0, fy * (1 - fx)), (y1, x1, fy * fx)))
    dM = (plane(z1) - plane(z0)).reshape(H, W, 3, 4)
    M = M.reshape(H, W, 3, 4)
    d_rgb = (M[..., :3] * d[..., :, None]).sum(-2)
    dgz = (d[..., :, None] * dM * cin[..., None, :]).sum((-1, -2)) * (L - 1)
    d_rgb = d_rgb + torch.where(inside, dgz, torch.zeros_like(dgz))[..., None] * torch.tensor(GRAY, dtype=torch.float64, device=dev)
    return d_rgb.cpu().numpy(), d_grid.cpu().numpy()


def tv_ref64(grids: torch.Tensor) -> torch.Tensor:
    """Total variation of grids [N, 12, L, Hg, Wg], differentiable."""
    n = grids.shape[0]
    tv = grids.new_zeros(())
    for axis in (2, 3, 4):
        if grids.shape[axis] > 1:
            tv = tv + torch.diff(grids, dim=axis).pow(2).mean()
    return tv / n
