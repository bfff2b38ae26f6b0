"""Per-image appearance correction with bilateral grids (Wang et al., "Bilateral Guided Radiance Field Processing",
SIGGRAPH 2024), as gsplat ships it (``use_bilateral_grid``), on this library's kernels (csrc/bilagrid.cu).

A driving log's cameras each have their own exposure, white balance and vignetting, drifting over the drive.  Without a
per-image correction the Gaussians absorb those differences as view-dependent colour and floaters.  Every training image k gets
a small grid of affine colour transforms that is trained beside the scene:

    grids [N_img, 12, L, Hg, Wg] float32 (defaults L = 8, Hg = 16, Wg = 16): a 3x4 affine per node, row-major by output
          channel (r, g, b) over the inputs (r, g, b, 1); every node starts as the identity.  The layout of the published
          implementation, so its grids load here and the other way round.
    slice, pixel (i, j) of an H x W image with rendered colour c = (r, g, b):
          gx = (j + 0.5) / W * (Wg - 1),  gy = (i + 0.5) / H * (Hg - 1),  gz = clamp(0.299 r + 0.587 g + 0.114 b, 0, 1) * (L - 1)
          M = [A | t] = the grid interpolated trilinearly at (gx, gy, gz), corners clamped to the grid;  out = A c + t
          -- exactly F.grid_sample(grids[k][None], 2 [x, y, gray] - 1, mode="bilinear", padding_mode="border",
          align_corners=True) followed by the affine, ties and borders included: the gradient through gz passes only where
          the gray is strictly inside (0, 1).
    slice gradients: d grids[k] = the trilinear scatter of d_out (x) (c, 1);
          d c = A^T d_out + (d_out . dM/dgz (c, 1)) (L - 1) (0.299, 0.587, 0.114).
    total variation: tv(grids) = (1 / N_img) sum over the axes L, Hg, Wg of mean((forward difference along the axis)^2), each
          mean over all images and all 12 coefficients.  An axis of size 1 (L = 1 is allowed) has no differences and adds 0.
          The model's loss term is losses["bilagrid_tv"] = 10 tv, every training step.

The slice backward reduces the grid gradient without float atomics (two runs give the same bits); it supports L <= 32.  There
is no torch path here: the torch form (F.grid_sample) is the tests' float64 reference.

    model = SceneGraphRasterModel(..., bilateral_grid=BilateralGrid(num_train_images))
    opt = FusedAdam(model.optimizer_params(), extra={"bilateral_grid.grids": (model.bilateral_grid.grids, 2e-3)})
"""
from __future__ import annotations

import torch

from . import _lib
from .raster import _ptr, _stream

IDENTITY = (1.0, 0.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 0.0, 1.0, 0.0)


def _check_image(rgb: torch.Tensor, device) -> torch.Tensor:
    if not rgb.is_cuda:
        raise _lib.SgnError("the bilateral-grid slice needs a CUDA image: it has no CPU path")
    if rgb.dim() != 3 or rgb.shape[2] != 3:
        raise ValueError(f"rgb must be [H, W, 3], got {tuple(rgb.shape)}")
    if rgb.device != device:
        raise ValueError(f"rgb is on {rgb.device}, the grids on {device}")
    return rgb.detach().to(torch.float32).contiguous()


class _Slice(torch.autograd.Function):
    """out [H, W, 3] = the slice of ``rgb`` with ``grid`` [12, L, Hg, Wg]: sgn_bilagrid_slice_fwd forward, one
    sgn_bilagrid_slice_bwd backward for both gradients."""

    @staticmethod
    def forward(ctx, grid: torch.Tensor, rgb: torch.Tensor):
        g = grid.detach()
        c = _check_image(rgb, g.device)
        H, W = c.shape[:2]
        L, Hg, Wg = g.shape[1:]
        out = torch.empty_like(c)
        with torch.cuda.device(g.device):
            _lib.check(_lib.load().sgn_bilagrid_slice_fwd(_ptr(g), L, Hg, Wg, _ptr(c), H, W, _ptr(out), _stream()),
                       "sgn_bilagrid_slice_fwd")
        ctx.save_for_backward(grid)  # autograd's version check: an in-place change before backward is an error
        ctx.rgb = c
        return out

    @staticmethod
    def backward(ctx, v_out):
        if v_out is None:
            return None, None
        (grid,) = ctx.saved_tensors
        g, c = grid.detach(), ctx.rgb
        H, W = c.shape[:2]
        L, Hg, Wg = g.shape[1:]
        v = v_out.to(torch.float32).contiguous()
        d_rgb = torch.empty_like(c)
        d_grid = torch.empty_like(g)
        lib = _lib.load()
        sb = lib.sgn_bilagrid_slice_bwd_scratch_bytes(L, Hg, Wg, H, W)
        scratch = torch.empty(sb, device=g.device, dtype=torch.uint8)
        with torch.cuda.device(g.device):
            _lib.check(lib.sgn_bilagrid_slice_bwd(_ptr(g), L, Hg, Wg, _ptr(c), _ptr(v), H, W, _ptr(d_rgb), _ptr(d_grid), _ptr(scratch),
                                                  sb, _stream()), "sgn_bilagrid_slice_bwd")
        return (d_grid if ctx.needs_input_grad[0] else None), (d_rgb if ctx.needs_input_grad[1] else None)


class _TotalVariation(torch.autograd.Function):
    """tv (0-d) of grids [N, 12, L, Hg, Wg]: sgn_bilagrid_tv_fwd forward, sgn_bilagrid_tv_bwd backward (a dense gradient)."""

    @staticmethod
    def forward(ctx, grids: torch.Tensor):
        g = grids.detach()
        N, _, L, Hg, Wg = g.shape
        lib = _lib.load()
        out = torch.empty((), device=g.device, dtype=torch.float32)
        sb = lib.sgn_bilagrid_tv_scratch_bytes()
        scratch = torch.empty(sb, device=g.device, dtype=torch.uint8)
        with torch.cuda.device(g.device):
            _lib.check(lib.sgn_bilagrid_tv_fwd(_ptr(g), N, L, Hg, Wg, _ptr(out), _ptr(scratch), sb, _stream()), "sgn_bilagrid_tv_fwd")
        ctx.save_for_backward(grids)
        return out

    @staticmethod
    def backward(ctx, v):
        if v is None:
            return None
        (grids,) = ctx.saved_tensors
        g = grids.detach()
        N, _, L, Hg, Wg = g.shape
        vv = v.reshape(1).to(torch.float32).contiguous()
        d = torch.empty_like(g)
        with torch.cuda.device(g.device):
            _lib.check(_lib.load().sgn_bilagrid_tv_bwd(_ptr(g), N, L, Hg, Wg, _ptr(vv), _ptr(d), _stream()), "sgn_bilagrid_tv_bwd")
        return d


class BilateralGrid(torch.nn.Module):
    """One bilateral grid per training image (see the module docstring).  ``shape`` = (Hg, Wg, L), gsplat's
    ``(grid_Y, grid_X, grid_W)`` order; the parameter is ``grids`` [num_images, 12, L, Hg, Wg], identity-initialised."""

    def __init__(self, num_images: int, shape=(16, 16, 8)):
        super().__init__()
        Hg, Wg, L = (int(s) for s in shape)
        if num_images < 1 or min(Hg, Wg, L) < 1:
            raise ValueError(f"BilateralGrid needs num_images >= 1 and a positive shape, got {num_images}, {tuple(shape)}")
        if L > 32:
            raise ValueError(f"BilateralGrid supports grid depths L <= 32, got {L}")
        self.num_images = int(num_images)
        ident = torch.tensor(IDENTITY, dtype=torch.float32).reshape(1, 12, 1, 1, 1)
        self.grids = torch.nn.Parameter(ident.repeat(self.num_images, 1, L, Hg, Wg))

    def _checked(self) -> torch.Tensor:
        g = self.grids
        if not (g.is_cuda and g.dtype == torch.float32 and g.is_contiguous()):
            raise _lib.SgnError(f"grids must be a contiguous float32 CUDA tensor; got {g.dtype} on {g.device} "
                                "(move the module with .to('cuda'))")
        return g

    def slice(self, rgb: torch.Tensor, image_index: int) -> torch.Tensor:
        """The corrected image [H, W, 3] of ``rgb`` [H, W, 3] with the grid of image ``image_index``, differentiable in both."""
        k = int(image_index)
        if not 0 <= k < self.num_images:
            raise IndexError(f"image index {k} outside [0, {self.num_images})")
        return _Slice.apply(self._checked()[k], rgb)

    def tv_loss(self) -> torch.Tensor:
        """The total variation of all grids (0-d, differentiable; without the model's weight of 10)."""
        return _TotalVariation.apply(self._checked())
