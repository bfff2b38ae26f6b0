"""Lidar depth supervision (csrc/depth.cu): a sweep projected into a sparse depth map for the camera the render uses, the L1
depth term on the rendered depth with its gradient, and the depth metrics of eval.

Street Gaussians supervises the rendered depth with lidar; the reference's datamanager carries the target as
``batch["depth_image"]`` (sgn_datamanager.py:360-361) and its eval calls a ``depth_result`` (sgn_splatfacto.py:1160-1168) that
it never defines.  There is no CPU path: every function launches the library's kernels and reads nothing back."""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np
import torch

from . import _lib
from .raster import RenderSettings, _ptr, _stream, camera_struct

METRIC_NAMES = ("abs_rel", "sq_rel", "rmse", "rmse_log", "a1", "a2", "a3", "n_valid")


def _image(t: Optional[torch.Tensor], what: str, H: int, W: int, device) -> Optional[torch.Tensor]:
    if t is None:
        return None
    if not t.is_cuda:
        raise _lib.SgnError(f"{what} must be a CUDA tensor: the depth kernels have no CPU path")
    if t.numel() != H * W:
        raise ValueError(f"{what} has {t.numel()} elements, the depth map has {H}x{W}")
    return t.detach().to(device=device, dtype=torch.float32).contiguous()


def lidar_depth_map(points: torch.Tensor, camera, to_world=None, settings: Optional[RenderSettings] = None) -> torch.Tensor:
    """Project the lidar ``points`` [M, 3] into a sparse float32 depth map [H, W, 1] for ``camera``: the camera-space z of the
    nearest return on each pixel, 0 where no point lands.

    ``camera`` is a ``scene.Camera`` (its struct is built as the render builds it, with ``settings``' clip_thresh) or a
    ``_lib.CameraStruct``.  ``to_world``: None when the points are in the world frame, else the sweep's 3x4 (or 4x4)
    sweep-to-world matrix (the lidar pose times the dataparser transform and scale), read on the host.  A point goes to pixel
    (floor(u), floor(v)) of the projection's own pixel centre; points with z <= clip_thresh or off the image are dropped."""
    cs = camera if isinstance(camera, _lib.CameraStruct) else camera_struct(camera, settings or RenderSettings())
    if not points.is_cuda:
        raise _lib.SgnError("lidar points must be a CUDA tensor: the depth map has no CPU path")
    pts = points.detach().to(torch.float32).contiguous()
    if pts.dim() != 2 or pts.shape[1] != 3:
        raise ValueError(f"lidar points must have shape [M, 3], got {tuple(points.shape)}")
    tw = None
    if to_world is not None:
        m = torch.as_tensor(to_world).detach().cpu().to(torch.float64).numpy()
        if m.shape not in ((3, 4), (4, 4)):
            raise ValueError(f"to_world must be 3x4 or 4x4, got {m.shape}")
        tw = (C.c_float * 12)(*np.asarray(m[:3, :4], np.float32).reshape(-1).tolist())
    L = _lib.load()
    out = torch.empty(cs.height, cs.width, 1, device=pts.device, dtype=torch.float32)
    with torch.cuda.device(pts.device):
        _lib.check(L.sgn_lidar_depth_map(_ptr(pts) if pts.numel() else None, pts.shape[0], C.byref(cs), tw, _ptr(out), _stream()),
                   "sgn_lidar_depth_map")
    return out


class _FusedDepthLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, depth, target, mask, weight: float):
        H, W = depth.shape[0], depth.shape[1]
        dev = depth.device
        d = _image(depth, "depth", H, W, dev)
        t = _image(target, "target", H, W, dev)
        m = _image(mask, "mask", H, W, dev)
        L = _lib.load()
        loss = torch.empty((), device=dev, dtype=torch.float32)
        n_valid = torch.empty((), device=dev, dtype=torch.int32)
        sb = L.sgn_depth_scratch_bytes()
        scratch = torch.empty(sb, device=dev, dtype=torch.uint8)
        _lib.check(L.sgn_depth_loss_fwd(H, W, _ptr(d), _ptr(t), _ptr(m), weight, _ptr(loss), _ptr(n_valid), _ptr(scratch), sb, _stream()),
                   "sgn_depth_loss_fwd")
        ctx.keep, ctx.n_valid, ctx.weight = (d, t, m), n_valid, weight
        return loss

    @staticmethod
    def backward(ctx, g):
        d, t, m = ctx.keep
        H, W = d.shape[0], d.shape[1]
        g = g.reshape(()).float().contiguous()
        v = torch.empty_like(d)
        _lib.check(_lib.load().sgn_depth_loss_bwd(H, W, _ptr(d), _ptr(t), _ptr(m), ctx.weight, _ptr(ctx.n_valid), _ptr(g), _ptr(v),
                                                  _stream()), "sgn_depth_loss_bwd")
        return v, None, None, None


def fused_depth_loss(depth: torch.Tensor, target: torch.Tensor, mask: Optional[torch.Tensor] = None, weight: float = 1.0) -> torch.Tensor:
    """``weight * sum |depth - target| / n_valid`` over the valid pixels (``target > 0`` and ``mask != 0``) as a 0-d tensor;
    exactly 0, with a zero gradient, when no pixel is valid.  ``depth``, ``target`` and ``mask`` (1 = keep, or None) are
    [H, W, 1] (or [H, W]) CUDA tensors.  The gradient flows to ``depth`` only; the count of valid pixels stays on the device."""
    return _FusedDepthLoss.apply(depth, target, mask, float(weight))


def depth_loss_torch(depth: torch.Tensor, target: torch.Tensor, mask: Optional[torch.Tensor] = None, weight: float = 1.0) -> torch.Tensor:
    """The same term as torch operations (the model's ``fused_loss=False`` path)."""
    valid = target > 0
    if mask is not None:
        valid = valid & (mask != 0)
    n = valid.sum().clamp(min=1).to(depth.dtype)
    return weight * torch.where(valid, (depth - target).abs(), torch.zeros((), device=depth.device, dtype=depth.dtype)).sum() / n


def depth_metrics(depth: torch.Tensor, target: torch.Tensor, mask: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Depth metrics over the valid pixels as a float32 device tensor [8] = ``METRIC_NAMES``: abs_rel, sq_rel, rmse, rmse_log,
    a1, a2, a3 (the fraction with max(d/t, t/d) < 1.25^k) and n_valid, with the prediction clamped to at least 1e-3.  Summed in
    fp64 in a fixed order; the means are NaN when no pixel is valid.  Nothing is read back."""
    H, W = depth.shape[0], depth.shape[1]
    dev = depth.device
    d = _image(depth, "depth", H, W, dev)
    t = _image(target, "target", H, W, dev)
    m = _image(mask, "mask", H, W, dev)
    L = _lib.load()
    out = torch.empty(8, device=dev, dtype=torch.float32)
    sb = L.sgn_depth_scratch_bytes()
    scratch = torch.empty(sb, device=dev, dtype=torch.uint8)
    _lib.check(L.sgn_depth_metrics(H, W, _ptr(d), _ptr(t), _ptr(m), _ptr(out), _ptr(scratch), sb, _stream()), "sgn_depth_metrics")
    return out
