"""Fused loss epilogue (SURVEY.md 8f rank 2): the image-space terms of the reference's ``get_loss_dict``
(street_gaussians_ns/sgn_splatfacto.py:1042-1094, sgn_splatfacto_scene_graph.py:376-391) that re-read the
rasterizer's outputs -- L1, sky accumulation, object-accumulation entropy -- as two HBM-bound kernels of
libsgn_raster.so (forward sums, backward cotangents) behind one autograd node; and the SSIM term
(sgn_splatfacto.py:1085-1087) as its own forward / backward pair (csrc/ssim.cu) behind a second one.  The per-step metrics
of ``get_metrics_dict`` (sgn_splatfacto.py:1015-1040) are one reduction kernel (csrc/metrics.cu, ``fused_metrics``)."""
from __future__ import annotations

import ctypes as C
from typing import Optional, Tuple

import torch

from . import _lib
from .raster import _ptr, _stream


def _loss_in(rgb, gt, mask, accumulation, sky_mask, object_acc, w) -> Tuple[_lib.LossIn, list]:
    li = _lib.LossIn()
    keep = []

    def f32(t):
        if t is None:
            return None
        t = t.detach()
        if t.dtype != torch.float32 or not t.is_contiguous():
            t = t.float().contiguous()
        keep.append(t)
        return t.data_ptr()

    li.rgb = f32(rgb)
    if gt is not None:
        if gt.dtype == torch.uint8:
            g = gt.contiguous()
            keep.append(g)
            li.gt_u8 = g.data_ptr()
        else:
            li.gt_f32 = f32(gt)
    li.mask = f32(mask)
    li.accumulation = f32(accumulation)
    if sky_mask is not None:
        sm = sky_mask.to(torch.uint8).contiguous()
        keep.append(sm)
        li.sky_mask = sm.data_ptr()
    li.object_acc = f32(object_acc)
    li.w_l1, li.w_sky, li.w_entropy = w
    return li, keep


class _FusedImageLosses(torch.autograd.Function):
    @staticmethod
    def forward(ctx, rgb, accumulation, object_acc, gt, mask, sky_mask, w_l1: float, w_sky: float, w_entropy: float):
        L = _lib.load()
        if not rgb.is_cuda:
            raise _lib.SgnError("the fused loss epilogue has no CPU path")
        H, W = rgb.shape[0], rgb.shape[1]
        use_sky = sky_mask is not None and accumulation is not None and w_sky > 0
        li, keep = _loss_in(rgb, gt, mask, accumulation if use_sky else None, sky_mask if use_sky else None,
                            object_acc if w_entropy > 0 else None, (w_l1, w_sky if use_sky else 0.0, w_entropy))
        losses = torch.empty(3, device=rgb.device, dtype=torch.float32)
        sb = L.sgn_loss_scratch_bytes()
        scratch = torch.empty(sb, device=rgb.device, dtype=torch.uint8)
        _lib.check(L.sgn_loss_fwd(H, W, C.byref(li), _ptr(losses), _ptr(scratch), sb, _stream()), "sgn_loss_fwd")
        ctx.li, ctx.keep, ctx.shape = li, keep, (H, W)
        ctx.need = (rgb.requires_grad, accumulation is not None and accumulation.requires_grad and use_sky,
                    object_acc is not None and object_acc.requires_grad and w_entropy > 0)
        ctx.set_materialize_grads(False)
        return losses[0], losses[1], losses[2]

    @staticmethod
    def backward(ctx, g_l1, g_sky, g_ent):
        L = _lib.load()
        H, W = ctx.shape
        dev = ctx.keep[0].device
        gs = [g if g is not None else torch.zeros((), device=dev) for g in (g_l1, g_sky, g_ent)]
        g = torch.stack([x.reshape(()).float() for x in gs])
        v_rgb = torch.empty(H, W, 3, device=dev) if ctx.need[0] else None
        v_acc = torch.empty(H, W, 1, device=dev) if ctx.need[1] else None
        v_obj = torch.empty(H, W, 1, device=dev) if ctx.need[2] else None
        _lib.check(L.sgn_loss_bwd(H, W, C.byref(ctx.li), _ptr(g), _ptr(v_rgb), _ptr(v_acc), _ptr(v_obj), _stream()), "sgn_loss_bwd")
        return v_rgb, v_acc, v_obj, None, None, None, None, None, None


def fused_image_losses(rgb: torch.Tensor, gt: torch.Tensor, accumulation: Optional[torch.Tensor] = None,
                       object_acc: Optional[torch.Tensor] = None, mask: Optional[torch.Tensor] = None,
                       sky_mask: Optional[torch.Tensor] = None, w_l1: float = 1.0, w_sky: float = 0.0,
                       w_entropy: float = 0.0):
    """Returns (Ll1, sky_accumulation, object_acc_entropy) 0-d tensors, already weighted; terms without
    inputs / with zero weight are exact zeros with no gradient.  ``gt`` may be float32 or uint8 (gt/255)."""
    return _FusedImageLosses.apply(rgb, accumulation, object_acc, gt, mask, sky_mask, float(w_l1), float(w_sky), float(w_entropy))


class _FusedSSIM(torch.autograd.Function):
    @staticmethod
    def forward(ctx, rgb, gt, mask, weight: float):
        L = _lib.load()
        if not rgb.is_cuda:
            raise _lib.SgnError("the fused SSIM term has no CPU path")
        H, W = rgb.shape[0], rgb.shape[1]
        li, keep = _loss_in(rgb, gt, mask, None, None, None, (0.0, 0.0, 0.0))
        loss = torch.empty((), device=rgb.device, dtype=torch.float32)
        wb = L.sgn_ssim_workspace_bytes(H, W)
        ws = torch.empty(max(wb, 1), device=rgb.device, dtype=torch.uint8)  # the derivative maps the backward reads
        _lib.check(L.sgn_ssim_fwd(H, W, C.byref(li), weight, _ptr(loss), _ptr(ws), wb, _stream()), "sgn_ssim_fwd")
        ctx.li, ctx.keep, ctx.ws, ctx.shape, ctx.weight = li, keep, ws, (H, W), weight
        return loss

    @staticmethod
    def backward(ctx, g):
        L = _lib.load()
        H, W = ctx.shape
        g = g.reshape(()).float().contiguous()
        v_rgb = torch.empty(H, W, 3, device=ctx.ws.device)
        _lib.check(L.sgn_ssim_bwd(H, W, C.byref(ctx.li), ctx.weight, _ptr(g), _ptr(ctx.ws), _ptr(v_rgb), _stream()), "sgn_ssim_bwd")
        return v_rgb, None, None, None


def fused_ssim_loss(rgb: torch.Tensor, gt: torch.Tensor, mask: Optional[torch.Tensor] = None, weight: float = 1.0) -> torch.Tensor:
    """``weight * (1 - SSIM(gt * mask, rgb * mask))`` as a 0-d tensor: pytorch_msssim.SSIM(data_range=1, size_average=True,
    channel=3) as the reference applies it (sgn_splatfacto.py:1081-1087).  ``rgb`` is [H,W,3] float32, ``gt`` [H,W,3] float32
    or uint8 (gt/255), ``mask`` [H,W,1] or None; H and W must be at least 11.  The gradient flows to ``rgb`` only.  With
    ``weight == 0`` the result is an exact zero and nothing is launched."""
    if float(weight) == 0.0:
        return torch.zeros((), device=rgb.device)
    return _FusedSSIM.apply(rgb, gt, mask, float(weight))


METRIC_NAMES = ("psnr", "scale_mean", "log_scale_mean", "sigmoid_opacity", "radii_mean")


def fused_metrics(rgb: Optional[torch.Tensor] = None, gt: Optional[torch.Tensor] = None, mask: Optional[torch.Tensor] = None,
                  table=None, radii: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The per-step metrics of the reference's ``get_metrics_dict`` (sgn_splatfacto.py:1015-1040) from one ``sgn_metrics``
    call (csrc/metrics.cu): a float32 device tensor [5] = ``METRIC_NAMES``.

    * psnr: ``10 log10(1 / mean((gt*mask - rgb*mask)^2))`` over H*W*3 (torchmetrics PeakSignalNoiseRatio, data_range 1), +inf
      for equal images; ``rgb`` [H,W,3] float32, ``gt`` [H,W,3] float32 or uint8 (gt/255), ``mask`` [H,W,1] or None.
    * scale_mean, log_scale_mean, sigmoid_opacity: means of exp(scales), scales and sigmoid(opacities) over the rows of
      ``table`` (a ``raster.SegmentTable`` with its device rows: the frame's visible sub-models, read in place).
    * radii_mean: mean of ``radii`` [N] int32.
    A term without its inputs is NaN, as is a mean over zero rows.  Nothing is read back to the host."""
    L = _lib.load()
    ref = rgb if rgb is not None else radii
    dev = ref.device if ref is not None else table.dev.device
    if dev.type != "cuda":
        raise _lib.SgnError("the fused metrics have no CPU path")
    li, keep, H, W = None, [], 0, 0
    if rgb is not None:
        H, W = rgb.shape[0], rgb.shape[1]
        li, keep = _loss_in(rgb, gt, mask, None, None, None, (0.0, 0.0, 0.0))
    if radii is not None:
        assert radii.dtype == torch.int32
        radii = radii.contiguous()
    tab, nseg, N, chunks = None, 0, 0, 0
    if table is not None:
        tab, nseg, N, chunks = table.dev, table.nseg, table.N, table.num_chunks
    elif radii is not None:
        N = radii.shape[0]
    if radii is not None:
        assert radii.shape[0] == N, "radii must have one entry per row of the table"
    out = torch.empty(5, device=dev, dtype=torch.float32)
    sb = L.sgn_metrics_scratch_bytes()
    scratch = torch.empty(sb, device=dev, dtype=torch.uint8)
    _lib.check(L.sgn_metrics(H, W, C.byref(li) if li is not None else None, _ptr(tab), nseg, N, chunks, _ptr(radii), _ptr(out),
                             _ptr(scratch), sb, _stream()), "sgn_metrics")
    return out
