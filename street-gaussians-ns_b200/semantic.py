"""Per-Gaussian semantic logits (csrc/semantic.cu): the cross-entropy term of the rendered semantic map against a 2D
segmentation with its gradient, the eval metrics (pixel accuracy and mean IoU from one confusion-matrix pass) and the carry of
a per-row tensor through a refinement.

Street Gaussians gives every Gaussian a vector of class logits, alpha-blends them into a semantic map and supervises it with
cross-entropy; the reference's loader carries the segmentation as ``batch["semantic"]`` (data/sgn_dataset.py:125, classes
DEFAULT / GROUND / SKY, data/utils/data_utils.py:26-29).  A pixel is valid when ``0 <= label < C`` and ``mask != 0``; any other
label (e.g. 255) is ignored.  There is no CPU path: the fused functions launch the library's kernels and read nothing back."""
from __future__ import annotations

import ctypes as C
import math
from typing import Dict, Optional, Tuple

import torch
import torch.nn.functional as F

from . import _lib
from .raster import _ptr, _stream

MAX_CLASSES = 64


def _logits(t: torch.Tensor) -> Tuple[torch.Tensor, int, int, int]:
    if not t.is_cuda:
        raise _lib.SgnError("the semantic logits must be a CUDA tensor: the semantic kernels have no CPU path")
    if t.dim() != 3:
        raise ValueError(f"semantic logits must have shape [H, W, C], got {tuple(t.shape)}")
    H, W, Cn = t.shape
    if not 1 <= Cn <= MAX_CLASSES:
        raise ValueError(f"{Cn} semantic classes: 1..{MAX_CLASSES} are supported")
    return t.detach().to(torch.float32).contiguous(), H, W, Cn


def _labels(labels: torch.Tensor, H: int, W: int, device) -> torch.Tensor:
    """[H, W] or [H, W, 1] -> contiguous int64 [H, W] on ``device`` (the loader's dtype is read as it is; other integer dtypes
    are converted once)."""
    if labels.numel() != H * W:
        raise ValueError(f"the labels have {labels.numel()} elements, the semantic map has {H}x{W}")
    if labels.is_floating_point():
        raise TypeError(f"semantic labels must be integers, got {labels.dtype}")
    return labels.detach().reshape(H, W).to(device=device, dtype=torch.int64).contiguous()


def _mask(mask: Optional[torch.Tensor], H: int, W: int, device) -> Optional[torch.Tensor]:
    if mask is None:
        return None
    if mask.numel() != H * W:
        raise ValueError(f"the mask has {mask.numel()} elements, the semantic map has {H}x{W}")
    return mask.detach().reshape(H, W).to(device=device, dtype=torch.float32).contiguous()


class _FusedSemanticLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, labels, mask, weight: float):
        s, H, W, Cn = _logits(logits)
        dev = s.device
        lab = _labels(labels, H, W, dev)
        m = _mask(mask, H, W, dev)
        L = _lib.load()
        loss = torch.empty((), device=dev, dtype=torch.float32)
        n_valid = torch.empty((), device=dev, dtype=torch.int32)
        sb = L.sgn_semantic_scratch_bytes()
        scratch = torch.empty(sb, device=dev, dtype=torch.uint8)
        _lib.check(L.sgn_semantic_loss_fwd(H, W, Cn, _ptr(s), _ptr(lab), _ptr(m), weight, _ptr(loss), _ptr(n_valid), _ptr(scratch), sb,
                                           _stream()), "sgn_semantic_loss_fwd")
        ctx.keep, ctx.n_valid, ctx.weight = (s, lab, m), n_valid, weight
        return loss

    @staticmethod
    def backward(ctx, g):
        s, lab, m = ctx.keep
        H, W, Cn = s.shape
        g = g.reshape(()).float().contiguous()
        v = torch.empty_like(s)
        _lib.check(_lib.load().sgn_semantic_loss_bwd(H, W, Cn, _ptr(s), _ptr(lab), _ptr(m), ctx.weight, _ptr(ctx.n_valid), _ptr(g),
                                                     _ptr(v), _stream()), "sgn_semantic_loss_bwd")
        return v, None, None, None


def fused_semantic_loss(logits: torch.Tensor, labels: torch.Tensor, mask: Optional[torch.Tensor] = None,
                        weight: float = 1.0) -> torch.Tensor:
    """``weight * sum CE / n_valid`` over the valid pixels as a 0-d tensor, CE = logsumexp(logits[p]) - logits[p, label];
    exactly 0, with a zero gradient, when no pixel is valid.  ``logits`` [H, W, C] (CUDA), ``labels`` [H, W] or [H, W, 1]
    integers, ``mask`` (1 = keep) [H, W] / [H, W, 1] or None.  The gradient flows to ``logits`` only; the count of valid pixels
    stays on the device, and two runs give the same bits."""
    return _FusedSemanticLoss.apply(logits, labels, mask, float(weight))


def semantic_loss_torch(logits: torch.Tensor, labels: torch.Tensor, mask: Optional[torch.Tensor] = None,
                        weight: float = 1.0) -> torch.Tensor:
    """The same term as torch operations (the model's ``fused_loss=False`` path): ``F.cross_entropy`` summed over the valid
    pixels, divided by their count (0 when there is none)."""
    H, W, Cn = logits.shape
    lab = labels.reshape(H, W).to(device=logits.device, dtype=torch.int64)
    valid = (lab >= 0) & (lab < Cn)
    if mask is not None:
        valid = valid & (mask.reshape(H, W).to(logits.device) != 0)
    target = torch.where(valid, lab, torch.full_like(lab, -100))  # F.cross_entropy's ignore_index
    ce = F.cross_entropy(logits.reshape(H * W, Cn), target.reshape(-1), ignore_index=-100, reduction="sum")
    n = valid.sum().clamp(min=1).to(logits.dtype)
    return weight * ce / n


def semantic_confusion(logits: torch.Tensor, labels: torch.Tensor, mask: Optional[torch.Tensor] = None) -> torch.Tensor:
    """int64 [C, C] device tensor: entry (label, argmax logits) counts the valid pixels with that pair (ties to the lowest
    class; the first NaN logit wins, as in torch.argmax).  One launch; nothing is read back."""
    s, H, W, Cn = _logits(logits)
    dev = s.device
    lab = _labels(labels, H, W, dev)
    m = _mask(mask, H, W, dev)
    out = torch.empty(Cn, Cn, device=dev, dtype=torch.int64)
    _lib.check(_lib.load().sgn_semantic_metrics(H, W, Cn, _ptr(s), _ptr(lab), _ptr(m), _ptr(out), _stream()), "sgn_semantic_metrics")
    return out


def metrics_from_confusion(conf: torch.Tensor) -> Dict[str, float]:
    """Pixel accuracy (NaN without a valid pixel) and mean IoU over the classes whose union is > 0 (NaN when none is)."""
    cm = conf.detach().to("cpu", torch.float64)
    total = float(cm.sum())
    tp = torch.diagonal(cm)
    union = cm.sum(0) + cm.sum(1) - tp
    seen = union > 0
    acc = float(tp.sum()) / total if total > 0 else float("nan")
    miou = float((tp[seen] / union[seen]).mean()) if bool(seen.any()) else float("nan")
    return {"semantic_acc": acc, "semantic_miou": miou}


def semantic_metrics(logits: torch.Tensor, labels: torch.Tensor, mask: Optional[torch.Tensor] = None) -> Dict[str, float]:
    """``{"semantic_acc", "semantic_miou"}`` of the semantic map against the labels over the valid pixels (one read-back of the
    [C, C] confusion matrix)."""
    return metrics_from_confusion(semantic_confusion(logits, labels, mask))


def refine_carry(plan, src: torch.Tensor, dst: torch.Tensor, src_moments: Optional[Tuple[torch.Tensor, torch.Tensor]] = None,
                 dst_moments: Optional[Tuple[torch.Tensor, torch.Tensor]] = None) -> None:
    """``sgn_refine_carry``: rebuild the per-row tensor ``src`` [plan.n, width] into ``dst`` [plan.out_rows, width] (and its
    (exp_avg, exp_avg_sq) moments, or None) with ``plan``'s row map -- what ``refine.apply_plan`` does to features_dc."""
    width = int(math.prod(src.shape[1:]))
    for t, rows in ((src, plan.n), (dst, plan.out_rows)):
        assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and t.shape[0] == rows, (tuple(t.shape), rows)
    assert tuple(src.shape[1:]) == tuple(dst.shape[1:])
    pm = [None] * 4
    if src_moments is not None:
        assert dst_moments is not None
        for j, (x, rows) in enumerate(((src_moments[0], plan.n), (src_moments[1], plan.n), (dst_moments[0], plan.out_rows),
                                       (dst_moments[1], plan.out_rows))):
            assert x.dtype == torch.float32 and x.is_contiguous() and x.shape[0] == rows and x.shape[1:] == src.shape[1:]
            pm[j] = _ptr(x)
    totals = (C.c_int32 * 4)(*plan.totals)
    _lib.check(_lib.load().sgn_refine_carry(plan.n, C.byref(plan.cfg), _ptr(plan.flags), _ptr(plan.scan), totals, _ptr(src), _ptr(dst),
                                            width, pm[0], pm[1], pm[2], pm[3], _stream()), "sgn_refine_carry")
