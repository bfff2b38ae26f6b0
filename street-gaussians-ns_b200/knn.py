"""Exact k-nearest-neighbour search on the GPU (csrc/knn.cu) and the lidar chamfer distance built on it.

``knn`` replaces the CPU KD-tree of ``SplatfactoModel.k_nearest_sklearn`` (street_gaussians_ns/sgn_splatfacto.py:439-457) that
``populate_modules`` runs over all seed points; ``chamfer_distance`` is ``calc_chamfer_distance``
(data/utils/geometric_metric.py:59-69, open3d on the CPU).
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Tuple

import torch

from . import _lib

MAX_K = 16
CD_UNIT = 1e-4  # geometric_metric.py:5


def _cloud(x: torch.Tensor, what: str, device) -> torch.Tensor:
    x = torch.as_tensor(x)
    if x.dim() != 2 or x.shape[1] != 3:
        raise ValueError(f"{what} must have shape [N, 3], got {tuple(x.shape)}")
    x = x.to(device=device, dtype=torch.float32).contiguous()
    if x.shape[0] and not bool(torch.isfinite(x).all()):
        raise ValueError(f"{what} has non-finite coordinates")
    return x


def _run(points: torch.Tensor, k: int, query: Optional[torch.Tensor], want_pairs: bool, want_scales: bool):
    if not 1 <= k <= MAX_K:
        raise ValueError(f"k = {k} outside 1..{MAX_K}")
    device = points.device if points.is_cuda else torch.device("cuda", torch.cuda.current_device())
    pts = _cloud(points, "points", device)
    n = pts.shape[0]
    if query is None:
        if n < k + 1:
            raise ValueError(f"{n} points cannot give {k} neighbours other than the point itself (need at least {k + 1})")
        q, m = None, n
    else:
        q = _cloud(query, "query", device)
        m = q.shape[0]
        if n < k:
            raise ValueError(f"{n} points cannot give {k} neighbours")
    L = _lib.load()
    scratch = torch.empty(L.sgn_knn_scratch_bytes(n, m if q is not None else 0), dtype=torch.uint8, device=device)
    dist = torch.empty(m, k, dtype=torch.float32, device=device) if want_pairs else None
    idx = torch.empty(m, k, dtype=torch.int32, device=device) if want_pairs else None
    scales = torch.empty(m, 3, dtype=torch.float32, device=device) if want_scales else None

    def ptr(t):
        return C.c_void_p(t.data_ptr()) if t is not None and t.numel() else None

    with torch.cuda.device(device):
        stream = torch.cuda.current_stream(device).cuda_stream
        _lib.check(L.sgn_knn(ptr(pts), n, ptr(q), m, k, ptr(dist), ptr(idx), ptr(scales), ptr(scratch), scratch.numel(),
                             C.c_void_p(stream)), "sgn_knn")
    return dist, idx, scales


def knn(points: torch.Tensor, k: int, query: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """The ``k`` nearest rows of ``points`` [N, 3] for every row of ``query`` [M, 3] (default: of ``points`` itself).

    Returns ``(dist, idx)``: float32 [M, k] Euclidean distances, ascending, and their int32 row indices into ``points``.  The
    search is exact (fp32 distances from the fp32 inputs); a tie goes to the smaller row, so the result is deterministic.
    Without ``query`` a point is never its own neighbour, while an exact duplicate of it is one at distance 0 -- sklearn's
    ``NearestNeighbors(k + 1).kneighbors(points)`` with its first column dropped.  1 <= k <= 16; host tensors are moved to the
    current CUDA device; non-finite coordinates raise ``ValueError``.
    """
    dist, idx, _ = _run(points, int(k), query, True, False)
    return dist, idx


def knn_log_scales(points: torch.Tensor, k: int = 3) -> torch.Tensor:
    """``log(mean distance to the k nearest other points)`` repeated over 3 columns, float32 [N, 3] on the device: the
    initial scales of ``populate_modules`` (sgn_splatfacto.py:260-264), written by the search kernel itself.  A point with k
    or more exact duplicates gets -inf, as in the reference."""
    return _run(points, int(k), None, False, True)[2]


def chamfer_distance(pred: torch.Tensor, gt: torch.Tensor) -> Tuple[float, float]:
    """``calc_chamfer_distance(pred, gt)``: the mean nearest distance pred -> gt and gt -> pred, each divided by CD_UNIT.

    The means are float64 sums of the per-point fp32 distances on the device (a fixed reduction order, so repeated calls agree
    to the bit)."""
    d1, _ = knn(gt, 1, query=pred)
    d2, _ = knn(pred, 1, query=gt)
    if d1.numel() == 0 or d2.numel() == 0:
        raise ValueError("chamfer_distance of an empty cloud")
    return float(d1.double().mean()) / CD_UNIT, float(d2.double().mean()) / CD_UNIT
