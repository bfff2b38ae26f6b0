"""Float64 brute-force k-nearest neighbours in numpy: the checker of csrc/knn.cu (sgn_knn) and of knn.chamfer_distance.

Same contract as the kernel: for every query row the k nearest rows of ``points``, ascending by distance, a tie going to the
smaller row; without a query set a row is never its own neighbour (an exact duplicate of it is one, at distance 0).  The
distances are float64 from the coordinates as given (pass the fp32 inputs to check an fp32 search)."""
from __future__ import annotations

import numpy as np

CD_UNIT = 1e-4  # street_gaussians_ns/data/utils/geometric_metric.py:5


def knn_ref64(points, k: int, query=None, chunk: int = 512):
    """Returns (dist float64 [M, k], idx int64 [M, k])."""
    P = np.asarray(points, np.float64)
    self_query = query is None
    Q = P if self_query else np.asarray(query, np.float64)
    n, m = P.shape[0], Q.shape[0]
    assert 1 <= k <= n - (1 if self_query else 0)
    dist = np.empty((m, k), np.float64)
    idx = np.empty((m, k), np.int64)
    for c0 in range(0, m, chunk):
        q = Q[c0:c0 + chunk]
        diff = q[:, None, :] - P[None, :, :]
        d2 = (diff * diff).sum(-1)
        if self_query:
            d2[np.arange(q.shape[0]), np.arange(c0, c0 + q.shape[0])] = np.inf
        kth = np.partition(d2, k - 1, axis=1)[:, k - 1]
        for r in range(q.shape[0]):
            cand = np.nonzero(d2[r] <= kth[r])[0]  # ascending rows: the stable sort keeps the smaller row first in a tie
            sel = cand[np.argsort(d2[r, cand], kind="stable")[:k]]
            idx[c0 + r] = sel
            dist[c0 + r] = np.sqrt(d2[r, sel])
    return dist, idx


def chamfer_ref64(pred, gt, chunk: int = 512):
    """``calc_chamfer_distance(pred, gt)`` in float64: (mean nearest distance pred -> gt, gt -> pred), each / CD_UNIT."""
    d1, _ = knn_ref64(gt, 1, query=pred, chunk=chunk)
    d2, _ = knn_ref64(pred, 1, query=gt, chunk=chunk)
    return float(d1.mean()) / CD_UNIT, float(d2.mean()) / CD_UNIT
