"""The GPU k-nearest-neighbour search (csrc/knn.cu through knn.py) against float64 brute force: full at 1 k and 100 k
points, a sample of query rows at 1 M and 2 M; directed clouds; determinism; the chamfer distance."""
import math

import numpy as np
import pytest
import torch

import street_gaussians_ns_b200.synthetic as syn
from oracle.knn_ref64 import chamfer_ref64, knn_ref64
from street_gaussians_ns_b200.knn import chamfer_distance, knn, knn_log_scales

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
KS = (1, 3, 8, 16)


def brute64(points, queries, k, self_rows=None, chunk=256):
    """float64 brute force on the device: (dist [m, k+1], idx [m, k+1]) ordered by (distance, row)."""
    P = points.to(DEV, torch.float64)
    Q = queries.to(DEV, torch.float64)
    ds, ix = [], []
    for c0 in range(0, Q.shape[0], chunk):
        q = Q[c0:c0 + chunk]
        d2 = (q[:, 0:1] - P[:, 0]) ** 2 + (q[:, 1:2] - P[:, 1]) ** 2 + (q[:, 2:3] - P[:, 2]) ** 2
        if self_rows is not None:
            d2[torch.arange(q.shape[0], device=DEV), self_rows[c0:c0 + chunk].to(DEV)] = math.inf
        v, i = torch.topk(d2, k + 1, dim=1, largest=False)
        o = torch.sort(i, dim=1, stable=True).indices  # a tie goes to the smaller row
        v, i = v.gather(1, o), i.gather(1, o)
        o = torch.sort(v, dim=1, stable=True).indices
        ds.append(v.gather(1, o).sqrt())
        ix.append(i.gather(1, o))
    return torch.cat(ds), torch.cat(ix)


def check(dist, idx, rd, ri, k):
    """Distances within 1e-6 relative (+1e-12) of float64; the index set equal wherever the k-th and (k+1)-th neighbours are
    apart by more than 1e-5 relative (fp32 may order a closer pair inside the k the other way)."""
    dist, idx = dist.double(), idx.long()
    rd_k, ri_k = rd[:, :k], ri[:, :k]
    err = (dist - rd_k).abs() - (1e-6 * rd_k + 1e-12)
    assert float(err.max()) <= 0, float(((dist - rd_k).abs() / rd_k.clamp_min(1e-30)).max())
    sep = (rd[:, k] - rd[:, k - 1]) > 1e-5 * rd[:, k]
    same = (idx.sort(dim=1).values == ri_k.sort(dim=1).values).all(1)
    assert bool(same[sep].all()), int((~same & sep).sum())
    assert float(sep.float().mean()) > 0.5


_CLOUDS = {}


def cloud(n):
    if n not in _CLOUDS:
        _CLOUDS[n] = (syn.street_points(n, seed=n % 9973).to(DEV), syn.street_points(max(1000, n // 2), seed=n % 9973 + 1).to(DEV))
    return _CLOUDS[n]


@pytest.mark.parametrize("with_query", [False, True])
@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("n", [1000, 100_000])
def test_full_brute_force(n, k, with_query):
    P, Q = cloud(n)
    if with_query:
        dist, idx = knn(P, k, query=Q)
        rd, ri = brute64(P, Q, k)
    else:
        dist, idx = knn(P, k)
        rd, ri = brute64(P, P, k, self_rows=torch.arange(n))
    assert dist.shape == (Q.shape[0] if with_query else n, k) and idx.dtype == torch.int32
    assert bool((dist[:, 1:] >= dist[:, :-1]).all())
    check(dist, idx, rd, ri, k)


@pytest.mark.parametrize("with_query", [False, True])
@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("n", [1_000_000, 2_000_000])
def test_sampled_brute_force(n, k, with_query):
    P, Q = cloud(n)
    rows = torch.randperm(Q.shape[0] if with_query else n, generator=torch.Generator().manual_seed(k))[:3000]
    if with_query:
        dist, idx = knn(P, k, query=Q)
        rd, ri = brute64(P, Q[rows.to(DEV)], k, chunk=16)
    else:
        dist, idx = knn(P, k)
        rd, ri = brute64(P, P[rows.to(DEV)], k, self_rows=rows, chunk=16)
    check(dist[rows.to(DEV)], idx[rows.to(DEV)], rd, ri, k)


def oracle_check(P, k, query=None):
    dist, idx = knn(torch.as_tensor(P), k, query=None if query is None else torch.as_tensor(query))
    rd, ri = knn_ref64(np.asarray(P, np.float32), k, query=None if query is None else np.asarray(query, np.float32))
    assert np.allclose(dist.cpu().numpy(), rd, rtol=1e-6, atol=1e-12)
    return dist.cpu().numpy(), idx.cpu().numpy(), rd, ri


def test_all_points_identical():
    P = torch.full((3000, 3), 2.5)
    dist, idx, _, ri = oracle_check(P, 16)
    assert (dist == 0).all() and np.array_equal(idx, ri)  # the 16 smallest other rows
    s = knn_log_scales(P)
    assert torch.isneginf(s).all()


@pytest.mark.parametrize("k", KS)
def test_k_plus_one_points(k):
    P = torch.randn(k + 1, 3, generator=torch.Generator().manual_seed(k))
    _, idx, _, ri = oracle_check(P, k)
    assert np.array_equal(idx, ri)


@pytest.mark.parametrize("shape", ["line", "plane"])
def test_degenerate_extent(shape):
    g = torch.Generator().manual_seed(4)
    P = torch.zeros(20000, 3)
    P[:, 0] = torch.rand(20000, generator=g) * 50
    if shape == "plane":
        P[:, 2] = torch.rand(20000, generator=g) * 30
    for k in (3, 16):
        oracle_check(P, k)


def test_cluster_with_far_outliers():
    g = torch.Generator().manual_seed(5)
    P = torch.cat([torch.rand(100_000, 3, generator=g), torch.tensor([[1e5, 0, 0], [0, -1e5, 0], [0, 0, 1e5], [1e5, 1e5, 1.0]])])
    dist, idx = knn(P, 3)
    rd, ri = brute64(P, P, 3, self_rows=torch.arange(P.shape[0]), chunk=512)
    check(dist, idx, rd, ri, 3)
    assert float(dist[-4:].min()) > 1e4


def test_two_far_clusters_one_a_singleton():
    g = torch.Generator().manual_seed(6)
    P = torch.cat([torch.rand(5000, 3, generator=g), torch.tensor([[1e4, 1e4, 1e4]])])
    dist, idx = knn(P, 8)
    rd, ri = brute64(P, P, 8, self_rows=torch.arange(P.shape[0]))
    check(dist, idx, rd, ri, 8)  # the singleton's neighbours lie within fp32 rounding of each other: only distances bind there
    assert float(dist[-1, 0]) > 1.7e4 and float(dist[:-1, -1].max()) < 1.0
    oracle_check(P, 4, query=torch.tensor([[1e4, 1e4, 1e4 + 1.0], [0.5, 0.5, 0.5]]))


def test_duplicates_mixed_with_distinct_points():
    g = torch.Generator().manual_seed(7)
    base = torch.rand(4000, 3, generator=g) * 10
    P = torch.cat([base, base[:500], base[:100], base[:10]])
    P = P[torch.randperm(P.shape[0], generator=g)]
    for k in KS:
        dist, idx, rd, ri = oracle_check(P, k)
        sep = rd[:, k - 1] < 1e-30
        assert np.array_equal(idx[sep], ri[sep])  # all-zero rows: the k smallest duplicate rows, in order


def test_errors():
    P = torch.rand(50, 3)
    for k in (0, 17):
        with pytest.raises(ValueError):
            knn(P, k)
    with pytest.raises(ValueError):
        knn(P[:3], 3)
    with pytest.raises(ValueError):
        knn(P[:3], 4, query=P)
    bad = P.clone()
    bad[10, 2] = float("nan")
    with pytest.raises(ValueError):
        knn(bad, 3)
    with pytest.raises(ValueError):
        knn(P, 3, query=bad)


def test_deterministic_bytes():
    P, Q = cloud(1_000_000)
    a, b = knn(P, 8), knn(P, 8)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    s1, s2 = knn_log_scales(P), knn_log_scales(P)
    assert torch.equal(s1, s2)
    c, d = knn(P, 3, query=Q), knn(P, 3, query=Q)
    assert torch.equal(c[0], d[0]) and torch.equal(c[1], d[1])


def test_log_scales_epilogue_matches_the_distances():
    P, _ = cloud(100_000)
    dist, _ = knn(P, 3)
    s = knn_log_scales(P)
    ref = torch.log(dist.mean(dim=-1, keepdim=True)).repeat(1, 3)
    assert s.shape == (P.shape[0], 3) and float((s - ref).abs().max()) <= 1e-6


def test_chamfer_distance():
    g = torch.Generator().manual_seed(8)
    pred = torch.rand(6000, 3, generator=g) * 5
    gt = torch.rand(4000, 3, generator=g) * 5 + 0.1
    d1, d2 = chamfer_distance(pred, gt)
    r1, r2 = chamfer_ref64(pred.numpy(), gt.numpy())
    assert d1 == pytest.approx(r1, rel=1e-6) and d2 == pytest.approx(r2, rel=1e-6)
    assert chamfer_distance(pred, gt) == (d1, d2)
