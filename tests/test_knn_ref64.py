"""CPU checks of the float64 brute-force kNN oracle (oracle/knn_ref64.py) that the GPU search is tested against."""
import numpy as np
import pytest

from oracle.knn_ref64 import CD_UNIT, chamfer_ref64, knn_ref64


def test_matches_a_sorted_distance_matrix():
    rng = np.random.RandomState(0)
    P = rng.randn(300, 3)
    d2 = ((P[:, None] - P[None]) ** 2).sum(-1)
    np.fill_diagonal(d2, np.inf)
    for k in (1, 3, 8, 16):
        dist, idx = knn_ref64(P, k, chunk=64)
        ref = np.argsort(d2, axis=1, kind="stable")[:, :k]
        assert np.array_equal(idx, ref)
        assert np.allclose(dist, np.sqrt(np.take_along_axis(d2, ref, 1)), rtol=0, atol=0)
        assert (np.diff(dist, axis=1) >= 0).all()


def test_self_exclusion_duplicates_and_ties():
    P = np.array([[0, 0, 0], [1, 0, 0], [0, 0, 0], [-1, 0, 0], [0, 2, 0]], np.float64)
    dist, idx = knn_ref64(P, 3)
    assert idx[0].tolist() == [2, 1, 3]  # the duplicate at 0, then the tie at 1 in row order
    assert idx[2].tolist() == [0, 1, 3]
    assert dist[0].tolist() == [0.0, 1.0, 1.0]
    assert 0 not in idx[0] and 2 not in idx[2]


def test_query_set_and_chamfer():
    rng = np.random.RandomState(1)
    P, Q = rng.rand(400, 3), rng.rand(250, 3) + 0.2
    dist, idx = knn_ref64(P, 4, query=Q)
    d2 = ((Q[:, None] - P[None]) ** 2).sum(-1)
    assert np.array_equal(idx, np.argsort(d2, axis=1, kind="stable")[:, :4])
    c1, c2 = chamfer_ref64(Q, P)
    assert c1 == pytest.approx(np.sqrt(d2.min(1)).mean() / CD_UNIT, rel=1e-12)
    assert c2 == pytest.approx(np.sqrt(d2.min(0)).mean() / CD_UNIT, rel=1e-12)


def test_matches_sklearn_kneighbors():
    sk = pytest.importorskip("sklearn.neighbors")
    rng = np.random.RandomState(2)
    P = (rng.rand(2000, 3) * [80, 20, 88]).astype(np.float32)
    d_sk, _ = sk.NearestNeighbors(n_neighbors=4).fit(P).kneighbors(P)
    dist, _ = knn_ref64(P, 3)
    assert np.allclose(dist, d_sk[:, 1:], rtol=1e-12, atol=1e-12)
