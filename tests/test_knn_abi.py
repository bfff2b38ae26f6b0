"""CPU checks of sgn_knn's host-side argument validation (no device work is started for a refused call) and of knn.py's
input checks that come before any device work."""
import ctypes

import pytest
import torch


@pytest.fixture(scope="module")
def L():
    import street_gaussians_ns_b200.build as b
    from street_gaussians_ns_b200 import _lib
    b.build()
    return _lib.load()


def call(L, n=100, k=3, points=16, query=None, m=0, dist=16, idx=16, scales=None, scratch=16, nbytes=1 << 30):
    p = lambda v: ctypes.c_void_p(v) if v else None  # noqa: E731
    return L.sgn_knn(p(points), n, p(query), m, k, p(dist), p(idx), p(scales), p(scratch), nbytes, None)


@pytest.mark.parametrize("kw, msg", [
    (dict(k=0), b"k = 0"), (dict(k=17), b"k = 17"),
    (dict(n=3, k=3), b"cannot give"), (dict(n=2, k=3, query=16, m=5), b"cannot give"),
    (dict(points=0), b"null"), (dict(scratch=0), b"null"), (dict(dist=0, idx=0), b"no output"),
])
def test_invalid_arguments_are_refused(L, kw, msg):
    assert call(L, **kw) == -1
    assert msg in L.sgn_last_error()


def test_scratch_size_is_checked(L):
    need = L.sgn_knn_scratch_bytes(100, 0)
    assert need > 0 and L.sgn_knn_scratch_bytes(100, 1000) > need
    assert call(L, nbytes=need - 1) == -3


def test_python_surface_rejects_bad_input_before_the_device():
    from street_gaussians_ns_b200 import knn
    with pytest.raises(ValueError, match="outside"):
        knn._run(torch.zeros(10, 3), 0, None, True, False)
    with pytest.raises(ValueError, match="outside"):
        knn._run(torch.zeros(10, 3), 17, None, True, False)
    with pytest.raises(ValueError, match=r"\[N, 3\]"):
        knn._cloud(torch.zeros(10, 2), "points", "cpu")
    bad = torch.zeros(10, 3)
    bad[4, 1] = float("nan")
    with pytest.raises(ValueError, match="non-finite"):
        knn._cloud(bad, "points", "cpu")
