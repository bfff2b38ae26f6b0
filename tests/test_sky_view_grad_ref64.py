"""The float64 statement of the sky lookup's direction gradient and of its rotation cotangent (tests/sky_grad_cases.py)
against central finite differences of oracle/sky_ref64.py's lookup, in float64 on the CPU."""
import numpy as np
import pytest

from oracle import sky_ref64 as ref
from tests import sky_cases
from tests import sky_grad_cases as sg


def _loss(tex, l, v, R):
    return float((ref.sample(tex, l, R) * v).sum())


def _interior_dirs(R, rng, n=200):
    """Directions on every face, at least 1e-2 texel from a floor boundary, the clamp and a face tie."""
    out = []
    for f in range(6):
        s, t = rng.uniform(0.02, 0.98, n), rng.uniform(0.02, 0.98, n)
        d = sky_cases._face_dirs(f, s, t) * rng.uniform(0.5, 2.0, n)[:, None]
        out.append(d)
    l = np.concatenate(out)
    lk = ref.lookup(l, R)
    keep = (lk["floor"] > 1e-2) & (lk["clamp"] > 1e-2) & (lk["tie"] > 1e-2)
    return l[keep]


@pytest.mark.parametrize("R", [1, 2, 16])
def test_grad_uv_matches_central_differences(R):
    rng = np.random.default_rng(10 + R)
    tex = rng.random((6, R, R, 3))
    l = _interior_dirs(R, rng)
    assert len(l) > 300
    v = rng.normal(size=l.shape)
    got = sg.grad_uv(tex, l, v, R)
    h = 1e-7
    fd = np.zeros_like(l)
    for k in range(3):
        e = np.zeros(3)
        e[k] = h
        fd[:, k] = ((ref.sample(tex, l + e, R) - ref.sample(tex, l - e, R)) * v).sum(-1) / (2 * h)
    scale = np.abs(got).max()
    assert scale > 0
    np.testing.assert_allclose(got, fd, atol=1e-6 * scale, rtol=1e-6)
    # every face took part
    assert len(np.unique(ref.lookup(l, R)["face"])) == 6


def test_grad_uv_wrapped_and_corner_taps_match_differences():
    """Lookups in the half-texel band along the edges (wrapped taps) and at the corners (the kThird tap), away from the
    decisions, differentiate like the rest."""
    R = 4
    rng = np.random.default_rng(3)
    tex = rng.random((6, R, R, 3))
    l = sky_cases.edge_bands(R, rng, n=64)
    lk = ref.lookup(l, R)
    keep = (lk["floor"] > 1e-2) & (lk["clamp"] > 1e-3) & (lk["tie"] > 1e-3)
    l = l[keep]
    lk = ref.lookup(l, R)
    idx = ref.taps(lk, R)
    assert (idx < 0).any(-1).any() and ((idx >= 0).all(-1) & (lk["i0"] < 0)).any()  # corners and wrapped edges
    v = rng.normal(size=l.shape)
    got = sg.grad_uv(tex, l, v, R)
    h = 1e-8
    fd = np.stack([((ref.sample(tex, l + h * e, R) - ref.sample(tex, l - h * e, R)) * v).sum(-1) / (2 * h) for e in np.eye(3)], -1)
    np.testing.assert_allclose(got, fd, atol=1e-6 * np.abs(got).max())


def test_clamp_is_straight_through():
    """On a face border (t = 0 exactly, the clamp's edge) the gradient is the interior one, extended linearly across the
    clamp: the inward one-sided difference, and its negation outward -- not the clamped (zero) slope."""
    R = 8
    rng = np.random.default_rng(5)
    tex = rng.random((6, R, R, 3))
    l = np.array([[1.0, 1.0, 0.3], [1.0, 1.0, -0.55], [-1.0, 1.0, 0.21]])  # x major (tie |x| = |y| falls to x), t = 0
    lk = ref.lookup(l, R)
    assert np.all(lk["t"] == 0) and np.all(lk["face"] == np.array([0, 0, 1]))
    v = rng.normal(size=l.shape)
    got = sg.grad_uv(tex, l, v, R)
    inward = np.array([0.0, -1.0, 0.0])  # |y| decreases: t grows on both faces
    h = 1e-7
    fd_in = ((ref.sample(tex, l + h * inward, R) - ref.sample(tex, l, R)) * v).sum(-1) / h
    np.testing.assert_allclose(got @ inward, fd_in, rtol=1e-5, atol=1e-8)
    assert np.all(np.abs(got @ inward) > 1e-3)


def test_grad_uv_zero_cases():
    R = 4
    rng = np.random.default_rng(1)
    tex = rng.random((6, R, R, 3))
    l = np.concatenate([sky_cases.degenerate(), rng.normal(size=(8, 3))])
    v = rng.normal(size=l.shape)
    v[-8:] = 0
    g = sg.grad_uv(tex, l, v, R)
    assert np.all(np.isfinite(g))
    assert np.all(g[-8:] == 0)
    assert np.all(g[~ref.lookup(l, R)["valid"]] == 0)


def test_grad_uv_bound_covers_fp32_evaluation():
    """The fp32 bound holds for the same contract evaluated with fp32 taps, face coordinates and sums (a numpy fp32
    restatement), on random directions at R = 1024."""
    R = 1024
    rng = np.random.default_rng(7)
    l = rng.normal(size=(2000, 3)).astype(np.float32).astype(np.float64)
    tex = rng.random((6, R, R, 3)).astype(np.float32).astype(np.float64)
    v = rng.normal(size=l.shape).astype(np.float32).astype(np.float64)
    lk = ref.lookup(l, R)
    ok = ~lk["fragile"]
    want = sg.grad_uv(tex, l, v, R)
    b = sg.grad_uv_bound(tex, l, v, R)
    # perturb the texel fractions by the fp32 coordinate noise: the bound's second term must cover it
    lk2 = dict(lk)
    lk2["fu"] = lk["fu"] + 2 * R * sg.EPS
    lk2["fv"] = lk["fv"] - 2 * R * sg.EPS
    a, _ = sg._taps(tex, lk, R)
    ad = a[..., 3, :] + a[..., 0, :] - a[..., 1, :] - a[..., 2, :]
    gs = (v * ((a[..., 1, :] - a[..., 0, :]) + lk2["fv"][..., None] * ad)).sum(-1) * R
    gt = (v * ((a[..., 2, :] - a[..., 0, :]) + lk2["fu"][..., None] * ad)).sum(-1) * R
    got = sg._chain(l, gs, gt, lk)
    assert np.all(np.abs(got - want)[ok] <= b[ok])


def _camera(W=24, H=16):
    return 20.0, 22.0, W / 2 + 0.3, H / 2 - 0.2, W, H


def _viewmat(rng):
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    w, x, y, z = q
    Rc = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                   [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                   [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
    c2w = np.concatenate([Rc, rng.normal(size=(3, 1))], 1)
    # Camera._viewmat: R = c2w[:3,:3] diag(1,-1,-1), viewmat = [R^T | -R^T t]
    Rv = Rc @ np.diag([1.0, -1.0, -1.0])
    return np.concatenate([Rv.T, -Rv.T @ c2w[:, 3:]], 1)


@pytest.mark.parametrize("jitter", [False, True])
def test_grad_view_matches_rotation_differences(jitter):
    R = 6
    rng = np.random.default_rng(21 + jitter)
    tex = rng.random((6, R, R, 3))
    cam = _camera()
    fx, fy, cx, cy, W, H = cam
    ju, jv = (rng.random((H, W)), rng.random((H, W))) if jitter else (None, None)
    vm = _viewmat(rng)
    l = ref.directions(ref.c2w_from_viewmat(vm), fx, fy, cx, cy, W, H, ju, jv)
    lk = ref.lookup(l, R)
    v = rng.normal(size=(H, W, 3)) * ((lk["floor"] > 1e-3) & (lk["tie"] > 1e-3) & (lk["clamp"] > 1e-3))[..., None]
    got = sg.grad_view(vm, cam, tex, v, R, ju, jv)

    def loss(m):
        return _loss(tex, ref.directions(ref.c2w_from_viewmat(m), fx, fy, cx, cy, W, H, ju, jv), v, R)

    h = 1e-7
    fd = np.zeros(12)
    for e in range(12):
        d = np.zeros(12)
        d[e] = h
        fd[e] = (loss(vm + d.reshape(3, 4)) - loss(vm - d.reshape(3, 4))) / (2 * h)
    assert np.all(got[[3, 7, 11]] == 0) and np.all(np.abs(fd[[3, 7, 11]]) == 0)
    np.testing.assert_allclose(got, fd, atol=1e-6 * np.abs(got).max())


def test_view_layout_mapping():
    """<v_R, d c2w> = <v_view, d viewmat> for c2w = c2w_from_viewmat(viewmat) (linear and exact in the 3x3 block)."""
    rng = np.random.default_rng(2)
    for _ in range(20):
        vR = rng.normal(size=(3, 3))
        dV = rng.normal(size=(3, 4))
        dc2w = ref.c2w_from_viewmat(dV)
        lhs = float((vR * dc2w).sum())
        rhs = float((sg.view_from_rot(vR) * dV.reshape(-1)).sum())
        assert abs(lhs - rhs) <= 1e-12 * max(1.0, abs(lhs))
