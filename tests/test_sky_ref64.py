"""CPU checks of the sky cube map specification (oracle/sky_ref64.py) and of the host side of the feature:

  * the direction formula against the reference's own EnvLight, executed on the CPU (tests/golden/reference_sky.npz);
  * the derived edge / corner wrap against the geometric rule at R = 1, 2, 3, 16;
  * continuity of a smooth function across the seams, an adjoint identity and central differences for the gradient;
  * the exact recovery of c2w[:3,:3] from the camera's viewmat;
  * argument validation of the four C entry points (no launch);
  * TrainStep handing the optimizer's further tensors (the sky) their gradient, and refusing it in data-parallel runs."""
import ctypes
import os
import types

import numpy as np
import pytest
import torch

from oracle import sky_ref64 as ref

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "reference_sky.npz")


def test_directions_match_the_reference_envlight():
    g = np.load(GOLDEN)
    assert int(g["num_cases"]) >= 6 and any(bool(g[f"train_{k}"]) for k in range(int(g["num_cases"])))
    for k in range(int(g["num_cases"])):
        W, H = (int(x) for x in g[f"size_{k}"])
        fx, fy, cx, cy = (float(x) for x in g[f"intr_{k}"])
        train = bool(g[f"train_{k}"])
        ju, jv = (g[f"ju_{k}"], g[f"jv_{k}"]) if train else (None, None)
        mine = ref.directions(g[f"c2w_{k}"][:, :3], fx, fy, cx, cy, W, H, ju, jv)
        got = g[f"l_{k}"]
        assert got.shape == (H, W, 3)
        np.testing.assert_allclose(mine, got, rtol=0, atol=2e-6)  # the reference's fp32 arithmetic against float64


def _edge_texels(R):
    F, I, J = [], [], []
    for f in range(6):
        for k in range(R):
            for i, j in ((-1, k), (R, k), (k, -1), (k, R)):
                F.append(f)
                I.append(i)
                J.append(j)
    return np.array(F), np.array(I), np.array(J)


@pytest.mark.parametrize("R", [1, 2, 3, 16])
def test_derived_wrap_is_the_nearest_texel_centre_on_the_adjacent_face(R):
    F, I, J = _edge_texels(R)
    got = ref.wrap(F, I, J, R)
    assert np.array_equal(got, ref.wrap_geometric(F, I, J, R))
    g = got // (R * R)
    assert np.all(g != F) and np.all(g // 2 != F // 2)  # always a neighbour, never the opposite face
    # the texels reached are exactly the border ring of every face
    assert np.array_equal(np.unique(got), np.flatnonzero(_ring(R)))


def _ring(R):
    m = np.zeros((6, R, R), bool)
    m[:, 0, :] = m[:, -1, :] = m[:, :, 0] = m[:, :, -1] = True
    return m.reshape(-1)


@pytest.mark.parametrize("R", [1, 2, 3, 16])
def test_corner_lookups_miss_exactly_one_tap(R):
    # the 8 cube corners, approached from inside each of the three faces that meet there
    rng = np.random.default_rng(R)
    for sx in (-1, 1):
        for sy in (-1, 1):
            for sz in (-1, 1):
                for bump in range(3):
                    d = np.array([sx, sy, sz], np.float64)
                    d[bump] *= 1 + 1e-3 * rng.random()
                    lk = ref.lookup(d[None], R)
                    idx = ref.taps(lk, R)[0]
                    assert (idx < 0).sum() == 1, (R, d, idx)
                    assert len(set(idx[idx >= 0] // (R * R))) == 3  # the three faces meeting at the corner


def _smooth_tex(R, a=np.array([0.3, -0.7, 0.5]), b=0.2):
    """Texel value = a . (direction of the texel centre, normalised) + b, per channel scaled."""
    f = np.arange(6)[:, None, None]
    j, i = np.meshgrid(np.arange(R), np.arange(R), indexing="ij")
    s, t = (i + 0.5) / R, (j + 0.5) / R
    B = ref.BASIS[f[:, 0, 0]].astype(np.float64)
    d = B[:, None, None, 0] + (2 * s - 1)[None, ..., None] * B[:, None, None, 1] + (2 * t - 1)[None, ..., None] * B[:, None, None, 2]
    d /= np.linalg.norm(d, axis=-1, keepdims=True)
    v = d @ a + b
    return np.stack([v, 2 * v, -v], -1)


@pytest.mark.parametrize("R", [4, 16])
def test_sampling_is_continuous_across_seams(R):
    tex = _smooth_tex(R)
    # great circles through edges and corners, stepped finely
    th = np.linspace(0, 2 * np.pi, 20001)
    for axis_a, axis_b in ((np.array([1.0, 0, 0]), np.array([0, 1.0, 0])), (np.array([1.0, 1, 0]) / np.sqrt(2), np.array([0, 0, 1.0])),
                           (np.array([1.0, 1, 1]) / np.sqrt(3), np.array([1.0, -1, 0]) / np.sqrt(2))):
        l = np.cos(th)[:, None] * axis_a + np.sin(th)[:, None] * axis_b
        out = ref.sample(tex, l, R)
        step = np.abs(np.diff(out, axis=0)).max()
        # a texel spans at least 2 / R of tangent, about 1 / R radian at the worst; a jump would be O(1 / R)
        assert step < 20.0 * (2 * np.pi / 20000) * R / 4 + 1e-9, step


def test_adjoint_and_central_differences():
    R = 3
    rng = np.random.default_rng(5)
    l = rng.normal(size=(400, 3))
    l[:8] = [[1, 1, 1], [-1, 1, 1], [1, -1, 0.5], [0, 0, 0], [np.nan, 1, 0], [1, 1, 0], [1e30, 1, 1], [1e-30, 0, 0]]
    T = rng.normal(size=(6, R, R, 3))
    y = rng.normal(size=(400, 3))
    g = ref.grad(T.shape, l, y, R)
    assert np.isclose((ref.sample(T, l, R) * y).sum(), (T * g).sum(), rtol=1e-12, atol=1e-12)
    assert np.all(ref.sample(T, l[3:5], R) == 0)  # zero and NaN directions sample 0
    for e in rng.choice(T.size, 12, replace=False):
        d = np.zeros(T.size)
        d[e] = 1e-3
        d = d.reshape(T.shape)
        fd = ((ref.sample(T + d, l, R) - ref.sample(T - d, l, R)) * y).sum() / 2e-3
        assert np.isclose(fd, g.reshape(-1)[e], rtol=1e-9, atol=1e-9)


def test_c2w_is_recovered_exactly_from_the_viewmat():
    from street_gaussians_ns_b200.scene import Camera
    rng = np.random.default_rng(9)
    for _ in range(50):
        q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
        c2w = np.concatenate([q, rng.normal(size=(3, 1)) * 10], 1).astype(np.float32)
        cam = Camera(c2w=c2w, fx=100.0, fy=100.0, cx=10.0, cy=10.0, width=20, height=20)
        assert np.array_equal(ref.c2w_from_viewmat(cam.viewmat()), cam.c2w[:3, :3])


@pytest.fixture(scope="module")
def lib():
    import street_gaussians_ns_b200.build as b
    from street_gaussians_ns_b200 import _lib
    b.build()
    return _lib.load(), _lib


def test_argument_validation_without_gpu(lib):
    L, mod = lib
    p = ctypes.c_void_p(256)
    cam = mod.CameraStruct()
    cam.width, cam.height, cam.fx, cam.fy = 64, 48, 50.0, 50.0
    launches = L.sgn_launch_count()

    def fwd(c=cam, ju=None, jv=None, tex=p, R=4, sky=p):
        return L.sgn_sky_fwd(ctypes.byref(c) if c is not None else None, ju, jv, tex, R, sky, None, None)

    def bwd(c=cam, ju=None, jv=None, R=4, v=p, vt=p):
        return L.sgn_sky_bwd(ctypes.byref(c) if c is not None else None, ju, jv, R, v, vt, None)

    for R in (0, -3):
        assert fwd(R=R) == -1 and b"resolution" in L.sgn_last_error()
        assert bwd(R=R) == -1
        assert L.sgn_cube_texture_fwd(4, p, p, R, p, None) == -1
        assert L.sgn_cube_texture_bwd(4, p, R, p, p, None) == -1
    assert fwd(R=20000) == -1 and b"32-bit" in L.sgn_last_error()
    assert fwd(c=None) == -1 and bwd(c=None) == -1
    assert fwd(tex=None) == -1 and fwd(sky=None) == -1
    assert bwd(v=None) == -1 and bwd(vt=None) == -1
    assert fwd(ju=p) == -1 and b"jitter" in L.sgn_last_error()
    assert bwd(jv=p) == -1 and b"jitter" in L.sgn_last_error()
    big = mod.CameraStruct()
    big.width, big.height = 40000, 40000
    assert fwd(c=big) == -1 and b"32-bit" in L.sgn_last_error()
    empty = mod.CameraStruct()
    assert fwd(c=empty) == -1
    assert L.sgn_cube_texture_fwd(-1, p, p, 4, p, None) == -1
    assert L.sgn_cube_texture_fwd(1 << 30, p, p, 4, p, None) == -1 and b"32-bit" in L.sgn_last_error()
    assert L.sgn_cube_texture_fwd(4, None, p, 4, p, None) == -1
    assert L.sgn_cube_texture_bwd(4, p, 4, None, p, None) == -1
    assert L.sgn_cube_texture_fwd(0, p, p, 4, p, None) == 0 and L.sgn_cube_texture_bwd(0, p, 4, p, p, None) == 0
    assert L.sgn_launch_count() == launches  # nothing was launched


class _Sky(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.base = torch.nn.Parameter(torch.full((6, 2, 2, 3), 0.5))


def _step_with_sky(monkeypatch, world):
    from street_gaussians_ns_b200.model import _FullArenaSink
    from street_gaussians_ns_b200.optim import FusedAdam
    from street_gaussians_ns_b200.training import TrainStep
    from tests.test_refine import build_model
    model, _ = build_model()
    model.env_map = _Sky()
    opt = FusedAdam(model.optimizer_params(), chunk_elems=4096, extra={"sky": (model.env_map.base, 0.005)})
    step_fn = TrainStep(model, opt, refine_every=0)
    calls = []
    monkeypatch.setattr(model, "get_outputs", lambda camera: {"sky": model.env_map.base.sum() * 2})
    monkeypatch.setattr(model, "get_loss_dict", lambda out, batch: {"main_loss": out["sky"]})
    monkeypatch.setattr(model, "after_train", lambda step: None)
    model._holder = types.SimpleNamespace(grad_arena=torch.zeros(8))
    monkeypatch.setattr(opt, "step", lambda arena, **kw: calls.append(kw))
    if world > 1:
        model._grad_sink = _FullArenaSink()
        monkeypatch.setattr(step_fn, "world_size", lambda: world)
        monkeypatch.setattr(step_fn, "_ensure_exchange", lambda: None)
    return model, step_fn, calls


def test_train_step_steps_the_sky_with_its_gradient(monkeypatch):
    model, step_fn, calls = _step_with_sky(monkeypatch, 1)
    model.env_map.base.grad = torch.ones_like(model.env_map.base)  # stale: zeroed before the step
    step_fn(700, camera=None, batch={})
    assert len(calls) == 1
    g = calls[0]["extra_grads"]["sky"]
    assert g is model.env_map.base.grad and torch.equal(g, torch.full_like(g, 2.0))


def test_train_step_without_a_sky_gradient_passes_none(monkeypatch):
    model, step_fn, calls = _step_with_sky(monkeypatch, 1)
    monkeypatch.setattr(model, "get_outputs", lambda camera: {"sky": model.all_models["background"].gauss_params["means"].sum()})
    step_fn(700, camera=None, batch={})
    assert calls[0]["extra_grads"] is None


def test_data_parallel_refuses_a_sky_before_rendering(monkeypatch):
    model, step_fn, calls = _step_with_sky(monkeypatch, 2)
    rendered = []
    monkeypatch.setattr(model, "get_outputs", lambda camera: rendered.append(camera))
    monkeypatch.setattr(step_fn, "_ensure_exchange", lambda: rendered.append("exchange"))
    with pytest.raises(NotImplementedError, match="sky"):
        step_fn(700, camera=None, batch={}, all_cameras=[None, None])
    assert calls == [] and rendered == []  # nothing rendered, no exchange set up or started
