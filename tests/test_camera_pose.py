"""The camera pose correction's float64 restatement (tests/camera_cases.py) and the module's host side, without a GPU:
the exponential map on both sides of its clamp, finite differences against autograd, the view of a zero correction
against Camera.viewmat(), the regulariser and metrics, and the argument checks that run before any launch."""
import numpy as np
import pytest
import torch

from street_gaussians_ns_b200 import _lib
from street_gaussians_ns_b200.camera_pose import CameraPoseOptimizer
from street_gaussians_ns_b200.scene import Camera
from tests import camera_cases as cc

F64 = torch.float64


def _rodrigues(axis, angle):
    k = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(angle) * K + (1 - np.cos(angle)) * K @ K


def test_zero_tangent_is_the_identity_and_translation_passes_through():
    A = cc.exp_map_so3xr3(torch.zeros(6, dtype=F64))
    assert torch.equal(A, torch.cat([torch.eye(3, dtype=F64), torch.zeros(3, 1, dtype=F64)], 1))
    A = cc.exp_map_so3xr3(torch.tensor([0.3, -0.2, 0.05, 0, 0, 0], dtype=F64))
    assert torch.equal(A[:, :3], torch.eye(3, dtype=F64)) and torch.equal(A[:, 3], torch.tensor([0.3, -0.2, 0.05], dtype=F64))


def test_rotation_about_z_matches_rodrigues_above_the_clamp():
    for angle in (0.02, 0.3, 1.2, -2.5):
        A = cc.exp_map_so3xr3(torch.tensor([0, 0, 0, 0, 0, angle], dtype=F64))
        assert np.abs(A[:, :3].numpy() - _rodrigues([0, 0, 1], angle)).max() <= 1e-12


def test_below_the_clamp_the_factors_are_constants():
    w = torch.tensor([0.002, -0.004, 0.003], dtype=F64)  # |w| = 5.4e-3 < 0.01 rad
    A = cc.exp_map_so3xr3(torch.cat([torch.zeros(3, dtype=F64), w]))
    th = 0.01
    K = cc.skew(w)
    want = torch.eye(3, dtype=F64) + np.sin(th) / th * K + (1 - np.cos(th)) / th ** 2 * (K @ K)
    assert torch.allclose(A[:, :3], want, rtol=0, atol=1e-15)


@pytest.mark.parametrize("x", [[0.1, -0.2, 0.3, 0.2, -0.5, 0.4], [0.01, 0.02, -0.03, 0.003, -0.002, 0.004]])
def test_finite_differences_agree_with_autograd(x):
    c2w = torch.tensor(np.array([[0.8, -0.6, 0.0, 1.0], [0.6, 0.8, 0.0, -2.0], [0.0, 0.0, 1.0, 0.5]]), dtype=F64)
    x = torch.tensor(x, dtype=F64, requires_grad=True)
    g = torch.randn(15, generator=torch.Generator().manual_seed(0), dtype=F64)
    (grad,) = torch.autograd.grad((cc.view_of(c2w, x) * g).sum(), x)
    h = 1e-6
    fd = []
    for k in range(6):
        e = torch.zeros(6, dtype=F64)
        e[k] = h
        with torch.no_grad():
            fd.append(float(((cc.view_of(c2w, x + e) - cc.view_of(c2w, x - e)) * g).sum()) / (2 * h))
    assert np.allclose(grad.numpy(), fd, rtol=1e-6, atol=1e-8)


def test_zero_adjustment_gives_the_cameras_viewmat():
    c2w = np.array([[0.36, 0.48, -0.8, 3.0], [-0.8, 0.6, 0.0, -1.0], [0.48, 0.64, 0.6, 2.0]])
    cam = Camera(c2w, 500.0, 500.0, 320.0, 240.0, 640, 480)
    v = cc.view_of(cam.c2w.astype(np.float64), torch.zeros(6, dtype=F64))
    assert np.abs(v[:12].numpy().reshape(3, 4) - cam.viewmat()).max() <= 1e-6
    assert np.abs(v[12:].numpy() - cam.cam_pos()).max() == 0


def test_regularizer_and_metrics_values_and_gradients():
    x = torch.tensor([[0.3, 0.4, 0.0, 0.0, 0.0, 0.2], [0.0, 0.0, 0.0, 0.0, 0.0, 0.0], [1.0, 0.0, 0.0, 0.0, 0.6, 0.8]],
                     dtype=F64, requires_grad=True)
    r = cc.regularizer(x)
    assert abs(float(r.detach()) - ((0.5 + 0 + 1) / 3 * 1e-2 + (0.2 + 0 + 1) / 3 * 1e-3)) < 1e-15
    (g,) = torch.autograd.grad(r, x)
    assert torch.equal(g[1], torch.zeros(6, dtype=F64))  # a zero row's norm has a zero gradient
    assert torch.allclose(g[0, :3], torch.tensor([0.6, 0.8, 0.0], dtype=F64) * 1e-2 / 3)
    m = cc.metrics(x.detach())
    assert abs(float(m["camera_opt_translation"]) - np.sqrt(0.25 + 1)) < 1e-15
    assert abs(float(m["camera_opt_rotation"]) - np.sqrt(0.04 + 1)) < 1e-15


def test_modes_and_indices_are_checked_on_the_host():
    with pytest.raises(NotImplementedError, match="SE3"):
        CameraPoseOptimizer(4, mode="SE3")
    with pytest.raises(ValueError):
        CameraPoseOptimizer(4, mode="simple")
    off = CameraPoseOptimizer(4, mode="off")
    assert not list(off.parameters()) and not off.active
    on = CameraPoseOptimizer(4)
    assert on.pose_adjustment.shape == (4, 6) and not on.pose_adjustment.any()
    assert dict(on.named_parameters()).keys() == {"pose_adjustment"}
    cam = Camera(np.eye(3, 4), 100.0, 100.0, 50.0, 50.0, 100, 100)
    assert cam.index is None
    for bad in (None, -1, 4):
        cam.index = bad
        with pytest.raises(IndexError):
            on.view(cam)  # raised before the library is touched
    # a module left on the host (or of another dtype) is refused before any launch: the kernels read device float32
    cam.index = 1
    for mod in (on, CameraPoseOptimizer(4).double()):
        for call in (lambda: mod.view(cam), mod.regularizer, mod.metrics):
            with pytest.raises(_lib.SgnError, match="float32"):
                call()
    with pytest.raises(RuntimeError, match="off"):
        off.regularizer()
