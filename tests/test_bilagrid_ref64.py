"""The float64 statement of the bilateral-grid slice and total variation (oracle/bilagrid_ref64.py) against F.grid_sample and
torch autograd in float64, on the CPU; and the host logic around the grids (module, checkpoint key, data-parallel refusal)."""
import types

import numpy as np
import pytest
import torch

from oracle.bilagrid_ref64 import (GRAY, gray_of, guide_f32, identity_grids, slice_grads_ref64, slice_grid_sample, slice_ref64,
                                   tv_ref64)

SHAPES = [  # (L, Hg, Wg, H, W)
    (8, 16, 16, 11, 13),
    (8, 16, 16, 2, 3),
    (3, 4, 7, 9, 5),     # non-square grid
    (1, 5, 3, 6, 7),     # L = 1: no guidance gradient, no L differences
    (4, 1, 1, 3, 4),     # one node in x and y
    (5, 3, 9, 8, 8),
]


def _grid(L, Hg, Wg, seed, scale=0.3):
    g = torch.Generator().manual_seed(seed)
    return identity_grids(1, L, Hg, Wg, torch.float64)[0] + scale * torch.randn(12, L, Hg, Wg, generator=g, dtype=torch.float64)


def _rgb(H, W, seed):
    """Random colours in [-0.2, 1.3] (grays outside [0, 1] included), with gray exactly 0 (black), grays beyond both ends, and
    a pixel whose gray is exactly 1 in float64."""
    g = torch.Generator().manual_seed(seed + 100)
    c = torch.rand(H, W, 3, generator=g, dtype=torch.float64) * 1.5 - 0.2
    flat = c.view(-1, 3)
    flat[0] = 0.0
    if flat.shape[0] > 1:
        flat[1] = torch.tensor([1.4, 1.2, 1.3], dtype=torch.float64)
    if flat.shape[0] > 2:
        flat[2] = torch.tensor([-0.3, -0.1, -0.2], dtype=torch.float64)
    if flat.shape[0] > 3:
        flat[3] = torch.tensor([1.0, 1.0, 0.0], dtype=torch.float64)
        flat[3, 2] = (1.0 - GRAY[0] - GRAY[1]) / GRAY[2]
    return c


@pytest.mark.parametrize("shape", SHAPES)
def test_gather_equals_grid_sample_values_and_gradients(shape):
    L, Hg, Wg, H, W = shape
    grid, rgb = _grid(L, Hg, Wg, 1), _rgb(H, W, 2)
    d = torch.randn(H, W, 3, generator=torch.Generator().manual_seed(3), dtype=torch.float64)
    outs, grads = [], []
    for fn in (slice_ref64, slice_grid_sample):
        g, c = grid.clone().requires_grad_(True), rgb.clone().requires_grad_(True)
        out = fn(g, c)
        (out * d).sum().backward()
        outs.append(out.detach())
        grads.append((g.grad, c.grad))
    assert torch.allclose(outs[0], outs[1], rtol=0, atol=1e-12)
    assert torch.allclose(grads[0][0], grads[1][0], rtol=0, atol=1e-12)
    assert torch.allclose(grads[0][1], grads[1][1], rtol=0, atol=1e-12)
    d_rgb, d_grid = slice_grads_ref64(grid.numpy(), rgb.numpy(), d.numpy())
    np.testing.assert_allclose(d_rgb, grads[1][1].numpy(), rtol=0, atol=1e-12)
    np.testing.assert_allclose(d_grid, grads[1][0].numpy(), rtol=0, atol=1e-12)


def test_gray_on_the_clamp_boundaries_passes_no_guidance_gradient():
    """gray exactly 0, exactly 1 and beyond: only the affine's A^T d_out reaches the colour."""
    grid, d = _grid(8, 4, 4, 5, scale=0.5), torch.ones(1, 4, 3, dtype=torch.float64)
    rgb = torch.tensor([[[0.0, 0.0, 0.0], [1.0, 1.0, (1.0 - GRAY[0] - GRAY[1]) / GRAY[2]], [1.5, 1.5, 1.5], [-0.5, 0.2, 0.1]]],
                       dtype=torch.float64)
    gray = GRAY[0] * rgb[..., 0] + GRAY[1] * rgb[..., 1] + GRAY[2] * rgb[..., 2]
    assert float(gray[0, 0]) == 0.0 and float(gray[0, 1]) == 1.0
    c = rgb.clone().requires_grad_(True)
    (slice_grid_sample(grid, c) * d).sum().backward()
    d_rgb, _ = slice_grads_ref64(grid.numpy(), rgb.numpy(), d.numpy())
    np.testing.assert_allclose(d_rgb, c.grad.numpy(), rtol=0, atol=1e-12)
    # A^T d_out alone: M at the clamped gray, with no gradient through it
    at = slice_grads_ref64(grid.numpy(), rgb.numpy(), d.numpy(), guide=((gray.clamp(0, 1) * 7).numpy(), np.zeros((1, 4), bool)))[0]
    np.testing.assert_allclose(d_rgb, at, rtol=0, atol=1e-12)


def _blue_for_gray(t: float) -> float:
    """A blue value whose gray (with red = green = 0) is exactly ``t`` in float64."""
    b = t / GRAY[2]
    for _ in range(64):
        if GRAY[2] * b == t:
            return b
        b = float(np.nextafter(b, np.inf if GRAY[2] * b < t else -np.inf))
    raise AssertionError(t)


def test_pixels_on_grid_nodes():
    """W = 3, Wg = 7 and H = 2, Hg = 5 put every pixel centre on a node in x and y; gray = k / (L - 1) puts it on a node in z,
    where the guidance derivative is grid_sample's one-sided one."""
    L = 5
    grid = _grid(L, 5, 7, 9, scale=0.4)
    rgb = torch.zeros(2, 3, 3, dtype=torch.float64)
    for k, t in enumerate((0.25, 0.5, 0.75, 0.5, 0.25, 0.75)):
        rgb.view(-1, 3)[k] = torch.tensor([0.0, 0.0, _blue_for_gray(t)], dtype=torch.float64)
    assert (gray_of(rgb) * (L - 1) == torch.round(gray_of(rgb) * (L - 1))).all()
    d = torch.randn(2, 3, 3, generator=torch.Generator().manual_seed(4), dtype=torch.float64)
    c = rgb.clone().requires_grad_(True)
    g = grid.clone().requires_grad_(True)
    out = slice_grid_sample(g, c)
    (out * d).sum().backward()
    assert torch.allclose(slice_ref64(grid, rgb), out.detach(), rtol=0, atol=1e-12)
    d_rgb, d_grid = slice_grads_ref64(grid.numpy(), rgb.numpy(), d.numpy())
    np.testing.assert_allclose(d_rgb, c.grad.numpy(), rtol=0, atol=1e-12)
    np.testing.assert_allclose(d_grid, g.grad.numpy(), rtol=0, atol=1e-12)


def test_identity_grid_is_the_identity():
    rgb = _rgb(7, 9, 6)
    out = slice_ref64(identity_grids(1, 8, 16, 16, torch.float64)[0], rgb)
    assert torch.allclose(out, rgb, rtol=0, atol=1e-14)


@pytest.mark.parametrize("shape", [(3, 4, 5, 3, 4), (1, 2, 3, 2, 2)])
def test_gradcheck(shape):
    L, Hg, Wg, H, W = shape
    grid = _grid(L, Hg, Wg, 7).requires_grad_(True)
    rgb = (torch.rand(H, W, 3, generator=torch.Generator().manual_seed(8), dtype=torch.float64) * 0.8 + 0.1).requires_grad_(True)
    assert torch.autograd.gradcheck(slice_ref64, (grid, rgb), eps=1e-7, atol=1e-6)
    grids = torch.randn(2, 12, L, Hg, Wg, generator=torch.Generator().manual_seed(9), dtype=torch.float64, requires_grad=True)
    assert torch.autograd.gradcheck(tv_ref64, (grids,), eps=1e-6, atol=1e-6)


@pytest.mark.parametrize("shape", [(8, 16, 16), (3, 4, 5), (1, 3, 2), (2, 1, 1)])
def test_tv_equals_explicit_means(shape):
    L, Hg, Wg = shape
    grids = torch.randn(3, 12, L, Hg, Wg, generator=torch.Generator().manual_seed(10), dtype=torch.float64)
    want = 0.0
    for axis, n in ((2, L), (3, Hg), (4, Wg)):
        if n > 1:
            a = grids.narrow(axis, 1, n - 1) - grids.narrow(axis, 0, n - 1)
            want += float((a ** 2).sum()) / a.numel()
    assert float(tv_ref64(grids)) == pytest.approx(want / 3, rel=1e-14)
    assert float(tv_ref64(identity_grids(4, L, Hg, Wg, torch.float64))) == 0.0


def test_guide_f32_matches_the_float64_branch_away_from_ties():
    rgb = _rgb(5, 6, 11).numpy()
    gz, inside = guide_f32(rgb, 8)
    gray = rgb @ np.asarray(GRAY)
    far = np.abs(gray) > 1e-6
    far &= np.abs(gray - 1) > 1e-6
    assert np.array_equal(inside[far], ((gray > 0) & (gray < 1))[far])
    np.testing.assert_allclose(gz, np.clip(gray, 0, 1) * 7, atol=1e-5)


def test_module_layout_and_checkpoint_key():
    from street_gaussians_ns_b200.bilagrid import BilateralGrid
    bg = BilateralGrid(3, shape=(4, 6, 2))
    assert tuple(bg.grids.shape) == (3, 12, 2, 4, 6)
    assert torch.equal(bg.grids.detach(), identity_grids(3, 2, 4, 6))
    assert list(bg.state_dict()) == ["grids"]
    with pytest.raises(ValueError):
        BilateralGrid(2, shape=(16, 16, 33))
    with pytest.raises(ValueError):
        BilateralGrid(0)


def test_slice_refuses_cpu_tensors():
    from street_gaussians_ns_b200 import _lib
    from street_gaussians_ns_b200.bilagrid import BilateralGrid
    bg = BilateralGrid(2, shape=(4, 4, 2))
    with pytest.raises(_lib.SgnError):
        bg.slice(torch.zeros(3, 3, 3), 0)
    with pytest.raises(_lib.SgnError):
        bg.tv_loss()


def test_data_parallel_refuses_the_grids(monkeypatch):
    """A data-parallel TrainStep does not exchange the grids' gradient: it refuses them before rendering, with the message it
    gives every extra tensor."""
    from street_gaussians_ns_b200.bilagrid import BilateralGrid
    from street_gaussians_ns_b200.model import _FullArenaSink
    from street_gaussians_ns_b200.optim import FusedAdam
    from street_gaussians_ns_b200.training import TrainStep
    from tests.test_refine import build_model
    model, _ = build_model()
    model.bilateral_grid = BilateralGrid(4, shape=(4, 4, 2))
    opt = FusedAdam(model.optimizer_params(), chunk_elems=4096, extra={"bilateral_grid.grids": (model.bilateral_grid.grids, 2e-3)})
    step_fn = TrainStep(model, opt, refine_every=0)
    rendered = []
    monkeypatch.setattr(model, "get_outputs", lambda camera: rendered.append(camera))
    model._holder = types.SimpleNamespace(grad_arena=torch.zeros(8))
    model._grad_sink = _FullArenaSink()
    monkeypatch.setattr(step_fn, "world_size", lambda: 2)
    monkeypatch.setattr(step_fn, "_ensure_exchange", lambda: rendered.append("exchange"))
    with pytest.raises(NotImplementedError, match=r"data-parallel training does not exchange the gradients of \['bilateral_grid.grids'\]"):
        step_fn(700, camera=None, batch={}, all_cameras=[None, None])
    assert not rendered
