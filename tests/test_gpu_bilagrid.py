"""The bilateral-grid kernels (csrc/bilagrid.cu) through their C entry points, the autograd nodes, the model and training, on
the GPU.

Bars against the float64 statement (oracle/bilagrid_ref64.py, evaluated with the kernel's float32 guidance so that a pixel on a
level node or on the clamp takes the same branch): the slice within 2e-5 of the largest output; d_rgb within 1e-4 of the largest
|d_rgb| (the guidance term multiplies differences of nodes by L - 1); d_grid within 1e-5 relative L2 and 1e-4 of the largest
element; the total variation within 1e-6 relative, its gradient within 1e-6 of the largest element.  Identity grids: the output
equals the input and d_rgb equals d_out within 1e-6."""
import ctypes as C

import numpy as np
import pytest
import torch

import street_gaussians_ns_b200.synthetic as syn
from oracle.bilagrid_ref64 import guide_f32, slice_grads_ref64, slice_ref64, tv_ref64
from street_gaussians_ns_b200 import _lib, raster
from street_gaussians_ns_b200.bilagrid import BilateralGrid
from street_gaussians_ns_b200.model import SceneGraphConfig, SceneGraphRasterModel
from street_gaussians_ns_b200.optim import FusedAdam
from street_gaussians_ns_b200.scene import PARAM_NAMES
from street_gaussians_ns_b200.training import TrainStep
from tests.bilagrid_cases import SLICE_CASES, TV_CASES, colours, cotangent, identity, random_grid

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def slice_fwd(grid: torch.Tensor, rgb: torch.Tensor) -> torch.Tensor:
    L, Hg, Wg = grid.shape[1:]
    H, W = rgb.shape[:2]
    out = torch.full_like(rgb, float("nan"))
    _lib.check(_lib.load().sgn_bilagrid_slice_fwd(_ptr(grid), L, Hg, Wg, _ptr(rgb), H, W, _ptr(out), _stream()), "sgn_bilagrid_slice_fwd")
    return out


def slice_bwd(grid: torch.Tensor, rgb: torch.Tensor, d_out: torch.Tensor):
    L, Hg, Wg = grid.shape[1:]
    H, W = rgb.shape[:2]
    lib = _lib.load()
    d_rgb = torch.full_like(rgb, float("nan"))
    d_grid = torch.full_like(grid, float("nan"))  # every element is written
    sb = lib.sgn_bilagrid_slice_bwd_scratch_bytes(L, Hg, Wg, H, W)
    scratch = torch.full((sb,), 255, device=DEV, dtype=torch.uint8)
    _lib.check(lib.sgn_bilagrid_slice_bwd(_ptr(grid), L, Hg, Wg, _ptr(rgb), _ptr(d_out), H, W, _ptr(d_rgb), _ptr(d_grid), _ptr(scratch), sb,
                                          _stream()), "sgn_bilagrid_slice_bwd")
    return d_rgb, d_grid


def tv_fwd(grids: torch.Tensor) -> torch.Tensor:
    N, _, L, Hg, Wg = grids.shape
    lib = _lib.load()
    out = torch.full((1,), float("nan"), device=DEV)
    sb = lib.sgn_bilagrid_tv_scratch_bytes()
    scratch = torch.empty(sb, device=DEV, dtype=torch.uint8)
    _lib.check(lib.sgn_bilagrid_tv_fwd(_ptr(grids), N, L, Hg, Wg, _ptr(out), _ptr(scratch), sb, _stream()), "sgn_bilagrid_tv_fwd")
    return out


def tv_bwd(grids: torch.Tensor, v: float) -> torch.Tensor:
    N, _, L, Hg, Wg = grids.shape
    vt = torch.tensor([v], device=DEV, dtype=torch.float32)
    d = torch.full_like(grids, float("nan"))
    _lib.check(_lib.load().sgn_bilagrid_tv_bwd(_ptr(grids), N, L, Hg, Wg, _ptr(vt), _ptr(d), _stream()), "sgn_bilagrid_tv_bwd")
    return d


def rel_l2(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def _oracle(grid_np, rgb_np, d_np):
    """(out, d_rgb, d_grid) of the float64 statement at the kernel's float32 guidance, evaluated on the GPU in float64."""
    L = grid_np.shape[1]
    guide = guide_f32(rgb_np, L)
    g64, c64 = _dev(grid_np).double(), _dev(rgb_np).double()
    out = slice_ref64(g64, c64, guide=guide).cpu().numpy()
    d_rgb, d_grid = slice_grads_ref64(g64, c64, _dev(d_np), guide=guide)
    return out, d_rgb, d_grid


@pytest.mark.parametrize("name", sorted(SLICE_CASES))
@pytest.mark.parametrize("kind", ["identity", "random"])
def test_slice_against_float64(name, kind):
    L, Hg, Wg, H, W = SLICE_CASES[name]
    seed = sorted(SLICE_CASES).index(name)
    grid_np = identity(L, Hg, Wg) if kind == "identity" else random_grid(L, Hg, Wg, seed)
    rgb_np, d_np = colours(H, W, seed + 10), cotangent(H, W, seed + 20)
    grid, rgb, d = _dev(grid_np), _dev(rgb_np), _dev(d_np)
    out = slice_fwd(grid, rgb)
    d_rgb, d_grid = slice_bwd(grid, rgb, d)
    torch.cuda.synchronize()
    out, d_rgb, d_grid = out.cpu().numpy(), d_rgb.cpu().numpy(), d_grid.cpu().numpy()
    assert np.isfinite(out).all() and np.isfinite(d_rgb).all() and np.isfinite(d_grid).all()
    if kind == "identity":
        assert np.abs(out - rgb_np).max() <= 1e-6
        assert np.abs(d_rgb - d_np).max() <= 1e-6
    ref_out, ref_d_rgb, ref_d_grid = _oracle(grid_np, rgb_np, d_np)
    assert np.abs(out - ref_out).max() <= 2e-5 * max(1.0, np.abs(ref_out).max())
    assert np.abs(d_rgb - ref_d_rgb).max() <= 1e-4 * max(1.0, np.abs(ref_d_rgb).max())
    assert rel_l2(d_grid, ref_d_grid) < 1e-5
    assert np.abs(d_grid - ref_d_grid).max() <= 1e-4 * np.abs(ref_d_grid).max()


@pytest.mark.parametrize("name", ["default_97x211", "rig_1280x1920", "one_node_xy"])
def test_backward_is_bitwise_repeatable(name):
    L, Hg, Wg, H, W = SLICE_CASES[name]
    grid, rgb, d = _dev(random_grid(L, Hg, Wg, 5)), _dev(colours(H, W, 6)), _dev(cotangent(H, W, 7))
    a = slice_bwd(grid, rgb, d)
    b = slice_bwd(grid, rgb, d)
    torch.cuda.synchronize()
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_slice_argument_errors():
    lib = _lib.load()
    g, c = _dev(identity(8, 4, 4)), _dev(colours(4, 4, 0))
    assert lib.sgn_bilagrid_slice_fwd(_ptr(g), 0, 4, 4, _ptr(c), 4, 4, _ptr(c), _stream()) != 0
    assert lib.sgn_bilagrid_slice_fwd(None, 8, 4, 4, _ptr(c), 4, 4, _ptr(c), _stream()) != 0
    sb = lib.sgn_bilagrid_slice_bwd_scratch_bytes(33, 4, 4, 4, 4)
    s = torch.empty(max(sb, 1), device=DEV, dtype=torch.uint8)
    g33 = _dev(identity(33, 4, 4))
    assert lib.sgn_bilagrid_slice_bwd(_ptr(g33), 33, 4, 4, _ptr(c), _ptr(c), 4, 4, _ptr(c), _ptr(g33), _ptr(s), sb, _stream()) != 0
    assert b"33" in lib.sgn_last_error()


@pytest.mark.parametrize("name", sorted(TV_CASES))
def test_tv_against_float64(name):
    N, L, Hg, Wg = TV_CASES[name]
    rng = np.random.default_rng(sorted(TV_CASES).index(name))
    x_np = rng.standard_normal((N, 12, L, Hg, Wg)).astype(np.float32)
    x = _dev(x_np)
    val = tv_fwd(x)
    grad = tv_bwd(x, 0.37)
    torch.cuda.synchronize()
    x64 = x.double().requires_grad_(True)
    ref = tv_ref64(x64)
    (ref * 0.37).backward()
    assert float(val) == pytest.approx(float(ref), rel=1e-6)
    want = x64.grad.cpu().numpy()
    assert np.abs(grad.cpu().numpy() - want).max() <= 1e-6 * np.abs(want).max()
    assert torch.equal(tv_fwd(x), val) and torch.equal(tv_bwd(x, 0.37), grad)


def test_autograd_nodes_match_the_entry_points():
    bg = BilateralGrid(3, shape=(5, 6, 4)).to(DEV)
    with torch.no_grad():
        bg.grids.copy_(_dev(np.stack([random_grid(4, 5, 6, s) for s in range(3)])))
    rgb_np, d_np = colours(30, 41, 1), cotangent(30, 41, 2)
    rgb = _dev(rgb_np).requires_grad_(True)
    out = bg.slice(rgb, 1)
    tv = bg.tv_loss()
    torch.autograd.backward([out, tv], [_dev(d_np), torch.tensor(2.0, device=DEV)])
    g1 = bg.grids.detach()[1].contiguous()
    d_rgb, d_grid = slice_bwd(g1, _dev(rgb_np), _dev(d_np))
    assert torch.equal(out.detach(), slice_fwd(g1, _dev(rgb_np)))
    assert torch.equal(rgb.grad, d_rgb)
    want = tv_bwd(bg.grids.detach(), 2.0)
    want[1] += d_grid
    assert torch.equal(bg.grids.grad, want)
    assert torch.equal(tv.detach().reshape(1), tv_fwd(bg.grids.detach()))


# ---- the model -----------------------------------------------------------------------------------------------------------


def _scene(seed=3):
    return syn.make_frame(n_background=20000, n_actors=0, width=320, height=240, seed=seed)


def _model(fr, bilateral_grid=None, **cfg):
    model = SceneGraphRasterModel(fr.segments[0].params.to(DEV), {}, SceneGraphConfig(use_sky_sphere=False, **cfg),
                                  bilateral_grid=bilateral_grid).to(DEV)
    model.train()
    return model


def _grid_module(n=4, seed=0):
    bg = BilateralGrid(n)
    with torch.no_grad():
        bg.grids.copy_(torch.from_numpy(np.stack([random_grid(8, 16, 16, seed + k, scale=0.05) for k in range(n)])))
    return bg


def _run(model, camera, gt):
    for p in model.parameters():
        p.grad = None
    out = model.get_outputs(camera)
    losses = model.get_loss_dict(out, {"image": gt})
    sum(losses.values()).backward()
    torch.cuda.synchronize()
    grads = {n: (None if p.grad is None else p.grad.clone()) for n, p in model.named_parameters()}
    return out, losses, grads


def test_model_without_a_grid_is_unchanged(monkeypatch):
    """A grid that does not apply (camera without an index) and an absent one render and train with the same bits as a model
    built without the argument; only ``bilagrid_tv`` is added by the grid that is present."""
    monkeypatch.setattr(raster, "DETERMINISTIC", True)
    fr = _scene()
    gt = torch.rand(240, 320, 3, generator=torch.Generator().manual_seed(2)).to(DEV)
    cam = fr.camera
    assert cam.index is None
    res = {}
    for key, bg in (("plain", "absent"), ("none", None), ("unindexed", _grid_module())):
        model = _model(fr) if bg == "absent" else _model(fr, bilateral_grid=bg)
        res[key] = _run(model, cam, gt)
    out0, l0, g0 = res["plain"]
    for key in ("none", "unindexed"):
        out, losses, grads = res[key]
        assert out.keys() == out0.keys() and all(torch.equal(out[k], out0[k]) for k in out0), key
        assert all(torch.equal(losses[k], l0[k]) for k in l0), key
        assert all(torch.equal(grads[k], g0[k]) for k in g0 if g0[k] is not None), key
    assert "bilagrid_tv" not in res["none"][1] and "bilagrid_tv" in res["unindexed"][1]


def test_training_render_is_the_slice_of_the_raw_render():
    fr = _scene()
    bg = _grid_module()
    model = _model(fr, bilateral_grid=bg)
    cam = fr.camera
    raw = model.get_outputs(cam)["rgb"].detach()
    cam.index = 2
    try:
        out = model.get_outputs(cam)
        assert out["rgb"].requires_grad
        want = bg.slice(raw, 2).detach()
        assert torch.equal(out["rgb"].detach(), want)
        assert not torch.equal(want, raw)
        losses = model.get_loss_dict(out, {"image": raw})
        assert "bilagrid_tv" in losses and losses["bilagrid_tv"].requires_grad
        model.eval()
        with torch.no_grad():
            ev = model.get_outputs_for_camera(cam)
            assert "bilagrid_tv" not in model.get_loss_dict(ev, {"image": raw})
            cam.index = None
            assert torch.equal(ev["rgb"], model.get_outputs_for_camera(cam)["rgb"])
    finally:
        cam.index = None


def test_state_dict_round_trip():
    fr = _scene()
    a = _model(fr, bilateral_grid=_grid_module(seed=4))
    sd = a.state_dict()
    assert "bilateral_grid.grids" in sd
    b = _model(fr, bilateral_grid=BilateralGrid(4).to(DEV))
    b.load_state_dict(sd)
    assert torch.equal(b.bilateral_grid.grids, a.bilateral_grid.grids)


def test_grids_train_to_known_colour_maps():
    """Gaussians frozen (Adam at lr 0), four cameras whose targets are per-channel gains in [0.7, 1.3] plus a tint of their own
    render: training only the grids for 150 steps per camera brings the mean |corrected - target| below 0.01, from a start at
    least three times higher."""
    fr = _scene(seed=5)
    n = 4
    bg = BilateralGrid(n)
    model = _model(fr, bilateral_grid=bg, ssim_lambda=0.0, object_acc_entropy_loss_mult=0.0)
    rng = np.random.default_rng(8)
    cams, targets, raws = [], [], []
    for k in range(n):
        c2w = np.asarray(fr.camera.c2w, np.float32).copy()
        c2w[0, 3] += 0.3 * k
        cam = syn.make_camera(320, 240, c2w=c2w, time=fr.camera.time)
        with torch.no_grad():
            raw = model.get_outputs(cam)["rgb"].detach()
        gain = torch.tensor(rng.uniform(0.7, 1.3, 3), dtype=torch.float32, device=DEV)
        tint = torch.tensor(rng.uniform(-0.05, 0.05, 3), dtype=torch.float32, device=DEV)
        cam.index = k
        cams.append(cam)
        raws.append(raw)
        targets.append(raw * gain + tint)
    opt = FusedAdam(model.optimizer_params(), lrs={k: 0.0 for k in PARAM_NAMES}, extra={"bilateral_grid.grids": (bg.grids, 5e-3)})
    step_fn = TrainStep(model, opt, refine_every=1_000_000)
    params0 = {k: p.detach().clone() for k, p in model.all_models.named_parameters()}

    def err():
        with torch.no_grad():
            return float(np.mean([float((bg.slice(raws[k], k) - targets[k]).abs().mean()) for k in range(n)]))
    start = err()
    for s in range(150 * n):
        step_fn(s, cams[s % n], {"image": targets[s % n]})
    torch.cuda.synchronize()
    end = err()
    assert start > 0.03, start
    assert end < 0.01, (start, end)
    assert all(torch.equal(p.detach(), params0[k]) for k, p in model.all_models.named_parameters())
