"""Lidar depth supervision on the GPU (csrc/depth.cu through depth.py, and the model surface built on it) against the float64
statement (oracle/depth_ref64.py) and torch autograd.

Bars: the map equals the float64 map pixel for pixel (which pixels have a return), with depths within 1e-6 relative, once the
points whose pixel coordinate lies within 1e-3 px of an integer are left out (float32 and float64 may floor those differently);
a point at a Gaussian's mean lands on that Gaussian's xy with its depth record, bit for bit; the loss and its cotangent agree
with float64 and with torch autograd to fp32 rounding; the model's gradient arena from the fused term agrees with the one from
the torch expression within 1e-5 relative L2; eval's depth metrics agree with float64 within 1e-5 relative."""
import math

import numpy as np
import pytest
import torch

import street_gaussians_ns_b200.synthetic as syn
from oracle import depth_ref64 as ref
from street_gaussians_ns_b200 import _lib, raster
from street_gaussians_ns_b200.depth import METRIC_NAMES, depth_loss_torch, depth_metrics, fused_depth_loss, lidar_depth_map
from street_gaussians_ns_b200.model import SceneGraphConfig, SceneGraphRasterModel

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def rel_l2(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / max(float(b.norm()), 1e-30))


def hand_camera(W=8, H=6, f=10.0, clip=0.01):
    cs = _lib.CameraStruct()
    for i, v in enumerate([1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0]):
        cs.viewmat[i] = float(v)
    cs.fx = cs.fy = f
    cs.cx, cs.cy = W / 2, H / 2
    cs.width, cs.height, cs.clip_thresh, cs.block_width = W, H, clip, 16
    return cs


def oracle_map(points, cs, to_world=None):
    V = np.array(list(cs.viewmat), np.float64).reshape(3, 4)
    A = ref.compose(V, to_world)
    if to_world is not None:  # the kernel rounds the composed matrix once to fp32
        A = A.astype(np.float32).astype(np.float64)
    return ref.lidar_depth_map_ref64(points, A, cs.fx, cs.fy, cs.cx, cs.cy, cs.width, cs.height, cs.clip_thresh)


def off_edges(points, cs, to_world=None, margin=1e-3):
    """The points whose pixel coordinates lie more than ``margin`` px from an integer."""
    V = np.array(list(cs.viewmat), np.float64).reshape(3, 4)
    _, u, v = ref.project_points_ref64(points, ref.compose(V, to_world), cs.fx, cs.fy, cs.cx, cs.cy)
    du, dv = np.abs(u - np.round(u)), np.abs(v - np.round(v))
    return ~((du < margin) | (dv < margin))


def check_map(got, want):
    got = got.cpu().numpy()[..., 0].astype(np.float64)
    assert np.array_equal(got > 0, want > 0), int(((got > 0) != (want > 0)).sum())
    hit = want > 0
    assert np.all(np.abs(got[hit] - want[hit]) <= 1e-6 * want[hit]), float(np.max(np.abs(got[hit] - want[hit]) / want[hit]))


HAND_CASES = {
    "two_on_one_pixel": [[0.25, 0.25, 5.0], [0.1, 0.1, 2.0]],
    "edge_u": [[0.0, 0.0, 3.0], [0.0, 0.5, 7.0]],  # u exactly 4 = cx: the pixel right of the edge
    "dropped": [[0.0, 0.0, -2.0], [5.0, 0.0, 1.0], [0.0, 0.0, 0.01], [0.0, -1.0, 2.0], [0.0, 0.0, 0.015]],
    "empty": np.zeros((0, 3)),
}


@pytest.mark.parametrize("case", list(HAND_CASES))
def test_map_hand_built(case):
    cs = hand_camera()
    pts = np.asarray(HAND_CASES[case], np.float32).reshape(-1, 3)
    got = lidar_depth_map(torch.from_numpy(pts).to(DEV), cs)
    want, _ = oracle_map(pts.astype(np.float64), cs)
    assert got.shape == (cs.height, cs.width, 1)
    assert np.array_equal(got.cpu().numpy()[..., 0], want.astype(np.float32))  # these depths are exact in fp32


def _cfg3_camera():
    return raster.camera_struct(syn.make_camera(1920, 1280), raster.RenderSettings())


@pytest.mark.parametrize("with_to_world", [False, True])
def test_map_street_sweep(with_to_world):
    cs = _cfg3_camera()
    pts = syn.street_points(170_000, seed=3).numpy()
    tw = None
    if with_to_world:  # the same sweep handed over in a lidar frame 1.5 m up and 0.3 rad around y
        a = 0.3
        R = np.array([[math.cos(a), 0, math.sin(a)], [0, 1, 0], [-math.sin(a), 0, math.cos(a)]])
        t = np.array([0.2, 1.5, -0.7])
        tw = np.concatenate([R, t[:, None]], axis=1)
        pts = ((pts.astype(np.float64) - t) @ R).astype(np.float32)  # to_world @ pts = the world cloud
    keep = off_edges(pts.astype(np.float64), cs, tw)
    pts = pts[keep]
    got = lidar_depth_map(torch.from_numpy(pts).to(DEV), cs, to_world=tw)
    want, pix = oracle_map(pts.astype(np.float64), cs, tw)
    assert (pix >= 0).sum() > 50_000
    check_map(got, want)
    again = lidar_depth_map(torch.from_numpy(pts).to(DEV), cs, to_world=tw)
    assert torch.equal(got, again)
    shuffled = lidar_depth_map(torch.from_numpy(pts[::-1].copy()).to(DEV), cs, to_world=tw)
    assert torch.equal(got, shuffled)


def test_point_at_a_mean_gets_the_depth_record():
    fr = syn.make_frame(n_background=20000, n_actors=0, width=320, height=240, seed=3)
    frame = raster.Frame(fr.camera, [s.__class__(s.params.to(DEV), s.cls, s.rot, s.center, s.idft, s.name) for s in fr.segments])
    with torch.no_grad():
        _, holder = raster.render_frame(frame)
    rec = holder.records.cpu().numpy()
    radii = holder.radii.cpu().numpy()
    means = frame.segments[0].params.means.detach().cpu().numpy()
    xy, z = rec[:, 0:2], rec[:, 9]
    ok = (radii > 0) & (xy[:, 0] >= 0) & (xy[:, 0] < 320) & (xy[:, 1] >= 0) & (xy[:, 1] < 240)
    pix = np.floor(xy[:, 1]).astype(np.int64) * 320 + np.floor(xy[:, 0]).astype(np.int64)
    _, first = np.unique(np.where(ok, pix, -1), return_index=True)
    rows = np.array([r for r in first if ok[r]])  # one Gaussian per pixel
    assert rows.size > 1000
    got = lidar_depth_map(torch.from_numpy(means[rows]).to(DEV), fr.camera).cpu().numpy().reshape(-1)
    assert np.array_equal(got[pix[rows]], z[rows])  # bit for bit
    assert np.count_nonzero(got) == rows.size


def _loss_case(H, W, seed, mask_kind=None):
    g = torch.Generator().manual_seed(seed)
    D = torch.rand(H, W, 1, generator=g) * 30 + 0.5
    T = torch.where(torch.rand(H, W, 1, generator=g) < 0.1, torch.rand(H, W, 1, generator=g) * 30 + 0.5, torch.zeros(()))
    mask = None
    if mask_kind == "binary":
        mask = (torch.rand(H, W, 1, generator=g) > 0.3).float()
    elif mask_kind == "none_kept":
        mask = (T == 0).float()
    return D, T, mask


@pytest.mark.parametrize("H,W", [(7, 9), (1280, 1920)])
@pytest.mark.parametrize("mask_kind", [None, "binary", "none_kept", "no_target"])
def test_loss_against_float64_and_autograd(H, W, mask_kind):
    D, T, mask = _loss_case(H, W, 5, mask_kind if mask_kind != "no_target" else None)
    if mask_kind == "no_target":
        T = torch.zeros_like(T)
    w, gscale = 0.25, 1.5
    d = D.to(DEV).requires_grad_(True)
    t, m = T.to(DEV), None if mask is None else mask.to(DEV)
    loss = fused_depth_loss(d, t, m, w)
    (gscale * loss).backward()
    L64, n = ref.depth_loss_ref64(D.numpy(), T.numpy(), None if mask is None else mask.numpy(), w)
    g64 = ref.depth_loss_grad_ref64(D.numpy(), T.numpy(), None if mask is None else mask.numpy(), w, gscale)
    got_l, got_g = float(loss.detach()), d.grad.cpu().numpy().astype(np.float64)
    assert np.isfinite(got_l) and np.isfinite(got_g).all()
    if n == 0:
        assert got_l == 0.0 and not got_g.any()
    else:
        assert got_l == pytest.approx(L64, rel=1e-6)
        assert np.all(np.abs(got_g - g64) <= 1e-6 * np.abs(g64).max())
        assert np.array_equal(got_g == 0, g64 == 0)
    d2 = D.to(DEV).requires_grad_(True)
    lt = depth_loss_torch(d2, t, m, w)
    (gscale * lt).backward()
    assert float(lt.detach()) == pytest.approx(got_l, rel=2e-6, abs=0)
    assert torch.allclose(d.grad, d2.grad, rtol=1e-6, atol=0)
    d.grad = None
    (gscale * fused_depth_loss(d, t, m, w)).backward()  # the same bits on a second run
    again = d.grad.clone()
    assert float(fused_depth_loss(d, t, m, w)) == got_l and np.array_equal(again.cpu().numpy(), got_g.astype(np.float32))


@pytest.mark.parametrize("mask_kind", [None, "binary", "none_kept"])
def test_metrics_against_float64(mask_kind):
    D, T, mask = _loss_case(1280, 1920, 9, mask_kind)
    D[:5] = 0.0  # clamped to 1e-3
    got = depth_metrics(D.to(DEV), T.to(DEV), None if mask is None else mask.to(DEV)).cpu().numpy().astype(np.float64)
    want = ref.depth_metrics_ref64(D.numpy(), T.numpy(), None if mask is None else mask.numpy())
    for i, name in enumerate(METRIC_NAMES):
        if math.isnan(want[i]):
            assert math.isnan(got[i]), name
        else:
            assert abs(got[i] - want[i]) <= 1e-6 * abs(want[i]) + 1e-7, (name, got[i], want[i])


# ---- model -----------------------------------------------------------------------------------------------------------

def _model(sky=False, w=0.05, seed=3, **cfg):
    fr = syn.make_frame(n_background=20000, n_actors=0, width=320, height=240, seed=seed)
    env = None
    if sky:
        from street_gaussians_ns_b200.sky import CubeMapSky
        torch.manual_seed(0)
        env = CubeMapSky(16)
        with torch.no_grad():
            env.base.copy_(torch.rand(6, 16, 16, 3))
    model = SceneGraphRasterModel(fr.segments[0].params.to(DEV), {}, SceneGraphConfig(use_sky_sphere=sky, depth_loss_mult=w, **cfg),
                                  sky=env).to(DEV)
    model.train()
    gt = torch.rand(240, 320, 3, generator=torch.Generator().manual_seed(2)).to(DEV)
    lidar = syn.street_points(30_000, seed=4).to(DEV)
    return fr, model, gt, lidar


def _arena(model, loss, retain_graph=False):
    for p in model.parameters():
        p.grad = None
    loss.backward(retain_graph=retain_graph)
    torch.cuda.synchronize()
    return model._holder.grad_arena.clone()


@pytest.mark.parametrize("sky", [False, True])
@pytest.mark.parametrize("async_binning", [False, True])
def test_model_fused_term_matches_torch_expression(sky, async_binning):
    """Backward passes over ONE render (the sky's jitter is drawn per render): the fused term, the torch expression of the
    term on out["depth"], and no term."""
    fr, model, gt, lidar = _model(sky=sky)
    mask = (torch.rand(240, 320, 1, generator=torch.Generator().manual_seed(6)) > 0.2).float().to(DEV)
    batch = {"image": gt, "lidar_points": lidar, "mask": mask}
    raster._ASYNC_STATE.clear()
    model.config.async_binning = async_binning
    try:
        for _ in range(2 if async_binning else 1):  # the first frame learns the count
            out = model.get_outputs(fr.camera)
        if async_binning:
            assert isinstance(model._holder.M, raster.LazyCount)
        losses = model.get_loss_dict(out, batch)
        assert "depth_loss" in losses and float(losses["depth_loss"]) > 0
        a_fused = _arena(model, sum(losses.values()), retain_graph=True)
        target = model._depth_target(batch)
        assert int((target > 0).sum()) > 1000
        model.config.depth_loss_mult = 0.0
        losses2 = model.get_loss_dict(out, batch)
        assert "depth_loss" not in losses2
        term = depth_loss_torch(out["depth"], target, mask, 0.05)
        assert float(term) == pytest.approx(float(losses["depth_loss"]), rel=2e-6)
        a_torch = _arena(model, sum(losses2.values()) + term, retain_graph=True)
        assert rel_l2(a_fused, a_torch) < 1e-5
        a_none = _arena(model, sum(losses2.values()))  # the term moves the geometry
        assert rel_l2(a_none, a_torch) > 1e-3
    finally:
        raster._ASYNC_STATE.clear()
        model.config.async_binning = None


def test_depth_image_target_and_torch_path():
    fr, model, gt, lidar = _model()
    out = model.get_outputs(fr.camera)
    target = lidar_depth_map(lidar, fr.camera)
    a = model.get_loss_dict(out, {"image": gt, "lidar_points": lidar})["depth_loss"]
    b = model.get_loss_dict(out, {"image": gt, "depth_image": target})["depth_loss"]
    assert float(a) == float(b)
    model.config.fused_loss = False
    c = model.get_loss_dict(out, {"image": gt, "depth_image": target})["depth_loss"]
    assert float(c) == pytest.approx(float(a), rel=2e-6)


def test_zero_weight_ignores_the_sweep(monkeypatch):
    monkeypatch.setattr(raster, "DETERMINISTIC", True)  # two renders give the same bits only without float atomics
    fr, model, gt, lidar = _model(w=0.0)
    res = []
    for batch in ({"image": gt}, {"image": gt, "lidar_points": lidar}):
        out = model.get_outputs(fr.camera)
        losses = model.get_loss_dict(out, batch)
        res.append(({k: v.detach().clone() for k, v in losses.items()}, _arena(model, sum(losses.values()))))
    (l0, a0), (l1, a1) = res
    assert l0.keys() == l1.keys() and all(torch.equal(l0[k], l1[k]) for k in l0)
    assert torch.equal(a0, a1)


def _train(steps):
    from street_gaussians_ns_b200.optim import FusedAdam
    from street_gaussians_ns_b200.training import TrainStep
    fr, model, gt, _ = _model(w=0.1)
    opt = FusedAdam(model.optimizer_params())
    step_fn = TrainStep(model, opt, refine_every=100)
    for s in steps:
        losses = step_fn(s, fr.camera, {"image": gt, "lidar_points": syn.street_points(30_000, seed=s).to(DEV)})
        assert "depth_loss" in losses
    torch.cuda.synchronize()
    return {f"{n}.{k}": p.detach().clone() for n, sub in model.all_models.items() for k, p in sub.gauss_params.items()}


def test_train_steps_repeat_bit_for_bit(monkeypatch):
    monkeypatch.setattr(raster, "DETERMINISTIC", True)
    a, b = _train([10, 11, 12]), _train([10, 11, 12])
    assert a.keys() == b.keys()
    assert not [k for k in a if not torch.equal(a[k], b[k])]


def test_train_step_full_gradient_arena():
    """The arena layout of data-parallel training (all sub-models): the term only changes the image cotangent."""
    from street_gaussians_ns_b200.optim import FusedAdam
    from street_gaussians_ns_b200.training import TrainStep
    fr, model, gt, lidar = _model(w=0.1, full_gradient_arena=True)
    step_fn = TrainStep(model, FusedAdam(model.optimizer_params()), refine_every=100)
    before = model.all_models["background"].gauss_params["means"].detach().clone()
    losses = step_fn(10, fr.camera, {"image": gt, "lidar_points": lidar})
    assert "depth_loss" in losses and math.isfinite(float(losses["depth_loss"]))
    assert not torch.equal(before, model.all_models["background"].gauss_params["means"].detach())


def test_eval_depth_metrics():
    fr, model, gt, lidar = _model()
    model.eval()
    out = model.get_outputs(fr.camera)
    batch = {"image": gt, "lidar_points": lidar}
    metrics, images = model.get_image_metrics_and_images(out, batch)
    assert set(images) == {"img", "accumulation", "depth"}
    target = lidar_depth_map(lidar, fr.camera)
    want = ref.depth_metrics_ref64(out["depth"].detach().cpu().numpy(), target.cpu().numpy())
    assert want[7] > 1000
    for i, name in enumerate(METRIC_NAMES[:7]):
        got = metrics[f"depth_{name}"]
        assert isinstance(got, float)
        assert abs(got - want[i]) <= 1e-5 * abs(want[i]) + 1e-7, (name, got, want[i])
    plain, _ = model.get_image_metrics_and_images(out, {"image": gt})
    assert not any(k.startswith("depth_") for k in plain)
