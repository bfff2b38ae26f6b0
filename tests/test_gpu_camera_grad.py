"""The gradient of the camera pose on the GPU: the device view through the projection (sgn_project_fwd_view /
sgn_project_bwd_view + sgn_view_grad_reduce), the adjust kernels, the sky with a device view, and
``camera_pose.CameraPoseOptimizer`` through the model and the training step.

  * plumbing: the camera's own view passed as a device view renders and differentiates bit for bit as the host view; without
    an optimizer, in mode "off", in eval or without a camera index the model's launches and outputs are today's;
  * directed: hand-built frames -- every cut of the projection -- with v_view within 1e-3 relative L2 of float64 autograd with
    the view as the leaf over the same record cotangents, exact zeros when nothing is visible, v_pose unchanged beside it;
  * config 3: along 3 translations and 3 rotations of the camera, the contraction of v_view equals float64 sums of the
    parameter gradients (background) and pose cotangents (actors) for the inverse motion of the world; reproducibility;
  * adjust kernels against float64; the sky; the model, FusedAdam, gradient accumulation; a perturbed camera pulled back.
"""
import numpy as np
import pytest
import torch

import street_gaussians_ns_b200.synthetic as syn
from street_gaussians_ns_b200 import _lib, raster
from street_gaussians_ns_b200.camera_pose import CameraPoseOptimizer
from street_gaussians_ns_b200.model import SceneGraphConfig, SceneGraphRasterModel
from street_gaussians_ns_b200.optim import FusedAdam
from street_gaussians_ns_b200.scene import Camera, Frame, Segment
from street_gaussians_ns_b200.sky import CubeMapSky
from street_gaussians_ns_b200.training import TrainStep
from tests import camera_cases as cc
from tests import pose_cases as pz
from tests import project_cases as pc

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
TOL = 1e-3
F64 = torch.float64


def _settings(case):
    st = case.st
    return raster.RenderSettings(sh_degree=st.sh_degree, sh_degree_to_use=st.deg_use, block_width=st.block_width, clip_thresh=st.clip_thresh)


def _cuda_frame(frame):
    return Frame(frame.camera, [Segment(s.params.to("cuda"), s.cls, s.rot, s.center, s.idft, s.name) for s in frame.segments])


def own_view(camera: Camera) -> torch.Tensor:
    return torch.from_numpy(np.concatenate([camera.viewmat().reshape(-1), camera.cam_pos()]).astype(np.float32)).to(DEV)


def _weights(H, W, seed=5):
    g = torch.Generator().manual_seed(seed)
    return {"rgb": torch.rand(H, W, 3, generator=g).to(DEV), "accumulation": torch.rand(H, W, 1, generator=g).to(DEV),
            "object_acc": torch.rand(H, W, 1, generator=g).to(DEV)}


def off_screen_all(seed=305):
    b = pc._cam(160, 96, seed)
    s = b.segment(0)
    b.scatter(s, 150, px=(30.0 * b.cam.width, 40.0 * b.cam.width), py=(0.0, 96.0), z=(2.0, 6.0), scale=(0.01, 0.05))
    return b.settle("off_screen_all")


def background_only(seed=306):
    b = pc._cam(160, 96, seed)
    pz._on_screen(b, b.segment(0), 300)
    return b.settle("background_only")


CASES = {"background_only": background_only, "actors_and_background": lambda: pz.get("actors_and_background"),
         "near_plane": pc.near_plane, "fov_clamp": pc.fov_clamp, "clip_plane": lambda: pz.get("clip_plane"),
         "off_screen_all": off_screen_all}


@pytest.mark.parametrize("name", list(CASES))
def test_directed_against_float64(name):
    case = CASES[name]()
    frc = _cuda_frame(case.frame)
    st = _settings(case)
    base = pz.frame_poses(case.frame)
    pose = torch.from_numpy(base).to(DEV).requires_grad_(True) if base.shape[0] else None
    view = own_view(frc.camera).requires_grad_(True)
    w = _weights(frc.camera.height, frc.camera.width)
    out, h = raster.render_frame(frc, st, pose=pose, view=view)
    sum((out[k] * w[k]).sum() for k in w if k in out).backward()
    torch.cuda.synchronize()
    got = view.grad.cpu().numpy().astype(np.float64)
    assert not np.any(got[12:])  # cam_pos: no cotangent
    want = cc.v_view_ref(case.frame, case.st, h.v_records.cpu().numpy())
    if not np.any(want):
        assert not np.any(got[:12]), f"{name}: nothing visible, v_view must be exactly zero"
    else:
        e = pz.rel_l2(got[:12], want)
        assert e <= TOL, f"{name}: relative L2 {e:.2e}\n{got[:12]}\n{want}"
        print(f"[view] {name}: relative L2 {e:.2e}")
    if pose is not None:  # v_pose beside it: what the pose-only render gives
        pose2 = torch.from_numpy(base).to(DEV).requires_grad_(True)
        out2, _ = raster.render_frame(frc, st, pose=pose2)
        sum((out2[k] * w[k]).sum() for k in w if k in out2).backward()
        want_p = pz.v_pose_ref(case.frame, case.st, h.v_records.cpu().numpy())
        gp = pose.grad.cpu().numpy().astype(np.float64)
        for a in range(want_p.shape[0]):
            if np.any(want_p[a]):
                assert pz.rel_l2(gp[a], want_p[a]) <= TOL
        assert np.allclose(gp, pose2.grad.cpu().numpy(), rtol=1e-4, atol=1e-6 * float(np.abs(gp).max() + 1e-30))


def _config3():
    fr = syn.config_frame(3)
    return fr, _cuda_frame(fr)


def _skewt(w):
    return cc.skew(torch.as_tensor(w, dtype=F64, device=DEV))


def test_full_size_plumbing_invariance_and_reproducibility():
    L = _lib.load()
    fr, frc = _config3()
    st = raster.RenderSettings()
    cs = raster.camera_struct(frc.camera, st)
    params = [s.params.tensors() for s in frc.segments]
    view = own_view(frc.camera)

    # the camera's own view on the device: same launches, same bits
    n0 = L.sgn_launch_count()
    out0, h0 = raster.render_frame(frc, st)
    n1 = L.sgn_launch_count()
    out1, h1 = raster.render_frame(frc, st, view=view)
    n2 = L.sgn_launch_count()
    assert n1 - n0 == n2 - n1
    for k in out0:
        assert torch.equal(out0[k], out1[k]), k
    assert torch.equal(h0.records, h1.records) and torch.equal(h0.radii, h1.radii)
    p0 = raster.project_fwd(h0.table, cs, DEV)
    p1 = raster.project_fwd(h0.table, cs, DEV, view)
    for a, b in zip((p0.tiles_touched, p0.touch_mask, p0.bbox, p0.tiles_hit), (p1.tiles_touched, p1.touch_mask, p1.bbox, p1.tiles_hit)):
        assert torch.equal(a, b)

    w, v = syn.cotangents(cs.height, cs.width)
    cot = {"rgb": w.to(DEV), "accumulation": v[..., None].to(DEV), "object_acc": (0.1 * v)[..., None].to(DEV)}
    _, hb = raster.forward_backward(frc, st, cot, want_param_grads=True)
    v_records, flat, arena = hb.v_records, hb.param_grads, hb.grad_arena.clone()
    v_view = torch.empty(12, device=DEV)
    v_pose = torch.empty(len(frc.segments), 16, device=DEV)
    a0 = L.sgn_launch_count()
    _, arena_v = raster.project_bwd(h0.table, params, cs, h0.records, h0.radii, v_records, make_views=False, view=view, v_view=v_view,
                                    v_pose=v_pose)
    assert L.sgn_launch_count() - a0 == 3
    assert torch.equal(arena, arena_v)
    vp_only = torch.empty_like(v_pose)
    raster.project_bwd(h0.table, params, cs, h0.records, h0.radii, v_records, make_views=False, v_pose=vp_only)
    assert torch.equal(v_pose, vp_only)
    again = torch.empty_like(v_view)
    raster.project_bwd(h0.table, params, cs, h0.records, h0.radii, v_records, make_views=False, view=view, v_view=again)
    assert torch.equal(v_view, again)
    nc = h0.table.num_chunks
    cuts = [0, 1, nc // 3, int(h0.table.host["chunk0"][1]) + 7, nc - 1, nc]
    ranged = torch.empty_like(v_view)
    _, arena_r = raster.project_bwd(h0.table, params, cs, h0.records, h0.radii, v_records, make_views=False, view=view, v_view=ranged,
                                    chunk_ranges=list(zip(cuts[:-1], cuts[1:])))
    assert torch.equal(v_view, ranged) and torch.equal(arena, arena_r)

    # invariance: camera motion p_c -> (I + e Omega) p_c + e tau  ==  world motion p_w -> (I + e Omega_w) p_w + e d,
    # Omega_w = W^T Omega W, d = W^T (Omega c + tau)
    Wc = torch.from_numpy(frc.camera.viewmat().astype(np.float64)).to(DEV)
    Wm, c = Wc[:, :3], Wc[:, 3]
    vW = v_view.double().reshape(3, 4)
    worst = 0.0
    for kind in range(6):
        omega = torch.zeros(3, dtype=F64, device=DEV)
        tau = torch.zeros(3, dtype=F64, device=DEV)
        (omega if kind >= 3 else tau)[kind % 3] = 1.0
        Om = _skewt(omega)
        lhs = float((vW[:, :3] * (Om @ Wm)).sum() + (vW[:, 3] * (Om @ c + tau)).sum())
        ow = Wm.T @ omega
        Omw = _skewt(ow)
        d = Wm.T @ (Om @ c + tau)
        dq = torch.cat([torch.zeros(1, dtype=F64, device=DEV), 0.5 * ow])
        rhs, mag = 0.0, 0.0
        for i, seg in enumerate(frc.segments):
            if not seg.has_pose:
                m, q = seg.params.means.double(), seg.params.quats.double()
                gm, gq = flat[6 * i].double(), flat[6 * i + 2].double()
                t1 = gm * (m @ Omw.T + d)
                t2 = gq * pz_quat_mul(dq[None].expand_as(q), q)
            else:
                R, t, a = (torch.from_numpy(x.astype(np.float64)).to(DEV) for x in seg.pose_f32())
                R = R.reshape(3, 3)
                vp = v_pose[i].double()
                t1 = torch.cat([(vp[0:9].reshape(3, 3) * (Omw @ R)).reshape(-1), vp[9:12] * (Omw @ t + d)])
                t2 = vp[12:16] * pz_quat_mul(dq, a)
            rhs += float(t1.sum() + t2.sum())
            mag += float(t1.abs().sum() + t2.abs().sum())
        err = abs(lhs - rhs) / max(abs(rhs), 1e-3 * mag)
        worst = max(worst, err)
        assert err <= TOL, f"direction {kind}: camera {lhs} vs world {rhs} (sum |terms| {mag})"
    print(f"[view] config 3 invariance: worst relative error {worst:.2e}")


def pz_quat_mul(a, b):
    aw, ax, ay, az = a.unbind(-1)
    bw, bx, by, bz = b.unbind(-1)
    return torch.stack([aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
                        aw * by - ax * bz + ay * bw + az * bx, aw * bz + ax * by - ay * bx + az * bw], -1)


def test_adjust_kernels_against_float64():
    cam = syn.make_camera(320, 240)
    co = CameraPoseOptimizer(5).to(DEV)
    g = torch.Generator().manual_seed(3)
    for x in (torch.zeros(6), torch.tensor([0.05, -0.02, 0.03, 0.002, -0.003, 0.001]), torch.randn(6, generator=g) * 0.3):
        with torch.no_grad():
            co.pose_adjustment.zero_()
            co.pose_adjustment[2] = x
        co.pose_adjustment.grad = None
        cam.index = 2
        view = co.view(cam)
        c2w = torch.from_numpy(cam.c2w.astype(np.float64))
        x64 = x.double().requires_grad_(True)
        want = cc.view_of(c2w, x64)
        got = view.detach().cpu().double()
        assert float((got - want.detach()).abs().max()) <= 1e-6 * float(want.detach().abs().max())
        gv = torch.randn(15, generator=g)
        gv[12:] = 0
        (view * gv.to(DEV)).sum().backward()
        (want_g,) = torch.autograd.grad((want * gv.double()).sum(), x64)
        grad = co.pose_adjustment.grad.cpu().double()
        assert not grad[[0, 1, 3, 4]].any()
        assert pz.rel_l2(grad[2].numpy(), want_g.numpy()) <= TOL


def test_sky_with_a_view_samples_the_corrected_camera():
    cam = syn.make_camera(160, 96)
    co = CameraPoseOptimizer(1).to(DEV)
    with torch.no_grad():
        co.pose_adjustment[0] = torch.tensor([0.1, 0.0, -0.2, 0.05, -0.1, 0.08])
    cam.index = 0
    view = co.view(cam)
    c2w = cc.adjusted_c2w(torch.from_numpy(cam.c2w.astype(np.float64)), co.pose_adjustment[0].detach().cpu().double())
    moved = Camera(c2w.numpy().astype(np.float32), cam.fx, cam.fy, cam.cx, cam.cy, cam.width, cam.height)
    sky = CubeMapSky(resolution=16).to(DEV)
    with torch.no_grad():
        sky.base.copy_(torch.rand(6, 16, 16, 3, generator=torch.Generator().manual_seed(1)))
    a = sky(cam, False, view=view)
    b = sky(moved, False)
    assert float((a - b).abs().max()) <= 1e-5
    assert not torch.equal(a, sky(cam, False))
    a.sum().backward()
    assert co.pose_adjustment.grad is None and float(sky.base.grad.abs().sum()) > 0


# ---- model level ------------------------------------------------------------------------------------------------------
W, H = 320, 240


def _scene(seed=3):
    return syn.make_frame(n_background=20000, n_actors=0, n_per_actor=0, width=W, height=H, seed=seed)


def _model(fr, co=None, sky=None):
    m = SceneGraphRasterModel(fr.segments[0].params.to(DEV), {}, SceneGraphConfig(use_sky_sphere=sky is not None, ssim_lambda=0.2),
                              sky=sky, camera_optimizer=co).to(DEV)
    m.train()
    return m


def _gt(seed=2):
    return (torch.rand(H, W, 3, generator=torch.Generator().manual_seed(seed)) * 0.5 + 0.25).to(DEV)


def test_unchanged_paths_launch_and_render_as_today(monkeypatch):
    """Training without an optimizer / in mode "off" / with a camera without an index, and eval with an optimizer against eval
    without one: the render's launches (the camera regulariser of get_loss_dict, a loss term of its own, is not counted) and
    every output are the same."""
    monkeypatch.setattr(raster, "DETERMINISTIC", True)
    fr = _scene()
    L = _lib.load()
    runs = []
    for co, index, train in ((None, 0, True), (CameraPoseOptimizer(3, "off"), 0, True), (CameraPoseOptimizer(3), None, True),
                             (None, 0, False), (CameraPoseOptimizer(3), 0, False)):
        m = _model(fr, co)
        m.train(train)
        cam = fr.camera
        cam.index = index
        n0 = L.sgn_launch_count()
        out = m.get_outputs(cam)
        n = L.sgn_launch_count() - n0
        arena = None
        if train:
            losses = m.get_loss_dict(out, {"image": _gt()})
            n1 = L.sgn_launch_count()
            sum(v for k, v in losses.items() if k != "camera_opt_regularizer").backward()
            torch.cuda.synchronize()
            n += L.sgn_launch_count() - n1
            arena = m._holder.grad_arena.clone()
        torch.cuda.synchronize()
        runs.append((n, {k: v.detach() for k, v in out.items()}, arena))
    cam.index = None
    for n, out, arena in runs[1:3]:
        assert n == runs[0][0] and all(torch.equal(out[k], runs[0][1][k]) for k in runs[0][1]) and torch.equal(arena, runs[0][2])
    (n_ev0, out_ev0, _), (n_ev1, out_ev1, _) = runs[3], runs[4]
    assert n_ev1 == n_ev0 and out_ev1.keys() == out_ev0.keys() and all(torch.equal(out_ev1[k], out_ev0[k]) for k in out_ev0)
    assert not out_ev1["rgb"].requires_grad


def test_regulariser_and_metrics_kernels_against_float64():
    """sgn_camera_adjust_fwd / _bwd over 600 cameras (more rows than the block has threads), some rows all zero, some with a
    zero translation or rotation only: the regulariser, the norms, and the gradient of view and regulariser together."""
    n = 600
    g = torch.Generator().manual_seed(9)
    x = torch.randn(n, 6, generator=g) * 0.05
    x[::7] = 0.0
    x[1::11, :3] = 0.0
    x[2::13, 3:] = 0.0
    co = CameraPoseOptimizer(n).to(DEV)
    with torch.no_grad():
        co.pose_adjustment.copy_(x)
    cam = syn.make_camera(320, 240)
    cam.index = 15
    L = _lib.load()
    n0 = L.sgn_launch_count()
    view, reg, norms = co.terms(cam)
    assert L.sgn_launch_count() - n0 == 1
    x64 = x.double().requires_grad_(True)
    want_reg = cc.regularizer(x64)
    want_m = cc.metrics(x64.detach())
    assert abs(float(reg) - float(want_reg.detach())) <= 1e-6 * float(want_reg.detach())
    assert abs(float(norms[0]) - float(want_m["camera_opt_translation"])) <= 1e-6 * float(want_m["camera_opt_translation"])
    assert abs(float(norms[1]) - float(want_m["camera_opt_rotation"])) <= 1e-6 * float(want_m["camera_opt_rotation"])
    assert not norms.requires_grad and reg.requires_grad and view.requires_grad
    gv = torch.randn(15, generator=g)
    gv[12:] = 0
    n0 = L.sgn_launch_count()
    ((view * gv.to(DEV)).sum() + 3.0 * reg).backward()
    assert L.sgn_launch_count() - n0 == 1
    want_view = cc.view_of(torch.from_numpy(cam.c2w.astype(np.float64)), x64[15])
    (want_g,) = torch.autograd.grad((want_view * gv.double()).sum() + 3.0 * want_reg, x64)
    got = co.pose_adjustment.grad.cpu().double()
    assert torch.equal(got[::7], torch.zeros_like(got[::7]))  # a zero row's norms have a zero gradient
    assert pz.rel_l2(got.numpy(), want_g.numpy()) <= TOL
    assert pz.rel_l2(got[15].numpy(), want_g[15].numpy()) <= TOL
    # the metrics and the regulariser alone: the same kernel without a view, no gradient for the norms
    m = co.metrics()
    assert torch.equal(m["camera_opt_translation"], norms[0]) and torch.equal(m["camera_opt_rotation"], norms[1])
    co.pose_adjustment.grad = None
    co.regularizer().backward()
    (want_r,) = torch.autograd.grad(cc.regularizer(x64), x64)
    assert pz.rel_l2(co.pose_adjustment.grad.cpu().double().numpy(), want_r.numpy()) <= 1e-5
    # an in-place change between forward and backward is caught by autograd's version check
    view, reg, _ = co.terms(cam)
    with torch.no_grad():
        co.pose_adjustment.add_(1.0)
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        (view.sum() + reg).backward()


def test_nothing_in_view_still_steps_the_camera_on_its_count():
    """A camera facing away from the whole scene: no render gradient, only the regulariser's.  With an accumulation of 2 the
    tensor moves at step 1 (step % 2 == 1), by Adam on the regulariser's gradient, as nerfstudio steps the group."""
    fr = _scene()
    co = CameraPoseOptimizer(2)
    m = _model(fr, co)
    m.config.async_binning = False  # the exact count: nothing in view takes the reference's early-out
    with torch.no_grad():
        co.pose_adjustment.copy_(torch.tensor([[0.1, -0.2, 0.05, 0.01, 0.02, -0.03], [0.0, 0.3, 0.0, 0.0, 0.0, 0.04]], device=DEV))
    away = np.concatenate([np.diag([-1.0, 1.0, -1.0]), np.zeros((3, 1))], 1)  # looks along +z: the scene lies behind it
    cam = syn.make_camera(W, H, c2w=away)
    cam.index = 0
    opt = FusedAdam(m.optimizer_params(), extra={"camera_opt.pose_adjustment": (co.pose_adjustment, 1e-3)})
    step_fn = TrainStep(m, opt, refine_every=0, gradient_accumulation_steps={"camera_opt.pose_adjustment": 2})
    ref = co.pose_adjustment.detach().clone().requires_grad_(True)
    twin = torch.optim.Adam([ref], lr=1e-3, eps=1e-15)
    before = co.pose_adjustment.detach().clone()
    step_fn(0, cam, {"image": _gt()})
    assert m._holder.grad_arena is None and torch.equal(co.pose_adjustment.detach(), before)
    step_fn(1, cam, {"image": _gt()})
    torch.cuda.synchronize()
    (g1,) = torch.autograd.grad(cc.regularizer(ref), ref)
    ref.grad = 2 * g1
    twin.step()
    assert not torch.equal(co.pose_adjustment.detach(), before)
    assert torch.allclose(co.pose_adjustment.detach(), ref.detach(), rtol=1e-5, atol=1e-9)


def test_sky_must_take_a_view():
    fr = _scene()
    with pytest.raises(TypeError):
        _model(fr, CameraPoseOptimizer(1), sky=lambda cam, train: torch.zeros(H, W, 3, device=DEV))
    _model(fr, CameraPoseOptimizer(1, "off"), sky=lambda cam, train: torch.zeros(H, W, 3, device=DEV))


def test_backward_regulariser_metrics_and_adam():
    fr = _scene()
    co = CameraPoseOptimizer(4)
    m = _model(fr, co, sky=CubeMapSky(resolution=32))
    with torch.no_grad():
        co.pose_adjustment.normal_(0, 0.01)
    cam = fr.camera
    cam.index = 1
    out = m.get_outputs(cam)
    losses = m.get_loss_dict(out, {"image": _gt()})
    assert "camera_opt_regularizer" in losses
    metrics = m.get_metrics_dict(out, {"image": _gt()})
    assert metrics["camera_opt_translation"].is_cuda and metrics["camera_opt_rotation"].is_cuda
    sum(losses.values()).backward()
    g = co.pose_adjustment.grad.clone()
    # the chain's share lands in row 1 only; the regulariser's everywhere
    x = co.pose_adjustment.detach().clone().requires_grad_(True)
    (g_reg,) = torch.autograd.grad(cc.regularizer(x), x)
    chain = g - g_reg
    assert float(chain[[0, 2, 3]].abs().max()) <= 1e-8 and float(chain[1].abs().max()) > 0
    view = co.view(cam)
    vv = m._holder.v_view
    (want,) = torch.autograd.grad(view, co.pose_adjustment, grad_outputs=torch.cat([vv, torch.zeros(3, device=DEV)]))
    assert torch.allclose(chain, want, rtol=1e-5, atol=1e-9)

    # FusedAdam moves the tensor as torch.optim.Adam does
    co.pose_adjustment.grad = None
    opt = FusedAdam(m.optimizer_params(), extra={"camera_opt.pose_adjustment": (co.pose_adjustment, 1e-3),
                                                 "sky": (m.env_map.base, 0.005)})
    step_fn = TrainStep(m, opt, refine_every=0)
    ref = co.pose_adjustment.detach().clone().requires_grad_(True)
    twin = torch.optim.Adam([ref], lr=1e-3, eps=1e-15)
    for step in range(3):
        step_fn(step, cam, {"image": _gt()})
        ref.grad = co.pose_adjustment.grad.clone()
        twin.step()
    torch.cuda.synchronize()
    assert torch.allclose(co.pose_adjustment.detach(), ref.detach(), rtol=1e-5, atol=1e-9)


def test_gradient_accumulation_steps():
    fr = _scene()
    co = CameraPoseOptimizer(2)
    m = _model(fr, co)
    cam = fr.camera
    cam.index = 0
    opt = FusedAdam(m.optimizer_params(), extra={"camera_opt.pose_adjustment": (co.pose_adjustment, 1e-3)})
    with pytest.raises(ValueError):
        TrainStep(m, opt, gradient_accumulation_steps={"camera_opt": 4})
    step_fn = TrainStep(m, opt, refine_every=0, gradient_accumulation_steps={"camera_opt.pose_adjustment": 4})
    ref = co.pose_adjustment.detach().clone().requires_grad_(True)
    twin = torch.optim.Adam([ref], lr=1e-3, eps=1e-15)
    acc = torch.zeros_like(ref)
    prev = co.pose_adjustment.detach().clone()
    for step in range(8):
        step_fn(step, cam, {"image": _gt(step)})
        torch.cuda.synchronize()
        acc = co.pose_adjustment.grad.clone()
        now = co.pose_adjustment.detach().clone()
        if step % 4 == 3:
            ref.grad = acc.clone()
            twin.step()
            assert not torch.equal(now, prev)
            assert torch.allclose(now, ref.detach(), rtol=1e-5, atol=1e-9)
        else:
            assert torch.equal(now, prev)
        prev = now
    assert opt.steps[opt.extra_index["camera_opt.pose_adjustment"]] == 2


def _train_det(steps):
    torch.manual_seed(0)
    fr = _scene()
    co = CameraPoseOptimizer(2)
    m = _model(fr, co, sky=CubeMapSky(resolution=32))
    cam = fr.camera
    cam.index = 1
    opt = FusedAdam(m.optimizer_params(), extra={"camera_opt.pose_adjustment": (co.pose_adjustment, 1e-3),
                                                 "sky": (m.env_map.base, 0.005)})
    step_fn = TrainStep(m, opt, refine_every=0)
    for step in range(steps):
        step_fn(step, cam, {"image": _gt()})
    torch.cuda.synchronize()
    return {"pa": co.pose_adjustment.detach().clone(), "grad": co.pose_adjustment.grad.clone(), "v_view": m._holder.v_view.clone(),
            "means": m.all_models["background"].gauss_params["means"].detach().clone(), "exp_avg": opt.exp_avg.clone()}


def test_deterministic_training_steps_repeat_bit_for_bit(monkeypatch):
    monkeypatch.setattr(raster, "DETERMINISTIC", True)
    a, b = _train_det(4), _train_det(4)
    diff = [k for k in a if not torch.equal(a[k], b[k])]
    assert not diff, diff
    assert float(a["pa"].abs().max()) > 0


def test_perturbed_camera_is_pulled_back():
    """Targets rendered from the true camera; the dataset camera is off by 5 cm and 0.5 degree; the Gaussians are frozen and
    pose_adjustment alone is optimised: the loss falls and both errors end below a quarter of where they started."""
    fr = syn.make_frame(n_background=30000, n_actors=0, n_per_actor=0, width=W, height=H, seed=7)
    true = fr.camera
    m = _model(fr)
    m.config.ssim_lambda = 0.0
    m.step = 30000
    with torch.no_grad():
        target = m.get_outputs(true)["rgb"].detach()
    axis = np.array([0.3, -0.5, 0.8]) / np.linalg.norm([0.3, -0.5, 0.8])
    ang = np.deg2rad(0.5)
    dt = np.array([0.03, -0.03, 0.028])
    dt = 0.05 * dt / np.linalg.norm(dt)
    x_err = torch.tensor(np.concatenate([dt, axis * ang]), dtype=F64)
    c2w = cc.adjusted_c2w(torch.from_numpy(true.c2w.astype(np.float64)), x_err).numpy()
    cam = Camera(c2w.astype(np.float32), true.fx, true.fy, true.cx, true.cy, true.width, true.height, index=0)
    co = CameraPoseOptimizer(1).to(DEV)
    m.camera_optimizer = co
    for p in m.all_models.parameters():
        p.requires_grad_(False)
    opt = torch.optim.Adam([co.pose_adjustment], lr=1e-3, eps=1e-15)

    def errors():
        got = cc.adjusted_c2w(torch.from_numpy(c2w), co.pose_adjustment.detach().cpu().double()[0])
        R = got[:, :3].T @ torch.from_numpy(true.c2w[:, :3].astype(np.float64))
        ang_err = float(torch.arccos(torch.clamp((torch.trace(R) - 1) / 2, -1, 1)))
        return float((got[:, 3] - torch.from_numpy(true.c2w[:, 3].astype(np.float64))).norm()), ang_err

    t0, r0 = errors()
    first = None
    for it in range(300):
        opt.zero_grad()
        out = m.get_outputs(cam)
        loss = torch.abs(out["rgb"] - target).mean()
        first = float(loss) if first is None else first
        loss.backward()
        opt.step()
    t1, r1 = errors()
    print(f"[camera] translation {t0:.4f} -> {t1:.4f} m, rotation {r0:.5f} -> {r1:.5f} rad, loss {first:.4f} -> {float(loss):.4f}")
    assert float(loss) < first and t1 < 0.25 * t0 and r1 < 0.25 * r0
