"""The gradient of the actor boxes on the GPU: pose cotangents out of the projection backward (sgn_project_bwd_pose +
sgn_pose_grad_reduce), poses as a differentiable input of the render, and ``box_pose.BoxPoseOptimizer`` through the model.

  * directed: hand-built frames (tests/pose_cases.py: one actor; a background and actors of 300 / 50 / 128 / 0 rows; an actor
    entirely off screen; an actor cut by the near plane) rendered with rgb / accumulation / object_acc cotangents -- each of
    v_R, v_t, v_q of every actor within 1e-3 relative L2 of float64 autograd over the same record cotangents (the blend
    backward that produces them has its own directed tests), exact zeros where no row is visible; the same with random
    record cotangents straight through ``raster.project_bwd``;
  * full size (config 3): since R is orthonormal and q_box a unit quaternion, vmw_i = R g_means_i and vqr_i = q_box (x) g_quats_i,
    so v_pose must equal float64 sums built from the parameter gradients the library already returns;
  * unchanged paths: without ``pose`` the launch count and every output are what they are with the frame's own poses passed
    in; the pose form writes a bit-identical gradient arena; the range form gives a bit-identical v_pose;
  * reproducibility: v_pose repeats bit for bit over the same v_records; in deterministic mode whole training steps with the box
    corrections on repeat bit for bit;
  * model: ``loss.backward()`` leaves the chain poses-autograd o v_pose on delta_center / delta_yaw, only in the frame's rows;
    ``FusedAdam(extra=...)`` moves them as ``torch.optim.Adam`` does;
  * purpose: from boxes displaced by 0.2 m and a yaw parameter off by 0.05, optimising the corrections alone brings the loss
    down and both errors below a quarter of where they started.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import street_gaussians_ns_b200.synthetic as syn
from street_gaussians_ns_b200 import _lib, raster
from street_gaussians_ns_b200.box_pose import BoxPoseOptimizer
from street_gaussians_ns_b200.model import ActorPose, SceneGraphConfig, SceneGraphRasterModel
from street_gaussians_ns_b200.optim import FusedAdam
from street_gaussians_ns_b200.scene import CLS_OBJECT, Frame, GaussianSet, Segment
from street_gaussians_ns_b200.training import TrainStep
from tests import pose_cases as pz

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
TOL = 1e-3  # the project's gradient bar: relative L2 against float64


def _settings(case):
    st = case.st
    return raster.RenderSettings(sh_degree=st.sh_degree, sh_degree_to_use=st.deg_use, block_width=st.block_width, clip_thresh=st.clip_thresh)


def _cuda_frame(frame):
    return Frame(frame.camera, [Segment(s.params.to("cuda"), s.cls, s.rot, s.center, s.idft, s.name) for s in frame.segments])


def _weights(H, W, seed=5):
    g = torch.Generator().manual_seed(seed)
    return {"rgb": torch.rand(H, W, 3, generator=g).to(DEV), "accumulation": torch.rand(H, W, 1, generator=g).to(DEV),
            "object_acc": torch.rand(H, W, 1, generator=g).to(DEV)}


def _render_backward(frame, settings, pose, **kw):
    out, h = raster.render_frame(frame, settings, pose=pose, **kw)
    w = _weights(frame.camera.height, frame.camera.width)
    sum((out[k] * w[k]).sum() for k in w).backward()
    return out, h


def _check_groups(name, got, want):
    worst = 0.0
    for a in range(want.shape[0]):
        for label, g, r in zip(("v_R", "v_t", "v_q"), pz.groups(got[a:a + 1]), pz.groups(want[a:a + 1])):
            if not np.any(r):
                assert not np.any(g), f"{name}: {label} of actor {a} must be exactly zero"
                continue
            e = pz.rel_l2(g, r)
            worst = max(worst, e)
            assert e <= TOL, f"{name}: {label} of actor {a}: relative L2 {e:.2e}\n{g}\n{r}"
    return worst


@pytest.mark.parametrize("name", list(pz.CASES))
def test_directed_against_float64(name):
    case = pz.get(name)
    frc = _cuda_frame(case.frame)
    base = pz.frame_poses(case.frame)
    pose = torch.from_numpy(base).to(DEV).requires_grad_(True)
    _, h = _render_backward(frc, _settings(case), pose)
    torch.cuda.synchronize()
    got = pose.grad.cpu().numpy().astype(np.float64)
    assert got.shape == base.shape and np.isfinite(got).all()
    want = pz.v_pose_ref(case.frame, case.st, h.v_records.cpu().numpy())
    worst = _check_groups(name, got, want)
    assert np.abs(want).max() > 0
    # holder.v_pose: one row per segment, zeros for the segments without a pose
    posed = np.array([s.has_pose for s in case.frame.segments])
    vp = h.v_pose.cpu().numpy()
    assert np.array_equal(vp[posed], pose.grad.cpu().numpy()) and not np.any(vp[~posed])
    # random record cotangents straight through the stage wrapper
    params = [s.params.tensors() for s in frc.segments]
    v = torch.from_numpy(pz.pc.v_records(case, "all")).to(DEV)
    v_pose = torch.full((len(frc.segments), 16), float("nan"), device=DEV)
    raster.project_bwd(h.table, params, raster.camera_struct(frc.camera, _settings(case)), h.records, h.radii, v, v_pose=v_pose)
    want2 = pz.v_pose_ref(case.frame, case.st, v.cpu().numpy())
    worst2 = _check_groups(name + " [random v_records]", v_pose.cpu().numpy().astype(np.float64)[posed], want2)
    print(f"[pose] {name}: worst relative L2 {worst:.2e} (render), {worst2:.2e} (random record cotangents)")


def test_off_screen_actor_and_empty_actor_get_exact_zeros():
    for name, actor in (("off_screen", 1), ("actors_and_background", 3)):
        case = pz.get(name)
        pose = torch.from_numpy(pz.frame_poses(case.frame)).to(DEV).requires_grad_(True)
        _render_backward(_cuda_frame(case.frame), _settings(case), pose)
        g = pose.grad.cpu().numpy()
        assert not np.any(g[actor]) and np.any(g[0])


def _config3():
    fr = syn.config_frame(3)
    return fr, _cuda_frame(fr)


def test_full_size_self_consistency_and_unchanged_paths():
    """Config 3 (1 M background + 32 x 10 k actor Gaussians, 1920 x 1280)."""
    L = _lib.load()
    fr, frc = _config3()
    st = raster.RenderSettings()
    cs = raster.camera_struct(frc.camera, st)
    params = [s.params.tensors() for s in frc.segments]
    base = torch.from_numpy(pz.frame_poses(fr)).to(DEV)

    # without pose / with the frame's own poses as a constant: same launches, same bits
    n0 = L.sgn_launch_count()
    out0, h0 = raster.render_frame(frc, st)
    n1 = L.sgn_launch_count()
    out1, h1 = raster.render_frame(frc, st, pose=base)
    n2 = L.sgn_launch_count()
    assert n1 - n0 == n2 - n1
    for k in out0:
        assert torch.equal(out0[k], out1[k]), k
    assert torch.equal(h0.records, h1.records) and torch.equal(h0.radii, h1.radii)
    assert h1.table.dev.data_ptr() != h0.table.dev.data_ptr() and torch.equal(h1.table.dev, h0.table.dev)

    # backward: sgn_project_bwd vs the pose form -- the arena is bit-identical, the pose form adds one launch and v_pose
    w, v = syn.cotangents(cs.height, cs.width)
    cot = {"rgb": w.to(DEV), "accumulation": v[..., None].to(DEV), "object_acc": (0.1 * v)[..., None].to(DEV)}
    _, hb = raster.forward_backward(frc, st, cot, want_param_grads=True)
    v_records, flat, arena = hb.v_records, hb.param_grads, hb.grad_arena.clone()
    a0 = L.sgn_launch_count()
    _, again0 = raster.project_bwd(h0.table, params, cs, h0.records, h0.radii, v_records, make_views=False)
    assert torch.equal(arena, again0)
    a1 = L.sgn_launch_count()
    v_pose = torch.empty(len(frc.segments), 16, device=DEV)
    _, arena_p = raster.project_bwd(h0.table, params, cs, h0.records, h0.radii, v_records, make_views=False, v_pose=v_pose)
    a2 = L.sgn_launch_count()
    assert (a1 - a0, a2 - a1) == (1, 2)
    assert torch.equal(arena, arena_p)

    # two passes over the same v_records, and the range form: the same bits
    again = torch.empty_like(v_pose)
    raster.project_bwd(h0.table, params, cs, h0.records, h0.radii, v_records, make_views=False, v_pose=again)
    assert torch.equal(v_pose, again)
    nc = h0.table.num_chunks
    cuts = [0, 1, nc // 3, int(h0.table.host["chunk0"][1]) + 7, nc - 1, nc]
    ranged = torch.empty_like(v_pose)
    _, arena_r = raster.project_bwd(h0.table, params, cs, h0.records, h0.radii, v_records, make_views=False, v_pose=ranged,
                                    chunk_ranges=list(zip(cuts[:-1], cuts[1:])))
    assert torch.equal(v_pose, ranged) and torch.equal(arena, arena_r)

    # self-consistency: float64 sums built from the parameter gradients.  Each of the 16 values is a float32 sum of n = 10 000
    # products in a fixed tree (32 lanes, 4 warps, 79 chunks): its error is bounded by (depth of the tree + the rounding of
    # a term) x eps x sum |terms|; the terms rebuilt from the returned gradients (R g, q_box (x) g) carry a few eps of their
    # own.  Bar: 64 eps sum |terms|.
    eps = float(np.finfo(np.float32).eps)
    assert not np.any(v_pose[0].cpu().numpy())  # the background has no pose
    worst, in_view = 0.0, 0
    for i, seg in enumerate(frc.segments):
        if not seg.has_pose:
            continue
        R, _, a = (torch.from_numpy(x.astype(np.float64)).to(DEV) for x in seg.pose_f32())
        g_m, g_q = flat[6 * i].double(), flat[6 * i + 2].double()
        m, q = seg.params.means.double(), seg.params.quats.double()
        vmw = g_m @ R.reshape(3, 3).T
        vqr = _quat_mul(a[None, :].expand_as(g_q), g_q)
        conj = q * torch.tensor([1.0, -1.0, -1.0, -1.0], device=DEV, dtype=torch.float64)
        terms = torch.cat([(vmw[:, :, None] * m[:, None, :]).reshape(-1, 9), vmw], 1)
        want = torch.cat([terms.sum(0), _quat_mul(vqr, conj).sum(0)])
        mag = torch.cat([terms.abs().sum(0), (vqr.abs().sum(1) * q.abs().amax(1)).sum(0).expand(4)])
        err = (v_pose[i].double() - want).abs()
        ratio = float((err / (64 * eps * mag + 1e-30)).max())
        worst = max(worst, ratio)
        assert ratio <= 1.0, f"segment {i}: {v_pose[i].tolist()} vs {want.tolist()}"
        in_view += int(float(want.abs().max()) > 0)
    assert in_view >= 8  # the camera sees part of the 4 x 8 grid of actors; the others get exact zeros
    print(f"[pose] config 3 self-consistency: {in_view} actors in view, worst error {worst:.3f} of 64 eps sum|terms|")


def _quat_mul(a, b):
    aw, ax, ay, az = a.unbind(-1)
    bw, bx, by, bz = b.unbind(-1)
    return torch.stack([aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
                        aw * by - ax * bz + ay * bw + az * bx, aw * bz + ax * by - ay * bx + az * bw], -1)


def test_pose_argument_is_validated_and_resident_rows_are_not_written():
    case = pz.get("actors_and_background")
    frc = _cuda_frame(case.frame)
    st = _settings(case)
    base = torch.from_numpy(pz.frame_poses(case.frame)).to(DEV)
    for bad in (base[:2], base.double(), base.cpu(), base[:, :12]):
        with pytest.raises(_lib.SgnError):
            raster.render_frame(frc, st, pose=bad)
    params = [s.params.tensors() for s in frc.segments]
    table = raster.SegmentTable(frc, params, DEV)
    before = table.dev.clone()
    moved = base.clone()
    moved[:, 9:12] += 0.25
    posed = raster.with_poses(table, moved)
    assert torch.equal(table.dev, before) and not torch.equal(posed.dev, before)
    rows = posed.dev.view(torch.float32).view(-1, raster.SEG_FLOATS)
    assert torch.equal(rows[1:, raster.POSE_OFFSET:raster.POSE_OFFSET + 16], moved)
    # everything but the 16 floats of the posed rows is the original
    keep = torch.ones_like(rows, dtype=torch.bool)
    keep[1:, raster.POSE_OFFSET:raster.POSE_OFFSET + 16] = False
    assert torch.equal(rows[keep].view(torch.int32), before.view(torch.float32).view(-1, raster.SEG_FLOATS)[keep].view(torch.int32))
    # a moved pose moves the render
    a, _ = raster.render_frame(frc, st)
    b, _ = raster.render_frame(frc, st, pose=moved)
    assert not torch.equal(a["rgb"], b["rgb"])


def test_null_and_range_checks_launch_nothing():
    L = _lib.load()
    cs = _lib.CameraStruct()
    p = C.c_void_p(256)
    before = L.sgn_launch_count()
    assert L.sgn_project_bwd_pose(p, p, 1, 10, 1, C.byref(cs), p, p, p, 0, 1, None, None) == -1
    assert b"pose_partials" in L.sgn_last_error()
    assert L.sgn_project_bwd_pose(p, p, 1, 10, 1, C.byref(cs), p, p, p, 0, 2, p, None) == -1
    assert b"chunk range" in L.sgn_last_error()
    assert L.sgn_project_bwd_pose(p, p, 0, 10, 1, C.byref(cs), p, p, p, 0, 1, p, None) == -1
    assert L.sgn_pose_grad_reduce(None, 1, 1, p, p, None) == -1
    assert L.sgn_pose_grad_reduce(p, 1, 1, None, p, None) == -1
    assert L.sgn_pose_grad_reduce(p, 2000, 1, p, p, None) == -1
    assert L.sgn_launch_count() == before


# ---- model level ------------------------------------------------------------------------------------------------------
W, H, FRAME, NUM_FRAMES = 320, 240, 21, 85


def _scene(seed=3):
    fr = syn.make_frame(n_background=20000, n_actors=3, n_per_actor=1500, width=W, height=H, seed=seed, frame=FRAME,
                        actor_shift=np.array([2.0, 0.0, -3.0]))  # all three actors in view
    return fr


def _model(fr, mode="simple", cfg=None, boxes=None):
    bg = fr.segments[0].params.to(DEV)
    names = [s.name.replace("object_", "") for s in fr.segments[1:]]
    actors = {n: s.params.to(DEV) for n, s in zip(names, fr.segments[1:])}
    poses = boxes or [ActorPose(n, s.rot, s.center, FRAME, list(range(NUM_FRAMES)), frame_id=FRAME) for n, s in zip(names, fr.segments[1:])]
    bo = None if mode is None else BoxPoseOptimizer(NUM_FRAMES, names + ["never_seen"], {f: f for f in range(NUM_FRAMES)}, mode=mode)
    model = SceneGraphRasterModel(bg, actors, cfg or SceneGraphConfig(use_sky_sphere=False, ssim_lambda=0.2), poses_at=lambda t: poses,
                                  bbox_optimizer=bo).to(DEV)
    model.train()
    return model


def _gt(seed=2):
    return (torch.rand(H, W, 3, generator=torch.Generator().manual_seed(seed)) * 0.5 + 0.25).to(DEV)


def _extra(bo, lr=1e-3):
    return {"bbox_opt.delta_center": (bo.delta_center, lr), "bbox_opt.delta_yaw": (bo.delta_yaw, lr)}


def test_off_and_none_render_what_the_model_renders_today(monkeypatch):
    monkeypatch.setattr(raster, "DETERMINISTIC", True)  # fixed-point accumulation: two backward passes can be compared bit for bit
    fr = _scene()
    cam = fr.camera
    outs = []
    for mode in (None, "off"):
        m = _model(fr, mode)
        L = _lib.load()
        n0 = L.sgn_launch_count()
        out = m.get_outputs(cam)
        sum(m.get_loss_dict(out, {"image": _gt()}).values()).backward()
        torch.cuda.synchronize()
        outs.append((L.sgn_launch_count() - n0, out, m._holder.grad_arena.clone()))
    assert outs[0][0] == outs[1][0]
    assert all(torch.equal(outs[0][1][k], outs[1][1][k]) for k in outs[0][1]) and torch.equal(outs[0][2], outs[1][2])
    # mode "simple" with zero corrections: the same picture up to the float32 rounding of R -> q -> R
    m = _model(fr, "simple")
    out = m.get_outputs(cam)
    assert float((out["rgb"] - outs[0][1]["rgb"]).abs().mean()) < 1e-5


def test_backward_reaches_the_box_parameters():
    fr = _scene()
    m = _model(fr)
    bo = m.bbox_optimizer
    with torch.no_grad():
        bo.delta_center.normal_(0, 0.02, generator=None)
        bo.delta_yaw.normal_(0, 0.01)
    out = m.get_outputs(fr.camera)
    sum(m.get_loss_dict(out, {"image": _gt()}).values()).backward()
    gc, gy = bo.delta_center.grad, bo.delta_yaw.grad
    assert gc is not None and gy is not None
    rows = torch.zeros(NUM_FRAMES, bo.num_bboxes, dtype=torch.bool, device=DEV)
    rows[FRAME, :3] = True
    assert float(gc[~rows].abs().sum()) == 0 and float(gy[~rows].abs().sum()) == 0
    assert float(gc[FRAME, :3].abs().amax(1).min()) > 0 and float(gy[FRAME, :3].abs().min()) > 0  # every actor in view
    for sub in m.all_models.values():  # the Gaussians still receive theirs
        assert float(sub.gauss_params["means"].grad.abs().max()) > 0
    # the chain: autograd of poses() applied to the kernel's v_pose
    v_pose = m._holder.v_pose[1:].clone()
    staged = bo.stage(*bo.indices(m.poses_at(fr.camera.time)), [s.rot for s in fr.segments[1:]], [s.center for s in fr.segments[1:]], device=DEV)
    want_c, want_y = torch.autograd.grad(bo(staged), [bo.delta_center, bo.delta_yaw], grad_outputs=v_pose)
    assert torch.allclose(gc, want_c, rtol=1e-6, atol=0) and torch.allclose(gy, want_y, rtol=1e-6, atol=0)
    # a second backward without zero_grad accumulates, as autograd does
    out = m.get_outputs(fr.camera)
    sum(m.get_loss_dict(out, {"image": _gt()}).values()).backward()
    # (float atomics in the blend backward: the second pass repeats the first to rounding only)
    assert float((bo.delta_center.grad - 2 * want_c).abs().max()) <= 1e-3 * float(want_c.abs().max())
    # eval applies the corrections too, without a graph
    m.eval()
    with torch.no_grad():
        ev = m.get_outputs(fr.camera)
    assert ev["object_rgb"].shape == (H, W, 3) and not ev["rgb"].requires_grad


def test_fused_adam_moves_the_corrections_as_torch_adam():
    fr = _scene()
    m = _model(fr)
    bo = m.bbox_optimizer
    opt = FusedAdam(m.optimizer_params(), extra=_extra(bo))
    step_fn = TrainStep(m, opt, refine_every=0)
    ref_c, ref_y = (p.detach().clone().requires_grad_(True) for p in (bo.delta_center, bo.delta_yaw))
    twin = torch.optim.Adam([ref_c, ref_y], lr=1e-3, eps=1e-15)
    for step in range(3):
        step_fn(step, fr.camera, {"image": _gt()})
        ref_c.grad, ref_y.grad = bo.delta_center.grad.clone(), bo.delta_yaw.grad.clone()
        twin.step()
    torch.cuda.synchronize()
    assert float(bo.delta_center.detach()[FRAME, :3].abs().amax(1).min()) > 1e-4
    assert torch.allclose(bo.delta_center.detach(), ref_c.detach(), rtol=1e-5, atol=1e-9)
    assert torch.allclose(bo.delta_yaw.detach(), ref_y.detach(), rtol=1e-5, atol=1e-9)
    assert float(bo.delta_center.detach()[FRAME + 1].abs().sum()) == 0  # rows of other frames: zero gradient, no motion


def _train(steps):
    torch.manual_seed(0)
    fr = _scene()
    m = _model(fr)
    bo = m.bbox_optimizer
    opt = FusedAdam(m.optimizer_params(), extra=_extra(bo))
    step_fn = TrainStep(m, opt, refine_every=0)
    for step in range(steps):
        step_fn(step, fr.camera, {"image": _gt()})
    torch.cuda.synchronize()
    state = {f"{n}.{k}": p.detach().clone() for n, sub in m.all_models.items() for k, p in sub.gauss_params.items()}
    state.update(delta_center=bo.delta_center.detach().clone(), delta_yaw=bo.delta_yaw.detach().clone(),
                 grad_center=bo.delta_center.grad.clone(), grad_yaw=bo.delta_yaw.grad.clone(), v_pose=m._holder.v_pose.clone(),
                 exp_avg=opt.exp_avg.clone(), exp_avg_sq=opt.exp_avg_sq.clone())
    return state


def test_deterministic_training_steps_repeat_bit_for_bit(monkeypatch):
    monkeypatch.setattr(raster, "DETERMINISTIC", True)
    a, b = _train(4), _train(4)
    diff = [k for k in a if not torch.equal(a[k], b[k])]
    assert not diff, diff
    assert float(a["grad_center"].abs().max()) > 0 and float(a["delta_yaw"].abs().max()) > 0


def _rz(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])


def displaced_scene():
    """3 actors x 2000 Gaussians (blobs of about 15 cm in boxes of 4.6 x 1.9 x 1.7 m, the long axis along the box's x, the box's
    z axis pointing up; the colour varies smoothly over the box) in front of a dim background of 4000, 640 x 480.  Returns
    (camera, background, actors, true boxes, displaced boxes, the centre corrections that undo the displacement): every
    displaced box is off by 0.2 m and turned by -0.1 rad about its own z axis, i.e. a yaw parameter of 0.05 restores it."""
    g = torch.Generator().manual_seed(11)
    rng = np.random.default_rng(12)
    K = 16

    def blobs(n, lo, hi, scale, dc):
        lo, hi = torch.tensor(lo), torch.tensor(hi)
        means = torch.rand(n, 3, generator=g) * (hi - lo) + lo
        colour = dc(2.0 * (means - lo) / (hi - lo) - 1.0) + 0.1 * torch.randn(n, 3, generator=g)
        return GaussianSet(means.float().contiguous(), (float(np.log(scale)) + 0.2 * torch.randn(n, 3, generator=g)).contiguous(),
                           syn.random_quats(n, g).contiguous(), colour.reshape(n, 1, 3).float().contiguous(),
                           torch.zeros(n, K - 1, 3), (1.5 + 0.5 * torch.randn(n, 1, generator=g)).contiguous())

    bg = blobs(4000, (-9.0, -3.5, -30.0), (9.0, 3.5, -16.0), 0.2, lambda u: torch.full_like(u, -1.2))
    acts, true, start, d_center = {}, [], [], []
    for a in range(3):
        mix = torch.from_numpy(rng.normal(size=(3, 3))).float()
        acts[str(a)] = blobs(2000, (-2.3, -0.95, -0.85), (2.3, 0.95, 0.85), 0.15, lambda u, mix=mix: 1.2 * torch.sin(1.5 * u @ mix) + 0.6)
        yaw = rng.uniform(-0.4, 0.4)
        c, s = np.cos(yaw), np.sin(yaw)
        rot = np.array([[c, 0.0, s], [0.0, 1.0, 0.0], [-s, 0.0, c]]) @ np.array([[1.0, 0, 0], [0, 0, 1.0], [0, -1.0, 0]])
        center = np.array([-2.5 + 2.5 * a, -0.3, -10.0 - 1.5 * a])
        d = rng.normal(size=3)
        d = 0.2 * d / np.linalg.norm(d)
        true.append((rot, center))
        start.append((rot @ _rz(-0.1), center - d))
        d_center.append(d)
    return syn.make_camera(640, 480, time=float(FRAME)), bg, acts, true, start, np.stack(d_center)


def test_displaced_boxes_are_pulled_back():
    """The target is rendered with the true boxes of ``displaced_scene``; the model starts from the displaced ones.  300 Adam
    steps on the corrections alone (Gaussians frozen), rates decayed to a tenth: the L1 loss falls and the centre / yaw errors
    end below a quarter of where they started (0.2 m, 0.05)."""
    steps = 300
    cam, bg, acts, true, start, d_center = displaced_scene()

    def model_with(boxes, mode):
        poses = [ActorPose(str(a), r, c, FRAME, list(range(NUM_FRAMES)), frame_id=FRAME) for a, (r, c) in enumerate(boxes)]
        bo = BoxPoseOptimizer(NUM_FRAMES, ["0", "1", "2"], {f: f for f in range(NUM_FRAMES)}, mode=mode)
        m = SceneGraphRasterModel(bg.to(DEV), {k: v.to(DEV) for k, v in acts.items()},
                                  SceneGraphConfig(use_sky_sphere=False, ssim_lambda=0.0, fourier_features_dim=1),
                                  poses_at=lambda t: poses, bbox_optimizer=bo).to(DEV)
        m.train()
        m.step = 30000  # every SH order in use, as late in training
        return m

    with torch.no_grad():
        target = model_with(true, "off").get_outputs(cam)["rgb"].clone()
    m = model_with(start, "simple")
    bo = m.bbox_optimizer
    for sub in m.all_models.values():
        for p in sub.gauss_params.values():
            p.requires_grad_(False)
    opt = torch.optim.Adam([{"params": [bo.delta_center], "lr": 0.01}, {"params": [bo.delta_yaw], "lr": 0.003}], eps=1e-15)
    sched = torch.optim.lr_scheduler.ExponentialLR(opt, gamma=0.1 ** (1.0 / steps))
    want_c = torch.tensor(d_center, device=DEV, dtype=torch.float32)
    losses = []
    for _ in range(steps):
        opt.zero_grad(set_to_none=True)
        out = m.get_outputs(cam)
        loss = sum(m.get_loss_dict(out, {"image": target}).values())
        loss.backward()
        opt.step()
        sched.step()
        losses.append(loss.detach())
    losses = torch.stack(losses).cpu().numpy()
    err_c = (bo.delta_center.detach()[FRAME] - want_c).norm(dim=1).cpu().numpy()
    err_y = (bo.delta_yaw.detach()[FRAME] - 0.05).abs().cpu().numpy()
    print(f"[pose] L1 {losses[0]:.5f} -> {losses[-1]:.5f}; centre error 0.2 -> {err_c.tolist()}; yaw error 0.05 -> {err_y.tolist()}")
    assert losses[-1] < 0.5 * losses[0]
    assert np.all(err_c < 0.05) and np.all(err_y < 0.0125)
