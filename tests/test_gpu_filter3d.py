"""Mip-Splatting's 3D smoothing filter on the device: the filter sweep (sgn_filter3d) against the float64 statement
(oracle/filter3d_ref64.py) on hand-built scenes and on a config-4 scene; the filtered projection forward and backward
(sgn_camera.filter_3d) against float64 in every form; the filter off; a full render against the baked parameters; the zoom
property the filter exists for; and training with the filter recomputed through refinements."""
import copy

import numpy as np
import pytest
import torch

import street_gaussians_ns_b200.synthetic as syn
from oracle import filter3d_ref64 as f3
from oracle import project_ref64 as ref
from street_gaussians_ns_b200 import _lib, filter3d, ply_io, raster
from street_gaussians_ns_b200.model import ActorPose, SceneGraphConfig, SceneGraphRasterModel
from street_gaussians_ns_b200.optim import FusedAdam
from street_gaussians_ns_b200.refine import RefineSettings
from street_gaussians_ns_b200.scene import Camera, Frame, GaussianSet, Segment
from street_gaussians_ns_b200.training import TrainStep
from tests import project_cases as pc
from tests.test_gpu_parity import rel_l2, to_cuda

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
BOUNDARY = 1e-5  # rows whose sampling decision lies this close (relative) to a boundary may go either way
FWD_K, FWD_R = 8.0, 2e-6  # tests/test_gpu_project_directed.py
GRAD_TOL = 1e-3           # relative L2 per gradient tensor, tests/test_gpu_fullsize_parity.py


def _views(cams):
    return [dict(fx=c.fx, fy=c.fy, cx=c.cx, cy=c.cy, width=c.width, height=c.height) for c in cams]


def _check_sweep(model, cams, rows=None, seed=0):
    """compute_filter_3d against filter3d_ref64.sweep (on ``rows`` random rows of each sub-model when given)."""
    n = model.compute_filter_3d(cams)
    torch.cuda.synchronize()
    names = list(model.all_models._modules)
    tab = filter3d.transform_table(model, cams, names)
    rng = np.random.default_rng(seed)
    picks, means = [], []
    for nm in names:
        mu = model.all_models[nm].gauss_params["means"].detach().cpu().numpy()
        idx = np.arange(mu.shape[0]) if rows is None or mu.shape[0] <= rows else np.sort(rng.choice(mu.shape[0], rows, replace=False))
        picks.append(idx)
        means.append(mu[idx])
    c = model.config
    r = f3.sweep(means, _views(cams), tab["M"].reshape(len(cams), len(names), 3, 4), tab["present"], c.filter_3d_variance,
                 c.filter_3d_near)
    got_all = [model.all_models[nm].filter_3d.cpu().numpy().astype(np.float64) for nm in names]
    fill = max((g.max() for g in got_all if g.size), default=0.0)
    bad = 0
    for k, nm in enumerate(names):
        got = got_all[k][picks[k]]
        ok = r["margin"][k] > BOUNDARY
        bad += int((~ok).sum())
        s = r["sampled"][k] & ok
        assert np.allclose(got[s], r["sigma"][k][s], rtol=1e-6, atol=0), nm
        u = ~r["sampled"][k] & ok
        assert np.all(got[u] == fill), nm  # unsampled rows: the largest sampled sigma (the lowest rate)
        assert np.all(np.isfinite(got)) and np.all(got >= 0)
    if rows is None:
        assert abs(n - r["n_sampled"]) <= bad
        assert np.isclose(fill, r["fill"], rtol=1e-6) or bad > 0
    return n, r


def _hand_model(dev=DEV):
    gen = torch.Generator().manual_seed(1)

    def gs(n, F, spread):
        return GaussianSet((torch.rand(n, 3, generator=gen) - 0.5) * spread, torch.randn(n, 3, generator=gen) * 0.3 - 3,
                           torch.randn(n, 4, generator=gen), torch.randn(n, F, 3, generator=gen), torch.zeros(n, 15, 3),
                           torch.randn(n, 1, generator=gen)).to(dev)
    bg = gs(3000, 1, 60.0)
    bg.means[:50] += torch.tensor([0.0, 0.0, 500.0], device=dev)  # behind every camera: never sampled
    boxes = {0.0: [ActorPose("a", pc._yaw(0.4), np.array([1.0, 0.5, -8.0]), 0, [0, 1]),
                   ActorPose("b", pc._yaw(-1.0), np.array([-3.0, 0.0, -15.0]), 0, [0, 1])],
             1.0: [ActorPose("a", pc._yaw(0.5), np.array([1.5, 0.5, -9.0]), 1, [0, 1])]}
    cfg = SceneGraphConfig(filter_3d=True)
    return SceneGraphRasterModel(bg, {"a": gs(300, 5, 3.0), "b": gs(200, 5, 3.0), "c": gs(100, 5, 3.0)}, config=cfg,
                                 poses_at=lambda t: boxes.get(t, []))


def _hand_cams():
    cams = []
    for k, (f, W, H) in enumerate(((500.0, 640, 480), (1800.0, 640, 480), (300.0, 320, 200), (900.0, 960, 640))):
        c2w = np.concatenate([pc._yaw(0.3 * k - 0.4), np.array([[0.3 * k], [0.1], [2.0 - k]])], 1)
        cams.append(Camera(c2w, f, f * (1.0 + 0.1 * k), W * 0.5 + 3, H * 0.5 - 2, W, H, time=float(k % 2)))
    return cams


def test_sweep_hand_built():
    m = _hand_model()
    n, r = _check_sweep(m, _hand_cams())
    assert 0 < n < sum(s.num_points for s in m.all_models.values())
    assert not r["sampled"][0][:50].any()
    assert not r["sampled"][3].any()  # actor "c" never has a box: every row takes the widest filter
    # no camera at all: nothing sampled, every sigma is 0
    with pytest.warns(UserWarning):
        assert m.compute_filter_3d([]) == 0
    assert all(float(s.filter_3d.abs().max()) == 0.0 for s in m.all_models.values())


def test_sweep_config4():
    sc = syn.WaymoScene(scale=1.0)

    def poses_at(t):
        f = int(t)
        return [ActorPose(str(a), rot, center, f, list(range(sc.num_frames))) for a, rot, center in sc.boxes_at(f)]
    m = SceneGraphRasterModel(sc.background.to(DEV), {k: v.to(DEV) for k, v in sc.actors.items()},
                              SceneGraphConfig(filter_3d=True), poses_at=poses_at)
    assert len(sc.cameras) == 425 and sum(s.num_points for s in m.all_models.values()) == 2_000_000
    m.compute_filter_3d(sc.cameras)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    n = m.compute_filter_3d(sc.cameras)
    e1.record()
    torch.cuda.synchronize()
    print(f"[filter3d] config 4: {n} of 2000000 rows sampled, compute_filter_3d {e0.elapsed_time(e1):.2f} ms")
    _check_sweep(m, sc.cameras, rows=20000)


# ---- the filtered projection ---------------------------------------------------------------------------------------------
def _case(seed=31, deg=3):
    b = pc._cam(160, 112, seed, ref.Settings(sh_degree=deg))
    s0, s1 = b.segment(0), b.segment(1, pose=(0.3, (0.2, -0.1, -3.0)), F=3)
    for s in (s0, s1):
        b.scatter(s, 150, z=(1.5, 12.0), scale=(0.002, 0.3))
    return b.settle("filter3d_proj")


def _sigmas(frame, seed=4, lo=1e-3, hi=0.05):
    rng = np.random.default_rng(seed)
    return [rng.uniform(lo, hi, s.params.num_points).astype(np.float32) for s in frame.segments]


def _with_filter(frame, sigmas):
    return Frame(frame.camera, [Segment(s.params, s.cls, s.rot, s.center, s.idft, s.name,
                                        filter_3d=None if sg is None else torch.as_tensor(sg).to(DEV).contiguous())
                                for s, sg in zip(frame.segments, sigmas)])


def _project(frc, st, mode, view=False):
    settings = raster.RenderSettings(sh_degree=st.sh_degree, sh_degree_to_use=st.deg_use, rasterize_mode=mode)
    cs = raster.camera_struct(frc.camera, settings)
    table = raster.SegmentTable(frc, [s.params.tensors() for s in frc.segments], DEV)
    v = None
    if view:
        v = torch.tensor(np.concatenate([frc.camera.viewmat().reshape(-1), frc.camera.cam_pos()]), device=DEV)
    return table, cs, raster.project_fwd(table, cs, DEV, v), v


@pytest.mark.parametrize("mode", ["classic", "antialiased"])
def test_projection_forward_against_float64(mode, monkeypatch):
    case = _case()
    sig = _sigmas(case.frame)
    frc = _with_filter(to_cuda(case.frame), sig)
    want = f3.forward(case.frame, case.st, sig, antialiased=mode == "antialiased")
    table, cs, p, _ = _project(frc, case.st, mode)
    rec = p.records.cpu().numpy().astype(np.float64)
    ok = want["margin"] > 1e-4
    radii = p.radii.cpu().numpy()
    assert np.array_equal(radii[ok], want["radii"][ok])
    vis = want["vis"] & ok
    assert vis.sum() > 100
    # the bars of tests/test_gpu_project_directed.py: FWD_K x the row's fp32 noise (the statement evaluated in float32) +
    # FWD_R x max|ref64| of the field group
    w = want["records"]
    w32 = f3.forward(case.frame, case.st, sig, antialiased=mode == "antialiased", dtype=torch.float32)["records"]
    for cols in ((0, 1), (2, 3, 4), (5,), (6, 7, 8), (9,)):
        c = list(cols)
        noise = np.abs(w32[vis][:, c] - w[vis][:, c]).max(1, keepdims=True)
        bar = FWD_K * noise + FWD_R * np.maximum(np.abs(w[vis][:, c]).max(1, keepdims=True), 1e-3)
        err = np.abs(rec[vis][:, c] - w[vis][:, c])
        assert (err <= bar).all(), (mode, cols, float((err / bar).max()))
    # every visible row is fainter than without the filter (coef < 1)
    assert (want["coef"][vis] < 1).all() and (rec[vis, 5] <= w[vis, 5] * (1 + 1e-5) + 1e-7).all()
    # the VIEW form and the staged form: the same bits as the plain direct form
    _, _, pv, _ = _project(frc, case.st, mode, view=True)
    assert torch.equal(pv.records, p.records) and torch.equal(pv.radii, p.radii) and torch.equal(pv.tiles_touched, p.tiles_touched)
    monkeypatch.setenv("SGN_PROJECT_STAGED", "1")
    _, _, ps, _ = _project(frc, case.st, mode)
    nz = p.radii > 0
    assert torch.equal(ps.records[nz], p.records[nz]) and torch.equal(ps.radii, p.radii)
    assert torch.equal(ps.tiles_touched, p.tiles_touched) and torch.equal(ps.touch_mask[nz], p.touch_mask[nz])


@pytest.mark.parametrize("mode", ["classic", "antialiased"])
def test_projection_backward_against_float64(mode):
    case = _case(33)
    sig = _sigmas(case.frame, 5)
    frc = _with_filter(to_cuda(case.frame), sig)
    want_fw = f3.forward(case.frame, case.st, sig, antialiased=mode == "antialiased")
    table, cs, p, _ = _project(frc, case.st, mode)
    rng = np.random.default_rng(9)
    vis = (p.radii.cpu().numpy() > 0) & (want_fw["margin"] > 1e-4)
    v = rng.normal(size=(case.frame.num_points, 12)) * vis[:, None]
    v[:, 10:] = 0
    vt = torch.tensor(v, dtype=torch.float32, device=DEV)
    params = [s.params.tensors() for s in frc.segments]
    flat, arena = raster.project_bwd(table, params, cs, p.records, p.radii, vt)
    want = f3.backward(case.frame, case.st, sig, v, antialiased=mode == "antialiased")
    names = ("means", "scales", "quats", "features_dc", "features_rest", "opacities")
    worst = 0.0
    for si in range(len(frc.segments)):
        for k, nm in enumerate(names):
            g = flat[6 * si + k].cpu().numpy()
            e = rel_l2(g, want[si][nm])
            worst = max(worst, e)
            assert np.all(np.isfinite(g)) and e <= GRAD_TOL, (mode, si, nm, e)
    print(f"[filter3d bwd] {mode}: worst relative L2 {worst:.2e}")
    # the same gradients from the pose and view forms, and from a second run (no atomics: deterministic); the arena's
    # alignment padding is not written, so the per-tensor views are compared
    g0 = [t.clone() for t in flat]
    f1, _ = raster.project_bwd(table, params, cs, p.records, p.radii, vt)
    assert all(torch.equal(a, b) for a, b in zip(g0, f1))
    v_pose = torch.empty(table.nseg, _lib.POSE_FLOATS, device=DEV)
    f2, _ = raster.project_bwd(table, params, cs, p.records, p.radii, vt, v_pose=v_pose)
    assert all(torch.equal(a, b) for a, b in zip(g0, f2)) and torch.isfinite(v_pose).all()
    _, _, pv, view = _project(frc, case.st, mode, view=True)
    v_view = torch.empty(_lib.VIEW_FLOATS, device=DEV)
    f3_, _ = raster.project_bwd(table, params, cs, pv.records, pv.radii, vt, view=view, v_view=v_view)
    assert all(torch.equal(a, b) for a, b in zip(g0, f3_)) and torch.isfinite(v_view).all()


def test_filter_off_and_zero_filter():
    case = _case(35)
    frc = to_cuda(case.frame)
    _, cs, p0, _ = _project(frc, case.st, "classic")
    assert cs.filter_3d is None
    zeros = [np.zeros(s.params.num_points, np.float32) for s in case.frame.segments]
    _, _, pz, _ = _project(_with_filter(frc, zeros), case.st, "classic")
    assert torch.equal(pz.radii, p0.radii)
    assert torch.allclose(pz.records, p0.records, rtol=1e-6, atol=0)
    # a frame where only some segments carry a filter is refused
    with pytest.raises(_lib.SgnError):
        _project(_with_filter(frc, [zeros[0], None]), case.st, "classic")
    # a render without filters passes NULL: the projection calls are the ones a camera without the field makes
    st = raster.RenderSettings(sh_degree=case.st.sh_degree)
    out, h = raster.render_frame(frc, st)
    assert h.table.filter_dev is None and torch.equal(h.records, p0.records)


def test_full_render_matches_baked_parameters():
    fr = syn.config_frame(3, scale=0.2)
    sig = _sigmas(fr, 6, 1e-3, 0.03)
    frc = _with_filter(to_cuda(fr), sig)
    baked = Frame(fr.camera, [Segment(ply_io.bake_filter_3d(s.params, torch.as_tensor(g)).to("cuda"), s.cls, s.rot, s.center,
                                      s.idft, s.name) for s, g in zip(fr.segments, sig)])
    # the antialiased mode too: comp of the baked s' is comp of the filtered covariance, and sigmoid(logit(sigmoid x coef))
    # is sigmoid x coef up to rounding
    for mode in ("classic", "antialiased"):
        st = raster.RenderSettings(rasterize_mode=mode)
        a, _ = raster.render_frame(frc, st)
        b, _ = raster.render_frame(baked, st)
        torch.cuda.synchronize()
        for k in ("rgb", "accumulation", "object_acc", "background_acc"):
            d = (a[k] - b[k]).abs().amax(-1)
            frac = float((d > 1e-4).float().mean())
            print(f"[filter3d bake] {mode} {k}: {frac:.4%} of pixels beyond 1e-4, max {float(d.max()):.2e}")
            assert frac <= 0.005, (mode, k, frac)


def test_zoom_property():
    """One Gaussian with s = 1e-4 at 10 m, filtered from a camera at f = 1000 and rendered at f = 8000."""
    z, s = 10.0, 1e-4
    train = Camera(np.concatenate([np.eye(3), np.zeros((3, 1))], 1), 1000.0, 1000.0, 320.0, 240.0, 640, 480)
    mean = torch.tensor([[0.0, 0.0, -z]])  # OpenGL camera: it looks along -z
    params = GaussianSet(mean, torch.full((1, 3), float(np.log(s))), torch.tensor([[1.0, 0.0, 0.0, 0.0]]), torch.zeros(1, 1, 3),
                         torch.zeros(1, 15, 3), torch.full((1, 1), 4.0)).to(DEV)
    m = SceneGraphRasterModel(params, {}, SceneGraphConfig(filter_3d=True))
    assert m.compute_filter_3d([train]) == 1
    sigma = float(m.all_models["background"].filter_3d[0])
    assert np.isclose(sigma, np.sqrt(0.2) * z / 1000.0, rtol=1e-6)
    zoom = Camera(train.c2w, 8000.0, 8000.0, 320.0, 240.0, 640, 480)
    g = m.all_models["background"].as_set()
    for filt, want_var in ((True, (s * s + sigma * sigma) * 8000.0 ** 2 / z ** 2 + 0.3), (False, s * s * 8000.0 ** 2 / z ** 2 + 0.3)):
        fr = Frame(zoom, [Segment(g, filter_3d=m.all_models["background"].filter_3d if filt else None)])
        _, _, p, _ = _project(fr, ref.Settings(), "classic")
        a, b, c = (float(x) for x in p.records[0, 2:5])
        det = a * c - b * b
        var_x, var_y = c / det, a / det  # the screen covariance from its inverse, the conic
        assert np.isclose(var_x, want_var, rtol=1e-4) and np.isclose(var_y, want_var, rtol=1e-4), (filt, var_x, want_var)
        if filt:
            assert 3.5 < np.sqrt(var_x) < 3.7
        else:  # about the 0.3 px^2 blur alone
            assert var_x < 0.31


def test_training_recomputes_the_filter():
    sc = syn.WaymoScene(scale=0.05)
    frame_list = list(range(sc.num_frames))

    def poses_at(t):
        f = int(t)
        return [ActorPose(str(a), rot, center, f, frame_list, frame_id=f) for a, rot, center in sc.boxes_at(f)]
    cfg = SceneGraphConfig(use_sky_sphere=False, ssim_lambda=0.0, refine=RefineSettings(refine_every=100),
                           object_refine=RefineSettings(refine_every=100, cull_alpha_thresh=0.005), num_train_data=len(sc.cameras),
                           filter_3d=True)
    model = SceneGraphRasterModel(sc.background.to(DEV), {k: v.to(DEV) for k, v in sc.actors.items()}, cfg, poses_at=poses_at).to(DEV)
    model.train()
    opt = FusedAdam(model.optimizer_params())
    step_fn = TrainStep(model, opt, refine_every=100, filter_cameras=sc.cameras)
    calls = []
    orig = model.compute_filter_3d
    model.compute_filter_3d = lambda cams: calls.append(model.step) or orig(cams)
    g = torch.Generator().manual_seed(5)
    gt = (torch.rand(sc.height, sc.width, 3, generator=g) * 255).to(torch.uint8).to(DEV)
    counts0 = [s.num_points for s in model.all_models.values()]
    start = 560
    for i in range(240):
        step = start + i
        losses = step_fn(step, sc.cameras[step % len(sc.cameras)], {"image": gt})
        assert all(torch.isfinite(v).all() for v in losses.values()), step
    torch.cuda.synchronize()
    counts1 = [s.num_points for s in model.all_models.values()]
    assert counts1 != counts0  # the refinements changed rows
    # the first step, then the refinements at 600 and 700 (which changed rows; also the 100-step schedule), once each
    assert calls == [start, 600, 700], calls
    for sub in model.all_models.values():
        assert sub.filter_3d.shape == (sub.num_points,) and torch.isfinite(sub.filter_3d).all() and (sub.filter_3d >= 0).all()
    assert float(model.all_models["background"].filter_3d.max()) > 0
    sd = copy.deepcopy(model.state_dict())
    other = SceneGraphRasterModel(sc.background.to(DEV), {k: v.to(DEV) for k, v in sc.actors.items()}, cfg, poses_at=poses_at).to(DEV)
    other.load_state_dict(sd)
    for a, b in zip(model.all_models.values(), other.all_models.values()):
        assert torch.equal(a.filter_3d, b.filter_3d)
    other.eval()
    out = other.get_outputs(sc.cameras[3])
    assert torch.isfinite(out["rgb"]).all()
