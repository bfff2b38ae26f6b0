"""CPU checks of the 3D smoothing filter: the float64 statement (oracle/filter3d_ref64.py) against closed forms, the host
tables the sweep reads (filter3d.py), the model's buffer and configuration, and the PLY export."""
import os

import numpy as np
import pytest
import torch

from oracle import filter3d_ref64 as f3
from oracle import project_ref64 as ref
from street_gaussians_ns_b200 import filter3d, ply_io
from street_gaussians_ns_b200.model import ActorPose, SceneGraphConfig, SceneGraphRasterModel
from street_gaussians_ns_b200.scene import Camera, GaussianSet
from tests import project_cases as pc

SQ = np.sqrt(0.2)


def _cam_view(f, W=100, H=80, cx=None, cy=None, fy=None):
    return dict(fx=f, fy=f if fy is None else fy, cx=W / 2 if cx is None else cx, cy=H / 2 if cy is None else cy, width=W, height=H)


def _M(b=(0.0, 0.0, 0.0), A=None):
    A = np.eye(3) if A is None else np.asarray(A, np.float64)
    return np.concatenate([A, np.asarray(b, np.float64).reshape(3, 1)], 1)


def _sweep(means, views, Ms, present=None, **kw):
    V, S = len(views), len(means)
    M = np.asarray(Ms, np.float64).reshape(V, S, 3, 4)
    pres = np.ones((V, S), bool) if present is None else np.asarray(present, bool)
    return f3.sweep(means, views, M, pres, **kw)


def test_one_gaussian_on_axis():
    for d, f in ((10.0, 1000.0), (3.5, 420.0), (0.25, 50.0)):
        r = _sweep([np.array([[0.0, 0.0, d]])], [_cam_view(f)], [_M()])
        assert r["sampled"][0][0] and r["n_sampled"] == 1
        assert np.isclose(r["sigma"][0][0], SQ * d / f, rtol=1e-14)


def test_margin_edges_inclusive_and_near_excluded():
    W, H = 60, 40  # sizes whose edges -0.15 W, 1.15 W are float32 numbers (the views' intrinsics are float32)
    lo_u, hi_u, lo_w, hi_w = -0.15 * W, 1.15 * W, -0.15 * H, 1.15 * H
    mean = np.array([[0.0, 0.0, 0.0]])
    # the projection of a mean on the axis is exactly (cx, cy): put cx / cy on the edges, depth from the translation
    views = [_cam_view(100.0, W, H, cx=lo_u), _cam_view(100.0, W, H, cx=hi_u), _cam_view(100.0, W, H, cy=lo_w),
             _cam_view(100.0, W, H, cy=hi_w)]
    for v in views:
        r = _sweep([mean], [v], [_M((0, 0, 5.0))])
        assert r["sampled"][0][0], v
    # just outside each edge
    for k, v in enumerate(views):
        key = "cx" if k < 2 else "cy"
        out = dict(v)
        out[key] = np.nextafter(np.float32(v[key]), np.float32(-np.inf if k % 2 == 0 else np.inf))
        r = _sweep([mean], [out], [_M((0, 0, 5.0))])
        assert not r["sampled"][0][0], out
    # z == near is not sampled, the next double above is
    assert not _sweep([mean], [_cam_view(100.0)], [_M((0, 0, 0.2))])["sampled"][0][0]
    assert _sweep([mean], [_cam_view(100.0)], [_M((0, 0, np.nextafter(0.2, 1.0)))])["sampled"][0][0]
    assert not _sweep([mean], [_cam_view(100.0)], [_M((0, 0, 0.5))], near=0.5)["sampled"][0][0]


def test_mixed_focal_lengths_take_max_rate_per_view():
    mean = [np.array([[0.0, 0.0, 0.0]])]
    views = [_cam_view(1000.0, 4000, 4000), _cam_view(2000.0, 4000, 4000)]
    r = _sweep(mean, views, [[_M((0, 0, 5.0))], [_M((0, 0, 20.0))]])
    # rates 1000 / 5 = 200 and 2000 / 20 = 100: sigma from 200, not from f_max / z_min = 400
    assert np.isclose(r["sigma"][0][0], SQ / 200.0, rtol=1e-14)
    assert not np.isclose(r["sigma"][0][0], SQ / 400.0)
    # fx != fy: max(fx, fy) / z
    r = _sweep(mean, [_cam_view(300.0, 4000, 4000, fy=900.0)], [_M((0, 0, 3.0))])
    assert np.isclose(r["sigma"][0][0], SQ * 3.0 / 900.0, rtol=1e-14)


def test_absent_actor_view_and_unsampled_rows_take_lowest_rate():
    bg = np.array([[0.0, 0.0, 0.0], [1e6, 0.0, 0.0]])      # the second row is never in view
    actor = np.array([[0.0, 0.0, 0.0]])
    views = [_cam_view(100.0), _cam_view(100.0)]
    Ms = [[_M((0, 0, 4.0)), _M((0, 0, 1.0))], [_M((0, 0, 8.0)), _M((0, 0, 2.0))]]
    r = _sweep([bg, actor], views, Ms, present=[[1, 1], [1, 0]])
    assert np.isclose(r["sigma"][1][0], SQ * 1.0 / 100.0)    # view 1 (z = 2) is absent for the actor: only z = 1 counts
    r2 = _sweep([bg, actor], views, Ms, present=[[1, 0], [1, 1]])
    assert np.isclose(r2["sigma"][1][0], SQ * 2.0 / 100.0)
    # unsampled rows: the lowest rate of all sampled rows (largest sigma), here the background's z = 8 in view 1 -- no,
    # z = 4 in view 0 is the higher rate for that row; the lowest over rows is min(100 / 4, 100 / 1) = 25
    assert not r["sampled"][0][1]
    assert np.isclose(r["sigma"][0][1], SQ * 4.0 / 100.0) and np.isclose(r["fill"], SQ * 4.0 / 100.0)
    # nothing sampled at all: every sigma is 0
    r0 = _sweep([bg], [_cam_view(100.0)], [_M((0, 0, -3.0))])
    assert r0["n_sampled"] == 0 and all((s == 0).all() for s in r0["sigma"])


def _model(filter_on=True, with_empty=True):
    gen = torch.Generator().manual_seed(0)

    def gs(n, F):
        return GaussianSet(torch.randn(n, 3, generator=gen), torch.randn(n, 3, generator=gen) * 0.3 - 3,
                           torch.randn(n, 4, generator=gen), torch.randn(n, F, 3, generator=gen), torch.zeros(n, 15, 3),
                           torch.randn(n, 1, generator=gen))
    R = pc._yaw(0.4)
    boxes = {0.0: [ActorPose("a", R, np.array([1.0, 2.0, -3.0]), 0, [0, 1])], 1.0: []}
    cfg = SceneGraphConfig(filter_3d=filter_on)
    actors = {"a": gs(7, 5), "b": gs(0, 5)} if with_empty else {"a": gs(7, 5)}
    return SceneGraphRasterModel(gs(20, 1), actors, config=cfg, poses_at=lambda t: boxes.get(t, []))


def test_transform_table_places_actors_by_box():
    m = _model()
    c2w = np.concatenate([pc._yaw(0.2), np.array([[0.5], [0.1], [2.0]])], 1)
    cams = [Camera(c2w, 500, 510, 320, 240, 640, 480, time=0.0), Camera(c2w, 500, 510, 320, 240, 640, 480, time=1.0)]
    names = list(m.all_models._modules)
    tab = filter3d.transform_table(m, cams, names)
    assert tab.dtype.itemsize == 104 and tab.shape == (2, 3)
    W = cams[0].viewmat().astype(np.float64)
    assert np.array_equal(tab["M"][0, 0].reshape(3, 4), W) and tab["present"][:, 0].tolist() == [1, 1]
    R, c = pc._yaw(0.4), np.array([1.0, 2.0, -3.0])
    want = np.concatenate([W[:, :3] @ R, (W[:, :3] @ c + W[:, 3])[:, None]], 1)
    assert np.allclose(tab["M"][0, 1].reshape(3, 4), want, rtol=0, atol=1e-12)
    assert tab["present"][:, 1].tolist() == [1, 0]       # no box at time 1
    assert tab["present"][:, 2].tolist() == [0, 0]       # no Gaussians (and no box)


def test_config_and_state_dict():
    c = SceneGraphConfig()
    assert (c.filter_3d, c.filter_3d_variance, c.filter_3d_near, c.filter_3d_every) == (False, 0.2, 0.2, 100)
    off = _model(False)
    assert not any("filter_3d" in k for k in off.state_dict())
    on = _model(True)
    keys = [k for k in on.state_dict() if "filter_3d" in k]
    assert sorted(keys) == ["all_models.background.filter_3d", "all_models.object_a.filter_3d", "all_models.object_b.filter_3d"]
    assert set(on.state_dict()) - set(keys) == set(off.state_dict())
    sd = on.state_dict()
    sd["all_models.background.filter_3d"] = torch.arange(20, dtype=torch.float32)
    other = _model(True)
    other.load_state_dict(sd)
    assert torch.equal(other.all_models["background"].filter_3d, torch.arange(20, dtype=torch.float32))


def test_coef_small_scales():
    ls = np.full(3, -20.0)
    sigma = 1e-3
    s = np.exp(ls)
    want = np.prod(s / np.sqrt(s * s + sigma * sigma))
    got = f3.coef(torch.tensor(ls)[None], torch.tensor([sigma]))[0].item()
    assert np.isclose(got, want, rtol=1e-12) and want > 0
    # the kernel's fp32 sequence (per-axis ratios) stays normal and correct; the plain ratio of products underflows
    s32 = np.float32(np.exp(np.float32(-20.0)))
    s2 = np.float32(s32 * s32)
    r = np.float32(s2 / np.float32(s2 + np.float32(sigma) * np.float32(sigma)))
    c32 = np.float32(np.float32(np.sqrt(r) * np.sqrt(r)) * np.sqrt(r))
    assert np.isfinite(c32) and c32 > 0 and abs(c32 / want - 1) < 1e-5
    with np.errstate(under="ignore"):
        assert np.float32(s2 * s2 * s2) == 0.0


def _frame(seed=3):
    b = pc._cam(96, 64, seed)
    s0, s1 = b.segment(0), b.segment(1, pose=(0.3, (0.2, -0.1, -3.0)), F=3)
    for s in (s0, s1):
        b.scatter(s, 25, z=(2.0, 9.0), scale=(0.003, 0.2))
    return b.settle("filter3d")


def test_zero_filter_is_the_plain_projection():
    case = _frame()
    fr = case.frame
    zeros = [np.zeros(s.params.num_points) for s in fr.segments]
    a = f3.forward(fr, case.st, zeros)
    b = ref.forward(fr, case.st)
    assert np.array_equal(a["radii"], b["radii"]) and np.allclose(a["records"][:, :10], b["records"][:, :10], rtol=1e-12, atol=1e-12)


def test_gradcheck_filtered_projection():
    case = _frame(5)
    fr = case.frame
    seg = fr.segments[0]
    n = seg.params.num_points
    rng = np.random.default_rng(1)
    sigma = torch.tensor(rng.uniform(0.001, 0.05, n))
    mw = seg.params.means.double()
    qr = seg.params.quats.double()
    logit = seg.params.opacities.double()[:, 0]
    vis = ref.project_core(mw, qr, f3.filtered_scales(seg.params.scales.double(), sigma), fr.camera, 16, 0.01, torch.float64)["vis"]
    vt = torch.from_numpy(vis)

    def fn(ls, lo):
        pr = ref.project_core(mw, qr, f3.filtered_scales(ls, sigma), fr.camera, 16, 0.01, torch.float64)
        return torch.cat([pr["conic"][vt].reshape(-1), (torch.sigmoid(lo) * f3.coef(ls, sigma))[vt]])

    ls = seg.params.scales.double().clone().requires_grad_(True)
    lo = logit.clone().requires_grad_(True)
    assert torch.autograd.gradcheck(fn, (ls, lo), eps=1e-6, atol=1e-6, rtol=1e-4)
    # the statement's VJP (backward) is autograd of the same records
    sigmas = [sigma.numpy(), np.full(fr.segments[1].params.num_points, 0.01)]
    v = rng.normal(size=(fr.num_points, 12))
    g = f3.backward(fr, case.st, sigmas, v)
    fw = f3.forward(fr, case.st, sigmas, grad=True)
    want = torch.autograd.grad((fw["rec"] * torch.tensor(v[:, :10])).sum(), fw["leaves"][0]["scales"])[0].numpy()
    assert np.allclose(g[0]["scales"], want, rtol=1e-12, atol=1e-14)
    # d log s' / d log s = r and d coef / d log s = coef (1 - r)
    ls1 = torch.tensor([[-2.0, -1.0, -3.0]], requires_grad=True)
    sg1 = torch.tensor([0.1], dtype=torch.float32)
    sp = torch.log(f3.filtered_scales(ls1.double(), sg1.double()))
    r = torch.exp(2 * ls1.double()) / (torch.exp(2 * ls1.double()) + 0.01)
    gd = torch.autograd.grad(sp.sum(), ls1)[0].double()
    assert torch.allclose(gd, r.detach(), rtol=1e-6)
    cf = f3.coef(ls1.double(), sg1.double())
    gc = torch.autograd.grad(cf.sum(), ls1)[0].double()
    assert torch.allclose(gc, (cf[:, None] * (1 - r)).detach(), rtol=1e-6)


def test_ply_bake_matches_filter_and_column_round_trips(tmp_path):
    case = _frame(7)
    fr = case.frame
    rng = np.random.default_rng(2)
    sigmas = [rng.uniform(0.001, 0.03, s.params.num_points) for s in fr.segments]
    want = f3.forward(fr, case.st, sigmas)
    baked_frame = type(fr)(fr.camera, [type(s)(ply_io.bake_filter_3d(s.params, torch.tensor(sig, dtype=torch.float32)), s.cls, s.rot,
                                               s.center, s.idft, s.name) for s, sig in zip(fr.segments, sigmas)])
    got = ref.forward(baked_frame, case.st)
    assert np.array_equal(got["vis"], want["vis"])
    vis = want["vis"]
    assert np.allclose(got["records"][vis, :10], want["records"][vis, :10], rtol=2e-6, atol=1e-7)
    ls, lo = f3.bake(fr.segments[0].params.scales.numpy(), fr.segments[0].params.opacities.numpy(), sigmas[0])
    b0 = ply_io.bake_filter_3d(fr.segments[0].params, torch.tensor(sigmas[0], dtype=torch.float32))
    assert np.allclose(b0.scales.numpy(), ls, rtol=1e-6) and np.allclose(b0.opacities.numpy(), lo, rtol=1e-5, atol=1e-6)
    # column: raw parameters plus filter_3D
    p = os.path.join(tmp_path, "x.ply")
    params = fr.segments[0].params
    f = torch.tensor(sigmas[0], dtype=torch.float32)
    n = ply_io.write_ply(p, params, filter_3d=f)
    assert n == params.num_points
    assert torch.equal(ply_io.read_filter_3d(p), f)
    back = ply_io.read_ply(p)
    assert torch.equal(back.scales, params.scales) and torch.equal(back.opacities, params.opacities)
    plain = os.path.join(tmp_path, "y.ply")
    ply_io.write_ply(plain, params)
    assert ply_io.read_filter_3d(plain) is None


def test_export_model_modes(tmp_path):
    m = _model(True, with_empty=False)
    for sub in m.all_models.values():
        sub.filter_3d = torch.full((sub.num_points,), 0.01)
    out = ply_io.export_model(m, os.path.join(tmp_path, "col"), filter_3d="column")
    assert out["background"] == 20
    f = ply_io.read_filter_3d(os.path.join(tmp_path, "col", "point_cloud_background.ply"))
    assert torch.allclose(f, torch.full((20,), 0.01))
    ply_io.export_model(m, os.path.join(tmp_path, "bake"), filter_3d="bake")
    baked = ply_io.read_ply(os.path.join(tmp_path, "bake", "point_cloud_background.ply"))
    raw = m.all_models["background"].gauss_params["scales"].detach()
    assert (baked.scales >= raw - 1e-6).all()
    with pytest.raises(ValueError):
        ply_io.export_model(m, os.path.join(tmp_path, "z"), filter_3d="mip")
    with pytest.raises(ValueError):
        ply_io.export_model(_model(False, with_empty=False), os.path.join(tmp_path, "w"), filter_3d="bake")


# ---- the filtered statements of tests/filter3d_cases.py ------------------------------------------------------------------
def test_filtered_pose_and_view_statements_at_zero_filter():
    from tests import antialias_cases as ac
    from tests import camera_cases as cc
    from tests import filter3d_cases as fc
    from tests import pose_cases as pz
    case = pc.get("fov_clamp")  # an unposed and a posed segment, FOV clamps on every side
    fr, st = case.frame, case.st
    zeros = fc.zero_filter(case)
    v = pc.v_records(case, "all")
    pairs = ((fc.v_pose_ref(fr, st, zeros, v), pz.v_pose_ref(fr, st, v)),
             (fc.v_pose_ref(fr, st, zeros, v, True), ac.v_pose_ref(fr, st, v)),
             (fc.v_view_ref(fr, st, zeros, v), cc.v_view_ref(fr, st, v)),
             (fc.v_view_ref(fr, st, zeros, v, True), ac.v_view_ref(fr, st, v)))
    for got, want in pairs:
        assert np.any(want) and np.allclose(got, want, rtol=1e-12, atol=1e-12 * np.abs(want).max())


@pytest.mark.parametrize("antialiased", [False, True])
def test_filtered_pose_and_view_statements_central_differences(antialiased):
    from tests import filter3d_cases as fc
    from tests import pose_cases as pz
    case = _frame(9)
    fr, st = case.frame, case.st
    rng = np.random.default_rng(4)
    sigmas = [np.float32(rng.uniform(0.3, 3.0, s.params.num_points)) * np.exp(s.params.scales.numpy()).max(1)
              for s in fr.segments]  # about the scales: both the covariance and coef move
    v = pc.v_records(case, "all")
    h = 1e-6
    pose0 = pz.frame_poses(fr).astype(np.float64)
    got = fc.v_pose_ref(fr, st, sigmas, v, antialiased)
    fd = np.zeros_like(pose0)
    for idx in np.ndindex(*pose0.shape):
        vals = []
        for sgn in (1, -1):
            p = pose0.copy()
            p[idx] += sgn * h
            vals.append(float(fc.pose_loss(fr, st, sigmas, v, torch.tensor(p), antialiased)))
        fd[idx] = (vals[0] - vals[1]) / (2 * h)
    assert np.abs(got - fd).max() <= 1e-5 * np.abs(fd).max()
    view0 = np.asarray(fr.camera.viewmat(), np.float64).reshape(-1)
    got = fc.v_view_ref(fr, st, sigmas, v, antialiased)
    fd = np.zeros(12)
    for k in range(12):
        vals = []
        for sgn in (1, -1):
            w = view0.copy()
            w[k] += sgn * h
            vals.append(float(fc.view_loss(fr, st, sigmas, v, torch.tensor(w), antialiased)[0]))
        fd[k] = (vals[0] - vals[1]) / (2 * h)
    assert np.abs(got - fd).max() <= 1e-5 * np.abs(fd).max()


def test_settled_cases():
    """Every filtered case of the directed tests: no filtered decision within the margin, and the families are what they say."""
    from tests import filter3d_cases as fc
    for name in fc.CONFIGS:
        c = fc.get(name)
        sig = np.concatenate(c.sigmas)
        fw = f3.forward(c.frame, c.st, c.sigmas)
        assert fw["margin"].min(initial=np.inf) >= pc.MARGIN, name
        assert np.all(sig[c.rows("zero")] == 0) and np.all(sig[~c.rows("zero")] >= 0), name
        idn = c.rows("identity") & c.thin.any(1)
        und = c.rows("underflow") & c.thin.any(1)
        assert np.all(sig[idn] == 0) and np.all(sig[und] > 0), name
        assert np.all(fw["coef"][idn] == 1.0), name
        f32 = f3.forward(c.frame, c.st, c.sigmas, dtype=torch.float32)
        assert np.all(f32["coef"][und] == 0), name  # in float32 an underflowed axis has r = 0
        assert np.all(np.isfinite(f32["records"])), name
        if name.startswith("comp_edges/") and not name.endswith("needle"):
            assert (idn | und).sum() == 6, name
        if name.endswith("/dominant"):
            assert np.all(fw["coef"][fw["vis"]] < 0.05), name
    mixed = fc.get("posed40/mixed")
    assert len(np.unique(mixed.fams)) == len(fc.FAMILIES)
