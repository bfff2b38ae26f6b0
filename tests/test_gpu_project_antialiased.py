"""The projection kernels in the antialiased rasterize mode (sgn_camera.antialiased = 1) on the hand-built Gaussians of
tests/project_cases.py and tests/antialias_cases.py, against the float64 reference with comp not detached
(oracle/project_aa_ref64.py) and the C oracle in the same mode (oracle/oracle_aa.py) -- the bars and helpers of
tests/test_gpu_project_directed.py.

Forward, every case through the direct and the staged kernel (SGN_PROJECT_STAGED):
  * the two forms agree bit for bit on every output array;
  * every record column but [5] and [11] is the classic mode's, bit for bit; classic records have [11] == 0; the antialiased
    [5] is float32(classic [5] x [11]);
  * the exact section and the integer outputs equal the C oracle's and the float64 reference's; record [5]
    (sigmoid x comp) and [11] (comp) of visible rows are within FWD_K x (the row's fp32 noise, at least eps32 kappa |ref|:
    tests/antialias_cases.py comp_condition) + FWD_R x max|ref| of float64;
  * touch mask: the property of the classic test with tau = ln(255 x record [5]), the compensated opacity;
  * comp_edges: its needles have comp == 0 exactly, opacity 0 and touch no tile; its wide Gaussians have comp > 0.99.
Backward, each cotangent alone (xy, conic, opacity, rgb, depth) and all of them, against float64 autograd with the bars of
the classic test, and for means, scales and quats at least COND_K eps32 kappa of the row's scale (tests/antialias_cases.py
comp_condition: comp's gradient reaches them through cov2d, which cancels by kappa, a needle's squared aspect ratio); the opacity-only cotangent must move means, scales and quats of rows with comp > 0; every gradient is
finite and the needles (comp == 0) get exactly zero geometry and opacity gradient from it.  The pose and view forms: the
parameter gradients are the plain form's bits, v_pose and v_view within relative L2 1e-3 of float64.  Range-backward
partitions are bit-identical to the single call.  Level-1: sgn_l1_project_bwd_comp with a compensation cotangent against
float64; without one it returns sgn_l1_project_bwd's bits, and gsplat_compat.project_gaussians picks the entry by whether
compensation has a cotangent.

Each of these one-token changes to project.cu fails tests here (on an H100 80GB HBM3 at a 700 W power limit): dropping comp's
cotangent from the backward (v_comp -> 0 in the VJP) 37 of 71, taking s (1 - s) from record [5] 30, leaving comp out of the
touch tau (the direct kernel's touch context built from the sigmoid) 28, making the staged kernel ignore the flag 28.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from street_gaussians_ns_b200 import _lib, gsplat_compat, raster
from oracle import oracle_aa
from oracle import project_aa_ref64 as aa
from oracle import project_ref64 as ref
from tests import antialias_cases as ac
from tests import pose_cases as pz
from tests import project_cases as pc
from tests.test_gpu_project_directed import (BWD_K, BWD_R, BWD_R_CONIC, DEV, FWD_K, FWD_R, KINDS, PARAMS, _cuda_frame, _l1_inputs,
                                             _partitions, _ptr, check_touch)

pytestmark = pytest.mark.gpu

CASES = {**pc.CASES, "comp_edges": ac.comp_edges}
_BUILT = {}


def get(name):
    if name not in _BUILT:
        _BUILT[name] = CASES[name]() if name == "comp_edges" else pc.get(name)
    return _BUILT[name]


def _settings(case, mode="antialiased"):
    st = case.st
    return raster.RenderSettings(sh_degree=st.sh_degree, sh_degree_to_use=st.deg_use, block_width=st.block_width,
                                 clip_thresh=st.clip_thresh, rasterize_mode=mode)


def run_forward(case, staged, monkeypatch, mode="antialiased"):
    monkeypatch.setenv("SGN_PROJECT_STAGED", "1" if staged else "0")
    frc = _cuda_frame(case)
    params = [s.params.tensors() for s in frc.segments]
    table = raster.SegmentTable(frc, params, DEV)
    cs = raster.camera_struct(frc.camera, _settings(case, mode))
    pr = raster.project_fwd(table, cs, DEV)
    torch.cuda.synchronize()
    out = dict(records=pr.records.cpu().numpy(), radii=pr.radii.cpu().numpy(), tiles_hit=pr.tiles_hit.cpu().numpy(),
               bbox=pr.bbox.cpu().numpy().view(np.uint16).astype(np.int64), tiles_touched=pr.tiles_touched.cpu().numpy(),
               touch_mask=pr.touch_mask.cpu().numpy().view(np.uint32))
    return table, params, cs, pr, out


_REF = {}


def ref_forward(case, dtype):
    key = (case.name, dtype)
    if key not in _REF:
        _REF[key] = aa.forward(case.frame, case.st, dtype)
    return _REF[key]


def check_forward(case, got, classic):
    rec, crec = got["records"], classic["records"]
    vis = case.fwd["vis"]
    # the mode touches [5] and [11] only
    keep = [0, 1, 2, 3, 4, 6, 7, 8, 9, 10]
    assert rec[:, keep].tobytes() == crec[:, keep].tobytes(), f"{case.name}: a column other than opacity / comp moved"
    for k in ("radii", "tiles_hit", "bbox"):
        assert got[k].tobytes() == classic[k].tobytes(), f"{case.name}: {k}"
    assert np.all(crec[:, 11] == 0)
    np.testing.assert_array_equal(rec[:, 5], (crec[:, 5] * rec[:, 11]).astype(np.float32))
    # exact section and the antialiased C oracle's opacity
    orc = oracle_aa.AntialiasedOracle(case.frame, case.st.sh_degree, case.st.deg_use, case.st.block_width,
                                      case.st.clip_thresh).project()
    np.testing.assert_array_equal(rec[:, 0:2], orc["xys"])
    np.testing.assert_array_equal(rec[:, 2:5], orc["conics"])
    np.testing.assert_array_equal(got["radii"], orc["radii"])
    np.testing.assert_array_equal(got["tiles_hit"], orc["num_tiles_hit"])
    assert np.all(orc["opac"][~vis] == 0)
    # opacity and comp against float64 (the oracle's opacity, float32(sigmoid x float64 comp), is no better a reference)
    fw, f32 = ref_forward(case, torch.float64), ref_forward(case, torch.float32)
    np.testing.assert_array_equal(got["radii"], fw["radii"])
    worst = 0.0
    kappa = ac.comp_condition(fw["records"])
    for col in (5, 11):
        r64 = fw["records"][:, col]
        noise = np.maximum(np.abs(f32["records"][:, col] - r64), ac.EPS32 * kappa * np.abs(r64))
        bar = FWD_K * noise + FWD_R * np.maximum(np.abs(r64), 1e-3)
        ratio = np.where(vis, np.abs(rec[:, col].astype(np.float64) - r64) / bar, 0.0)
        worst = max(worst, ratio.max(initial=0.0))
        g = int(np.argmax(ratio)) if ratio.size else 0
        assert ratio.max(initial=0.0) <= 1.0, f"{case.name}: record column {col} of row {g}: {rec[g, col]!r} vs {r64[g]!r}"
    assert np.all(rec[~vis][:, [5, 11]] == 0)
    return worst


@pytest.mark.parametrize("name", list(CASES))
def test_forward_direct_and_staged(name, monkeypatch):
    case = get(name)
    outs = [run_forward(case, staged, monkeypatch)[-1] for staged in (False, True)]
    for k in outs[0]:
        assert outs[0][k].tobytes() == outs[1][k].tobytes(), f"{name}: {k} differs between the direct and the staged kernel"
    classic = run_forward(case, False, monkeypatch, "classic")[-1]
    worst = check_forward(case, outs[0], classic)
    check_touch(case, outs[0])
    got = outs[0]
    if name == "comp_edges":
        needles = np.array(case.notes["needles"])
        assert np.all(case.fwd["vis"][needles])
        assert np.all(got["records"][needles, 11] == 0) and np.all(got["records"][needles, 5] == 0)
        assert np.all(got["tiles_touched"][needles] == 0) and np.all(got["touch_mask"][needles] == 0)
        assert np.all(classic["tiles_touched"][needles] > 0)
        wide = np.arange(len(needles) + 12, len(needles) + 16)
        assert np.all(got["records"][wide, 11] > 0.99)
    print(f"[fwd aa] {name}: worst {worst:.3f} of the bar, M {int(got['tiles_touched'].sum())} (classic "
          f"{int(classic['tiles_touched'].sum())})")


def check_backward(case, flat, v, tag=""):
    r64 = aa.backward(case.frame, case.st, v)
    r32 = aa.backward(case.frame, case.st, v, torch.float32)
    vis = case.fwd["vis"]
    kappa = ac.comp_condition(ref_forward(case, torch.float64)["records"]) if ("opacity" in tag or "all" in tag) else 0 * vis
    Kuse = (case.st.deg_use + 1) ** 2
    R = BWD_R_CONIC if ("conic" in tag or "all" in tag) else BWD_R
    worst, k, row0 = 0.0, 0, 0
    for i, seg in enumerate(case.frame.segments):
        n = seg.params.num_points
        geo = np.max([np.abs(r64[i][p].reshape(n, -1)).max(1) for p in PARAMS[:3]], 0) if n else None
        for name in PARAMS:
            k += 1
            if n == 0:
                continue
            got = flat[k - 1].detach().cpu().numpy().astype(np.float64).reshape(n, -1)
            assert np.all(np.isfinite(got)), f"{case.name}{tag}: {name} is not finite"
            assert np.all(got[~vis[row0:row0 + n]] == 0), f"{case.name}{tag}: {name} of an invisible row is not zero"
            a64, a32 = r64[i][name].reshape(n, -1), r32[i][name].reshape(n, -1)
            if got.shape[1] == 0:
                continue
            err = np.abs(got - a64).max(1)
            scale = np.maximum(np.abs(a64).max(1), geo) if name in PARAMS[:3] else np.abs(a64).max(1)
            bar = np.maximum(BWD_K * np.abs(a32 - a64).max(1), R * scale)
            if name in PARAMS[:3]:
                bar = np.maximum(bar, ac.COND_K * ac.EPS32 * kappa[row0:row0 + n] * scale)
            ratio = np.where(err == 0, 0.0, err / np.where(bar > 0, bar, 1e-300))
            worst = max(worst, ratio.max())
            r = int(np.argmax(ratio))
            assert ratio.max() <= 1.0, (f"{case.name}{tag}: {name} of row {r} of segment {i}: {got[r].tolist()} vs "
                                        f"{a64[r].tolist()} (fp32 noise {np.abs(a32 - a64)[r].max():.3e})")
            if name == "features_rest":
                assert np.all(got[:, 3 * (Kuse - 1):] == 0)
        row0 += n
    return worst


@pytest.mark.parametrize("name", list(CASES))
def test_backward_each_cotangent(name, monkeypatch):
    case = get(name)
    table, params, cs, pr, out = run_forward(case, False, monkeypatch)
    comp = out["records"][:, 11]
    worst = {}
    for kind in KINDS:
        v = pc.v_records(case, kind)
        flat, _ = raster.project_bwd(table, params, cs, pr.records, pr.radii, torch.from_numpy(v).to(DEV))
        torch.cuda.synchronize()
        worst[kind] = check_backward(case, flat, v, f" [{kind}]")
        if kind == "opacity":  # the opacity cotangent now moves the geometry, through comp
            geo = np.concatenate([np.concatenate([flat[6 * i + j].detach().cpu().numpy().reshape(s.params.num_points, w)
                                                  for j, w in enumerate((3, 3, 4))], 1) for i, s in enumerate(case.frame.segments)], 0)
            moved = np.abs(geo).max(1) > 0
            assert moved[comp > 0].mean() > 0.99 and not moved[comp == 0].any(), \
                f"{name}: the opacity cotangent must move the geometry of the rows with comp > 0, and only those"
            if name == "comp_edges":
                needles = np.array(case.notes["needles"])
                assert np.all(flat[5].detach().cpu().numpy()[needles] == 0)
    print(f"[bwd aa] {name}: " + " ".join(f"{k} {w:.3f}" for k, w in worst.items()))


@pytest.mark.parametrize("name", ["layout", "staged_mix", "posed40", "comp_edges"])
def test_range_backward(name, monkeypatch):
    case = get(name)
    table, params, cs, pr, _ = run_forward(case, False, monkeypatch)
    v = torch.from_numpy(pc.v_records(case, "all")).to(DEV)
    size = sum(raster.arena_layout(table.static)[0])
    _, full = raster.project_bwd(table, params, cs, pr.records, pr.radii, v, out=torch.zeros(size, device=DEV))
    full = full.cpu().numpy()
    for ranges in _partitions(table):
        _, arena = raster.project_bwd(table, params, cs, pr.records, pr.radii, v, make_views=False, chunk_ranges=ranges,
                                      out=torch.zeros(size, device=DEV))
        assert arena.cpu().numpy().tobytes() == full.tobytes(), f"{name}: partition {ranges} differs from the single call"


def _rel_l2(a, b):
    return pz.rel_l2(a, b)


@pytest.mark.parametrize("name", ["posed40", "layout", "comp_edges", "fov_clamp"])
def test_pose_and_view_forms(name, monkeypatch):
    case = get(name)
    table, params, cs, pr, _ = run_forward(case, False, monkeypatch)
    v_np = pc.v_records(case, "all")
    v = torch.from_numpy(v_np).to(DEV)
    size = sum(raster.arena_layout(table.static)[0])
    _, plain = raster.project_bwd(table, params, cs, pr.records, pr.radii, v, make_views=False, out=torch.zeros(size, device=DEV))
    plain = plain.cpu().numpy()
    vm = torch.from_numpy(np.concatenate([case.frame.camera.viewmat().reshape(-1), case.frame.camera.cam_pos()])).to(DEV)
    v_view = torch.zeros(_lib.VIEW_FLOATS, device=DEV)
    _, arena_v = raster.project_bwd(table, params, cs, pr.records, pr.radii, v, make_views=False, view=vm, v_view=v_view,
                                    out=torch.zeros(size, device=DEV))
    assert arena_v.cpu().numpy().tobytes() == plain.tobytes(), f"{name}: the view form's parameter gradients differ"
    want = ac.v_view_ref(case.frame, case.st, v_np)
    e = _rel_l2(v_view.cpu().numpy(), want)
    assert e <= 1e-3, f"{name}: v_view relative L2 {e:.2e}"
    if any(s.has_pose for s in case.frame.segments):
        v_pose = torch.empty(table.nseg, _lib.POSE_FLOATS, device=DEV)
        _, arena_p = raster.project_bwd(table, params, cs, pr.records, pr.radii, v, make_views=False, v_pose=v_pose,
                                        out=torch.zeros(size, device=DEV))
        assert arena_p.cpu().numpy().tobytes() == plain.tobytes(), f"{name}: the pose form's parameter gradients differ"
        got = v_pose.cpu().numpy()[[i for i, s in enumerate(case.frame.segments) if s.has_pose]].astype(np.float64)
        want_p = ac.v_pose_ref(case.frame, case.st, v_np)
        for a in range(want_p.shape[0]):
            if np.any(want_p[a]):
                assert _rel_l2(got[a], want_p[a]) <= 1e-3, f"{name}: v_pose of posed segment {a}"
            else:
                assert not np.any(got[a])


# ------------------------------------------------------------------------------------------------------------------
# Level-1
# ------------------------------------------------------------------------------------------------------------------
def _l1_call(L, fn, N, d, glob_scale, cs, radii, v, with_comp):
    outs = [torch.full((N, w), float("nan"), device=DEV) for w in (3, 3, 4)]
    args = [N, _ptr(d["m"]), _ptr(d["s"]), C.c_float(glob_scale), _ptr(d["q"]), C.byref(cs), _ptr(radii), _ptr(v["xys"]),
            _ptr(v["depths"]), _ptr(v["conics"])]
    if with_comp:
        args.append(_ptr(v["comp"]))
    _lib.check(getattr(L, fn)(*args, *[_ptr(t) for t in outs], None), fn)
    torch.cuda.synchronize()
    return [t.cpu().numpy() for t in outs]


@pytest.mark.parametrize("glob_scale", [1.0, 0.37])
@pytest.mark.parametrize("name", ["fov_clamp", "shapes", "comp_edges"])
def test_l1_compensation_cotangent(name, glob_scale):
    L = _lib.load()
    if name == "comp_edges":
        case = get(name)
        seg = case.frame.segments[0]
        m = seg.params.means.numpy().astype(np.float32)
        s = np.exp(seg.params.scales.numpy().astype(np.float64)).astype(np.float32)
        q = seg.params.quats.numpy().astype(np.float32)
    else:
        case, m, s, q = _l1_inputs(name)
    N = m.shape[0]
    cs = raster.camera_struct(case.frame.camera, _settings(case, "classic"))
    d = {k: torch.from_numpy(a).to(DEV) for k, a in (("m", m), ("s", s), ("q", q))}
    o = [torch.zeros(N, 2), torch.zeros(N), torch.zeros(N, dtype=torch.int32), torch.zeros(N, 3), torch.zeros(N),
         torch.zeros(N, dtype=torch.int32), torch.zeros(N, 6)]
    o = [t.to(DEV) for t in o]
    _lib.check(L.sgn_l1_project_fwd(N, _ptr(d["m"]), _ptr(d["s"]), C.c_float(glob_scale), _ptr(d["q"]), C.byref(cs),
                                    *[_ptr(t) for t in o], None), "sgn_l1_project_fwd")
    radii, comp = o[2], o[4].cpu().numpy()
    rng = np.random.default_rng(9)
    vs = dict(xys=rng.uniform(-1, 1, (N, 2)), depths=rng.uniform(-1, 1, N), conics=rng.uniform(-1, 1, (N, 3)),
              comp=rng.uniform(-1, 1, N))
    vs = {k: a.astype(np.float32) for k, a in vs.items()}
    fw = ref.l1_project(m, s, np.float32(glob_scale), q, case.frame.camera, case.st.block_width, case.st.clip_thresh)
    ok = fw["margin"] >= pc.MARGIN
    vis = ok & fw["vis"]
    rec64 = np.zeros((N, 12))
    rec64[:, 2:5] = fw["conics"].detach().double().numpy()
    rec64[:, 11] = fw["compensation"]
    kappa = ac.comp_condition(rec64)
    for drop_others in (True, False):  # the compensation cotangent alone, then with the other three
        v = {k: (None if drop_others and k != "comp" else a) for k, a in vs.items()}
        vd = {k: (None if a is None else torch.from_numpy(a).to(DEV)) for k, a in v.items()}
        got = _l1_call(L, "sgn_l1_project_bwd_comp", N, d, glob_scale, cs, radii, vd, True)
        r = aa.l1_project_bwd(m, s, np.float32(glob_scale), q, case.frame.camera, v["xys"], v["depths"], v["conics"], v["comp"],
                               case.st.block_width, case.st.clip_thresh)
        r32 = aa.l1_project_bwd(m, s, np.float32(glob_scale), q, case.frame.camera, v["xys"], v["depths"], v["conics"], v["comp"],
                                 case.st.block_width, case.st.clip_thresh, dtype=torch.float32)
        geo = np.max([np.abs(x).max(1) for x in r], 0)
        R = BWD_R if drop_others else BWD_R_CONIC
        for t, a64, a32, nm in zip(got, r, r32, ("means", "scales", "quats")):
            assert np.all(np.isfinite(t)), f"{name}: v_{nm}"
            g = t.astype(np.float64)
            assert np.all(g[~fw["vis"] & ok] == 0), f"{name}: v_{nm} of an invisible row"
            err = np.abs(g - a64).max(1)[vis]
            bar = np.maximum.reduce([BWD_K * np.abs(a32 - a64).max(1), R * geo, ac.COND_K * ac.EPS32 * kappa * geo])[vis]
            assert np.all(err <= bar), (f"{name} (comp alone: {drop_others}): v_{nm} worst "
                                        f"{np.max(err / np.maximum(bar, 1e-300)):.2f} of the bar")
            if drop_others:
                assert np.all(g[comp == 0] == 0), f"{name}: v_{nm} through a zero compensation"
    # no compensation cotangent: the old entry's bits, through either entry
    vd = {k: torch.from_numpy(a).to(DEV) for k, a in vs.items()}
    old = _l1_call(L, "sgn_l1_project_bwd", N, d, glob_scale, cs, radii, vd, False)
    vd["comp"] = None
    new = _l1_call(L, "sgn_l1_project_bwd_comp", N, d, glob_scale, cs, radii, vd, True)
    for a, b in zip(old, new):
        assert a.tobytes() == b.tobytes()


def test_gsplat_compat_routes_the_compensation_cotangent():
    case, m, s, q = _l1_inputs("shapes")
    cam = case.frame.camera
    vm = torch.eye(4)
    vm[:3, :] = torch.from_numpy(cam.viewmat())
    qn = q / np.linalg.norm(q, axis=1, keepdims=True)

    def grads(use_comp):
        leaves = [torch.from_numpy(a).to(DEV).requires_grad_(True) for a in (m, s, qn.astype(np.float32))]
        xys, depths, radii, conics, comp, _, _ = gsplat_compat.project_gaussians(
            leaves[0], leaves[1], 1.0, leaves[2], vm.to(DEV), cam.fx, cam.fy, cam.cx, cam.cy, cam.height, cam.width, 16)
        loss = xys.sum() + conics.sum() + (comp.sum() if use_comp else 0.0)
        loss.backward()
        return [t.grad.cpu().numpy() for t in leaves], comp.detach().cpu().numpy()

    g0, _ = grads(False)
    g1, comp = grads(True)
    assert g0[1].tobytes() != g1[1].tobytes()  # the compensation's cotangent reached the scales
    # without it: the Level-1 backward of before, bit for bit
    L = _lib.load()
    N = m.shape[0]
    cs = gsplat_compat._common.camera_struct(vm.to(DEV), cam.fx, cam.fy, cam.cx, cam.cy, cam.height, cam.width, 16)
    d = {k: torch.from_numpy(a).to(DEV) for k, a in (("m", m), ("s", s), ("q", qn.astype(np.float32)))}
    o = [torch.zeros(N, 2), torch.zeros(N), torch.zeros(N, dtype=torch.int32), torch.zeros(N, 3), torch.zeros(N),
         torch.zeros(N, dtype=torch.int32), torch.zeros(N, 6)]
    o = [t.to(DEV) for t in o]
    _lib.check(L.sgn_l1_project_fwd(N, _ptr(d["m"]), _ptr(d["s"]), C.c_float(1.0), _ptr(d["q"]), C.byref(cs),
                                    *[_ptr(t) for t in o], None), "sgn_l1_project_fwd")
    ones = {"xys": torch.ones(N, 2, device=DEV), "depths": None, "conics": torch.ones(N, 3, device=DEV)}
    want = _l1_call(L, "sgn_l1_project_bwd", N, d, 1.0, cs, o[2], ones, False)
    for a, b in zip(g0, want):
        assert a.tobytes() == b.tobytes()
