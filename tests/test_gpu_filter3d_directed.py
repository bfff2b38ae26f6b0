"""The 3D-filtered projection (sgn_camera.filter_3d, Mip-Splatting's smoothing filter) on hand-built Gaussians against the
float64 statement (oracle/filter3d_ref64.py), in the classic and the antialiased rasterize mode, with the helpers and the
bars of tests/test_gpu_project_directed.py and tests/test_gpu_project_antialiased.py.

Cases (tests/filter3d_cases.py): every case of tests/project_cases.py with the ``mixed`` sigma family; the pure families
zero, faint, even, dominant and needle on ``shapes``, ``posed40`` and ``layout``; tests/antialias_cases.py's ``comp_edges``
(needles whose thin axes of exp(-80) underflow in float32) with ``needle``, ``underflow`` and ``identity``; and
``thin_discs`` (one thin axis, two wide ones, comp > 0) with ``underflow`` and ``identity``.  Every filtered decision is at
least project_cases.MARGIN from its threshold (sigma re-drawn, the parameters untouched).

Forward, every case and mode through the direct and the staged kernel (SGN_PROJECT_STAGED):
  * the two forms agree bit for bit on every output array, on every row;
  * radii, num_tiles_hit, the tile AABB of visible rows and the aux bits equal the float64 statement's; each float record
    field group of a visible row is within FWD_K x (its fp32 noise: the statement run in float32; for the opacity and comp
    of the antialiased mode at least eps32 kappa |ref|, antialias_cases.comp_condition) + FWD_R x max|ref|;
  * invisible rows carry only the class bit and touch nothing; the touch mask holds against the kernel's own filtered record;
  * underflow rows (sigma > 0 beside a thin axis): record [5] == 0 exactly and no tile touched; identity rows (sigma 0 on a
    thin axis): record [5] is the unfiltered projection's, bit for bit (coef == 1).  In the antialiased mode these checks
    bite only on thin_discs: comp_edges' needles have comp == 0, so their opacity is 0 with or without the filter.
Backward, each cotangent alone (xy, conic, opacity, rgb, depth) and all of them, per Gaussian and per parameter row against
float64 autograd with the float32 run of the same statement as the noise: the classic bars BWD_K / BWD_R / BWD_R_CONIC, and in
the antialiased mode also COND_K eps32 kappa of the row's scale for means, scales and quats when the opacity cotangent takes
part; invisible rows and features_rest beyond sh_degree_to_use exactly zero.  Underflow rows get an exactly zero opacity
gradient and an exactly zero gradient on every underflowed axis' scale (r = 0 and coef = 0 there), while every axis that
did not underflow (a needle's long axis, a disc's wide ones) still gets its geometry gradient from a conic cotangent.
Zero filter, every project_cases case in both modes: an all-zero filter gives the unfiltered projection's bits -- forward
records, radii, tile boxes and touch masks of both forms, the backward arena, v_pose and v_view -- since sqrt(fl(s^2)) == s
for a normal s^2 and r = coef = 1 exactly.  The one difference allowed is the sign of a zero log-scale gradient, and only
in the log-scale slots of the arena: the filtered chain ends in g r + v (1 - r), which turns g = -0 into +0.
Range backward with the filter (layout, staged_mix, posed40, nseg1024, both modes): every partition is bit-identical to the
single call, and issued ranges write nothing outside their chunks.  The pose and view forms: their parameter gradients are
the plain form's bits; v_pose (each of v_R, v_t, v_q) and v_view within 1e-3 relative L2 of the float64 statements of
tests/filter3d_cases.py.

Every filter size is read from one device buffer holding all segments' sizes, padded by N floats: an index past a
segment's own rows reads another row's sigma, a wrong value the checks see, and never leaves the allocation.

Three bars are wider than the unfiltered files', each from a conditioning argument: the conic's forward noise is at least
the unfiltered row's relative float32 noise times the filtered conic's own size (_plain_conic_noise); the log-scale
gradient's bar is at least FILT_K eps32 |v_opacity x record [5]| (the coef term's 1 - r cancels as r -> 1); in the
antialiased mode the opacity gradient's bar is at least BWD_K eps32 kappa of its size, as record [5]'s is in the forward.

Observed on an H100 80GB HBM3 (700 W power limit), 260 tests in 93 s: the forward's float fields at most 0.75 of their bar,
the backward at most 0.41 (opacity cotangent; xy 0.10, conic 0.13, rgb 0.10, depth 0.01, all five 0.13), v_pose / v_view at
most 1.5e-5 relative L2 (of 1e-3); with a zero filter 4951 log-scale gradients over the classic cases (none in the
antialiased mode) differ from the unfiltered ones only in the sign of a zero.  One-token changes to project.cu /
sgn_exact.cuh and the tests each fails: r and 1 - r swapped in the scale gradient 148, v_coef taken after f has taken coef
88, v_comp *= coef dropped 47, the direct form's touch context built from the opacity before coef 79, sgn_filter_axis
returning r = 0 when s^2 + sigma^2 == 0 6, sigma indexed by the global row in the backward 56 and in the staged forward 48,
the staged form's ge[9] and ge[10] swapped 145, one sign of the pose partials' v_q 8.
"""
import types

import numpy as np
import pytest
import torch

from oracle import filter3d_ref64 as f3
from oracle import project_ref64 as ref
from street_gaussians_ns_b200 import _lib, raster
from street_gaussians_ns_b200.scene import Frame, Segment
from tests import antialias_cases as ac
from tests import filter3d_cases as fc
from tests import pose_cases as pz
from tests import project_cases as pc
from tests.test_gpu_project_directed import (BWD_K, BWD_R, BWD_R_CONIC, DEV, FWD_K, FWD_R, KINDS, PARAMS, _partitions,
                                             _written_mask, check_touch)

pytestmark = pytest.mark.gpu

MODES = ("classic", "antialiased")
TOL = 1e-3  # v_pose / v_view: relative L2 against float64 (tests/test_gpu_pose_grad.py, tests/test_gpu_camera_grad.py)
F32, F64 = torch.float32, torch.float64
# The coef term of a log-scale's gradient is v_c (1 - r), v_c = v_opacity x record [5].  r = fl(fl(s^2) / fl(s^2 + sigma^2))
# is within three half-ulps of its value, so 1 - r carries an absolute error of up to 1.5 eps32 whatever its size -- a
# relative error of eps32 / (1 - r) once sigma << s and r -> 1 -- and the term an error of 1.5 eps32 |v_c|.  FILT_K: the
# bar's multiple of eps32 |v_c| (the float32 statement's autograd rounds the same cancellation differently, so its noise
# does not bound the kernel's).
FILT_K = 4.0


def _settings(case, mode):
    st = case.st
    return raster.RenderSettings(sh_degree=st.sh_degree, sh_degree_to_use=st.deg_use, block_width=st.block_width,
                                 clip_thresh=st.clip_thresh, rasterize_mode=mode)


def _cuda_frame(case, sigmas):
    """The frame on the device; sigmas None: no filter, else every segment's sizes as a view of one padded buffer."""
    views = [None] * len(case.frame.segments)
    if sigmas is not None:
        sizes = [len(s) for s in sigmas]
        N = sum(sizes)
        buf = torch.zeros(2 * N + 1, dtype=torch.float32, device=DEV)
        buf[:N] = torch.from_numpy(np.concatenate(sigmas) if N else np.zeros(0, np.float32)).to(DEV)
        offs = np.concatenate([[0], np.cumsum(sizes)])
        views = [buf[offs[i]:offs[i + 1]] for i in range(len(sizes))]
    return Frame(case.frame.camera, [Segment(s.params.to("cuda"), s.cls, s.rot, s.center, s.idft, filter_3d=f)
                                     for s, f in zip(case.frame.segments, views)])


def run_forward(case, sigmas, mode, staged, monkeypatch):
    monkeypatch.setenv("SGN_PROJECT_STAGED", "1" if staged else "0")
    frc = _cuda_frame(case, sigmas)
    params = [s.params.tensors() for s in frc.segments]
    table = raster.SegmentTable(frc, params, DEV)
    cs = raster.camera_struct(frc.camera, _settings(case, mode))
    pr = raster.project_fwd(table, cs, DEV)
    torch.cuda.synchronize()
    out = dict(records=pr.records.cpu().numpy(), radii=pr.radii.cpu().numpy(), tiles_hit=pr.tiles_hit.cpu().numpy(),
               bbox=pr.bbox.cpu().numpy().view(np.uint16).astype(np.int64), tiles_touched=pr.tiles_touched.cpu().numpy(),
               touch_mask=pr.touch_mask.cpu().numpy().view(np.uint32))
    return dict(frc=frc, table=table, params=params, cs=cs, pr=pr, out=out)


_FWD = {}


def ref_forward(fcase, mode, dtype):
    key = (fcase.name, mode, dtype)
    if key not in _FWD:
        _FWD[key] = f3.forward(fcase.frame, fcase.st, fcase.sigmas, antialiased=mode == "antialiased", dtype=dtype)
    return _FWD[key]


_BWD = {}


def ref_backward(fcase, mode, kind, v, dtype):
    key = (fcase.name, mode, kind, dtype)
    if key not in _BWD:
        _BWD[key] = f3.backward(fcase.frame, fcase.st, fcase.sigmas, v, antialiased=mode == "antialiased", dtype=dtype)
    return _BWD[key]


def _outs_equal(a, b, what):
    for k in a:
        assert a[k].tobytes() == b[k].tobytes(), f"{what}: {k}"


_PLAIN = {}


def _plain_conic_noise(fcase):
    """Per row, the unfiltered projection's float32 noise of the conic relative to the row's largest conic entry,
    max |conic32 - conic64| / max |conic64|.  One float32 run of the filtered statement can land unusually close to float64
    on a row (it did for a conic of layout by 5x).  The filter only adds sigma^2 to the covariance's eigenvalues, so the row
    is no worse conditioned than without it: the conic's relative error is no larger, and this relative noise times the
    filtered conic's own size is a floor of its noise.  xy and depth need no floor: the filter does not move them, and the
    filtered statement's float32 noise of them is the unfiltered one."""
    name = fcase.base.name
    if name not in _PLAIN:
        c64 = ref.forward(fcase.frame, fcase.st)["records"][:, 2:5]
        c32 = ref.forward(fcase.frame, fcase.st, F32)["records"][:, 2:5]
        mag = np.abs(c64).max(1)
        _PLAIN[name] = np.where(mag > 0, np.abs(c32 - c64).max(1) / np.where(mag > 0, mag, 1.0), 0.0)
    return _PLAIN[name]


def check_forward(fcase, mode, got):
    fw, f32 = ref_forward(fcase, mode, F64), ref_forward(fcase, mode, F32)
    vis, rec, aa_ = fw["vis"], got["records"], mode == "antialiased"
    np.testing.assert_array_equal(got["radii"], fw["radii"])
    np.testing.assert_array_equal(got["tiles_hit"], fw["num_tiles_hit"])
    np.testing.assert_array_equal(got["bbox"][vis], np.concatenate([fw["tmin"], fw["tmax"]], 1)[vis])
    np.testing.assert_array_equal(rec[:, 10].view(np.int32), fw["aux"])
    if not aa_:
        assert np.all(rec[:, 11] == 0)
    kappa = ac.comp_condition(fw["records"]) if aa_ else np.zeros(len(vis))
    worst = 0.0
    for cols in ([0, 1], [2, 3, 4], [5], [6, 7, 8], [9]) + (([11],) if aa_ else ()):
        r64 = fw["records"][:, cols]
        noise = np.abs(f32["records"][:, cols] - r64).max(1, keepdims=True)
        if cols[0] == 2:  # the conic: at least the unfiltered row's relative noise times its own size (_plain_conic_noise)
            noise = np.maximum(noise, _plain_conic_noise(fcase)[:, None] * np.abs(r64).max(1, keepdims=True))
        if aa_ and cols[0] in (5, 11):
            noise = np.maximum(noise, ac.EPS32 * kappa[:, None] * np.abs(r64))
        bar = FWD_K * noise + FWD_R * np.maximum(np.abs(r64).max(1, keepdims=True), 1e-3)
        ratio = np.where(vis[:, None], np.abs(rec[:, cols].astype(np.float64) - r64) / bar, 0.0)
        worst = max(worst, ratio.max(initial=0.0))
        g = np.unravel_index(np.argmax(ratio), ratio.shape) if ratio.size else (0, 0)
        assert ratio.max(initial=0.0) <= 1.0, (f"{fcase.name} [{mode}]: record column {cols[g[1]]} of row {g[0]}: "
                                               f"{rec[g[0], cols[g[1]]]!r} vs {r64[g]!r}")
    inv = ~vis
    assert np.all(rec[inv][:, [0, 1, 5, 6, 7, 8, 9, 11]] == 0)
    cls_bit = np.concatenate([np.full(s.params.num_points, s.cls) for s in fcase.frame.segments]) == 1
    np.testing.assert_array_equal(rec[inv, 10].view(np.int32), np.where(cls_bit[inv], 8, 0))
    assert np.all(got["tiles_touched"][inv] == 0) and np.all(got["touch_mask"][inv] == 0)
    return worst


def _touch_case(fcase, mode):
    return types.SimpleNamespace(name=f"{fcase.name} [{mode}]", frame=fcase.frame, st=fcase.st,
                                 fwd={"vis": ref_forward(fcase, mode, F64)["vis"]})


def _underflow_rows(fcase):
    return fcase.rows("underflow") & fcase.thin.any(1)


def _identity_rows(fcase):
    return fcase.rows("identity") & fcase.thin.any(1)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", fc.CONFIGS)
def test_forward_direct_and_staged(name, mode, monkeypatch):
    fcase = fc.get(name)
    outs = [run_forward(fcase, fcase.sigmas, mode, staged, monkeypatch)["out"] for staged in (False, True)]
    _outs_equal(outs[0], outs[1], f"{name} [{mode}]: the direct and the staged kernel differ")
    got = outs[0]
    worst = check_forward(fcase, mode, got)
    check_touch(_touch_case(fcase, mode), got)
    vis = ref_forward(fcase, mode, F64)["vis"]
    u = _underflow_rows(fcase) & vis
    if u.any():
        assert np.all(got["records"][u, 5] == 0), f"{name} [{mode}]: an underflow row has a non-zero opacity"
        assert np.all(got["tiles_touched"][u] == 0) and np.all(got["touch_mask"][u] == 0)
    idn = _identity_rows(fcase) & vis
    if idn.any():
        plain = run_forward(fcase, None, mode, False, monkeypatch)["out"]["records"]
        assert got["records"][idn, 5].tobytes() == plain[idn, 5].tobytes(), f"{name} [{mode}]: coef != 1 on an identity row"
    if name.startswith("comp_edges/"):
        assert (u | idn).sum() >= (6 if name.endswith(("underflow", "identity")) else 0)
    if name.startswith("thin_discs/"):  # discs keep comp > 0: the antialiased mode's checks above can fail there too
        assert (u | idn).sum() == 20
        if mode == "antialiased":
            assert np.all(got["records"][u | idn, 11] > 0.5)
    print(f"[fwd filter3d] {name} [{mode}]: worst {worst:.3f} of the bar")


def check_backward(fcase, mode, flat, v, kind):
    aa_ = mode == "antialiased"
    r64, r32 = ref_backward(fcase, mode, kind, v, F64), ref_backward(fcase, mode, kind, v, F32)
    vis = ref_forward(fcase, mode, F64)["vis"]
    use_kappa = aa_ and kind in ("opacity", "all")
    kappa = ac.comp_condition(ref_forward(fcase, mode, F64)["records"]) if use_kappa else np.zeros(len(vis))
    vc = np.abs(v[:, 5] * ref_forward(fcase, mode, F64)["records"][:, 5])
    Kuse = (fcase.st.deg_use + 1) ** 2
    R = BWD_R_CONIC if kind in ("conic", "all") else BWD_R
    tag = f"{fcase.name} [{mode}] [{kind}]"
    worst, k, row0 = 0.0, 0, 0
    for i, seg in enumerate(fcase.frame.segments):
        n = seg.params.num_points
        geo = np.max([np.abs(r64[i][p].reshape(n, -1)).max(1) for p in PARAMS[:3]], 0) if n else None
        for name in PARAMS:
            k += 1
            if n == 0:
                continue
            got = flat[k - 1].detach().cpu().numpy().astype(np.float64).reshape(n, -1)
            assert np.all(np.isfinite(got)), f"{tag}: {name} is not finite"
            assert np.all(got[~vis[row0:row0 + n]] == 0), f"{tag}: {name} of an invisible row is not zero"
            a64, a32 = r64[i][name].reshape(n, -1), r32[i][name].reshape(n, -1)
            if got.shape[1] == 0:
                continue
            err = np.abs(got - a64).max(1)
            scale = np.maximum(np.abs(a64).max(1), geo) if name in PARAMS[:3] else np.abs(a64).max(1)
            bar = np.maximum(BWD_K * np.abs(a32 - a64).max(1), R * scale)
            if name in PARAMS[:3]:
                bar = np.maximum(bar, ac.COND_K * ac.EPS32 * kappa[row0:row0 + n] * scale)
            if name == "scales":  # the coef term v_c (1 - r): see FILT_K
                bar = np.maximum(bar, FILT_K * ac.EPS32 * vc[row0:row0 + n])
            if name == "opacities" and use_kappa:  # proportional to comp, which carries about eps32 kappa of relative error
                bar = np.maximum(bar, BWD_K * ac.EPS32 * kappa[row0:row0 + n] * np.abs(a64).max(1))
            ratio = np.where(err == 0, 0.0, err / np.where(bar > 0, bar, 1e-300))
            worst = max(worst, ratio.max())
            r = int(np.argmax(ratio))
            assert ratio.max() <= 1.0, (f"{tag}: {name} of row {r} of segment {i}: {got[r].tolist()} vs {a64[r].tolist()} "
                                        f"(fp32 noise {np.abs(a32 - a64)[r].max():.3e})")
            if name == "features_rest":
                assert np.all(got[:, 3 * (Kuse - 1):] == 0)
        row0 += n
    return worst


def _rows(flat, fcase, j, width):
    return np.concatenate([flat[6 * i + j].detach().cpu().numpy().reshape(s.params.num_points, width)
                           for i, s in enumerate(fcase.frame.segments)], 0)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", fc.CONFIGS)
def test_backward_each_cotangent(name, mode, monkeypatch):
    fcase = fc.get(name)
    run = run_forward(fcase, fcase.sigmas, mode, False, monkeypatch)
    u = _underflow_rows(fcase) & ref_forward(fcase, mode, F64)["vis"]
    worst = {}
    for kind in KINDS:
        v = pc.v_records(fcase.base, kind)
        flat, _ = raster.project_bwd(run["table"], run["params"], run["cs"], run["pr"].records, run["pr"].radii,
                                     torch.from_numpy(v).to(DEV))
        torch.cuda.synchronize()
        worst[kind] = check_backward(fcase, mode, flat, v, kind)
        if u.any():
            assert np.all(_rows(flat, fcase, 5, 1)[u] == 0), f"{name} [{mode}] [{kind}]: opacity gradient of an underflow row"
            gs = _rows(flat, fcase, 1, 3)
            assert np.all(gs[u][fcase.thin[u]] == 0), f"{name} [{mode}] [{kind}]: scale gradient of an underflowed axis"
            if kind in ("conic", "all"):  # a needle's long axis, a disc's two wide axes
                assert np.all(np.abs(gs[u][~fcase.thin[u]]) > 0), \
                    f"{name} [{mode}] [{kind}]: an axis that did not underflow lost its geometry gradient"
    print(f"[bwd filter3d] {name} [{mode}]: " + " ".join(f"{k} {w:.3f}" for k, w in worst.items()))


# ------------------------------------------------------------------------------------------------------------------
# an all-zero filter is no filter
# ------------------------------------------------------------------------------------------------------------------
def _scale_slots(table):
    """Arena floats that hold log-scale gradients."""
    sizes, shapes, _ = raster.arena_layout(table.static)
    off = np.concatenate([[0], np.cumsum(sizes)])
    mask = np.zeros(int(off[-1]), bool)
    for si in range(len(sizes) // 6):
        n = int(np.prod(shapes[6 * si + 1]))
        mask[off[6 * si + 1]: off[6 * si + 1] + n] = True
    return mask


def _same_up_to_zero_sign_of_scales(a, b, scales, what):
    """a and b bit for bit, except that a log-scale gradient (``scales``) may be +0 in one and -0 in the other."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    same = (a.view(np.uint32) == b.view(np.uint32)) | (scales & (a == 0) & (b == 0))
    assert same.all(), f"{what}: {int((~same).sum())} values differ"
    return int(((a.view(np.uint32) != b.view(np.uint32))).sum())


def _grads(run, v, pose=False, view=None):
    size = sum(raster.arena_layout(run["table"].static)[0])
    kw = {}
    if pose:
        kw["v_pose"] = torch.zeros(run["table"].nseg, _lib.POSE_FLOATS, device=DEV)
    if view is not None:
        kw["view"], kw["v_view"] = view, torch.zeros(_lib.VIEW_FLOATS, device=DEV)
    _, arena = raster.project_bwd(run["table"], run["params"], run["cs"], run["pr"].records, run["pr"].radii, v,
                                  make_views=False, out=torch.zeros(size, device=DEV), **kw)
    torch.cuda.synchronize()
    return arena.cpu().numpy(), {k: t.cpu().numpy() for k, t in kw.items() if k in ("v_pose", "v_view")}


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", list(pc.CASES))
def test_zero_filter_is_no_filter(name, mode, monkeypatch):
    case = pc.get(name)
    zeros = fc.zero_filter(case)
    for staged in (False, True):
        a = run_forward(case, zeros, mode, staged, monkeypatch)["out"]
        b = run_forward(case, None, mode, staged, monkeypatch)["out"]
        _outs_equal(a, b, f"{name} [{mode}] staged={staged}: zero filter vs no filter")
    fz, fn = run_forward(case, zeros, mode, False, monkeypatch), run_forward(case, None, mode, False, monkeypatch)
    assert fz["table"].filter_dev is not None and fn["table"].filter_dev is None
    vm = torch.from_numpy(np.concatenate([case.frame.camera.viewmat().reshape(-1), case.frame.camera.cam_pos()])).to(DEV)
    scales = _scale_slots(fz["table"])
    flips = 0
    for kind in KINDS:
        v = torch.from_numpy(pc.v_records(case, kind)).to(DEV)
        az, pz_ = _grads(fz, v, pose=True, view=vm)
        an, pn = _grads(fn, v, pose=True, view=vm)
        flips += _same_up_to_zero_sign_of_scales(az, an, scales, f"{name} [{mode}] [{kind}]: backward arena")
        for k in pz_:
            assert pz_[k].tobytes() == pn[k].tobytes(), f"{name} [{mode}] [{kind}]: {k}"
    print(f"[zero filter] {name} [{mode}]: {flips} log-scale gradients differ only in the sign of a zero")


# ------------------------------------------------------------------------------------------------------------------
# range backward, pose and view forms
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", ["layout/mixed", "staged_mix/mixed", "posed40/mixed", "nseg1024/mixed"])
def test_range_backward(name, mode, monkeypatch):
    fcase = fc.get(name)
    run = run_forward(fcase, fcase.sigmas, mode, False, monkeypatch)
    table, params, cs, pr = run["table"], run["params"], run["cs"], run["pr"]
    v = torch.from_numpy(pc.v_records(fcase.base, "all")).to(DEV)
    size = sum(raster.arena_layout(table.static)[0])
    _, full = raster.project_bwd(table, params, cs, pr.records, pr.radii, v, out=torch.zeros(size, device=DEV))
    full = full.cpu().numpy()
    for ranges in _partitions(table):
        _, arena = raster.project_bwd(table, params, cs, pr.records, pr.radii, v, make_views=False, chunk_ranges=ranges,
                                      out=torch.zeros(size, device=DEV))
        assert arena.cpu().numpy().tobytes() == full.tobytes(), f"{name} [{mode}]: partition {ranges} differs from the single call"
    nc = table.num_chunks
    for issued in ([(0, 0)], [(1, min(3, nc))], [(0, 1), (nc - 1, nc)]):
        arena = torch.full_like(torch.from_numpy(full), float("nan")).to(DEV)
        raster.project_bwd(table, params, cs, pr.records, pr.radii, v, make_views=False, out=arena, chunk_ranges=issued)
        got = arena.cpu().numpy()
        mask = _written_mask(table, issued)
        assert np.all(np.isnan(got[~mask])), f"{name} [{mode}]: ranges {issued} wrote outside their chunks"
        assert got[mask].tobytes() == full[mask].tobytes(), f"{name} [{mode}]: ranges {issued}"


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", ["posed40/mixed", "posed40/even", "layout/mixed", "fov_clamp/mixed", "comp_edges/underflow"])
def test_pose_and_view_forms(name, mode, monkeypatch):
    fcase = fc.get(name)
    aa_ = mode == "antialiased"
    run = run_forward(fcase, fcase.sigmas, mode, False, monkeypatch)
    v_np = pc.v_records(fcase.base, "all")
    v = torch.from_numpy(v_np).to(DEV)
    plain, _ = _grads(run, v)
    cam = fcase.frame.camera
    vm = torch.from_numpy(np.concatenate([cam.viewmat().reshape(-1), cam.cam_pos()])).to(DEV)
    arena_v, outs = _grads(run, v, view=vm)
    assert arena_v.tobytes() == plain.tobytes(), f"{name} [{mode}]: the view form's parameter gradients differ"
    want = fc.v_view_ref(fcase.frame, fcase.st, fcase.sigmas, v_np, aa_)
    e = pz.rel_l2(outs["v_view"], want)
    assert e <= TOL, f"{name} [{mode}]: v_view relative L2 {e:.2e}"
    worst = e
    posed = [i for i, s in enumerate(fcase.frame.segments) if s.has_pose]
    if posed:
        arena_p, outs = _grads(run, v, pose=True)
        assert arena_p.tobytes() == plain.tobytes(), f"{name} [{mode}]: the pose form's parameter gradients differ"
        got = outs["v_pose"][posed].astype(np.float64)
        want_p = fc.v_pose_ref(fcase.frame, fcase.st, fcase.sigmas, v_np, aa_)
        for a in range(want_p.shape[0]):
            for label, g, r in zip(("v_R", "v_t", "v_q"), pz.groups(got[a:a + 1]), pz.groups(want_p[a:a + 1])):
                if not np.any(r):
                    assert not np.any(g), f"{name} [{mode}]: {label} of posed segment {a} must be exactly zero"
                    continue
                e = pz.rel_l2(g, r)
                worst = max(worst, e)
                assert e <= TOL, f"{name} [{mode}]: {label} of posed segment {a}: relative L2 {e:.2e}"
    print(f"[pose/view filter3d] {name} [{mode}]: worst relative L2 {worst:.2e}")
