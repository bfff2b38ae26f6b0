"""The projection kernels on hand-built Gaussians (tests/project_cases.py) against the float64 reference
(oracle/project_ref64.py) and the C oracle.

Forward, every case through the direct and the staged kernel (SGN_PROJECT_STAGED):
  * the two forms agree bit for bit on every output array;
  * the exact section (xy, conic, depth, radii, num_tiles_hit, tile AABB of visible rows) is bit-equal to the C oracle;
  * the integer outputs and aux bits equal the reference's (every decision is >= 1e-4 from its threshold), and every
    float record field of a visible row is within FWD_K x (the row's fp32 noise: the reference run in float32) +
    FWD_R x max|ref| of its field group;
  * invisible rows carry zero xy, opacity, colour and depth, and only the class bit;
  * touch mask: every AABB tile whose float64 min sigma (from the kernel's own record) is <= tau is kept, every kept tile has
    min sigma <= tau + 2e-3 + 1e-5 |terms|; AABBs over 32 tiles are checked through tiles_touched between the two counts.
Backward, each cotangent alone (xy, conic, opacity, rgb, depth) and all of them: per Gaussian and per parameter row,
max|got - ref64| <= max(BWD_K max|ref32 - ref64|, R max|ref64|) over the row (for means / scales / quats, max|ref64| over
the Gaussian's three geometry rows), R = BWD_R, or BWD_R_CONIC when a conic cotangent takes part; invisible rows and the
features_rest columns beyond sh_degree_to_use are exactly zero.  The range backward over several partitions of the chunks is bit-identical
to the single call and leaves every arena slot outside the issued ranges untouched.  Level-1: project_gaussians forward and
backward (glob_scale 1 and 0.37, each cotangent NULL in turn, compensation, cov3d) and spherical_harmonics (K x degree).

Observed on an H100 80GB HBM3 (400 W power limit), 79 tests in 22 s: the forward's float fields at most 0.75 of their bar
(posed40), the backward at most 0.26 of its bar (opacity cotangent; conic 0.08, all five 0.13).  With only the row's fp32
noise and 2e-6 of its max as the bar, the conic gradients of needles (scale ratio 1e4) missed it by up to 2.6x: the
kernel's hand-derived VJP rounds differently from autograd there, hence BWD_R_CONIC.  Ten one-token changes to project.cu /
sgn_touch.cuh (FOV-clamp sign and axis in the VJP, quaternion normalisation, posed quaternion product, Fourier weight in the
DC gradient, glob_scale in the Level-1 scale gradient, the staged gather row, the range backward's chunk offset, the touch
margin's sign, the touch rectangle's image clip) each fail 3 to 33 of these tests.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from street_gaussians_ns_b200 import _lib, raster
from street_gaussians_ns_b200.scene import Frame, Segment
from oracle import oracle_c
from oracle import project_ref64 as ref
from tests import project_cases as pc

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
FWD_K, FWD_R = 8.0, 2e-6
BWD_K, BWD_R = 8.0, 8e-6
BWD_R_CONIC = 5e-4  # with a conic cotangent: the inverse of cov2d amplifies fp32 rounding by its condition number
TOUCH_A, TOUCH_R = 2e-3, 1e-5
KINDS = ["xy", "conic", "opacity", "rgb", "depth", "all"]
PARAMS = ("means", "scales", "quats", "features_dc", "features_rest", "opacities")


def _settings(case):
    st = case.st
    return raster.RenderSettings(sh_degree=st.sh_degree, sh_degree_to_use=st.deg_use, block_width=st.block_width,
                                 clip_thresh=st.clip_thresh)


def _cuda_frame(case):
    return Frame(case.frame.camera, [Segment(s.params.to("cuda"), s.cls, s.rot, s.center, s.idft) for s in case.frame.segments])


def run_forward(case, staged, monkeypatch):
    monkeypatch.setenv("SGN_PROJECT_STAGED", "1" if staged else "0")
    frc = _cuda_frame(case)
    params = [s.params.tensors() for s in frc.segments]
    table = raster.SegmentTable(frc, params, DEV)
    cs = raster.camera_struct(frc.camera, _settings(case))
    pr = raster.project_fwd(table, cs, DEV)
    torch.cuda.synchronize()
    out = dict(records=pr.records.cpu().numpy(), radii=pr.radii.cpu().numpy(), tiles_hit=pr.tiles_hit.cpu().numpy(),
               bbox=pr.bbox.cpu().numpy().view(np.uint16).astype(np.int64), tiles_touched=pr.tiles_touched.cpu().numpy(),
               touch_mask=pr.touch_mask.cpu().numpy().view(np.uint32))
    return table, params, cs, pr, out


_REF32 = {}


def ref32_forward(case):
    if case.name not in _REF32:
        _REF32[case.name] = ref.forward(case.frame, case.st, torch.float32)
    return _REF32[case.name]


def check_forward(case, got):
    fw, vis = case.fwd, case.fwd["vis"]
    rec = got["records"]
    orc = oracle_c.Oracle(case.frame, case.st.sh_degree, case.st.deg_use, case.st.block_width, case.st.clip_thresh).project()
    np.testing.assert_array_equal(rec[:, 0:2], orc["xys"])
    np.testing.assert_array_equal(rec[:, 2:5], orc["conics"])
    np.testing.assert_array_equal(rec[:, 9], orc["depths"])
    np.testing.assert_array_equal(got["radii"], orc["radii"])
    np.testing.assert_array_equal(got["tiles_hit"], orc["num_tiles_hit"])
    np.testing.assert_array_equal(got["bbox"][vis], orc["tile_bbox"][vis])
    # decisions against the float64 reference
    np.testing.assert_array_equal(got["radii"], fw["radii"])
    np.testing.assert_array_equal(got["tiles_hit"], fw["num_tiles_hit"])
    np.testing.assert_array_equal(got["bbox"][vis], np.concatenate([fw["tmin"], fw["tmax"]], 1)[vis])
    np.testing.assert_array_equal(rec[:, 10].view(np.int32), fw["aux"])
    assert np.all(rec[:, 11] == 0)
    # float fields of visible rows
    f32 = ref32_forward(case)["records"]
    r64 = fw["records"]
    worst = 0.0
    for cols in ([0, 1], [2, 3, 4], [5], [6, 7, 8], [9]):
        noise = np.abs(f32[:, cols] - r64[:, cols]).max(1, keepdims=True)
        bar = FWD_K * noise + FWD_R * np.maximum(np.abs(r64[:, cols]).max(1, keepdims=True), 1e-3)
        err = np.abs(rec[:, cols].astype(np.float64) - r64[:, cols])
        ratio = np.where(vis[:, None], err / bar, 0.0)
        worst = max(worst, ratio.max(initial=0.0))
        g = np.unravel_index(np.argmax(ratio), ratio.shape) if ratio.size else (0, 0)
        assert ratio.max(initial=0.0) <= 1.0, f"{case.name}: record column {cols[g[1]]} of row {g[0]}: {rec[g[0], cols[g[1]]]!r} vs {r64[g[0], cols[g[1]]]!r}"
    # invisible rows: nothing but the class bit
    inv = ~vis
    assert np.all(rec[inv][:, [0, 1, 5, 6, 7, 8, 9]] == 0)
    np.testing.assert_array_equal(rec[inv, 10].view(np.int32), np.where(fw["cls"][inv] == 1, ref.AUX_OBJECT, 0))
    assert np.all(got["tiles_touched"][inv] == 0) and np.all(got["touch_mask"][inv] == 0)
    return worst


def check_touch(case, got):
    cam, bw = case.frame.camera, case.st.block_width
    rec = got["records"]
    for g in np.nonzero(case.fwd["vis"])[0]:
        x0, y0, x1, y1 = got["bbox"][g]
        tx, ty, d, mag = ref.touch_min_sigma(rec[g, 0:2].astype(np.float64), rec[g, 2:5].astype(np.float64),
                                             float(rec[g, 5]), (x0, y0), (x1, y1), cam.width, cam.height, bw)
        need = d <= 0
        allow = d <= TOUCH_A + TOUCH_R * mag
        area = len(d)
        if area <= 32:
            bits = (int(got["touch_mask"][g]) >> np.arange(area)) & 1
            assert np.all(bits[need] == 1), f"{case.name}: row {g} drops a tile some pixel centre reaches"
            assert np.all(allow[bits == 1]), f"{case.name}: row {g} keeps a tile no pixel centre reaches"
            assert got["tiles_touched"][g] == bits.sum()
        else:
            assert need.sum() <= got["tiles_touched"][g] <= allow.sum(), f"{case.name}: row {g}"


@pytest.mark.parametrize("name", list(pc.CASES))
def test_forward_direct_and_staged(name, monkeypatch):
    case = pc.get(name)
    outs = [run_forward(case, staged, monkeypatch)[-1] for staged in (False, True)]
    for k in outs[0]:
        assert outs[0][k].tobytes() == outs[1][k].tobytes(), f"{name}: {k} differs between the direct and the staged kernel"
    worst = check_forward(case, outs[0])
    check_touch(case, outs[0])
    print(f"[fwd] {name}: worst {worst:.3f} of the bar")


def check_backward(case, flat, v, tag=""):
    r64 = ref.backward(case.frame, case.st, v)
    r32 = ref.backward(case.frame, case.st, v, torch.float32)
    vis = case.fwd["vis"]
    Kuse = (case.st.deg_use + 1) ** 2
    R = BWD_R_CONIC if ("conic" in tag or "all" in tag) else BWD_R
    worst, k, row0 = 0.0, 0, 0
    for i, seg in enumerate(case.frame.segments):
        n = seg.params.num_points
        # geometry rows share one scale: the gradient of an isotropic Gaussian's quaternion is 0 up to rounding of terms
        # the size of its scale gradient
        geo = np.max([np.abs(r64[i][p].reshape(n, -1)).max(1) for p in PARAMS[:3]], 0) if n else None
        for name in PARAMS:
            k += 1
            if n == 0:
                continue
            assert np.all(flat[k - 1].detach().cpu().numpy().reshape(n, -1)[~vis[row0:row0 + n]] == 0), \
                f"{case.name}{tag}: {name} of an invisible row is not zero"
            got = flat[k - 1].detach().cpu().numpy().astype(np.float64).reshape(n, -1)
            a64, a32 = r64[i][name].reshape(n, -1), r32[i][name].reshape(n, -1)
            if got.shape[1] == 0:
                continue
            err = np.abs(got - a64).max(1)
            scale = np.maximum(np.abs(a64).max(1), geo) if name in PARAMS[:3] else np.abs(a64).max(1)
            bar = np.maximum(BWD_K * np.abs(a32 - a64).max(1), R * scale)
            ratio = np.where(err == 0, 0.0, err / np.where(bar > 0, bar, 1e-300))
            worst = max(worst, ratio.max())
            r = int(np.argmax(ratio))
            assert ratio.max() <= 1.0, (f"{case.name}{tag}: {name} of row {r} of segment {i}: {got[r].tolist()} vs "
                                        f"{a64[r].tolist()} (fp32 noise {np.abs(a32 - a64)[r].max():.3e})")
            if name == "features_rest":
                assert np.all(got[:, 3 * (Kuse - 1):] == 0)
        row0 += n
    return worst


@pytest.mark.parametrize("name", list(pc.CASES))
def test_backward_each_cotangent(name, monkeypatch):
    case = pc.get(name)
    table, params, cs, pr, _ = run_forward(case, False, monkeypatch)
    worst = {}
    for kind in KINDS:
        v = pc.v_records(case, kind)
        flat, _ = raster.project_bwd(table, params, cs, pr.records, pr.radii, torch.from_numpy(v).to(DEV))
        torch.cuda.synchronize()
        worst[kind] = check_backward(case, flat, v, f" [{kind}]")
    print(f"[bwd] {name}: " + " ".join(f"{k} {w:.3f}" for k, w in worst.items()))


def _partitions(table):
    nc = table.num_chunks
    edges = sorted(set(int(c) for c in table.host["chunk0"]) | {nc})
    inside = sorted({1, nc // 2, nc - 1} - set(edges))
    cuts = [
        [(0, 0), (0, nc), (nc, nc)],
        [(0, 1), (1, 1), (1, nc)] if nc > 1 else [(0, nc)],
        [(a, b) for a, b in zip([0] + edges, edges + [nc]) if a <= b],
        [(a, b) for a, b in zip([0] + inside, inside + [nc])],
        [(c, c + 1) for c in reversed(range(nc))],
    ]
    return cuts


def _written_mask(table, ranges):
    """Arena floats that the chunk ranges write (dense gradient rows of their chunks)."""
    sizes, shapes, _ = raster.arena_layout(table.static)
    mask = np.zeros(sum(sizes), bool)
    host = table.host
    off = np.concatenate([[0], np.cumsum(sizes)])
    for c0, c1 in ranges:
        for c in range(c0, c1):
            si = int(np.nonzero(host["chunk0"] <= c)[0][-1])
            while host["count"][si] == 0 or c >= host["chunk0"][si] + (host["count"][si] + 127) // 128:
                si -= 1
            r0 = (c - int(host["chunk0"][si])) * 128
            rows = min(128, int(host["count"][si]) - r0)
            for j in range(6):
                w = int(np.prod(shapes[6 * si + j][1:]))
                base = off[6 * si + j]
                mask[base + r0 * w: base + (r0 + rows) * w] = True
    return mask


@pytest.mark.parametrize("name", ["layout", "staged_mix", "posed40"])
def test_range_backward(name, monkeypatch):
    case = pc.get(name)
    table, params, cs, pr, _ = run_forward(case, False, monkeypatch)
    v = torch.from_numpy(pc.v_records(case, "all")).to(DEV)
    size = sum(raster.arena_layout(table.static)[0])
    _, full = raster.project_bwd(table, params, cs, pr.records, pr.radii, v, out=torch.zeros(size, device=DEV))
    full = full.cpu().numpy()
    for ranges in _partitions(table):
        _, arena = raster.project_bwd(table, params, cs, pr.records, pr.radii, v, make_views=False, chunk_ranges=ranges,
                                      out=torch.zeros(size, device=DEV))
        assert arena.cpu().numpy().tobytes() == full.tobytes(), f"{name}: partition {ranges} differs from the single call"
    nc = table.num_chunks
    for issued in ([(0, 0)], [(1, min(3, nc))], [(0, 1), (nc - 1, nc)]):
        arena = torch.full_like(torch.from_numpy(full), float("nan")).to(DEV)
        raster.project_bwd(table, params, cs, pr.records, pr.radii, v, make_views=False, out=arena, chunk_ranges=issued)
        got = arena.cpu().numpy()
        mask = _written_mask(table, issued)
        assert np.all(np.isnan(got[~mask])), f"{name}: ranges {issued} wrote outside their chunks"
        assert got[mask].tobytes() == full[mask].tobytes(), f"{name}: ranges {issued}"


# ------------------------------------------------------------------------------------------------------------------
# Level-1 entry points
# ------------------------------------------------------------------------------------------------------------------
def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _l1_inputs(name):
    case = pc.get(name)
    seg = case.frame.segments[0]
    m = seg.params.means.numpy().astype(np.float32)
    s = np.exp(seg.params.scales.numpy().astype(np.float64)).astype(np.float32)
    q = seg.params.quats.numpy().astype(np.float32)
    return case, m, s, q


@pytest.mark.parametrize("glob_scale", [1.0, 0.37])
@pytest.mark.parametrize("name", ["fov_clamp", "near_plane", "shapes"])
def test_l1_project(name, glob_scale):
    L = _lib.load()
    case, m, s, q = _l1_inputs(name)
    N = m.shape[0]
    cs = raster.camera_struct(case.frame.camera, _settings(case))
    d = {k: torch.from_numpy(a).to(DEV) for k, a in (("m", m), ("s", s), ("q", q))}
    o = dict(xys=torch.zeros(N, 2), depths=torch.zeros(N), radii=torch.zeros(N, dtype=torch.int32), conics=torch.zeros(N, 3),
             comp=torch.zeros(N), tiles=torch.zeros(N, dtype=torch.int32), cov3d=torch.zeros(N, 6))
    o = {k: t.to(DEV) for k, t in o.items()}
    _lib.check(L.sgn_l1_project_fwd(N, _ptr(d["m"]), _ptr(d["s"]), C.c_float(glob_scale), _ptr(d["q"]), C.byref(cs), _ptr(o["xys"]),
                                    _ptr(o["depths"]), _ptr(o["radii"]), _ptr(o["conics"]), _ptr(o["comp"]), _ptr(o["tiles"]),
                                    _ptr(o["cov3d"]), None), "sgn_l1_project_fwd")
    torch.cuda.synchronize()
    g = {k: t.cpu().numpy() for k, t in o.items()}
    fw = ref.l1_project(m, s, np.float32(glob_scale), q, case.frame.camera, case.st.block_width, case.st.clip_thresh)
    ok = fw["margin"] >= pc.MARGIN
    assert ok.mean() > 0.8
    np.testing.assert_array_equal(g["radii"][ok], fw["radii"][ok])
    np.testing.assert_array_equal(g["tiles"][ok], fw["num_tiles_hit"][ok])
    vis = ok & fw["vis"]
    f32 = ref.l1_project(m, s, np.float32(glob_scale), q, case.frame.camera, case.st.block_width, case.st.clip_thresh,
                         dtype=torch.float32)
    for k, rk in (("xys", "xys"), ("depths", "depths"), ("conics", "conics"), ("comp", "compensation"), ("cov3d", "cov3d")):
        r, r32 = (np.asarray(x[rk].detach().double() if torch.is_tensor(x[rk]) else x[rk], np.float64).reshape(N, -1)
                  for x in (fw, f32))
        sel = ok if k == "cov3d" else vis
        gv, rv, nv = g[k].reshape(N, -1)[sel].astype(np.float64), r[sel], np.abs(r32 - r)[sel]
        tol = FWD_K * nv.max(1, keepdims=True) + FWD_R * np.maximum(np.abs(rv).max(1, keepdims=True), 1e-6)
        assert np.all(np.abs(gv - rv) <= tol), f"{name}: {k} worst {np.max(np.abs(gv - rv) / tol):.2f} of the bar"
    assert np.all(g["cov3d"][~fw["unclipped"] & ok] == 0)
    assert np.all(g["comp"][~fw["vis"] & ok] == 0) and np.all(g["depths"][~fw["vis"] & ok] == 0)
    # backward: all cotangents, then each pointer NULL in turn
    rng = np.random.default_rng(5)
    vs = dict(xys=rng.uniform(-1, 1, (N, 2)).astype(np.float32), depths=rng.uniform(-1, 1, N).astype(np.float32),
              conics=rng.uniform(-1, 1, (N, 3)).astype(np.float32))
    for drop in (None, "xys", "depths", "conics"):
        v = {k: (None if k == drop else a) for k, a in vs.items()}
        vd = {k: (None if a is None else torch.from_numpy(a).to(DEV)) for k, a in v.items()}
        outs = [torch.full((N, w), float("nan"), device=DEV) for w in (3, 3, 4)]
        _lib.check(L.sgn_l1_project_bwd(N, _ptr(d["m"]), _ptr(d["s"]), C.c_float(glob_scale), _ptr(d["q"]), C.byref(cs),
                                        _ptr(o["radii"]), _ptr(vd["xys"]), _ptr(vd["depths"]), _ptr(vd["conics"]),
                                        *[_ptr(t) for t in outs], None), "sgn_l1_project_bwd")
        torch.cuda.synchronize()
        r = ref.l1_project_bwd(m, s, np.float32(glob_scale), q, case.frame.camera, v["xys"], v["depths"], v["conics"],
                               case.st.block_width, case.st.clip_thresh)
        r32 = _l1_bwd32(m, s, glob_scale, q, case, v)
        for t, a64, a32, nm in zip(outs, r, r32, ("means", "scales", "quats")):
            got = t.cpu().numpy().astype(np.float64)
            assert np.all(got[~fw["vis"] & ok] == 0), f"{name}: v_{nm} of an invisible row"
            err = np.abs(got - a64).max(1)[vis]
            geo = np.max([np.abs(x).max(1) for x in r], 0)
            R = BWD_R_CONIC if v["conics"] is not None else BWD_R
            bar = np.maximum(BWD_K * np.abs(a32 - a64).max(1), R * geo)[vis]
            assert np.all(err <= bar), f"{name} (drop {drop}): v_{nm} worst {np.max(err / np.maximum(bar, 1e-300)):.2f} of the bar"


def _l1_bwd32(m, s, glob_scale, q, case, v):
    fw = ref.l1_project(m, s, np.float32(glob_scale), q, case.frame.camera, case.st.block_width, case.st.clip_thresh,
                        dtype=torch.float32, grad=True)
    loss = 0.0
    for out, k in ((fw["xys"], "xys"), (fw["depths"], "depths"), (fw["conics"], "conics")):
        if v[k] is not None:
            loss = loss + (out * torch.from_numpy(v[k]).reshape(out.shape)).sum()
    gs = torch.autograd.grad(loss, fw["leaves"], allow_unused=True)
    return [np.zeros(np.shape(x)) if g is None else g.double().numpy() for g, x in zip(gs, (m, s, q))]


@pytest.mark.parametrize("K", [1, 4, 9, 16])
@pytest.mark.parametrize("degree", [0, 1, 2, 3])
def test_l1_sh(degree, K):
    L = _lib.load()
    rng = np.random.default_rng(100 * degree + K)
    N = 300
    dirs = rng.normal(size=(N, 3))
    dirs = (dirs / np.linalg.norm(dirs, axis=1, keepdims=True)).astype(np.float32)
    coeffs = rng.normal(size=(N, K, 3)).astype(np.float32)
    vcol = rng.uniform(-1, 1, (N, 3)).astype(np.float32)
    rc, rv = ref.l1_sh(degree, dirs, coeffs, vcol)
    dd, cd, vd = (torch.from_numpy(a).to(DEV) for a in (dirs, coeffs, vcol))
    colors = torch.full((N, 3), float("nan"), device=DEV)
    _lib.check(L.sgn_l1_sh(N, K, degree, _ptr(dd), _ptr(cd), None, _ptr(colors), None, None), "sgn_l1_sh forward")
    v_coeffs = torch.full((N, K, 3), float("nan"), device=DEV)
    _lib.check(L.sgn_l1_sh(N, K, degree, _ptr(dd), None, _ptr(vd), None, _ptr(v_coeffs), None), "sgn_l1_sh backward")
    torch.cuda.synchronize()
    Kuse = min((degree + 1) ** 2, K)
    Y = ref.sh_basis(degree, torch.from_numpy(dirs.astype(np.float64))).numpy()[:, :Kuse]
    scale = (np.abs(Y)[:, :, None] * np.abs(coeffs[:, :Kuse].astype(np.float64))).sum(1)
    assert np.all(np.abs(colors.cpu().numpy() - rc) <= 1e-6 * scale + 1e-7)
    got = v_coeffs.cpu().numpy()
    assert np.all(got[:, Kuse:] == 0)
    assert np.all(np.abs(got - rv) <= 1e-6 * np.abs(rv) + 1e-7)
