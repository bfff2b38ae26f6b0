"""The extra-channel blend (sgn_blend_extra_fwd / _bwd / _bwd_det, render_frame(extra=...)) and the Level-1
gsplat_compat.rasterize_gaussians on hand-built inputs, against the channel form of the float64 blend reference
(oracle/blend_ref64.py forward_channels / backward_channels).

Extra channels run on the tiles of tests/blend_cases.py, under every execution variant of the main forward (the extra
pass reads its final_T / final_idx), for C in {1, 3, 8, 9, 17} (partial last groups, one to three groups of 8):
  * the forward writes every pixel (the output is prefilled with NaN), each within IMG_TOL max(1, S), S the pixel's sum of
    absolute terms (values up to 1e3 in magnitude, of both signs);
  * with extra = records[:, 6:10] the output is the main pass's raw sums bit for bit (a zero of either sign equals a
    zero: the paired body keeps negated sums).  The extra pass repeats the main pass's sigma, ex2 and T fma in the same
    order; the paired and row-skip bodies differ from it only by exact negations and exact zero addends.  Two exceptions,
    both within fp32 rounding and excluded from the bit comparison (they are still compared with the reference):
      - a tile the main forward splits into strips: the strip's first row is folded into the pixel centre (dy =
        y - (row0 + 0.5) - 2s rounds differently from the extra pass's y - (tile row + 0.5) - 2(s + row offset));
      - a pixel that blends a clamped alpha under the paired body (SGN_TUNE_FWD_PACKED): its clamp is
        in_register(-clamp_fwd) = -(1 - (1 + 0.999f)), which rounds to -0.99900007 (1 - x is exact only for x in
        [0.5, 2]), where the scalar bodies and the extra pass clamp at 0.999f;
  * the backward ADDS to prefilled v_extra / v_records: pattern plus gradient within GRAD_R |ref| + GRAD_A (S + |pattern|)
    per element, columns 6..11 untouched, no NaN from the degenerate entries;
  * the deterministic form gives the same bits twice and the reference's values within the same bars plus its grid's
    rounding.

Level-1 rasterize_gaussians: hand-built gsplat inputs (xys, conics, opacity, depths, radii), lists from
oracle/bin_ref64.py (gsplat's AABB lists in depth order; entries the touch test drops are valid for no pixel), C from 1
to 12 (the fourth channel of each group of 4 rides in the depth slot), with and without a background, cotangents on the
image, the alpha and both; uint8 colours, the empty scene and the block-width check.

Observed on an H100 80GB HBM3: see DESIGN.md section 4, "Directed extra-channel tests".
"""
import ctypes as C

import numpy as np
import pytest
import torch

import street_gaussians_ns_b200.synthetic as syn
from street_gaussians_ns_b200 import _lib, gsplat_compat, raster
from oracle import bin_ref64
from oracle import blend_ref64 as ref
from tests import blend_cases as bc
from tests.test_gpu_blend_directed import GRAD_A, GRAD_R, IMG_TOL, TUNINGS, fixed_shift, run_forward

pytestmark = pytest.mark.gpu

CHANNELS = [1, 3, 8, 9, 17]
EXTRA_CG = 8  # channels per traversal (csrc/blend.cu)
_p = raster._ptr


def L():
    return _lib.load()


def extra_values(case, Cn, seed=0):
    """Seeded values of both signs, magnitudes from 1e-2 to 1e3."""
    rng = np.random.default_rng(1000 * case.seed + 10 * Cn + seed)
    N = case.inp.records.shape[0]
    mag = 10.0 ** rng.uniform(-2.0, 3.0, (N, Cn))
    return (rng.choice([-1.0, 1.0], (N, Cn)) * mag).astype(np.float32)


def v_out_seed(case, Cn):
    rng = np.random.default_rng(case.seed)
    return rng.uniform(-1.0, 1.0, (case.inp.height, case.inp.width, Cn)).astype(np.float32)


_REF = {}


def reference(case, Cn):
    key = (case.name, Cn)
    if key not in _REF:
        vals = extra_values(case, Cn)
        fw = ref.forward_channels(case.inp, case.opts, vals)
        bw = ref.backward_channels(case.inp, case.opts, vals, v_out_seed(case, Cn))
        _REF[key] = (vals, fw, bw)
    return _REF[key]


def extra_fwd(cs, bo, d, out, ex):
    res = torch.full((cs.height, cs.width, ex.shape[1]), float("nan"), device="cuda")
    _lib.check(L().sgn_blend_extra_fwd(C.byref(cs), C.byref(bo), _p(d["records"]), _p(d["sorted_ids"]), _p(d["tile_bins"]),
                                       _p(out["final_T"]), _p(out["final_idx"]), _p(ex), ex.shape[1], _p(res), None),
               "sgn_blend_extra_fwd")
    torch.cuda.synchronize()
    return res.cpu().numpy()


def extra_bwd(cs, bo, d, out, ex, v_out, vrec0, vex0, det=False):
    """(v_records, v_extra) after the backward has added to the prefilled vrec0 / vex0."""
    v_rec = torch.from_numpy(vrec0).cuda()
    v_ex = torch.from_numpy(vex0).cuda()
    vo = torch.from_numpy(np.ascontiguousarray(v_out)).cuda()
    args = (C.byref(cs), C.byref(bo), _p(d["records"]), _p(d["sorted_ids"]), _p(d["tile_bins"]), _p(out["final_T"]),
            _p(out["final_idx"]), _p(ex), ex.shape[1])
    if det:
        N = ex.shape[0]
        fg = torch.zeros(N, 6, dtype=torch.int64, device="cuda")
        fe = torch.zeros(N, ex.shape[1], dtype=torch.int64, device="cuda")
        fs = torch.empty(2, device="cuda")
        rc = L().sgn_blend_extra_bwd_det(*args, N, _p(vo), _p(v_ex), _p(v_rec), _p(fg), _p(fe), _p(fs), None)
    else:
        rc = L().sgn_blend_extra_bwd(*args, _p(vo), _p(v_ex), _p(v_rec), None)
    _lib.check(rc, "sgn_blend_extra_bwd")
    torch.cuda.synchronize()
    return v_rec.cpu().numpy(), v_ex.cpu().numpy()


def excess(got, want, S):
    """|got - want| / (GRAD_R |want| + GRAD_A S) per element; <= 1 passes."""
    bound = GRAD_R * np.abs(want) + GRAD_A * S
    err = np.abs(got.astype(np.float64) - want)
    with np.errstate(all="ignore"):
        return np.where(err == 0, 0.0, err / np.where(bound > 0, bound, 1e-300))


def check_forward(case, Cn, got):
    _, fw, _ = reference(case, Cn)
    assert not np.isnan(got).any(), f"{case.name} C={Cn}: pixels left unwritten at {np.argwhere(np.isnan(got))[:3].tolist()}"
    err = np.abs(got.astype(np.float64) - fw["out"])
    tol = IMG_TOL * np.maximum(1.0, fw["abs"])
    assert (err <= tol).all(), f"{case.name} C={Cn}: out differs at {np.argwhere(err > tol)[:5].tolist()} ({(err / tol).max():.2f} of the bar)"
    return float((err / tol).max())


def quantization_floor_extra(case, vals, v_out):
    """The deterministic grids' rounding: half a unit per addend, one addend per tile that lists the Gaussian and channel
    group (geometry) or per tile (channels); units as csrc/blend.cu extra_fixed_scale_kernel sets them."""
    Cn = vals.shape[1]
    mv = float(np.abs(v_out).max())
    me = max(1.0, float(np.abs(vals).max()))
    eg, ev = np.ceil(np.log2(mv * me * Cn)), np.ceil(np.log2(mv))
    ids = np.asarray(case.inp.sorted_ids, np.int64) & 0x7FFFFFFF
    ntiles = np.bincount(ids, minlength=vals.shape[0]).astype(np.float64)
    groups = -(-Cn // EXTRA_CG)
    geom = 0.5 * ntiles[:, None] * groups * np.ldexp(1.0, fixed_shift(case.inp.records)[:, :6] - 32 + int(eg))
    chan = 0.5 * ntiles[:, None] * np.ldexp(1.0, -32 + int(ev)) * np.ones((1, Cn))
    return geom, chan


def check_backward(case, Cn, vrec0, vex0, got_rec, got_ex, det=False):
    vals, _, (vv, vr, vva, vra) = reference(case, Cn)
    assert np.isfinite(got_rec).all() and np.isfinite(got_ex).all(), f"{case.name} C={Cn}: non-finite gradient"
    assert np.array_equal(got_rec[:, 6:].view(np.int32), vrec0[:, 6:].view(np.int32)), f"{case.name}: columns 6..11 changed"
    Sg, Se = vra[:, :6] + np.abs(vrec0[:, :6]), vva + np.abs(vex0)
    if det:
        fg, fe = quantization_floor_extra(case, vals, v_out_seed(case, Cn))
        Sg, Se = Sg + fg / GRAD_A, Se + fe / GRAD_A
    worst = 0.0
    for what, got, want, S in (("v_extra", got_ex, vex0 + vv, Se), ("geometry", got_rec[:, :6], vrec0[:, :6] + vr[:, :6], Sg)):
        ex = excess(got, want, S)
        w = np.unravel_index(np.argmax(ex), ex.shape)
        assert ex.max() <= 1.0, f"{case.name} C={Cn} {what}: Gaussian {w[0]} component {w[1]}: {got[w]!r} vs {want[w]!r}"
        worst = max(worst, float(ex.max()))
    return worst


def bit_equality_exemptions(case, tuning):
    """[H,W] pixels of tiles the main forward splits into strips, and (paired body) pixels that blend a clamped alpha."""
    inp, opts = case.inp, case.opts
    H, W = inp.height, inp.width
    split = case.splits.get("SGN_SPLIT_FWD_MAIN") or 768
    lens = inp.tile_bins[:, 1] - inp.tile_bins[:, 0]
    ex = np.zeros(H * W, bool)
    if tuning & 4:  # SGN_TUNE_FWD_PACKED
        _, streams, _ = ref._run(inp, opts)
        for e in streams:
            m, pid, inside = e["main"], e["pid"], e["inside"]
            clamped = (m.blended & (m.raw >= opts.clamp_fwd)).any(2)
            ex[pid[inside & clamped]] = True
    ex = ex.reshape(H, W)
    for t in np.nonzero([ref.strips_for(int(n), split) > 1 for n in lens])[0]:
        tx, ty = t % inp.tiles_x, t // inp.tiles_x
        ex[16 * ty:16 * ty + 16, 16 * tx:16 * tx + 16] = True
    return ex


@pytest.mark.parametrize("tuning", TUNINGS)
@pytest.mark.parametrize("name", list(bc.CASES))
def test_extra_against_reference(name, tuning, monkeypatch):
    case = bc.get(name)
    cs, bo, d, out = run_forward(case, tuning, monkeypatch)
    torch.cuda.synchronize()
    # extra = the colour and depth columns: the main pass's raw sums, bit for bit (a zero of either sign equals a zero)
    ex4 = d["records"][:, 6:10].contiguous()
    got4 = extra_fwd(cs, bo, d, out, ex4)
    raw = out["raw"].cpu().numpy().reshape(got4.shape)
    same = (got4.view(np.int32) == raw.view(np.int32)) | ((got4 == 0) & (raw == 0))
    exempt = bit_equality_exemptions(case, tuning)
    bad = ~same & ~exempt[..., None]
    assert not bad.any(), f"{name}: extra != raw at {np.argwhere(bad)[:5].tolist()}: {got4[bad][:4]} vs {raw[bad][:4]}"
    rng = np.random.default_rng(case.seed + tuning)
    N = case.inp.records.shape[0]
    wf = wb = 0.0
    for Cn in CHANNELS:
        vals, _, _ = reference(case, Cn)
        ex = torch.from_numpy(vals).cuda()
        wf = max(wf, check_forward(case, Cn, extra_fwd(cs, bo, d, out, ex)))
        vrec0 = rng.uniform(-1.0, 1.0, (N, 12)).astype(np.float32)
        vex0 = rng.uniform(-1.0, 1.0, (N, Cn)).astype(np.float32)
        got_rec, got_ex = extra_bwd(cs, bo, d, out, ex, v_out_seed(case, Cn), vrec0, vex0)
        wb = max(wb, check_backward(case, Cn, vrec0, vex0, got_rec, got_ex))
    print(f"[worst] {name} tuning {tuning}: forward {wf:.3g}, backward {wb:.3g} of the bar")


@pytest.mark.parametrize("name", list(bc.CASES))
def test_extra_deterministic_against_reference_and_repeatable(name, monkeypatch):
    case = bc.get(name)
    cs, bo, d, out = run_forward(case, raster.DEFAULT_TUNING, monkeypatch)
    N = case.inp.records.shape[0]
    rng = np.random.default_rng(case.seed)
    for Cn in (3, 9):
        vals, _, _ = reference(case, Cn)
        ex = torch.from_numpy(vals).cuda()
        vrec0 = rng.uniform(-1.0, 1.0, (N, 12)).astype(np.float32)
        vex0 = rng.uniform(-1.0, 1.0, (N, Cn)).astype(np.float32)
        runs = [extra_bwd(cs, bo, d, out, ex, v_out_seed(case, Cn), vrec0, vex0, det=True) for _ in range(2)]
        assert np.array_equal(runs[0][0].view(np.int32), runs[1][0].view(np.int32)), f"{name}: v_records differ between runs"
        assert np.array_equal(runs[0][1].view(np.int32), runs[1][1].view(np.int32)), f"{name}: v_extra differs between runs"
        w = check_backward(case, Cn, vrec0, vex0, *runs[0], det=True)
        print(f"[worst] {name} deterministic C={Cn}: backward {w:.3g} of the bar")


@pytest.mark.parametrize("Cn", [64, 4096])
def test_extra_channel_limits(Cn, monkeypatch):
    """Many groups on a small image (blockIdx.y up to 511), forward and backward."""
    case = bc.get("shape_17x3")
    cs, bo, d, out = run_forward(case, raster.DEFAULT_TUNING, monkeypatch)
    vals, _, _ = reference(case, Cn)
    ex = torch.from_numpy(vals).cuda()
    check_forward(case, Cn, extra_fwd(cs, bo, d, out, ex))
    N = case.inp.records.shape[0]
    vrec0, vex0 = np.zeros((N, 12), np.float32), np.zeros((N, Cn), np.float32)
    check_backward(case, Cn, vrec0, vex0, *extra_bwd(cs, bo, d, out, ex, v_out_seed(case, Cn), vrec0, vex0))


def test_extra_argument_errors(monkeypatch):
    case = bc.get("shape_17x3")
    cs, bo, d, out = run_forward(case, raster.DEFAULT_TUNING, monkeypatch)
    torch.cuda.synchronize()
    N = case.inp.records.shape[0]
    ex = torch.zeros(N, 4097, device="cuda")
    res = torch.zeros(cs.height, cs.width, 4097, device="cuda")
    v_rec = torch.zeros(N, 12, device="cuda")
    fg = torch.zeros(N, 6, dtype=torch.int64, device="cuda")
    fe = torch.zeros(N, 4097, dtype=torch.int64, device="cuda")
    fs = torch.zeros(2, device="cuda")
    mis = torch.zeros(N * 12 + 4, device="cuda")
    rec, ids, bins, fT, fi = (_p(d["records"]), _p(d["sorted_ids"]), _p(d["tile_bins"]), _p(out["final_T"]), _p(out["final_idx"]))

    def fwd(C_, r=rec, i=ids, b=bins, t=fT, x=fi, e=_p(ex), o=_p(res)):
        return L().sgn_blend_extra_fwd(C.byref(cs), C.byref(bo), r, i, b, t, x, e, C_, o, None)

    def bwd(C_, r=rec, e=_p(ex), vo=_p(res), ve=_p(ex), vr=_p(v_rec)):
        return L().sgn_blend_extra_bwd(C.byref(cs), C.byref(bo), r, ids, bins, fT, fi, e, C_, vo, ve, vr, None)

    def det(C_, n=N, r=rec, g=_p(fg), x=_p(fe), s=_p(fs)):
        return L().sgn_blend_extra_bwd_det(C.byref(cs), C.byref(bo), r, ids, bins, fT, fi, _p(ex), C_, n, _p(res), _p(ex),
                                           _p(v_rec), g, x, s, None)

    before = L().sgn_launch_count()
    for call in (fwd, bwd, det):
        assert call(0) == -1 and b"out of range" in L().sgn_last_error()
        assert call(4097) == -1 and b"out of range" in L().sgn_last_error()
        assert call(4, r=C.c_void_p(mis.data_ptr() + 4)) == -1 and b"aligned" in L().sgn_last_error()
        assert call(4, r=None) == -1
    for k in ("i", "b", "t", "x", "e", "o"):
        assert fwd(4, **{k: None}) == -1, k
    for k in ("e", "vo", "ve", "vr"):
        assert bwd(4, **{k: None}) == -1, k
    for k in ("g", "x", "s"):
        assert det(4, **{k: None}) == -1, k
    assert det(4, n=0) == -1
    bad = _lib.CameraStruct.from_buffer_copy(cs)
    bad.block_width = 8
    assert L().sgn_blend_extra_fwd(C.byref(bad), C.byref(bo), rec, ids, bins, fT, fi, _p(ex), 4, _p(res), None) == -1
    assert L().sgn_launch_count() == before, "an argument error launched a kernel"


# ---- render_frame(extra=...) in deterministic mode ----------------------------------------------------------------
def _render_extra_grads(settings, Cn=9, seed=31):
    from tests.test_gpu_parity import SCENES, to_cuda
    fr = syn.make_frame(**SCENES["small_actors"])
    frc = to_cuda(fr, requires_grad=True)
    N = sum(s.params.num_points for s in fr.segments)
    g = torch.Generator().manual_seed(seed)
    ex = (torch.randn(N, Cn, generator=g) * 3).cuda().requires_grad_(True)
    out, holder = raster.render_frame(frc, settings, extra=ex)
    H, W = fr.camera.height, fr.camera.width
    w = torch.rand(H, W, Cn, generator=g).cuda()
    ((out["extra"] * w).sum() + out["rgb"].sum() + out["object_acc"].sum()).backward()
    torch.cuda.synchronize()
    params = [t.grad.detach().cpu().numpy() for s in frc.segments for t in s.params.tensors()]
    return ex.grad.cpu().numpy(), holder.v_records.cpu().numpy(), params


def test_render_frame_extra_deterministic_is_bit_repeatable():
    """Deterministic mode with extra channels: v_extra, v_records and every parameter gradient the same bits twice, and
    within 1e-5 relative L2 of the float-atomic gradients."""
    a = _render_extra_grads(raster.RenderSettings(deterministic=True))
    b = _render_extra_grads(raster.RenderSettings(deterministic=True))
    assert np.array_equal(a[0].view(np.int32), b[0].view(np.int32)), "v_extra differs between runs"
    assert np.array_equal(a[1].view(np.int32), b[1].view(np.int32)), "v_records differ between runs"
    for k, (x, y) in enumerate(zip(a[2], b[2])):
        assert np.array_equal(x.view(np.int32), y.view(np.int32)), f"parameter gradient {k} differs between runs"
    f = _render_extra_grads(raster.RenderSettings(deterministic=False))
    for what, x, y in (("v_extra", a[0], f[0]), ("v_records", a[1][:, :10], f[1][:, :10])):
        rel = np.linalg.norm(x.astype(np.float64) - y) / np.linalg.norm(y)
        assert rel <= 1e-5, f"{what}: deterministic vs float atomics relative L2 {rel:.3e}"


# ---- Level-1 rasterize_gaussians ------------------------------------------------------------------------------------
L1_W, L1_H = 40, 24


def _l1_lists(rec, radii, W, H):
    """gsplat's lists: every tile of the AABB get_tile_bbox gives (xys, radii), in (tile, depth) order."""
    bw = np.float32(16)
    tc = rec[:, 0:2] / bw
    tr = (radii.astype(np.float32) / bw)[:, None]
    lim = np.array([(W + 15) // 16, (H + 15) // 16], np.float32)
    tmin = np.minimum(np.maximum(np.trunc(tc - tr), 0), lim)
    tmax = np.minimum(np.maximum(np.trunc(tc + tr + np.float32(1)), 0), lim)
    bbox = np.concatenate([tmin, tmax], 1).astype(np.int64)
    z = np.zeros(len(radii), np.int64)
    h = bin_ref64.rows(rec, radii, bbox, z, z)
    tile, row = bin_ref64.list_order(h, *bin_ref64.entries(h, W, H, 16, touch_filter=False))
    ids, bins = bin_ref64.lists(h, int(lim[0] * lim[1]), tile, row)
    nth = ((bbox[:, 2] - bbox[:, 0]) * (bbox[:, 3] - bbox[:, 1])).astype(np.int32)
    return ids, bins.astype(np.int32), nth


L1_OPTS = ref.Opts(raw_mode=True, class_streams=False)


def l1_scene(Cn, seed, n=70, W=L1_W, H=L1_H):
    """gsplat-style inputs; opacities nudged until no skip / stop decision is within bc.MARGIN of its threshold."""
    rng = np.random.default_rng(seed)
    xys = rng.uniform(-4.0, W + 4.0, (n, 2))
    sx, sy = rng.uniform(1.0, 5.0, (2, n))
    rho = rng.uniform(-0.6, 0.6, n)
    cov = np.stack([np.stack([sx * sx, rho * sx * sy], -1), np.stack([rho * sx * sy, sy * sy], -1)], -2)
    inv = np.linalg.inv(cov)
    conics = np.stack([inv[:, 0, 0], inv[:, 0, 1], inv[:, 1, 1]], 1).astype(np.float32)
    radii = np.ceil(3.0 * np.sqrt(np.linalg.eigvalsh(cov)[:, 1])).astype(np.int32)
    depths = (1.0 + 0.1 * rng.permutation(n) + rng.uniform(0.0, 0.05, n)).astype(np.float32)
    opac = rng.uniform(0.05, 0.9, n).astype(np.float32)
    colors = rng.uniform(-0.5, 1.5, (n, Cn)).astype(np.float32)
    rec = np.zeros((n, 12), np.float32)
    rec[:, 0:2], rec[:, 2:5], rec[:, 9] = xys, conics, depths
    ids, bins, nth = _l1_lists(rec, radii, W, H)
    for _ in range(60):
        rec[:, 5] = opac
        inp = ref.Inputs(W, H, rec.copy(), ids, bins)
        fw = ref.forward_channels(inp, L1_OPTS, colors)
        bad = fw["gauss_margin"] < bc.MARGIN
        if not bad.any() and fw["margin"].min() >= bc.MARGIN:
            return dict(xys=rec[:, 0:2].copy(), conics=conics, opac=opac.copy(), depths=depths, radii=radii, nth=nth,
                        colors=colors, inp=inp)
        if not bad.any():  # a pixel-level decision: nudge everything listed in the offending tiles
            ys, xs = np.nonzero(fw["margin"] < bc.MARGIN)
            for y, x in zip(ys, xs):
                t = (y // 16) * ((W + 15) // 16) + x // 16
                bad[ids[bins[t, 0]:bins[t, 1]] & 0x7FFFFFFF] = True
        opac[bad] *= (1.0 + rng.uniform(-0.03, 0.03, int(bad.sum()))).astype(np.float32)
    raise AssertionError("could not move every decision away from its threshold")


def _cuda(x, grad=False):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda().requires_grad_(grad)


@pytest.mark.parametrize("with_bg", [True, False], ids=["background", "default_ones"])
@pytest.mark.parametrize("Cn", [1, 2, 3, 4, 5, 7, 8, 12])
def test_l1_rasterize_against_reference(Cn, with_bg):
    sc = l1_scene(Cn, seed=300 + Cn)
    rng = np.random.default_rng(Cn)
    bg = rng.uniform(-0.5, 1.5, Cn).astype(np.float32) if with_bg else np.ones(Cn, np.float32)
    fw = ref.forward_channels(sc["inp"], L1_OPTS, sc["colors"], background=bg)
    v_img = rng.uniform(-1.0, 1.0, (L1_H, L1_W, Cn)).astype(np.float32)
    v_alpha = rng.uniform(-1.0, 1.0, (L1_H, L1_W)).astype(np.float32)
    for cot in ("image", "alpha", "both"):
        xys, conics, colors = _cuda(sc["xys"], True), _cuda(sc["conics"], True), _cuda(sc["colors"], True)
        opac = _cuda(sc["opac"][:, None], True)
        img, alpha = gsplat_compat.rasterize_gaussians(xys, _cuda(sc["depths"]), _cuda(sc["radii"]), conics, _cuda(sc["nth"]),
                                                       colors, opac, L1_H, L1_W, 16,
                                                       background=_cuda(bg) if with_bg else None, return_alpha=True)
        got = img.detach().cpu().numpy()
        tol = IMG_TOL * np.maximum(1.0, fw["abs"])
        assert (np.abs(got - fw["out"]) <= tol).all(), f"C={Cn}: image off by {(np.abs(got - fw['out']) / tol).max():.2f} of the bar"
        assert np.abs(alpha.detach().cpu().numpy() - (1.0 - fw["final_T"])).max() <= IMG_TOL
        vo = v_img if cot != "alpha" else np.zeros_like(v_img)
        va = v_alpha if cot != "image" else None
        loss = 0.0
        if cot != "alpha":
            loss = loss + (img * _cuda(v_img)).sum()
        if cot != "image":
            loss = loss + (alpha * _cuda(v_alpha)).sum()
        gx, gc, gcol, gop = torch.autograd.grad(loss, [xys, conics, colors, opac], allow_unused=True)
        vv, vr, vva, vra = ref.backward_channels(sc["inp"], L1_OPTS, sc["colors"], vo, v_alpha=va, background=bg)
        pairs = (("v_xys", gx, vr[:, 0:2], vra[:, 0:2]), ("v_conics", gc, vr[:, 2:5], vra[:, 2:5]),
                 ("v_colors", gcol, vv, vva), ("v_opacity", gop, vr[:, 5:6], vra[:, 5:6]))
        for what, g, want, S in pairs:
            g = np.zeros_like(want, dtype=np.float32) if g is None else g.cpu().numpy().reshape(want.shape)
            ex = excess(g, want, S)
            w = np.unravel_index(np.argmax(ex), ex.shape)
            assert ex.max() <= 1.0, f"C={Cn} [{cot}] {what}: Gaussian {w[0]} component {w[1]}: {g[w]!r} vs {want[w]!r}"


def test_l1_rasterize_uint8_colors():
    sc = l1_scene(3, seed=307)
    rng = np.random.default_rng(8)
    u8 = rng.integers(0, 256, (len(sc["opac"]), 3)).astype(np.uint8)
    bg = np.array([0.1, 0.5, 0.9], np.float32)
    fw = ref.forward_channels(sc["inp"], L1_OPTS, u8.astype(np.float32) / np.float32(255), background=bg)
    img = gsplat_compat.rasterize_gaussians(_cuda(sc["xys"]), _cuda(sc["depths"]), _cuda(sc["radii"]), _cuda(sc["conics"]),
                                            _cuda(sc["nth"]), _cuda(u8), _cuda(sc["opac"][:, None]), L1_H, L1_W, 16,
                                            background=_cuda(bg))
    assert (np.abs(img.cpu().numpy() - fw["out"]) <= IMG_TOL * np.maximum(1.0, fw["abs"])).all()


def test_l1_rasterize_empty_scene():
    """Every num_tiles_hit 0: the background everywhere, alpha 0, zero gradients of the inputs' shapes."""
    sc = l1_scene(5, seed=305)
    n = len(sc["opac"])
    bg = np.linspace(-0.5, 1.5, 5).astype(np.float32)
    xys, conics, colors = _cuda(sc["xys"], True), _cuda(sc["conics"], True), _cuda(sc["colors"], True)
    opac = _cuda(sc["opac"][:, None], True)
    img, alpha = gsplat_compat.rasterize_gaussians(xys, _cuda(sc["depths"]), _cuda(sc["radii"]), conics,
                                                   torch.zeros(n, dtype=torch.int32, device="cuda"), colors, opac, L1_H, L1_W,
                                                   16, background=_cuda(bg), return_alpha=True)
    assert np.array_equal(img.detach().cpu().numpy(), np.broadcast_to(bg, (L1_H, L1_W, 5)))
    assert np.all(alpha.detach().cpu().numpy() == 0)
    grads = torch.autograd.grad((img * 2).sum() + alpha.sum(), [xys, conics, colors, opac])
    for g, t in zip(grads, (xys, conics, colors, opac)):
        assert g.shape == t.shape and torch.all(g == 0)


def test_l1_rasterize_refuses_other_block_widths():
    sc = l1_scene(3, seed=303)
    args = (_cuda(sc["xys"]), _cuda(sc["depths"]), _cuda(sc["radii"]), _cuda(sc["conics"]), _cuda(sc["nth"]),
            _cuda(sc["colors"]), _cuda(sc["opac"][:, None]), L1_H, L1_W)
    with pytest.raises(_lib.SgnError):
        gsplat_compat.rasterize_gaussians(*args, 8)
    with pytest.raises(AssertionError):
        gsplat_compat.rasterize_gaussians(*args, 17)
