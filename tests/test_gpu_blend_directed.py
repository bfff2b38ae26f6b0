"""The blend kernels on hand-built tiles (tests/blend_cases.py) against the float64 reference (oracle/blend_ref64.py).

Every case runs under each execution variant (SGN_TUNING 0, 1, 4, 8, 1|4, 4|8, 16, 4|8|32, with the heavy-first schedule
on and off) and is compared with the reference, never with another variant:
  * every pixel of rgb, accumulation, depth, object_acc, background_acc and the raw sums within IMG_TOL (depth: plus
    what the division by a small alpha makes of the fp32 error of 1 - T);
  * final_idx of all three slots exactly, and tile_depth exactly as the reference's indices imply;
  * every component of every per-Gaussian gradient within |got - ref| <= GRAD_R |ref| + GRAD_A S, element by element,
    where S is the element's sum of the absolute values of its terms (the reference computes it alongside): the scale of
    the fp32 rounding of a sum that cancels, such as the conic gradient of a symmetric Gaussian or the depth cotangent's
    terms of a Gaussian that alone makes up a pixel's depth.  Under each of the five cotangents alone, all five together
    (U(-1, 1)) and all five constant, with v_sky where the case has a sky; with float atomics and with the deterministic
    fixed-point accumulator (bit-repeatable; its rounding to the grid is allowed for on top, quantization_floor).

Observed on an H100 80GB HBM3 (every case, variant and cotangent, float atomics): rgb at most 1.2e-6 from the reference,
accumulation 4.2e-7, object_acc / background_acc 3.3e-7, the raw sums 4.8e-6, depth 1.7e-5 (1.5e-4 on the 1920x1280
frame, where depth is 20 and alpha is small at the Gaussian's edge); gradients at most 2.1e-6 |ref| + 2.1e-6 S.  The
bounds below leave a factor above 20.  A dropped, doubled or misplaced entry moves a Gaussian's components by a sizeable
fraction of S; each of six one-token changes to blend.cu (residual condition, object rank, replay depth, background
cotangent fold, paired row offset, row reach) fails between 34 and 221 of these tests.
"""
import numpy as np
import pytest
import torch

from street_gaussians_ns_b200 import _lib, raster
from oracle import blend_ref64 as ref
from tests import blend_cases as bc

pytestmark = pytest.mark.gpu

IMG_TOL = 1e-4
GRAD_R = 5e-5
GRAD_A = 5e-5
TUNINGS = [0, 1, 4, 8, 1 | 4, 4 | 8, 16, 4 | 8 | 32]
COT_SETS = ["rgb", "accumulation", "depth", "object_acc", "background_acc", "all", "const"]


def _setup(case, tuning, monkeypatch):
    for k in ("SGN_SPLIT_FWD_MAIN", "SGN_SPLIT_FWD_ACC", "SGN_SPLIT_BWD_MAIN", "SGN_SPLIT_BWD_ACC"):
        monkeypatch.setenv(k, str(case.splits.get(k, 0)))
    monkeypatch.setenv("SGN_TUNING", str(tuning))
    o = case.opts
    cs = _lib.CameraStruct()
    cs.width, cs.height, cs.block_width = case.inp.width, case.inp.height, 16
    bo = raster.blend_opts(raster.RenderSettings(class_streams=o.class_streams, training=not o.eval_clamp), o.has_sky)
    bo.raw_mode = int(o.raw_mode)
    for c in range(4):
        bo.background[c] = o.background[c]
    return cs, bo


def _dev(case):
    inp = case.inp
    d = dict(records=torch.from_numpy(np.ascontiguousarray(inp.records)).cuda(),
             sorted_ids=torch.from_numpy(inp.sorted_ids if len(inp.sorted_ids) else np.zeros(1, np.int32)).cuda(),
             tile_bins=torch.from_numpy(inp.tile_bins).cuda(),
             sky=torch.from_numpy(inp.sky).cuda() if inp.sky is not None else None)
    if case.opts.class_streams:
        d["cls_ids"] = torch.from_numpy(inp.cls_ids).cuda()
        d["cls_bins"] = torch.from_numpy(inp.cls_bins).cuda()
    return d


def run_forward(case, tuning, monkeypatch):
    cs, bo = _setup(case, tuning, monkeypatch)
    d = _dev(case)
    out = raster.blend_fwd(cs, bo, d["records"], d["sorted_ids"], d["tile_bins"], d["sky"], d.get("cls_ids"), d.get("cls_bins"))
    return cs, bo, d, out


def run_backward(case, cs, bo, d, out, cot, deterministic):
    v = {k: torch.from_numpy(np.ascontiguousarray(x)).cuda() for k, x in cot.items()}
    v_records, v_sky = raster.blend_bwd(cs, bo, d["records"], d["sorted_ids"], d["tile_bins"], out, d["sky"], v, d["sky"] is not None,
                                        d.get("cls_ids"), d.get("cls_bins"), deterministic=deterministic)
    torch.cuda.synchronize()
    return v_records.cpu().numpy(), (v_sky.cpu().numpy() if v_sky is not None else None)


def _cot(case, kind):
    full = bc.cotangents(case, "const" if kind == "const" else "rand")
    if kind in ("all", "const"):
        return full
    return {kind: full[kind]} if kind in full else None


_REF_BWD = {}


def reference_backward(case, kind):
    key = (case.name, kind)
    if key not in _REF_BWD:
        _REF_BWD[key] = ref.backward(case.inp, case.opts, _cot(case, kind))
    return _REF_BWD[key]


def check_forward(case, out):
    fw = case.fwd
    got = {k: t.cpu().numpy() for k, t in out.items() if isinstance(t, torch.Tensor)}
    alpha = fw["accumulation"]
    names = ["rgb", "accumulation", "depth", "raw"] + (["object_acc", "background_acc"] if case.opts.class_streams else [])
    for k in names:
        g = got[k].reshape(fw[k].shape)
        err = np.abs(g.astype(np.float64) - fw[k])
        tol = IMG_TOL
        if k == "depth" and not case.opts.raw_mode:  # d / alpha: the fp32 error of 1 - T (~1e-7) grows as 1 / alpha
            tol = IMG_TOL + 2e-6 * np.abs(fw[k]) / np.maximum(alpha, 1e-3)
        bad = err > tol
        assert not bad.any(), f"{case.name}: {k} differs at {np.argwhere(bad)[:5].tolist()} by up to {err.max():.3e}"
    S = fw["final_idx"].shape[0]
    for s in range(S):
        np.testing.assert_array_equal(got["final_idx"][s], fw["final_idx"][s], err_msg=f"{case.name}: final_idx slot {s}")
    np.testing.assert_array_equal(got["tile_depth"], fw["tile_depth"], err_msg=f"{case.name}: tile_depth")


def grad_excess(got, refv, absv):
    """|got - ref| / (GRAD_R |ref| + GRAD_A S) per element, S = the element's sum of absolute terms; <= 1 passes."""
    bound = GRAD_R * np.abs(refv) + GRAD_A * absv
    err = np.abs(got.astype(np.float64) - refv)
    with np.errstate(all="ignore"):
        return np.where(err == 0, 0.0, err / np.where(bound > 0, bound, 1e-300))


def fixed_shift(records):
    """[N,12] places the deterministic grid gives up per record component (csrc/blend.cu fixed_shift, same double ops)."""
    a, b, c = (records[:, k].astype(np.float64) for k in (2, 3, 4))
    with np.errstate(all="ignore"):
        det = a * c - b * b
        E = (a + c) / det
        e = np.frexp(np.fmin(np.where((det > 0) & (E > 0), E, 1.0), 1e18))[1]
    sh = np.where((det > 0) & (E > 0), np.clip(2 * e - 26, 0, 100), 0)
    out = np.zeros(records.shape, np.int64)
    out[:, 2:5] = sh[:, None]
    return out


def quantization_floor(case, cot):
    """Deterministic mode: every addend is rounded to the fixed-point grid (half a unit of 2^(shift - 32) max|cotangent|),
    and a Gaussian gets at most 24 addends per tile that lists it (8 strips x main, object residual, background)."""
    m = max(float(np.abs(v).max()) for v in cot.values())
    unit = np.ldexp(1.0, fixed_shift(case.inp.records) - 32 + int(np.ceil(np.log2(m))))
    ids = np.asarray(case.inp.sorted_ids, np.int64) & 0x7FFFFFFF
    ntiles = np.bincount(ids, minlength=case.inp.records.shape[0])
    return 12.0 * ntiles[:, None] * unit


def check_grads(case, kind, got, v_sky, deterministic=False):
    rv, rsky, _, rabs = reference_backward(case, kind)
    cols = list(range(10))
    if deterministic:
        rabs = rabs + quantization_floor(case, _cot(case, kind)) / GRAD_A
    ex = grad_excess(got[:, cols], rv[:, cols], rabs[:, cols])
    worst = np.unravel_index(np.argmax(ex), ex.shape)
    assert ex.max() <= 1.0, (f"{case.name} [{kind}]: gradient of Gaussian {worst[0]} component {worst[1]}: "
                             f"{got[worst[0], worst[1]]!r} vs {rv[worst[0], worst[1]]!r}")
    assert np.all(got[:, 10:] == 0)
    if rsky is not None:
        assert v_sky is not None
        assert np.abs(v_sky - rsky).max() <= IMG_TOL


@pytest.fixture(params=[True, False], ids=["heavy_first", "raster_order"])
def heavy(request, monkeypatch):
    monkeypatch.setattr(raster, "HEAVY_FIRST", request.param)
    return request.param


@pytest.mark.parametrize("tuning", TUNINGS)
@pytest.mark.parametrize("name", list(bc.CASES))
def test_case_against_reference(name, tuning, heavy, monkeypatch):
    case = bc.get(name)
    cs, bo, d, out = run_forward(case, tuning, monkeypatch)
    torch.cuda.synchronize()
    check_forward(case, out)
    for kind in COT_SETS:
        cot = _cot(case, kind)
        if cot is None:
            continue
        got, v_sky = run_backward(case, cs, bo, d, out, cot, deterministic=False)
        check_grads(case, kind, got, v_sky)


@pytest.mark.parametrize("name", list(bc.CASES))
def test_deterministic_against_reference_and_repeatable(name, monkeypatch):
    """Fixed-point accumulation: the same bits twice (with the schedule and without), and the reference's values at the
    float path's bounds plus the grid's rounding (quantization_floor) -- including the sigma-250 px Gaussian, whose conic
    gradient is -3.8e10 under unit cotangents (it wrapped to +2.3e8 before the conic grid of large Gaussians was coarsened)."""
    case = bc.get(name)
    for kind in ("all", "const"):
        cot = _cot(case, kind)
        runs = []
        for hf in (True, False):
            monkeypatch.setattr(raster, "HEAVY_FIRST", hf)
            cs, bo, d, out = run_forward(case, raster.DEFAULT_TUNING, monkeypatch)
            runs.append(run_backward(case, cs, bo, d, out, cot, deterministic=True))
        assert np.array_equal(runs[0][0], runs[1][0]), f"{case.name}: deterministic gradients differ between runs"
        check_grads(case, kind, runs[0][0], runs[0][1], deterministic=True)


def test_config3_deterministic_matches_float_atomics():
    """A full config-3 frame: fixed-point against float-atomic gradients, per record component, 1e-5 relative L2."""
    import street_gaussians_ns_b200.synthetic as syn
    from street_gaussians_ns_b200.scene import Frame, Segment
    fr = syn.config_frame(3)
    frc = Frame(fr.camera, [Segment(s.params.to("cuda"), s.cls, s.rot, s.center, s.idft) for s in fr.segments])
    H, W = fr.camera.height, fr.camera.width
    g = torch.Generator().manual_seed(3)
    cots = {"rgb": torch.rand(H, W, 3, generator=g).cuda(), "accumulation": torch.rand(H, W, 1, generator=g).cuda(),
            "object_acc": torch.rand(H, W, 1, generator=g).cuda()}
    res = {}
    for det in (True, False):
        _, h = raster.forward_backward(frc, raster.RenderSettings(deterministic=det), cots)
        res[det] = h.v_records.cpu().numpy().astype(np.float64)
    for c0, c1 in ((0, 2), (2, 5), (5, 6), (6, 9)):
        a, b = res[True][:, c0:c1], res[False][:, c0:c1]
        rel = np.linalg.norm(a - b) / np.linalg.norm(b)
        assert rel <= 1e-5, f"components {c0}:{c1}: deterministic vs float atomics relative L2 {rel:.3e}"
