"""The absolute screen-space gradient (sgn_blend_bwd_absgrad, sgn_densify_stats_abs, the model's absgrad switch) on the GPU.

  * every hand-built blend case (tests/blend_cases.py) under every execution variant and both schedules, against the
    float64 statement (oracle/absgrad_ref64.py): v_absxy within GRAD_R |ref| + GRAD_A S, S the element's sum of absolute
    factors; v_records and v_sky within the bounds of the directed blend tests, for the cotangents rgb, accumulation,
    depth, object_acc (whose stream adds nothing: v_absxy is exactly 0) and all of them but background_acc;
  * deterministic mode: the same bits over two runs (heavy-first and raster order), v_records bit-identical to
    sgn_blend_bwd's, values within the bounds plus the fixed-point grid's rounding;
  * a full config-3 frame: v_absxy >= |v_records[:, 0:2]| and fixed point against float atomics;
  * a large Gaussian over a 2-px checkerboard: split only with absgrad;
  * one training step of the model with absgrad, and the argument checks of both entry points.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import absgrad_ref64 as aref
from oracle import blend_ref64 as ref
from street_gaussians_ns_b200 import _lib, raster, refine
from tests import blend_cases as bc
from tests import test_gpu_blend_directed as bd

pytestmark = pytest.mark.gpu

ABS_SETS = ["rgb", "accumulation", "depth", "object_acc", "main"]


def _cot(case, kind):
    if kind == "main":  # every cotangent but background_acc's, which absgrad refuses
        return {k: v for k, v in bc.cotangents(case, "rand").items() if k != "background_acc"}
    return bd._cot(case, kind)


_REF = {}


def _ref(case, kind):
    key = (case.name, kind)
    if key not in _REF:
        cot = _cot(case, kind)
        _REF[key] = (aref.absgrad(case.inp, case.opts, cot), ref.backward(case.inp, case.opts, cot))
    return _REF[key]


def run_backward_abs(case, cs, bo, d, out, cot, deterministic):
    v = {k: torch.from_numpy(np.ascontiguousarray(x)).cuda() for k, x in cot.items()}
    v_records, v_sky, v_absxy = raster.blend_bwd(cs, bo, d["records"], d["sorted_ids"], d["tile_bins"], out, d["sky"], v,
                                                 d["sky"] is not None, d.get("cls_ids"), d.get("cls_bins"),
                                                 deterministic=deterministic, absgrad=True)
    torch.cuda.synchronize()
    return v_records.cpu().numpy(), (v_sky.cpu().numpy() if v_sky is not None else None), v_absxy.cpu().numpy()


def check_abs(case, kind, got_rec, got_sky, got_abs, deterministic=False):
    (want, bound, _), (rv, rsky, _, rabs) = _ref(case, kind)
    if deterministic:
        floor = bd.quantization_floor(case, _cot(case, kind)) / bd.GRAD_A
        bound, rabs = bound + floor[:, 0:2], rabs + floor
    ex = bd.grad_excess(got_abs, want, bound)
    w = np.unravel_index(np.argmax(ex), ex.shape)
    assert ex.max() <= 1.0, f"{case.name} [{kind}]: absgrad of Gaussian {w[0]} component {w[1]}: {got_abs[w]!r} vs {want[w]!r}"
    ex = bd.grad_excess(got_rec[:, :10], rv[:, :10], rabs[:, :10])
    w = np.unravel_index(np.argmax(ex), ex.shape)
    assert ex.max() <= 1.0, f"{case.name} [{kind}]: gradient of Gaussian {w[0]} component {w[1]}: {got_rec[w]!r} vs {rv[w]!r}"
    assert np.all(got_rec[:, 10:] == 0)
    if rsky is not None:
        assert got_sky is not None and np.abs(got_sky - rsky).max() <= bd.IMG_TOL


@pytest.mark.parametrize("tuning", bd.TUNINGS)
@pytest.mark.parametrize("name", list(bc.CASES))
def test_case_against_reference(name, tuning, heavy, monkeypatch):
    case = bc.get(name)
    cs, bo, d, out = bd.run_forward(case, tuning, monkeypatch)
    for kind in ABS_SETS:
        cot = _cot(case, kind)
        if cot is None:
            continue
        got_rec, got_sky, got_abs = run_backward_abs(case, cs, bo, d, out, cot, deterministic=False)
        check_abs(case, kind, got_rec, got_sky, got_abs)
        if kind == "object_acc":  # the objects-only stream adds nothing
            assert not got_abs.any()


@pytest.fixture(params=[True, False], ids=["heavy_first", "raster_order"])
def heavy(request, monkeypatch):
    monkeypatch.setattr(raster, "HEAVY_FIRST", request.param)
    return request.param


@pytest.mark.parametrize("name", list(bc.CASES))
def test_deterministic(name, monkeypatch):
    case = bc.get(name)
    cot = _cot(case, "main")
    runs = []
    for hf in (True, False):
        monkeypatch.setattr(raster, "HEAVY_FIRST", hf)
        cs, bo, d, out = bd.run_forward(case, raster.DEFAULT_TUNING, monkeypatch)
        runs.append(run_backward_abs(case, cs, bo, d, out, cot, deterministic=True))
        plain, plain_sky = bd.run_backward(case, cs, bo, d, out, cot, deterministic=True)
        assert np.array_equal(runs[-1][0], plain), f"{case.name}: v_records differ from sgn_blend_bwd's"
        assert (plain_sky is None) == (runs[-1][1] is None) and (plain_sky is None or np.array_equal(runs[-1][1], plain_sky))
    assert np.array_equal(runs[0][2], runs[1][2]), f"{case.name}: deterministic absgrad differs between runs"
    check_abs(case, "main", *runs[0], deterministic=True)


def _config3(det):
    import street_gaussians_ns_b200.synthetic as syn
    from street_gaussians_ns_b200.scene import Frame, Segment
    fr = syn.config_frame(3)
    frc = Frame(fr.camera, [Segment(s.params.to("cuda"), s.cls, s.rot, s.center, s.idft) for s in fr.segments])
    H, W = fr.camera.height, fr.camera.width
    g = torch.Generator().manual_seed(3)
    cots = {"rgb": torch.rand(H, W, 3, generator=g).cuda(), "accumulation": torch.rand(H, W, 1, generator=g).cuda()}
    _, h = raster.forward_backward(frc, raster.RenderSettings(deterministic=det, absgrad=True), cots)
    return (h.v_records.cpu().numpy().astype(np.float64), h.v_absxy.cpu().numpy().astype(np.float64),
            h.num_tiles_hit.cpu().numpy().astype(np.float64))


def test_config3_frame():
    """v_absxy >= |v_records[:, 0:2]| up to fp32 rounding (1e-5 relative) and, in deterministic mode, the grid's: each of the
    two sums rounds every addend to half a unit of 2^-32 (max|cotangent| < 1), at most 24 addends per tile listing the row."""
    rec_d, abs_d, tiles = _config3(True)
    rec_f, abs_f, _ = _config3(False)
    for det, rec, ab in ((True, rec_d, abs_d), (False, rec_f, abs_f)):
        vxy = np.abs(rec[:, 0:2])
        floor = (24.0 * tiles * 2.0 ** -32)[:, None] if det else 0.0
        short = vxy - ab - 1e-5 * (ab + vxy) - floor
        w = np.unravel_index(np.argmax(short), short.shape)
        assert short.max() <= 0, f"deterministic={det}: row {w[0]} component {w[1]}: absgrad {ab[w]!r} < |v_xy| {vxy[w]!r}"
    assert abs_f.max() > 0
    rel = np.linalg.norm(abs_d - abs_f) / np.linalg.norm(abs_f)
    assert rel <= 1e-5, f"absgrad: deterministic vs float atomics relative L2 {rel:.3e}"


def checkerboard():
    """One Gaussian of sigma 12 px and opacity 0.9 centred on a cell corner of a 64 x 64 image whose target is a 2-px
    checkerboard of 0 and 1; its colour (0.5) sits between them, so the L1 cotangent sign(rgb - target) / (3 H W)
    alternates from cell to cell and the per-pixel screen-space gradients cancel in their sum."""
    b = bc.Builder(64, 64, 11)
    g = b.gauss(32.0, 32.0, 12.0, o=0.9, rgb=(0.5, 0.5, 0.5), depth=5.0)
    for t in range(b.tiles):
        b.lists[t] = [g]
    inp = b.inputs()
    y, x = np.mgrid[0:64, 0:64]
    target = (((x // 2) + (y // 2)) % 2).astype(np.float32)
    return inp, np.repeat(target[:, :, None], 3, 2)


def test_checkerboard_split_only_with_absgrad(monkeypatch):
    inp, target = checkerboard()
    case = bc.Case("checkerboard", 11, inp, ref.Opts(class_streams=False))
    cs, bo, d, out = bd.run_forward(case, raster.DEFAULT_TUNING, monkeypatch)
    rgb = out["rgb"].cpu().numpy()
    v_rgb = (np.sign(rgb - target) / rgb.size).astype(np.float32)
    got_rec, _, got_abs = run_backward_abs(case, cs, bo, d, out, {"rgb": v_rgb}, deterministic=False)
    s = refine.RefineSettings()
    norm = 0.5 * 64
    signed, absolute = np.linalg.norm(got_rec[0, 0:2]) * norm, np.linalg.norm(got_abs[0]) * norm
    assert signed < s.densify_grad_thresh, signed
    assert absolute > s.densify_absgrad_thresh, absolute
    # sgn_refine_decide: a Gaussian larger than densify_size_thresh with a high statistic is split
    dev = torch.device("cuda")
    scales = torch.full((1, 3), float(np.log(0.5)), device=dev)
    opac = torch.full((1, 1), 2.0, device=dev)
    vis = torch.ones(1, device=dev)
    size = torch.full((1,), 0.01, device=dev)
    for absgrad, stat in ((False, np.linalg.norm(got_rec[0, 0:2])), (True, np.linalg.norm(got_abs[0]))):
        cfg = refine.make_config(s, 1000, (64, 64), True, absgrad=absgrad)
        flags, _ = refine.decide_submodel(scales, opac, torch.full((1,), float(stat), device=dev), vis, size, cfg)
        assert bool(int(flags[0]) & _lib.RF_SPLIT) == absgrad, (absgrad, int(flags[0]))


def test_model_train_step_uses_absgrad():
    import street_gaussians_ns_b200.synthetic as syn
    from street_gaussians_ns_b200.model import ActorPose, SceneGraphConfig, SceneGraphRasterModel
    from street_gaussians_ns_b200.optim import FusedAdam
    from street_gaussians_ns_b200.training import TrainStep
    sc = syn.WaymoScene(scale=0.02, num_frames=20, n_actors=4)
    frame_list = list(range(sc.num_frames))

    def poses_at(t):
        f = int(t)
        return [ActorPose(str(a), rot, center, f, frame_list, frame_id=f) for a, rot, center in sc.boxes_at(f)]
    cfg = SceneGraphConfig(use_sky_sphere=False, ssim_lambda=0.0, absgrad=True, refine_record=True)
    model = SceneGraphRasterModel(sc.background.to("cuda"), {k: v.to("cuda") for k, v in sc.actors.items()}, cfg,
                                  poses_at=poses_at).to("cuda")
    model.train()
    opt = FusedAdam(model.optimizer_params())
    fn = TrainStep(model, opt)
    g = torch.Generator().manual_seed(5)
    gt = (torch.rand(sc.height, sc.width, 3, generator=g) * 255).to(torch.uint8).to("cuda")
    cam = sc.cameras[1]
    fn(599, cam, {"image": gt})
    torch.cuda.synchronize()
    h = model._holder
    assert h.v_absxy is not None and h.v_absxy.shape == (h.v_records.shape[0], 2)
    subs = dict(model.all_models.items())
    for name in model.visible_model_names:
        sub = subs[name]
        sl = next(s for m, s in model._slices if m is sub)
        want = torch.linalg.vector_norm(h.v_absxy[sl], dim=1)
        assert torch.allclose(sub.xys_grad_norm, want, rtol=1e-6, atol=0), name
        xys = sub.xys
        assert torch.equal(xys.absgrad, h.v_absxy[sl]) and torch.equal(xys.grad, h.v_records[sl, 0:2])
    n0 = [s.num_points for s in subs.values()]
    fn(600, cam, {"image": gt})  # refine_every 100: a refinement
    torch.cuda.synchronize()
    assert any(s.refine_record_dict for s in subs.values())
    assert [s.num_points for s in subs.values()] != n0


def _bad_calls():
    """(description, callable) of argument errors of both entry points; nothing else about them is wrong."""
    L = _lib.load()
    cs = _lib.CameraStruct()
    cs.width, cs.height, cs.block_width = 32, 32, 16
    bo = raster.blend_opts(raster.RenderSettings(), False)
    dev = torch.device("cuda")
    records = torch.zeros(4, 12, device=dev)
    ids = torch.zeros(1, dtype=torch.int32, device=dev)
    bins = torch.zeros(4, 2, dtype=torch.int32, device=dev)
    buf = torch.zeros(64, device=dev)
    absxy = torch.zeros(4, 2, device=dev)
    fx = torch.zeros(4, 2, dtype=torch.int64, device=dev)
    keep = [records, ids, bins, buf, absxy, fx]

    def bwd_in(det=False, bg=False):
        bi = _lib.BlendBwdIn()
        bi.raw = bi.final_T = bi.final_idx = bi.tile_depth = buf.data_ptr()
        bi.v_rgb = buf.data_ptr()
        bi.num_gaussians = 4
        if det:
            bi.v_fixed, bi.fixed_scale = fx.data_ptr(), buf.data_ptr()
        if bg:
            bi.v_background_acc = buf.data_ptr()
        return bi

    def call(bi, v_absxy, fixed):
        return L.sgn_blend_bwd_absgrad(C.byref(cs), C.byref(bo), records.data_ptr(), ids.data_ptr(), bins.data_ptr(), 1, None, None,
                                       C.byref(bi), buf.data_ptr(), v_absxy, fixed, None)
    tab = torch.zeros(64, dtype=torch.uint8, device=dev)
    radii = torch.zeros(4, dtype=torch.int32, device=dev)
    keep += [tab, radii]
    return keep, [
        ("null v_absxy", lambda: call(bwd_in(), None, None)),
        ("misaligned v_absxy", lambda: call(bwd_in(), absxy.data_ptr() + 4, None)),
        ("fixed_absxy without v_fixed", lambda: call(bwd_in(), absxy.data_ptr(), fx.data_ptr())),
        ("v_fixed without fixed_absxy", lambda: call(bwd_in(det=True), absxy.data_ptr(), None)),
        ("v_background_acc", lambda: call(bwd_in(bg=True), absxy.data_ptr(), None)),
        ("stats: null v_absxy", lambda: L.sgn_densify_stats_abs(tab.data_ptr(), 1, 4, None, radii.data_ptr(), 32, 32, None)),
        ("stats: misaligned v_absxy", lambda: L.sgn_densify_stats_abs(tab.data_ptr(), 1, 4, absxy.data_ptr() + 4, radii.data_ptr(),
                                                                      32, 32, None)),
        ("stats: bad size", lambda: L.sgn_densify_stats_abs(tab.data_ptr(), 1, 4, absxy.data_ptr(), radii.data_ptr(), 0, 32, None)),
    ]


def test_argument_validation():
    L = _lib.load()
    keep, calls = _bad_calls()
    torch.cuda.synchronize()
    for what, fn in calls:
        n0 = L.sgn_launch_count()
        rc = fn()
        assert rc == -1, f"{what}: rc {rc}"  # SGN_ERR_INVALID
        assert L.sgn_launch_count() == n0, f"{what}: launched"
    del keep
