"""The frame's two entry points run one pipeline: ``forward_backward`` (no autograd graph) and ``render_frame`` + autograd's
backward give the same bits, in deterministic mode, for every output, v_records, the gradient arena, the sky's gradient and
the absolute screen-space gradient; they record the same StageTimer stages, in the same order and as often, and launch as
many kernels.  Classic and antialiased, absgrad off and on, no parameter term, the scale regularisation and MCMC's
regularisers, and the backward of a term alone (no image cotangent: the blend and projection backward are skipped)."""
import pytest
import torch

import street_gaussians_ns_b200.synthetic as syn
from street_gaussians_ns_b200 import _lib, raster
from tests.test_gpu_parity import SCENES, to_cuda

pytestmark = pytest.mark.gpu

IMAGES = ("rgb", "accumulation", "depth", "object_acc", "background_acc")


def _terms(kind):
    """(scale_reg, terms) for render_frame / forward_backward."""
    return {"none": (None, ()), "scale_reg": (10.0, ()), "mcmc": (None, (raster.MCMCRegTerm(0.01, 0.02),))}[kind]


@pytest.fixture(scope="module")
def frame():
    return syn.make_frame(**SCENES["small_actors"])


def _cotangents(frame, kind, absgrad, images=True):
    H, W = frame.camera.height, frame.camera.width
    w, v = syn.cotangents(H, W)
    w, v = w.cuda(), v.cuda()[..., None]
    cots = {}
    if images:
        cots = {"rgb": w, "accumulation": v, "depth": 0.05 * v, "object_acc": 0.1 * v}
        if not absgrad:  # absgrad refuses a background_acc cotangent
            cots["background_acc"] = 0.1 * v
    names = {"none": (), "scale_reg": ("scale_reg",), "mcmc": ("mcmc_opacity_reg", "mcmc_scale_reg")}[kind]
    for i, n in enumerate(names):
        cots[n] = torch.tensor(0.5 + 0.25 * i, device="cuda")
    return cots


def _run(autograd, frame, settings, cots, kind, monkeypatch):
    frc = to_cuda(frame, requires_grad=True)
    H, W = frame.camera.height, frame.camera.width
    sky = torch.rand(H, W, 3, generator=torch.Generator().manual_seed(11)).cuda().requires_grad_(True)
    scale_reg, terms = _terms(kind)
    L = _lib.load()
    timer = raster.StageTimer()
    monkeypatch.setattr(raster, "TIMER", timer)
    torch.cuda.synchronize()
    n0 = L.sgn_launch_count()
    if autograd:
        out, h = raster.render_frame(frc, settings, sky=sky, scale_reg=scale_reg, terms=terms)
        torch.autograd.backward([out[k] for k in cots], [cots[k] for k in cots])
        v_sky = sky.grad
    else:
        out, h = raster.forward_backward(frc, settings, cots, sky=sky.detach(), want_param_grads=True, scale_reg=scale_reg,
                                         terms=terms)
        v_sky = h.v_sky
    launches = L.sgn_launch_count() - n0
    torch.cuda.synchronize()
    arena = torch.cat([g.reshape(-1) for g in raster.arena_views(h.grad_arena, h.table.static)])
    return dict(out={k: t.detach() for k, t in out.items() if k != "sky"}, v_records=h.v_records, arena=arena, v_sky=v_sky,
                v_absxy=h.v_absxy, stages=[(k, len(e)) for k, e in timer.events.items()], launches=launches)


def _same(a, b):
    return (a is None and b is None) or (a is not None and b is not None and torch.equal(a, b))


def _check(frame, settings, cots, kind, monkeypatch):
    fb = _run(False, frame, settings, cots, kind, monkeypatch)
    ag = _run(True, frame, settings, cots, kind, monkeypatch)
    assert set(fb["out"]) == set(ag["out"]) and set(IMAGES) <= set(fb["out"])
    for k in fb["out"]:
        assert torch.equal(fb["out"][k], ag["out"][k]), k
    for k in ("v_records", "arena", "v_sky", "v_absxy"):
        assert _same(fb[k], ag[k]), k
    assert (fb["v_absxy"] is not None) == settings.absgrad
    assert fb["stages"] == ag["stages"]
    assert fb["launches"] == ag["launches"] > 0
    return fb


@pytest.mark.parametrize("kind", ["none", "scale_reg", "mcmc"])
@pytest.mark.parametrize("absgrad", [False, True], ids=["plain", "absgrad"])
@pytest.mark.parametrize("mode", raster.RASTERIZE_MODES)
def test_both_entry_points_agree(frame, mode, absgrad, kind, monkeypatch):
    settings = raster.RenderSettings(deterministic=True, rasterize_mode=mode, absgrad=absgrad)
    fb = _check(frame, settings, _cotangents(frame, kind, absgrad), kind, monkeypatch)
    assert fb["v_sky"] is not None and fb["arena"].any()


@pytest.mark.parametrize("kind", ["scale_reg", "mcmc"])
def test_both_entry_points_agree_on_a_params_only_backward(frame, kind, monkeypatch):
    settings = raster.RenderSettings(deterministic=True)
    fb = _check(frame, settings, _cotangents(frame, kind, False, images=False), kind, monkeypatch)
    stages = {k for k, _ in fb["stages"]}
    assert "blend_bwd:start" not in stages and "project_bwd:start" not in stages
    assert fb["v_sky"] is None and not fb["v_records"].any() and fb["arena"].any()


def test_forward_backward_refuses_a_mismatched_sh_degree(frame):
    frc = to_cuda(frame)
    assert frc.segments[0].params.features_rest.shape[1] == 15  # sh_degree 3
    with pytest.raises(_lib.SgnError):
        raster.forward_backward(frc, raster.RenderSettings(sh_degree=2, deterministic=True), {})
