"""Renders in the antialiased rasterize mode (RenderSettings.rasterize_mode / SceneGraphConfig.rasterize_mode).

  * full-size parity at BASELINE.json configs 2 and 3 against the C oracle in the same mode (oracle/oracle_aa.py),
    with the bars of tests/test_gpu_fullsize_parity.py: at most 0.5 % fragile pixels, 1e-4 on the others (rgb, accumulation,
    class streams), and relative L2 1e-3 per gradient tensor with the cotangents masked to the non-fragile pixels and unmasked;
  * the property the mode exists for: one small Gaussian rendered at 0.5x, 1x and 2x the resolution keeps its integrated
    accumulation (sum over the pixels / pixel area) within a few percent, where classic mode drifts by a large factor.  The
    tolerance is the float64 statement's own spread over the three scales (pixel-centre sums of o comp exp(-sigma), alpha
    clamped at 0.999 and truncated below 1/255) plus 1e-3; each render is within 1e-4 (relative) of that statement;
  * the model: an unknown mode raises ValueError; training steps with FusedAdam and a refinement stay finite, and repeat bit
    for bit under SGN_DETERMINISTIC=1; eval returns every output key of classic mode.
"""
import numpy as np
import pytest
import torch

import street_gaussians_ns_b200.synthetic as syn
from street_gaussians_ns_b200 import raster
from street_gaussians_ns_b200.model import SceneGraphConfig, SceneGraphRasterModel
from street_gaussians_ns_b200.optim import FusedAdam
from street_gaussians_ns_b200.refine import RefineSettings
from street_gaussians_ns_b200.training import TrainStep
from oracle import oracle_aa, oracle_c
from oracle import project_aa_ref64 as aa
from oracle import project_ref64 as ref
from tests import antialias_cases as ac
from tests import project_cases as pc
from tests.test_gpu_fullsize_parity import FRAGILE_MAX, GRAD_TOL, RGB_TOL, _oracle_grads
from tests.test_gpu_parity import rel_l2, to_cuda

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
AA = raster.RenderSettings(rasterize_mode="antialiased")


@pytest.fixture(scope="module", params=["cfg2", "cfg3"])
def full(request):
    import os
    oracle_c.lib().sgn_oracle_set_threads(max(1, len(os.sched_getaffinity(0))))
    fr = syn.config_frame(int(request.param[-1]))
    orc = oracle_aa.AntialiasedOracle(fr)
    return request.param, fr, orc, orc.forward()


def test_fullsize_forward(full):
    name, fr, orc, fw = full
    out, holder = raster.render_frame(to_cuda(fr), AA)
    torch.cuda.synchronize()
    rec = holder.records.cpu().numpy()
    np.testing.assert_array_equal(holder.radii.cpu().numpy(), fw.radii)
    vis = fw.radii > 0
    # float32 comp against the oracle's float64 one: a few eps32 kappa, relative (antialias_cases.comp_condition)
    r = np.zeros((len(vis), 12))
    r[:, 2:5], r[:, 11] = fw.conics, np.where(vis, orc.comp(), 0.0)
    o = fw.opac.astype(np.float64)
    assert np.all((np.abs(rec[:, 5] - o) <= 1e-6 + 8 * ac.EPS32 * ac.comp_condition(r) * o)[vis])
    assert 0 < holder.M <= fw.M
    alpha = 1 - fw.final_T
    rgb_ref, _, _ = oracle_c.post_ops(torch.from_numpy(fw.img), torch.from_numpy(alpha), None, True)
    ok = fw.fragile == 0
    err = np.abs(out["rgb"].cpu().numpy() - rgb_ref.numpy()).max(axis=2)
    acc_err = np.abs(out["accumulation"].cpu().numpy()[..., 0] - alpha)
    obj_err = np.abs(out["object_acc"].cpu().numpy()[..., 0] - (1 - fw.obj_T))
    bg_err = np.abs(out["background_acc"].cpu().numpy()[..., 0] - (1 - fw.bg_T))
    frag = 1 - ok.mean()
    print(f"[aa parity] {name}: fragile {frag:.4%}, rgb {err[ok].max():.2e}, acc {acc_err[ok].max():.2e}, M {holder.M} "
          f"(oracle AABB {fw.M})")
    assert frag <= FRAGILE_MAX and (fw.fragile_obj != 0).mean() <= FRAGILE_MAX and (fw.fragile_bg != 0).mean() <= FRAGILE_MAX
    assert err[ok].max() <= RGB_TOL and acc_err[ok].max() <= RGB_TOL
    assert obj_err[fw.fragile_obj == 0].max() <= RGB_TOL and bg_err[fw.fragile_bg == 0].max() <= RGB_TOL


@pytest.mark.parametrize("masked", [True, False])
def test_fullsize_gradients(full, masked):
    name, fr, orc, fw = full
    frc = to_cuda(fr, requires_grad=True)
    out, holder = raster.render_frame(frc, AA)
    H, W = fr.camera.height, fr.camera.width
    g = torch.Generator().manual_seed(7)
    ok = ((fw.fragile == 0) & (fw.fragile_obj == 0) & (fw.fragile_bg == 0)).astype(np.float32)
    okt = torch.from_numpy(ok) if masked else torch.ones(H, W)
    w_rgb = torch.rand(H, W, 3, generator=g) * okt[..., None]
    w_a = torch.rand(H, W, generator=g) * okt
    w_d = 0.05 * torch.rand(H, W, generator=g) * okt
    w_o = torch.rand(H, W, generator=g) * okt
    w_b = torch.rand(H, W, generator=g) * okt
    loss = ((out["rgb"] * w_rgb.cuda()).sum() + (out["accumulation"][..., 0] * w_a.cuda()).sum()
            + (out["depth"][..., 0] * w_d.cuda()).sum() + (out["object_acc"][..., 0] * w_o.cuda()).sum()
            + (out["background_acc"][..., 0] * w_b.cuda()).sum())
    loss.backward()
    torch.cuda.synchronize()
    grads, _ = _oracle_grads(orc, fw, w_rgb, w_a, w_d, w_o, w_b)
    worst = 0.0
    for si, (seg, gref) in enumerate(zip(frc.segments, grads)):
        for k in ("means", "scales", "quats", "features_dc", "features_rest", "opacities"):
            got = getattr(seg.params, k).grad
            if np.linalg.norm(gref[k]) == 0:
                assert float(got.abs().max()) == 0.0, (si, k)
                continue
            e = rel_l2(got.cpu().numpy(), gref[k])
            worst = max(worst, e)
            assert e <= GRAD_TOL, (name, masked, si, k, e)
    print(f"[aa grads] {name} masked={masked}: worst relative L2 {worst:.2e}")


# ---- the integrated density across resolutions ---------------------------------------------------------------------------
def _one_gaussian(k, sigma_px=0.6, logit=5.0):
    """A W x H camera scaled by k, and one isotropic Gaussian of sigma_px pixels (at k = 1) near the centre."""
    b = pc.Builder(int(64 * k), int(48 * k), 60.0 * k, 60.0 * k, 32.0 * k, 24.0 * k, 0, ref.Settings(sh_degree=0))
    z = 5.0
    w = pc.Builder(64, 48, 60.0, 60.0, 32.0, 24.0, 0, ref.Settings(sh_degree=0)).world(32.3, 24.2, z)
    s = b.segment(0)
    b.add(s, 0, 0, z, sigma_px * z / 60.0, quat=(1.0, 0.0, 0.0, 0.0), logit=logit, dc=0.0)
    b.segs[s]["rows"][0]["means"] = w
    return b.frame()


def _density64(fr, antialiased):
    """float64: sum over pixel centres of min(0.999, o exp(-sigma)) where >= 1/255, divided by the pixel area (1 / k^2)."""
    fw = (aa if antialiased else ref).forward(fr, ref.Settings(sh_degree=0))
    r = fw["records"][0]
    cam = fr.camera
    ys, xs = np.mgrid[0:cam.height, 0:cam.width] + 0.5
    dx, dy = xs - r[0], ys - r[1]
    sigma = 0.5 * (r[2] * dx * dx + r[4] * dy * dy) + r[3] * dx * dy
    alpha = np.minimum(0.999, r[5] * np.exp(-sigma))
    alpha = np.where((sigma >= 0) & (alpha >= 1 / 255), alpha, 0.0)
    return alpha.sum() * (64.0 / cam.width) ** 2


def test_integrated_density_keeps_across_resolutions():
    res = {}
    for mode in ("classic", "antialiased"):
        got, want = [], []
        for k in (0.5, 1.0, 2.0):
            fr = _one_gaussian(k)
            out, _ = raster.render_frame(to_cuda(fr), raster.RenderSettings(sh_degree=0, rasterize_mode=mode))
            got.append(float(out["accumulation"].double().sum()) * (64.0 / fr.camera.width) ** 2)
            want.append(_density64(fr, mode == "antialiased"))
        got, want = np.array(got), np.array(want)
        assert np.all(np.abs(got - want) <= 1e-4 * want), (mode, got, want)
        res[mode] = (got, want)
    got, want = res["antialiased"]
    tol = (want.max() - want.min()) / want.mean() + 1e-3
    spread = (got.max() - got.min()) / got.mean()
    print(f"[density] antialiased {got} spread {spread:.4f} (tol {tol:.4f}); classic {res['classic'][0]}")
    assert tol <= 0.05 and spread <= tol
    cl = res["classic"][0]
    assert cl.max() / cl.min() > 3.0  # classic: the blur's 0.3 px^2 inflates the sub-pixel renders


# ---- the model -----------------------------------------------------------------------------------------------------
W, H = 320, 240


def _model(mode, refine=False):
    fr = syn.make_frame(n_background=20000, n_actors=2, n_per_actor=1500, width=W, height=H, seed=3, frame=21,
                        actor_shift=np.array([2.0, 0.0, -3.0]))
    bg = fr.segments[0].params.to(DEV)
    actors = {s.name.replace("object_", ""): s.params.to(DEV) for s in fr.segments[1:]}
    cfg = SceneGraphConfig(use_sky_sphere=False, rasterize_mode=mode)
    if refine:
        cfg.refine = RefineSettings(cull_alpha_thresh=0.02, warmup_length=0, refine_every=2)
        cfg.object_refine = RefineSettings(cull_alpha_thresh=0.005, warmup_length=0, refine_every=2)
    from street_gaussians_ns_b200.model import ActorPose
    poses = [ActorPose(s.name.replace("object_", ""), s.rot, s.center, 21, list(range(85))) for s in fr.segments[1:]]
    m = SceneGraphRasterModel(bg, actors, cfg, poses_at=lambda t: poses).to(DEV)
    m.train()
    return fr, m


def _gt(seed=2):
    return (torch.rand(H, W, 3, generator=torch.Generator().manual_seed(seed)) * 0.5 + 0.25).to(DEV)


def test_unknown_mode_raises():
    with pytest.raises(ValueError):
        _model("mip")
    with pytest.raises(ValueError):
        raster.camera_struct(syn.make_camera(64, 48), raster.RenderSettings(rasterize_mode="Antialiased"))


def _train(steps=4):
    torch.manual_seed(0)
    fr, m = _model("antialiased", refine=True)
    n0 = sum(sub.num_points for sub in m.all_models.values())
    opt = FusedAdam(m.optimizer_params())
    step_fn = TrainStep(m, opt, refine_every=2)
    for step in range(1, steps + 1):
        losses = step_fn(step, fr.camera, {"image": _gt()})
        assert all(np.isfinite(float(v)) for v in losses.values())
    torch.cuda.synchronize()
    state = {f"{n}.{k}": p.detach().clone() for n, sub in m.all_models.items() for k, p in sub.gauss_params.items()}
    return state, n0, sum(sub.num_points for sub in m.all_models.values())


def test_training_with_fused_adam_and_refinement_repeats_bit_for_bit(monkeypatch):
    monkeypatch.setenv("SGN_DETERMINISTIC", "1")
    monkeypatch.setattr(raster, "DETERMINISTIC", True)
    (a, n0, n1), (b, _, _) = _train(), _train()
    assert n1 != n0  # the refinement changed the rows
    assert all(torch.isfinite(t).all() for t in a.values())
    assert a.keys() == b.keys() and not [k for k in a if not torch.equal(a[k], b[k])]


def test_eval_outputs():
    outs = {}
    for mode in ("classic", "antialiased"):
        fr, m = _model(mode)
        m.eval()
        with torch.no_grad():
            outs[mode] = m.get_outputs(fr.camera)
        assert all(torch.isfinite(v).all() for v in outs[mode].values() if torch.is_tensor(v))
    aa, classic = outs["antialiased"], outs["classic"]
    assert set(aa) == set(classic)
    assert aa["background_rgb"].shape == (H, W, 3) and aa["object_rgb"].shape == (H, W, 3)
    assert float((aa["accumulation"] - classic["accumulation"]).abs().max()) > 0
