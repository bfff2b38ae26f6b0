"""Densification by MCMC (csrc/mcmc.cu, mcmc.py, the model and TrainStep) on the GPU, against the float64 statement
(oracle/mcmc_ref64.py).

Bars: the update rule's stored logit and log-scale within 2 float32 ulps of the float64 statement, plus 1e-7 absolute near 0,
plus how far they move when the float32 opacity moves by one ulp (the device's expf and the host's exp may disagree by one);
sampler draws equal to the statement's, neighbours accepted only where u * total lies within 1e-12 (relative) of a prefix-sum
boundary; the noise within 1e-5 of each row's largest displacement plus 2 ulps of the means; the regularisers within 1e-6
relative, their gradients within 1e-5 relative."""
import numpy as np
import pytest
import torch
from scipy import stats

import street_gaussians_ns_b200.synthetic as syn
from oracle import mcmc_ref64 as R
from street_gaussians_ns_b200 import _lib, mcmc, raster
from street_gaussians_ns_b200.mcmc import MCMCSettings
from street_gaussians_ns_b200.model import ActorPose, SceneGraphConfig, SceneGraphRasterModel
from street_gaussians_ns_b200.optim import FusedAdam
from street_gaussians_ns_b200.scene import PARAM_NAMES, GaussianSet
from street_gaussians_ns_b200.training import TrainStep, warm_up_refinement

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
MIN_O = 0.005


def _ulp32(x):
    return np.spacing(np.abs(np.asarray(x, np.float32))).astype(np.float64)


def _logit32(o):
    o = np.float64(o)
    return np.float32(np.log(o / (1 - o)))


# ---- update rule -----------------------------------------------------------------------------------------------
def _one_ulp_of_o(logit, log_scale, count):
    """How far the stored values move when the float32 opacity moves by one ulp: the kernel's expf and the host's exp may give
    sigmoids one ulp apart, and near o = 1 the logit amplifies that."""
    o = R.sigmoid32(np.float32(logit))
    s = np.exp(np.asarray(log_scale, np.float32))
    lo, ls = R.relocation_params_o(o, s, count, MIN_O)
    d_o, d_s = 0.0, np.zeros(3)
    for oo in (np.nextafter(o, np.float32(0)), np.nextafter(o, np.float32(1))):
        if oo > 1:
            continue
        a, b = R.relocation_params_o(oo, s, count, MIN_O)
        d_o, d_s = max(d_o, abs(a - lo)), np.maximum(d_s, np.abs(b - ls))
    return d_o, d_s


def test_update_rule_against_float64():
    rng = np.random.default_rng(0)
    counts = list(range(1, 51)) + [51, 60, 200]  # every N = c + 1 up to 51, and clamped counts
    special = [_logit32(MIN_O), _logit32(MIN_O * 1.0001), np.float32(16.0), np.float32(40.0), _logit32(0.999), np.float32(0.0)]
    logits, cs = [], []
    for c in counts:
        for lg in special + list(rng.normal(0, 3, 4).astype(np.float32)):
            logits.append(lg)
            cs.append(c)
    n = len(logits)
    logits = np.array(logits, np.float32).reshape(n, 1)
    cs = np.array(cs, np.int32)
    cs[::7] = 0  # not drawn: untouched
    scales = rng.normal(-3, 1, (n, 3)).astype(np.float32)
    op, sc = torch.from_numpy(logits).to(DEV), torch.from_numpy(scales).to(DEV)
    m = torch.randn(n, 3, device=DEV) + 1
    v = torch.rand(n, 3, device=DEV) + 1
    m0, v0 = m.clone(), v.clone()
    mcmc.update_rows(op, sc, torch.from_numpy(cs).to(DEV), MIN_O, [m, v])
    got_o, got_s = op.cpu().numpy(), sc.cpu().numpy()
    for i in range(n):
        if cs[i] == 0:
            assert got_o[i, 0] == logits[i, 0] and np.array_equal(got_s[i], scales[i])
            assert torch.equal(m[i], m0[i]) and torch.equal(v[i], v0[i])
            continue
        lo, ls = R.relocation_params(logits[i, 0], scales[i], cs[i], MIN_O)
        dlo, dls = _one_ulp_of_o(logits[i, 0], scales[i], cs[i])
        assert abs(got_o[i, 0] - lo) <= 2 * _ulp32(lo) + 1e-7 + dlo, (i, cs[i], logits[i, 0], got_o[i, 0], lo)
        assert (np.abs(got_s[i] - ls) <= 2 * _ulp32(ls) + 1e-7 + dls).all(), (i, cs[i], got_s[i], ls)
        assert not m[i].any() and not v[i].any()
    # the clamps: every stored opacity is within [min_opacity, 1 - 2^-23] up to the logit's rounding
    o = R.sigmoid32(got_o[cs > 0])
    assert o.min() >= np.float32(MIN_O) * (1 - 1e-6) and o.max() < 1.0


# ---- sampler ---------------------------------------------------------------------------------------------------
def _device_sigmoid(lg):
    """1 / (1 + exp(-logit)) in float32 as the device evaluates it, same shape: the host's exp may differ by an ulp, which would
    move the weights and their sum by more than the 1e-12 the draws are held to, and which the logit of an opacity near 1
    amplifies in the update rule."""
    a = np.asarray(lg, np.float32)
    t = torch.from_numpy(np.ascontiguousarray(a.reshape(-1))).to(DEV)
    return (1.0 / (1.0 + torch.exp(-t))).cpu().numpy().reshape(a.shape)


def _device_o(lg):
    return _device_sigmoid(lg).astype(np.float64).ravel()


def _logits_with_dead(n, frac_dead, seed):
    g = np.random.default_rng(seed)
    lg = g.normal(0, 2.5, (n, 1)).astype(np.float32)
    dead = g.random(n) < frac_dead
    lg[dead, 0] = g.uniform(-12, float(_logit32(MIN_O)), int(dead.sum())).astype(np.float32)
    return lg


@pytest.mark.parametrize("n", [1, 37, 4096, 4097, 100_003])
def test_sampler_explicit_uniforms(n):
    lg = _logits_with_dead(n, 0.2, n)
    o = _device_o(lg)
    dead = o <= np.float32(MIN_O)
    w = np.where(dead, 0.0, o)
    if not w.any():
        lg[0, 0] = 2.0
        o = _device_o(lg)
        dead = o <= np.float32(MIN_O)
        w = np.where(dead, 0.0, o)
    g = np.random.default_rng(1)
    p = np.cumsum(w)
    u = np.concatenate([g.random(3000), p[g.integers(0, n, 200)] / p[-1], [0.0, np.nextafter(1.0, 0.0)]])
    u = np.minimum(u, np.nextafter(1.0, 0.0))
    ut = torch.from_numpy(u).to(DEV)
    r = mcmc.sample(torch.from_numpy(lg).to(DEV), MIN_O, True, len(u), 0, 0, 0, _lib.MCMC_RELOCATE, uniforms=ut, want_dead=True)
    draws = r["draws"].cpu().numpy()
    want = R.draws_from_uniforms(w, u)
    ok = R.acceptable_draws(w, u)
    for j in range(len(u)):
        assert draws[j] == want[j] or draws[j] in ok[j], (j, u[j], draws[j], want[j], ok[j])
    assert not dead[draws].any()
    assert np.array_equal(r["counts"].cpu().numpy(), np.bincount(draws, minlength=n))
    assert np.array_equal(r["dead_rows"].cpu().numpy()[:int(r["num_dead"])], np.nonzero(dead)[0])
    assert abs(float(r["total"]) - p[-1]) <= 1e-12 * p[-1]


def test_sampler_chi_square_and_determinism():
    n = 64
    lg = _logits_with_dead(n, 0.25, 3)
    o = _device_o(lg)
    w = np.where(o <= np.float32(MIN_O), 0.0, o)
    D = 1_000_000
    t = torch.from_numpy(lg).to(DEV)
    a = mcmc.sample(t, MIN_O, True, D, seed=11, step=600, sub=2, purpose=_lib.MCMC_ADD)
    counts = a["counts"].cpu().numpy()
    assert counts[w == 0].sum() == 0
    pos = w > 0
    chi = stats.chisquare(counts[pos], D * w[pos] / w.sum())
    assert chi.pvalue > 1e-4, chi
    b = mcmc.sample(t, MIN_O, True, D, seed=11, step=600, sub=2, purpose=_lib.MCMC_ADD)
    assert torch.equal(a["draws"], b["draws"]) and torch.equal(a["counts"], b["counts"])
    for kw in (dict(seed=11, step=700, sub=2), dict(seed=11, step=600, sub=3), dict(seed=12, step=600, sub=2)):
        c = mcmc.sample(t, MIN_O, True, D, purpose=_lib.MCMC_ADD, **kw)
        assert (c["draws"] != a["draws"]).float().mean() > 0.5, kw
    c = mcmc.sample(t, MIN_O, True, D, seed=11, step=600, sub=2, purpose=_lib.MCMC_RELOCATE)
    assert (c["draws"] != a["draws"]).float().mean() > 0.5


def test_sampler_without_live_rows_draws_nothing():
    lg = torch.full((100, 1), -9.0, device=DEV)
    r = mcmc.sample(lg, MIN_O, True, 100, 0, 0, 0, _lib.MCMC_RELOCATE, want_dead=True, draw_dead=True)
    assert int(r["num_dead"]) == 100 and (r["draws"] == -1).all() and not r["counts"].any()


# ---- noise -----------------------------------------------------------------------------------------------------
def _random_sub(n, seed, F=1):
    g = torch.Generator(device=DEV).manual_seed(seed)
    r = lambda *s: torch.randn(s, device=DEV, generator=g)  # noqa: E731
    op = r(n, 1) * 3
    op[: n // 10] = -7.0  # faint rows: the gate is open
    return GaussianSet(r(n, 3) * 20, r(n, 3) * 0.5 - 3, r(n, 4) * 2.5, r(n, F, 3), r(n, 15, 3), op)


def test_noise_explicit_normals_config4():
    subs = [_random_sub(2_000_000, 0)] + [_random_sub(10_000, 1 + a, 5) for a in range(32)]
    lr = 1.6e-4
    tab = mcmc.NoiseTable()
    entries = [(s.means, s.scales, s.quats, s.opacities, 5e5 if k == 0 else 2e5) for k, s in enumerate(subs)]
    rows = sum(s.means.shape[0] for s in subs)
    normals = torch.randn(rows, 3, device=DEV, generator=torch.Generator(device=DEV).manual_seed(9))
    before = [s.means.clone() for s in subs]
    mcmc.inject_noise(tab, entries, lr, seed=0, step=1, normals=normals)
    torch.cuda.synchronize()
    row0 = 0
    g = np.random.default_rng(0)
    for k, s in enumerate(subs):
        n = s.means.shape[0]
        idx = np.sort(g.choice(n, min(n, 200_000), replace=False))
        it = torch.from_numpy(idx).to(DEV)
        want = R.noise_delta(s.scales[it].cpu().numpy(), s.quats[it].cpu().numpy(), s.opacities[it].cpu().numpy(),
                             normals[row0:row0 + n][it].cpu().numpy(), float(np.float32(lr) * np.float32(entries[k][4])))
        got = s.means[it].cpu().numpy().astype(np.float64)
        old = before[k][it].cpu().numpy().astype(np.float64)
        err = np.abs(got - (old + want))
        bound = 1e-5 * np.abs(want).max(1, keepdims=True) + 2 * _ulp32(got)
        assert (err <= bound).all(), (k, float((err - bound).max()))
        row0 += n
    assert float((subs[0].means - before[0]).abs().max()) > 0


def test_noise_philox_is_deterministic():
    a, b = _random_sub(50_000, 3), _random_sub(50_000, 3)
    ta, tb = mcmc.NoiseTable(), mcmc.NoiseTable()
    mcmc.inject_noise(ta, [(a.means, a.scales, a.quats, a.opacities, 5e5)], 1.6e-4, seed=5, step=10)
    mcmc.inject_noise(tb, [(b.means, b.scales, b.quats, b.opacities, 5e5)], 1.6e-4, seed=5, step=10)
    assert torch.equal(a.means, b.means)
    mcmc.inject_noise(tb, [(b.means, b.scales, b.quats, b.opacities, 5e5)], 1.6e-4, seed=5, step=11)
    assert not torch.equal(a.means, b.means)


# ---- a model -----------------------------------------------------------------------------------------------------
def _model(strategy="mcmc", semantic=0, filter_3d=False, n_bg=20_000, n_act=3_000, actors=2, **cfg):
    bg = _random_sub(n_bg, 100)
    acts = {str(a): _random_sub(n_act, 200 + a, 5) for a in range(actors)}
    config = SceneGraphConfig(strategy=strategy, use_sky_sphere=False, semantic_classes=semantic, filter_3d=filter_3d, **cfg)
    m = SceneGraphRasterModel(bg, acts, config).to(DEV)
    m.train()
    return m


def test_refinement_under_fused_adam():
    """One refinement at step 600 against the float64 statement, with the draws the sampler makes for the same keys."""
    m = _model(semantic=3, filter_3d=True, mcmc=MCMCSettings(cap_max=20_500), object_mcmc=MCMCSettings(cap_max=100_000),
               refine_record=True)
    subs = list(m.all_models.values())
    for i, sub in enumerate(subs):
        sub.semantic_logits.data.normal_()
        sub.filter_3d.uniform_(0, 0.01)
    opt = FusedAdam(m.optimizer_params(), rows={"semantic": (m.semantic_params(), 1e-3)})
    opt.exp_avg.normal_()
    opt.exp_avg_sq.uniform_(0.1, 1.0)
    opt.steps[:] = np.arange(len(opt.steps)) + 3
    steps0 = opt.steps.copy()
    before = []
    for i, sub in enumerate(subs):
        rows = {k: sub.gauss_params[k].detach().cpu().numpy().copy() for k in PARAM_NAMES}
        rows["semantic_logits"] = sub.semantic_logits.detach().cpu().numpy().copy()
        rows["filter_3d"] = sub.filter_3d.cpu().numpy().copy()
        mom = {k: tuple(x.cpu().numpy().copy() for x in opt.moment_views(6 * i + j)) for j, k in enumerate(PARAM_NAMES)}
        mom["semantic_logits"] = tuple(x.cpu().numpy().copy() for x in opt.row_moment_views("semantic", i))
        before.append((rows, mom, sub.gauss_params["opacities"].detach().clone()))
    step, seed = 600, 7
    m.step = step
    m.refinement_after(opt, step, due_only=True, seed=seed)
    torch.cuda.synchronize()
    assert np.array_equal(opt.steps, steps0)  # step counts are kept
    for i, sub in enumerate(subs):
        rows, mom, op0 = before[i]
        st = m.config.mcmc if i == 0 else m.config.object_mcmc
        n = rows["means"].shape[0]
        r1 = mcmc.sample(op0, MIN_O, True, n, seed, step, i, _lib.MCMC_RELOCATE, want_dead=True, draw_dead=True)
        nd = int(r1["num_dead"])
        assert nd == len(R.dead_rows(rows["opacities"], MIN_O, _device_sigmoid)) and nd > 0
        want, wmom = R.relocate(rows, mom, r1["draws"][:nd].cpu().numpy(), MIN_O, _device_sigmoid)
        A = min(st.cap_max, int(1.05 * n)) - n
        lg = torch.from_numpy(want["opacities"].astype(np.float32)).to(DEV)
        r2 = mcmc.sample(lg, MIN_O, False, A, seed, step, i, _lib.MCMC_ADD)
        want, wmom = R.add(want, wmom, r2["draws"].cpu().numpy(), MIN_O, _device_sigmoid)
        assert sub.num_points == n + A == want["means"].shape[0]
        assert sub.refine_record_dict == {"mcmc_relocated": nd, "mcmc_added": A}
        got = {k: sub.gauss_params[k].detach().cpu().numpy() for k in PARAM_NAMES}
        got["semantic_logits"] = sub.semantic_logits.detach().cpu().numpy()
        got["filter_3d"] = sub.filter_3d.cpu().numpy()
        for k, w in want.items():
            if k in ("opacities", "scales"):
                assert (np.abs(got[k] - w) <= 2 * _ulp32(w) + 1e-7).all(), (i, k)
            else:
                assert np.array_equal(got[k], w.astype(np.float32)), (i, k)
        gm = {k: tuple(x.cpu().numpy() for x in opt.moment_views(6 * i + j)) for j, k in enumerate(PARAM_NAMES)}
        gm["semantic_logits"] = tuple(x.cpu().numpy() for x in opt.row_moment_views("semantic", i))
        for k, (wm, wv) in wmom.items():
            assert np.array_equal(gm[k][0], wm.astype(np.float32)) and np.array_equal(gm[k][1], wv.astype(np.float32)), (i, k)
        dead = R.dead_rows(rows["opacities"], MIN_O, _device_sigmoid)
        src = r1["draws"][:nd].cpu().numpy()
        for k in got:  # the relocated rows are bit copies of their sources (whose opacity and scales the add phase may change again)
            if k not in ("opacities", "scales"):
                assert np.array_equal(got[k][dead], got[k][src]), (i, k)
        assert np.array_equal(got["means"][n:], got["means"][r2["draws"].cpu().numpy()])
        # right after the refinement no row is dead, up to the clamp at min_opacity
        o = torch.sigmoid(sub.gauss_params["opacities"].detach())
        assert float(o.min()) >= MIN_O * (1 - 1e-6)
    assert subs[0].num_points == 20_500  # the background reached its cap


# ---- regularisers ---------------------------------------------------------------------------------------------------
def test_regularisers_through_the_render():
    m = _model()
    cam = syn.make_camera(320, 240)
    m.step = 0
    frame = m._frame(cam)
    term = raster.MCMCRegTerm(0.01, 0.02)
    out, h = raster.render_frame(frame, m._settings(class_streams=True), terms=(term,), scale_reg=10.0)
    ops = np.concatenate([seg.params.opacities.detach().cpu().numpy() for seg in frame.segments])
    scs = np.concatenate([seg.params.scales.detach().cpu().numpy() for seg in frame.segments])
    ro, rs = R.regularisers(ops, scs, 0.01, 0.02)
    assert abs(out["mcmc_opacity_reg"].item() - ro) <= 1e-6 * ro and abs(out["mcmc_scale_reg"].item() - rs) <= 1e-6 * rs
    alone, _ = raster.render_frame(frame, m._settings(class_streams=True), scale_reg=10.0)
    assert torch.equal(alone["scale_reg"], out["scale_reg"])  # the scale regularisation is the same bits beside another term
    # a backward of the two terms alone: the arena holds their gradients and nothing else
    (out["mcmc_opacity_reg"] * 2.0 + out["mcmc_scale_reg"] * 3.0).backward()
    go, gs = R.regulariser_grads(ops, scs, 0.01, 0.02, _device_sigmoid)
    got_o = torch.cat([seg.params.opacities.grad for seg in frame.segments]).cpu().numpy()
    got_s = torch.cat([seg.params.scales.grad for seg in frame.segments]).cpu().numpy()
    assert np.allclose(got_o, 2.0 * go, rtol=1e-5, atol=0) and np.allclose(got_s, 3.0 * gs, rtol=1e-5, atol=0)
    assert not torch.cat([seg.params.means.grad for seg in frame.segments]).any()
    assert h.params_only and h.term_kinds == [1, 5]


def test_fused_regularisers_match_torch_path():
    vals = {}
    for fused in (True, False):
        m = _model(fused_loss=fused, ssim_lambda=0.0)
        cam = syn.make_camera(320, 240)
        gt = torch.rand(240, 320, 3, device=DEV)
        m.step = 3
        out = m.get_outputs(cam)
        losses = m.get_loss_dict(out, {"image": gt})
        vals[fused] = (losses["mcmc_opacity_reg"].item(), losses["mcmc_scale_reg"].item())
    for a, b in zip(vals[True], vals[False]):
        assert abs(a - b) <= 1e-6 * abs(b)


# ---- training ---------------------------------------------------------------------------------------------------------
def _scene_model(seed_cap):
    sc = syn.WaymoScene(scale=0.02, num_frames=20, n_actors=4)
    frame_list = list(range(sc.num_frames))

    def poses_at(t):
        f = int(t)
        return [ActorPose(str(a), rot, center, f, frame_list, frame_id=f) for a, rot, center in sc.boxes_at(f)]
    sched = dict(refine_start=5, refine_stop=200, refine_every=10)
    cfg = SceneGraphConfig(use_sky_sphere=False, ssim_lambda=0.0, strategy="mcmc", mcmc=MCMCSettings(cap_max=seed_cap, **sched),
                           object_mcmc=MCMCSettings(cap_max=260, **sched), refine_record=True)
    bg = sc.background
    bg = GaussianSet(bg.means, bg.scales, bg.quats, bg.features_dc, bg.features_rest, bg.opacities - 3.0)  # some rows start dead
    model = SceneGraphRasterModel(bg.to(DEV), {k: v.to(DEV) for k, v in sc.actors.items()}, cfg, poses_at=poses_at).to(DEV)
    model.train()
    return sc, model


def _train(steps, seed=0):
    sc, model = _scene_model(36_000)
    opt = FusedAdam(model.optimizer_params())
    fn = TrainStep(model, opt, refine_seed=seed)
    g = torch.Generator().manual_seed(5)
    gt = (torch.rand(sc.height, sc.width, 3, generator=g) * 255).to(torch.uint8).to(DEV)
    history = []
    for step in range(1, steps + 1):
        n_before = [s.num_points for s in model.all_models.values()]
        losses = fn(step, sc.cameras[step % len(sc.cameras)], {"image": gt})
        assert all(torch.isfinite(v).all() for v in losses.values()), step
        if mcmc.due(model.config.mcmc, step):
            history.append((step, n_before, [s.num_points for s in model.all_models.values()],
                            [torch.sigmoid(s.gauss_params["opacities"].detach()).min().item() if s.num_points else 1.0
                             for s in model.all_models.values()]))
    torch.cuda.synchronize()
    return model, history


def test_short_training_run(monkeypatch):
    monkeypatch.setattr(raster, "DETERMINISTIC", True)
    model, history = _train(60)
    assert len(history) == 6  # steps 10 .. 60
    for step, before, after, omin in history:
        for name, b, a, o in zip(model.all_models._modules, before, after, omin):
            cap = (model.config.mcmc if name == "background" else model.config.object_mcmc).cap_max
            assert a == max(b, min(cap, int(1.05 * b))), (step, name, b, a)
            assert o >= MIN_O * (1 - 1e-6), (step, name, o)
    assert history[-1][2][0] > history[0][1][0]
    for sub in model.all_models.values():
        for k in PARAM_NAMES:
            assert torch.isfinite(sub.gauss_params[k]).all()
    other, _ = _train(60)
    for a, b in zip(model.all_models.values(), other.all_models.values()):
        for k in PARAM_NAMES:
            assert torch.equal(a.gauss_params[k], b.gauss_params[k]), k


def test_default_strategy_is_untouched_and_warm_up():
    m = _model(strategy="default")
    assert "mcmc_opacity_reg" not in m.get_loss_dict(m.get_outputs(syn.make_camera(160, 120)), {"image": torch.zeros(120, 160, 3, device=DEV)})
    m = _model()
    rec = warm_up_refinement(m)
    assert rec["rows_after"][0] == int(1.05 * rec["rows_before"][0])
    with pytest.raises(ValueError):
        _model(strategy="bogus")
