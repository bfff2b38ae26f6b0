"""Per-Gaussian semantic logits on the GPU (csrc/semantic.cu through semantic.py, and the model surface built on it) against
the float64 statement (tests/semantic_cases.py), torch autograd of F.cross_entropy, and sgn_refine_apply.

Bars: the loss within 1e-6 relative of float64 and its cotangent within fp32 rounding, the same bits on every run; the
confusion matrix equal to float64's; the carry bit-identical to sgn_refine_apply's features_dc rows and moments; the model's
gradients from the fused term within 1e-5 relative L2 of the torch expression's; with the term off the losses and the gradient
arena bit-identical to a model without semantics; accumulated steps equal to torch.optim.Adam over the same gradients."""
import numpy as np
import pytest
import torch

import street_gaussians_ns_b200.synthetic as syn
from street_gaussians_ns_b200 import raster, refine
from street_gaussians_ns_b200.model import ActorPose, SceneGraphConfig, SceneGraphRasterModel, _FullArenaSink
from street_gaussians_ns_b200.optim import FusedAdam
from street_gaussians_ns_b200.scene import PARAM_NAMES
from street_gaussians_ns_b200.semantic import (fused_semantic_loss, refine_carry, semantic_confusion, semantic_loss_torch,
                                               semantic_metrics)
from tests import semantic_cases as ref

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def rel_l2(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / max(float(b.norm()), 1e-30))


def _loss_case(H, W, C, seed, ignore, masked):
    g = torch.Generator().manual_seed(seed)
    logits = torch.randn(H, W, C, generator=g) * 3.0
    labels = torch.randint(0, C, (H, W, 1), generator=g)
    if ignore:
        labels[torch.rand(H, W, 1, generator=g) < 0.1] = 255
    mask = (torch.rand(H, W, 1, generator=g) > 0.25).float() if masked else None
    return logits.to(DEV), labels.to(DEV), None if mask is None else mask.to(DEV)


@pytest.mark.parametrize("C", [3, 19])
@pytest.mark.parametrize("ignore,masked", [(False, False), (True, False), (True, True)])
def test_loss_against_float64_and_autograd(C, ignore, masked):
    H, W = 1280, 1920
    logits, labels, mask = _loss_case(H, W, C, 7 + C, ignore, masked)
    x = logits.clone().requires_grad_(True)
    loss = fused_semantic_loss(x, labels, mask, 0.3)
    loss.backward()
    want, n = ref.loss_ref64(logits.cpu().numpy(), labels.cpu().numpy(), None if mask is None else mask.cpu().numpy(), 0.3)
    assert n > 1_000_000
    assert abs(float(loss.detach()) - want) <= 1e-6 * abs(want)
    v_ref = ref.grad_ref64(logits.cpu().numpy(), labels.cpu().numpy(), None if mask is None else mask.cpu().numpy(), 0.3)
    np.testing.assert_allclose(x.grad.cpu().numpy(), v_ref, rtol=1e-5, atol=1e-6 * 0.3 / n)
    y = logits.clone().requires_grad_(True)
    t = semantic_loss_torch(y, labels, mask, 0.3)
    t.backward()
    assert float(t.detach()) == pytest.approx(float(loss.detach()), rel=1e-5)  # torch sums the 2.4 M terms in fp32
    assert rel_l2(x.grad, y.grad) < 1e-5
    for _ in range(2):  # the same bits on every run
        z = logits.clone().requires_grad_(True)
        again = fused_semantic_loss(z, labels, mask, 0.3)
        again.backward()
        assert torch.equal(again, loss) and torch.equal(z.grad, x.grad)


def test_no_valid_pixel_and_label_dtypes():
    logits, labels, mask = _loss_case(64, 96, 3, 1, False, False)
    x = logits.clone().requires_grad_(True)
    loss = fused_semantic_loss(x, torch.full_like(labels, 255), None, 1.0)
    loss.backward()
    assert float(loss) == 0.0 and not x.grad.any()
    x.grad = None
    loss = fused_semantic_loss(x, labels, torch.zeros_like(mask if mask is not None else labels, dtype=torch.float32), 1.0)
    loss.backward()
    assert float(loss) == 0.0 and not x.grad.any()
    a = fused_semantic_loss(logits, labels[..., 0], None, 1.0)
    b = fused_semantic_loss(logits, labels.to(torch.uint8), None, 1.0)  # converted once in the wrapper
    assert torch.equal(a, b)
    from street_gaussians_ns_b200 import _lib
    with pytest.raises(ValueError):
        fused_semantic_loss(torch.zeros(4, 4, 65, device=DEV), torch.zeros(4, 4, dtype=torch.int64, device=DEV))
    with pytest.raises(_lib.SgnError):
        fused_semantic_loss(torch.zeros(4, 4, 3), torch.zeros(4, 4, dtype=torch.int64))


@pytest.mark.parametrize("C,masked", [(3, False), (19, True)])
def test_metrics_against_float64(C, masked):
    logits, labels, mask = _loss_case(1280, 1920, C, 3, True, masked)
    logits = torch.round(logits * 2) / 2  # many exact ties: the lowest class wins
    conf = semantic_confusion(logits, labels, mask).cpu().numpy()
    want = ref.confusion_ref64(logits.cpu().numpy(), labels.cpu().numpy(), None if mask is None else mask.cpu().numpy())
    assert np.array_equal(conf, want)
    got = semantic_metrics(logits, labels, mask)
    acc, miou = ref.metrics_ref64(want)
    assert got["semantic_acc"] == pytest.approx(acc, rel=1e-12) and got["semantic_miou"] == pytest.approx(miou, rel=1e-12)
    assert np.array_equal(semantic_confusion(logits, labels, mask).cpu().numpy(), conf)


@pytest.mark.parametrize("step,F", [(700, 1), (3400, 5), (25000, 1)])
def test_carry_is_bit_identical_to_refine_apply(step, F):
    g = torch.Generator(device=DEV).manual_seed(5)
    n = 50_000
    params = [torch.randn(n, 3, device=DEV, generator=g) * 5, torch.randn(n, 3, device=DEV, generator=g) * 1.5 - 4.0,
              torch.randn(n, 4, device=DEV, generator=g), torch.randn(n, F, 3, device=DEV, generator=g),
              torch.randn(n, 15, 3, device=DEV, generator=g), torch.randn(n, 1, device=DEV, generator=g) * 2.5 - 1.0]
    moments = [(torch.randn_like(p), torch.rand_like(p)) for p in params]
    vis = torch.randint(1, 9, (n,), device=DEV, generator=g).float()
    xgn = torch.rand(n, device=DEV, generator=g) * vis * 2.5e-6
    m2d = torch.rand(n, device=DEV, generator=g) * 0.2
    st = refine.RefineSettings(cull_alpha_thresh=0.02)
    densify, _, _ = refine.phase(st, step, 50)
    cfg = refine.make_config(st, step, (240, 320), densify)
    plan = refine.plan_submodel(params[1], params[5], xgn if densify else None, vis if densify else None,
                                m2d if cfg.use_screen_size else None, cfg, torch.Generator(device=DEV).manual_seed(1))
    assert plan.changed
    new = [torch.empty((plan.out_rows,) + tuple(p.shape[1:]), device=DEV) for p in params]
    new_m = [(torch.empty_like(a), torch.empty_like(a)) for a in new]
    refine.apply_plan(plan, params, new, moments, new_m)
    src = params[3].reshape(n, 3 * F)
    dst = torch.full((plan.out_rows, 3 * F), float("nan"), device=DEV)
    dm = (torch.full_like(dst, float("nan")), torch.full_like(dst, float("nan")))
    refine_carry(plan, src, dst, (moments[3][0].reshape(n, 3 * F), moments[3][1].reshape(n, 3 * F)), dm)
    assert torch.equal(dst, new[3].reshape(-1, 3 * F))
    assert torch.equal(dm[0], new_m[3][0].reshape(-1, 3 * F)) and torch.equal(dm[1], new_m[3][1].reshape(-1, 3 * F))
    logits = torch.randn(n, 3, device=DEV, generator=g)  # width 3 without moments against the float64 map
    out = torch.empty(plan.out_rows, 3, device=DEV)
    refine_carry(plan, logits, out)
    want, _ = ref.carry_ref(logits.cpu().numpy(), plan.flags.cpu().numpy(), cfg.n_split_samples)
    assert np.array_equal(out.cpu().numpy(), want)


# ---- model -----------------------------------------------------------------------------------------------------------

def _model(sky=False, classes=3, w=0.1, actors=True, seed=3, **cfg):
    fr = syn.make_frame(n_background=20000, n_actors=3 if actors else 0, n_per_actor=1500, width=320, height=240, seed=seed,
                        actor_shift=np.array([1.0, 0.0, -1.0]))
    env = None
    if sky:
        from street_gaussians_ns_b200.sky import CubeMapSky
        torch.manual_seed(0)
        env = CubeMapSky(16)
        with torch.no_grad():
            env.base.copy_(torch.rand(6, 16, 16, 3))
    poses = [ActorPose(s.name.replace("object_", ""), s.rot, s.center, 21, list(range(85))) for s in fr.segments[1:]]
    config = SceneGraphConfig(use_sky_sphere=sky, semantic_classes=classes, semantic_loss_mult=w, **cfg)
    model = SceneGraphRasterModel(fr.segments[0].params.to(DEV), {s.name.replace("object_", ""): s.params.to(DEV) for s in fr.segments[1:]},
                                  config, sky=env, poses_at=lambda t: poses).to(DEV)
    model.train()
    if classes:
        with torch.no_grad():
            for i, p in enumerate(model.semantic_params()):
                p.copy_(torch.randn(p.shape, generator=torch.Generator().manual_seed(40 + i)))
    gt = torch.rand(240, 320, 3, generator=torch.Generator().manual_seed(2)).to(DEV)
    labels = torch.randint(0, 3, (240, 320, 1), generator=torch.Generator().manual_seed(8))
    labels[torch.rand(240, 320, 1, generator=torch.Generator().manual_seed(9)) < 0.05] = 255
    return fr, model, gt, labels.to(DEV)


def _grads(model, loss, retain_graph=False):
    for p in model.parameters():
        p.grad = None
    loss.backward(retain_graph=retain_graph)
    torch.cuda.synchronize()
    sem = []
    if model.config.semantic_classes:  # a None gradient: nothing used the semantic map
        grads = [model.all_models[n].semantic_logits.grad for n in model.visible_model_names]
        sem = [None if g is None else g.clone() for g in grads]
    return model._holder.grad_arena.clone(), sem


@pytest.mark.parametrize("sky", [False, True])
@pytest.mark.parametrize("async_binning", [False, True])
def test_model_fused_term_matches_torch_expression(sky, async_binning):
    fr, model, gt, labels = _model(sky=sky)
    mask = (torch.rand(240, 320, 1, generator=torch.Generator().manual_seed(6)) > 0.2).float().to(DEV)
    batch = {"image": gt, "semantic": labels, "mask": mask}
    raster._ASYNC_STATE.clear()
    model.config.async_binning = async_binning
    try:
        for _ in range(2 if async_binning else 1):  # the first frame learns the count
            out = model.get_outputs(fr.camera)
        if async_binning:
            assert isinstance(model._holder.M, raster.LazyCount)
        assert out["semantic"].shape == (240, 320, 3) and len(model.visible_model_names) == 4
        losses = model.get_loss_dict(out, batch)
        assert "semantic_loss" in losses and float(losses["semantic_loss"]) > 0
        a_fused, s_fused = _grads(model, sum(losses.values()), retain_graph=True)
        model.config.semantic_loss_mult = 0.0
        losses2 = model.get_loss_dict(out, batch)
        assert "semantic_loss" not in losses2
        term = semantic_loss_torch(out["semantic"], labels, mask, 0.1)
        assert float(term) == pytest.approx(float(losses["semantic_loss"]), rel=2e-6)
        a_torch, s_torch = _grads(model, sum(losses2.values()) + term, retain_graph=True)
        assert rel_l2(a_fused, a_torch) < 1e-5
        assert float(s_torch[0].abs().max()) > 0
        for a, b in zip(s_fused, s_torch):  # an actor out of view has a zero gradient on both paths
            assert rel_l2(a, b) < 1e-5
        a_none, s_none = _grads(model, sum(losses2.values()))  # the term moves the geometry too
        assert all(g is None for g in s_none)
        assert rel_l2(a_none, a_torch) > 1e-4
    finally:
        raster._ASYNC_STATE.clear()
        model.config.async_binning = None


def test_off_path_is_bit_identical(monkeypatch):
    monkeypatch.setattr(raster, "DETERMINISTIC", True)
    res = []
    for cfg in ({"classes": 0, "w": 0.0}, {"classes": 0, "w": 0.5}, {"classes": 3, "w": 0.0}):
        fr, model, gt, labels = _model(**cfg)
        out = model.get_outputs(fr.camera)
        assert ("semantic" in out) == (cfg["classes"] > 0)
        losses = model.get_loss_dict(out, {"image": gt, "semantic": labels})
        assert "semantic_loss" not in losses
        arena, _ = _grads(model, sum(losses.values()))
        res.append(({k: v.detach().clone() for k, v in losses.items()}, arena, out["rgb"].detach().clone()))
    (l0, a0, r0) = res[0]
    for l1, a1, r1 in res[1:]:
        assert l0.keys() == l1.keys() and all(torch.equal(l0[k], l1[k]) for k in l0)
        assert torch.equal(a0, a1) and torch.equal(r0, r1)


def _step_model(accumulate, det=False):
    fr, model, gt, labels = _model(actors=False)
    opt = FusedAdam(model.optimizer_params(), rows={"semantic": (model.semantic_params(), 0.0025)})
    from street_gaussians_ns_b200.training import TrainStep
    step_fn = TrainStep(model, opt, refine_every=100000, gradient_accumulation_steps={"semantic": 10} if accumulate else None)
    return fr, model, gt, labels, opt, step_fn


def test_accumulated_steps_match_torch_adam():
    fr, model, gt, labels, opt, step_fn = _step_model(True)
    sem = model.semantic_params()[0]
    start = sem.detach().clone()
    seen = []
    real_step = opt.step

    def spy(*a, **k):
        if k.get("row_grads"):
            seen.append(k["row_grads"]["semantic"][0].clone())
        return real_step(*a, **k)
    opt.step = spy
    for s in range(10):
        step_fn(s, fr.camera, {"image": gt, "semantic": labels})
        torch.cuda.synchronize()
        moved = not torch.equal(sem.detach(), start)
        assert moved == (s == 9), s
    assert len(seen) == 1
    p = torch.nn.Parameter(start.clone())
    adam = torch.optim.Adam([p], lr=0.0025, eps=1e-15)
    p.grad = seen[0]
    adam.step()
    torch.testing.assert_close(sem.detach(), p.detach(), rtol=1e-6, atol=1e-7)
    st = adam.state[p]
    m, v = opt.row_moment_views("semantic", 0)
    torch.testing.assert_close(m, st["exp_avg"], rtol=1e-6, atol=0)
    torch.testing.assert_close(v, st["exp_avg_sq"], rtol=1e-6, atol=0)


def test_refinement_carries_logits_like_the_reference_optimizer_form():
    """One real refinement of the same model with FusedAdam and with the reference's dict of torch.optim.Adam (plus a
    "semantic" group): the carried logits and their moments agree bit for bit, and match the features_dc row map."""
    results = []
    for form in ("fused", "torch"):
        fr, model, gt, labels = _model(actors=True)
        model.config.num_train_data = 50
        subs = list(model.all_models.values())
        g = torch.Generator(device=DEV).manual_seed(11)
        for sub in subs:
            n, d = sub.num_points, sub.__dict__
            vis = torch.randint(1, 9, (n,), device=DEV, generator=g).float()
            d["vis_counts"], d["xys_grad_norm"] = vis, torch.rand(n, device=DEV, generator=g) * vis * 2.5e-6
            d["max_2Dsize"], d["last_size"] = torch.rand(n, device=DEV, generator=g) * 0.2, (240, 320)
        mom = {}
        gm = torch.Generator(device=DEV).manual_seed(12)
        for i, sub in enumerate(subs):
            for k in PARAM_NAMES + ("semantic",):
                t = sub.semantic_logits if k == "semantic" else sub.gauss_params[k]
                mom[(i, k)] = (torch.randn(t.shape, device=DEV, generator=gm), torch.rand(t.shape, device=DEV, generator=gm))
        if form == "fused":
            opt = FusedAdam(model.optimizer_params(), rows={"semantic": (model.semantic_params(), 0.0025)})
            for i in range(len(subs)):
                for j, k in enumerate(PARAM_NAMES):
                    for dst, src in zip(opt.moment_views(6 * i + j), mom[(i, k)]):
                        dst.copy_(src)
                for dst, src in zip(opt.row_moment_views("semantic", i), mom[(i, "semantic")]):
                    dst.copy_(src)
        else:
            opt = {k: torch.optim.Adam([sub.gauss_params[k] for sub in subs], lr=1e-3, eps=1e-15) for k in PARAM_NAMES}
            opt["semantic"] = torch.optim.Adam(model.semantic_params(), lr=0.0025, eps=1e-15)
            for k, o in opt.items():
                for i, p in enumerate(o.param_groups[0]["params"]):
                    m, v = mom[(i, k)]
                    o.state[p] = {"step": torch.tensor(1.0), "exp_avg": m.clone(), "exp_avg_sq": v.clone()}
        model.step = 3400
        before = [sub.num_points for sub in subs]
        model.refinement_after(opt, 3400, generator=torch.Generator(device=DEV).manual_seed(0))
        torch.cuda.synchronize()
        subs = list(model.all_models.values())
        assert [s.num_points for s in subs] != before
        out = []
        for i, sub in enumerate(subs):
            if form == "fused":
                m, v = opt.row_moment_views("semantic", i)
            else:
                st = opt["semantic"].state[sub.semantic_logits]
                m, v = st["exp_avg"], st["exp_avg_sq"]
                assert opt["semantic"].param_groups[0]["params"][i] is sub.semantic_logits
            out.append((sub.semantic_logits.detach().clone(), m.clone(), v.clone(), sub.gauss_params["features_dc"].detach().clone()))
        results.append(out)
    for (l0, m0, v0, f0), (l1, m1, v1, f1) in zip(*results):
        assert torch.equal(f0, f1) and torch.equal(l0, l1) and torch.equal(m0, m1) and torch.equal(v0, v1)


def test_deterministic_steps_repeat_bit_for_bit(monkeypatch):
    monkeypatch.setattr(raster, "DETERMINISTIC", True)
    runs = []
    for _ in range(2):
        fr, model, gt, labels, opt, step_fn = _step_model(False)
        for s in (10, 11, 12):
            losses = step_fn(s, fr.camera, {"image": gt, "semantic": labels})
            assert "semantic_loss" in losses
        torch.cuda.synchronize()
        runs.append({n: p.detach().clone() for n, p in model.named_parameters()})
    a, b = runs
    assert a.keys() == b.keys() and any("semantic_logits" in k for k in a)
    assert not [k for k in a if not torch.equal(a[k], b[k])]


def test_eval_outputs_and_metrics():
    fr, model, gt, labels = _model()
    model.eval()
    out = model.get_outputs_for_camera(fr.camera)
    assert out["semantic"].shape == (240, 320, 3)
    # the reference render script's branch for a "*semantic*" output of logits (scripts/render.py:231-236)
    img = (out["semantic"].argmax(dim=-1).cpu().numpy() * 100).astype(np.uint8)
    assert img.shape == (240, 320) and set(np.unique(img)) <= {0, 100, 200}
    metrics, _ = model.get_image_metrics_and_images(out, {"image": gt, "semantic": labels})
    acc, miou = ref.metrics_ref64(ref.confusion_ref64(out["semantic"].cpu().numpy(), labels.cpu().numpy()))
    assert metrics["semantic_acc"] == pytest.approx(acc, rel=1e-12) and metrics["semantic_miou"] == pytest.approx(miou, rel=1e-12)
    plain, _ = model.get_image_metrics_and_images(out, {"image": gt})
    assert not any(k.startswith("semantic") for k in plain)
    empty = SceneGraphConfig(semantic_classes=3)
    assert empty.semantic_loss_mult == 0.0


def test_data_parallel_refuses_semantics(monkeypatch):
    fr, model, gt, labels, opt, step_fn = _step_model(False)
    monkeypatch.setattr(step_fn, "world_size", lambda: 2)
    model.config.full_gradient_arena = True
    model._grad_sink = _FullArenaSink()
    called = []
    monkeypatch.setattr(model, "get_outputs", lambda camera: called.append(camera))
    with pytest.raises(NotImplementedError):
        step_fn(0, fr.camera, {"image": gt, "semantic": labels}, all_cameras=[fr.camera, fr.camera])
    assert not called
