"""The semantic term on the CPU: the float64 statement (tests/semantic_cases.py) against finite differences and the reference's
refinement restatement (oracle/oracle_refine.py), the torch expression of the term against it, the PLY columns, and the host
logic of the ``semantic`` row group in FusedAdam and TrainStep.  The kernels themselves are checked in tests/test_gpu_semantic.py."""
import numpy as np
import pytest
import torch

from oracle import oracle_refine as orc
from street_gaussians_ns_b200 import refine
from street_gaussians_ns_b200.scene import PARAM_NAMES, GaussianSet
from tests import semantic_cases as ref
from tests.test_refine import build_model, clone_state, make_state, run_oracle, to_settings


def case(H=6, W=7, C=4, seed=0, ignore=0.2, mask_frac=None):
    rng = np.random.default_rng(seed)
    logits = rng.normal(size=(H, W, C)) * 2.0
    labels = rng.integers(0, C, size=(H, W))
    labels[rng.random((H, W)) < ignore] = 255
    mask = None if mask_frac is None else (rng.random((H, W, 1)) > mask_frac).astype(np.float64)
    return logits, labels, mask


@pytest.mark.parametrize("mask_frac", [None, 0.3])
def test_gradient_matches_finite_differences(mask_frac):
    logits, labels, mask = case(mask_frac=mask_frac)
    v = ref.grad_ref64(logits, labels, mask, weight=0.7)
    eps = 1e-6
    fd = np.zeros_like(logits)
    for idx in np.ndindex(*logits.shape):
        a, b = logits.copy(), logits.copy()
        a[idx] += eps
        b[idx] -= eps
        fd[idx] = (ref.loss_ref64(a, labels, mask, 0.7)[0] - ref.loss_ref64(b, labels, mask, 0.7)[0]) / (2 * eps)
    np.testing.assert_allclose(v, fd, rtol=1e-6, atol=1e-9)


def test_ignored_labels_mask_and_no_valid_pixel():
    logits, labels, mask = case(mask_frac=0.4)
    loss, n = ref.loss_ref64(logits, labels, mask)
    keep = ref.valid_ref(labels, 4, mask)
    assert 0 < n == int(keep.sum()) < labels.size
    sub = logits.reshape(-1, 4)[keep][None]
    assert loss == pytest.approx(ref.loss_ref64(sub, labels.reshape(-1)[keep][None])[0], rel=1e-14)
    v = ref.grad_ref64(logits, labels, mask).reshape(-1, 4)
    assert not v[~keep].any() and v[keep].any()
    negative = labels.copy()
    negative[0, 0] = -1  # any label outside [0, C) is ignored, not only 255
    assert ref.loss_ref64(logits, negative)[1] == ref.loss_ref64(logits, labels)[1] - int(labels[0, 0] < 4)
    for lab, m in ((np.full_like(labels, 255), None), (labels, np.zeros_like(mask))):
        assert ref.loss_ref64(logits, lab, m) == (0.0, 0)
        assert not ref.grad_ref64(logits, lab, m).any()


@pytest.mark.parametrize("mask_frac", [None, 0.3])
def test_torch_expression_matches_float64(mask_frac):
    from street_gaussians_ns_b200.semantic import semantic_loss_torch
    logits, labels, mask = case(mask_frac=mask_frac)
    x = torch.tensor(logits, requires_grad=True)
    m = None if mask is None else torch.tensor(mask)
    loss = semantic_loss_torch(x, torch.tensor(labels)[..., None], m, 0.3)
    loss.backward()
    assert float(loss.detach()) == pytest.approx(ref.loss_ref64(logits, labels, mask, 0.3)[0], rel=1e-12)
    np.testing.assert_allclose(x.grad.numpy(), ref.grad_ref64(logits, labels, mask, 0.3), rtol=1e-10, atol=1e-14)
    y = torch.tensor(logits, requires_grad=True)
    none = semantic_loss_torch(y, torch.full(labels.shape, 255), None, 0.3)
    none.backward()
    assert float(none.detach()) == 0.0 and not y.grad.any()


def test_argmax_ties_go_to_the_lowest_class_and_the_metrics():
    from street_gaussians_ns_b200.semantic import metrics_from_confusion
    logits = np.array([[[1.0, 1.0, 0.0], [0.0, 2.0, 2.0], [3.0, 3.0, 3.0], [0.0, 0.0, 1.0]]])
    labels = np.array([[1, 2, 0, 255]])
    conf = ref.confusion_ref64(logits, labels)
    assert conf.tolist() == [[1, 0, 0], [1, 0, 0], [0, 1, 0]]
    acc, miou = ref.metrics_ref64(conf)
    assert acc == pytest.approx(1 / 3)
    assert miou == pytest.approx((1 / 2 + 0 + 0) / 3)  # IoU of class 0 = 1 / (2 + 1 - 1); every union is non-empty
    got = metrics_from_confusion(torch.tensor(conf))
    assert got["semantic_acc"] == pytest.approx(acc) and got["semantic_miou"] == pytest.approx(miou)
    only0 = metrics_from_confusion(torch.tensor([[5, 0, 0], [0, 0, 0], [0, 0, 0]]))
    assert only0 == {"semantic_acc": 1.0, "semantic_miou": 1.0}  # classes without a union are left out of the mean
    empty = metrics_from_confusion(torch.zeros(3, 3, dtype=torch.int64))
    assert np.isnan(empty["semantic_acc"]) and np.isnan(empty["semantic_miou"])


@pytest.fixture()
def host_backend(monkeypatch):
    from tests.host_harness import load_refine_harness
    harness = load_refine_harness()
    monkeypatch.setattr(refine, "_backend", lambda: harness)
    monkeypatch.setattr(refine, "_require_cuda", lambda t, what: None)
    return harness


@pytest.mark.parametrize("step,over", [(700, {}), (3400, {}), (7400, {"n_split_samples": 3}), (25000, {})])
def test_carry_row_map_matches_the_reference_refinement(host_backend, step, over):
    """Tag every row's features_dc with its row number: the reference's refinement then spells out the row map, which the
    float64 carry must equal for the flags the refinement rules decide."""
    cfg = orc.RefineConfig(stop_split_at=25000, cull_alpha_thresh=0.02, cull_scale_thresh=0.2, **over)
    st = make_state(1500, 1, seed=21, with_moments=True)
    st.params["features_dc"][:, 0, 0] = torch.arange(1500, dtype=torch.float32)
    settings = to_settings(cfg)
    densify, cull_only, _ = refine.phase(settings, step, 50)
    mcfg = refine.make_config(settings, step, (240, 320), densify)
    plan = refine.plan_submodel(st.params["scales"], st.params["opacities"], st.xys_grad_norm if densify else None,
                                st.vis_counts if densify else None, st.max_2Dsize if mcfg.use_screen_size else None, mcfg,
                                torch.Generator().manual_seed(3))
    ost, _ = run_oracle(clone_state(st), cfg, step, (240, 320), 50, seed=3)
    rows, kept = ref.carry_rows_ref(plan.flags.numpy(), mcfg.n_split_samples)
    assert plan.changed and rows.shape[0] == plan.out_rows
    assert ost.params["features_dc"][:, 0, 0].long().tolist() == rows.tolist()
    m_src, v_src = st.moments["features_dc"]
    out, (m, v) = ref.carry_ref(st.params["features_dc"].numpy(), plan.flags.numpy(), mcfg.n_split_samples,
                                (m_src.numpy(), v_src.numpy()))
    assert np.array_equal(out, ost.params["features_dc"].numpy())
    assert np.array_equal(m, ost.moments["features_dc"][0].numpy()) and np.array_equal(v, ost.moments["features_dc"][1].numpy())
    assert kept.sum() == plan.totals[0]


# ---- PLY ---------------------------------------------------------------------------------------------------------------------

def _set(n=9, seed=0):
    g = torch.Generator().manual_seed(seed)
    return GaussianSet(torch.randn(n, 3, generator=g), torch.randn(n, 3, generator=g), torch.randn(n, 4, generator=g),
                       torch.randn(n, 1, 3, generator=g), torch.randn(n, 15, 3, generator=g), torch.randn(n, 1, generator=g))


def test_ply_round_trip_with_and_without_semantics(tmp_path):
    from street_gaussians_ns_b200 import ply_io
    s = _set()
    plain_a, plain_b, sem_path = tmp_path / "a.ply", tmp_path / "b.ply", tmp_path / "s.ply"
    ply_io.write_ply(plain_a, s)
    ply_io.write_ply(plain_b, s, None)
    assert plain_a.read_bytes() == plain_b.read_bytes()
    assert ply_io.read_semantic(plain_a) is None
    assert ply_io.property_names(45) == ply_io.property_names(45, 0)
    logits = torch.randn(9, 3, generator=torch.Generator().manual_seed(1))
    logits[4, 1] = float("nan")  # a non-finite row is dropped like any other
    assert ply_io.write_ply(sem_path, s, logits) == 8
    cols = list(ply_io.read_ply_columns(sem_path))
    assert cols[cols.index("rot_3") + 1:] == ["semantic_0", "semantic_1", "semantic_2"]
    keep = torch.ones(9, dtype=torch.bool)
    keep[4] = False
    assert torch.equal(ply_io.read_semantic(sem_path), logits[keep])
    back = ply_io.read_ply(sem_path)
    assert torch.equal(back.means, s.means[keep])
    plain = ply_io.read_ply_columns(plain_a)  # the other columns are those of the file without semantics
    assert all(np.array_equal(v, plain[k][keep.numpy()]) for k, v in ply_io.read_ply_columns(sem_path).items() if k in plain)


# ---- optimizer and training step (host logic) ----------------------------------------------------------------------------------

def _params(rows=((10, 1), (7, 5), (5, 5))):
    return [[torch.zeros(n, *shape) for shape in ((3,), (3,), (4,), (F, 3), (15, 3), (1,))] for n, F in rows]


def test_fused_adam_without_rows_is_unchanged():
    from street_gaussians_ns_b200.optim import FusedAdam
    a, b = FusedAdam(_params(), chunk_elems=64), FusedAdam(_params(), chunk_elems=64, rows=None)
    assert a.moment_elems == b.moment_elems and a.arena_elems == b.arena_elems and b.row_index == {}
    assert np.array_equal(a.table[["arena_offset", "grad_offset", "numel", "chunk0"]], b.table[["arena_offset", "grad_offset", "numel", "chunk0"]])
    assert b.row_tensors() == {}


def test_fused_adam_row_group_tables():
    from street_gaussians_ns_b200.optim import FusedAdam
    params = _params()
    sky = torch.zeros(6, 4, 4, 3)
    sem = [torch.zeros(n, 3) for n in (10, 7, 5)]
    opt = FusedAdam(params, chunk_elems=64, extra={"sky": (sky, 0.005)}, rows={"semantic": (sem, 0.0025)})
    plain = FusedAdam(params, chunk_elems=64, extra={"sky": (sky, 0.005)})
    assert opt.arena_elems == plain.arena_elems                     # the gradient arena is the six tensors' only
    i0 = opt.row_index["semantic"]
    assert i0 == 18 + 1                                             # behind the extra tensors
    assert list(opt.offsets[:i0]) == list(plain.offsets)
    assert opt.moment_elems == plain.moment_elems + sum((t.numel() + 3) // 4 * 4 for t in sem)
    assert [opt.kinds[i0 + k] for k in range(3)] == ["row:semantic"] * 3
    arena = torch.zeros(opt.arena_elems + 64)
    grads = [arena[opt.arena_elems:opt.arena_elems + 30].view(10, 3), None, torch.zeros(5, 3)]
    tab = opt.step_table(present=[0, 2], grad_arena=arena, row_grads={"semantic": grads})
    assert len(tab) == 12 + 2                                       # sub-model 1 has no semantic gradient: skipped
    assert list(tab["arena_offset"][12:]) == [opt.offsets[i0], opt.offsets[i0 + 2]]
    assert int(tab["grad_offset"][12]) == opt.arena_elems
    assert int(tab["grad_offset"][13]) == (grads[2].data_ptr() - arena.data_ptr()) // 4
    assert list(opt.steps[i0:i0 + 3]) == [1, 0, 1]
    np.testing.assert_allclose(tab["step_size"][12], 0.0025 / (1 - 0.9), rtol=1e-6)
    # a refinement: sub-model 0's logits are a new tensor (zeroed moments, carried by the caller), the others keep theirs
    opt.exp_avg.fill_(1.0)
    new_sem = [torch.zeros(12, 3), sem[1], sem[2]]
    new_params = [[torch.zeros(12, *p.shape[1:]) for p in params[0]], params[1], params[2]]
    old_m, _, old_off = opt.rebuild(new_params, {"semantic": new_sem})
    m0, _ = opt.row_moment_views("semantic", 0)
    m1, _ = opt.row_moment_views("semantic", 1)
    assert m0.shape == (12, 3) and not m0.any() and bool((m1 == 1).all())
    assert bool((opt.moment_views(18)[0] == 1).all())               # the extra tensor's moments moved along
    assert opt.row_tensors()["semantic"][0] is new_sem[0]


def test_train_step_accumulates_the_row_group(monkeypatch):
    """nerfstudio's rule for {"semantic": 10}: zeroed at step % 10 == 0, stepped at step % 10 == 9 (sub-models whose gradient is
    None then are skipped), kept in between."""
    from street_gaussians_ns_b200.optim import FusedAdam
    from street_gaussians_ns_b200.training import TrainStep
    model, _ = build_model()
    with pytest.raises(AssertionError):
        model.semantic_params()
    states = [make_state(900, 1, 0), make_state(300, 5, 1), make_state(200, 5, 2)]
    from street_gaussians_ns_b200.model import SceneGraphConfig, SceneGraphRasterModel
    sets = [GaussianSet(*[s.params[k].clone() for k in PARAM_NAMES]) for s in states]
    model = SceneGraphRasterModel(sets[0], {"a": sets[1], "b": sets[2]}, SceneGraphConfig(use_sky_sphere=False, semantic_classes=3))
    assert [tuple(p.shape) for p in model.semantic_params()] == [(900, 3), (300, 3), (200, 3)]
    assert all(not p.any() for p in model.semantic_params())
    assert not any("semantic" in n for n in dict(model.all_models["background"].gauss_params.named_parameters()))
    opt = FusedAdam(model.optimizer_params(), chunk_elems=4096, rows={"semantic": (model.semantic_params(), 0.0025)})
    with pytest.raises(ValueError):
        TrainStep(model, opt, gradient_accumulation_steps={"semantics": 10})
    step_fn = TrainStep(model, opt, refine_every=100000, gradient_accumulation_steps={"semantic": 10})
    sem = model.semantic_params()
    due = []
    monkeypatch.setattr(model, "get_outputs", lambda camera: {})
    monkeypatch.setattr(model, "get_loss_dict", lambda out, batch: {"main_loss": torch.zeros(())})
    monkeypatch.setattr(model, "refinement_after", lambda *a, **k: None)
    launched = []
    monkeypatch.setattr(opt, "launch", lambda tab, arena: launched.append(tab.copy()))  # the table, not the kernel
    for s in range(12):
        if s in (0, 3):
            sem[0].grad = torch.ones(900, 3) if sem[0].grad is None else sem[0].grad + 1
        kept = sem[0].grad
        due.append(step_fn._due_row_grads(s))
        step_fn(s, camera=None, batch={})
        if s % 10 == 0:
            assert s == 0 or sem[0].grad is None          # zeroed at the start of the cycle (step 0 set it again above)
        elif kept is not None:
            assert sem[0].grad is kept                    # kept in between
    assert [bool(d) for d in due] == [False] * 9 + [True] + [False] * 2
    assert due[9]["semantic"][0] is not None and due[9]["semantic"][1] is None and due[9]["semantic"][2] is None
    assert len(launched) == 1 and len(launched[0]) == 1      # step 9 only, sub-model 0's logits only
    assert int(launched[0]["param"][0]) == sem[0].data_ptr() and int(launched[0]["numel"][0]) == 900 * 3


def test_model_refinement_carries_the_logits(host_backend, monkeypatch):
    """The model's refinement hands every changed sub-model's logits (and their FusedAdam moments) to the carry with its plan;
    the carry is the float64 map here (the kernel is checked on the GPU)."""
    from street_gaussians_ns_b200 import semantic
    from street_gaussians_ns_b200.model import SceneGraphConfig, SceneGraphRasterModel
    from street_gaussians_ns_b200.optim import FusedAdam

    def host_carry(plan, src, dst, ms=None, md=None):
        out, mom = ref.carry_ref(src.numpy(), plan.flags.numpy(), plan.cfg.n_split_samples,
                                 None if ms is None else (ms[0].numpy(), ms[1].numpy()))
        dst.copy_(torch.from_numpy(out))
        if mom is not None:
            md[0].copy_(torch.from_numpy(mom[0]))
            md[1].copy_(torch.from_numpy(mom[1]))
    monkeypatch.setattr(semantic, "refine_carry", host_carry)
    _, states = build_model()
    sets = [GaussianSet(*[s.params[k].clone() for k in PARAM_NAMES]) for s in states]
    model = SceneGraphRasterModel(sets[0], {"a": sets[1], "b": sets[2]},
                                  SceneGraphConfig(use_sky_sphere=False, num_train_data=50, semantic_classes=2))
    model.train()
    for sub, s in zip(model.all_models.values(), states):
        d = sub.__dict__
        d["xys_grad_norm"], d["vis_counts"], d["max_2Dsize"] = s.xys_grad_norm.clone(), s.vis_counts.clone(), s.max_2Dsize.clone()
        d["last_size"] = (240, 320)
        with torch.no_grad():  # logit 0 = the row's features_dc[:, 0, 0]: the carry must move it with its row
            sub.semantic_logits[:, 0] = sub.gauss_params["features_dc"][:, 0, 0]
            sub.semantic_logits[:, 1] = torch.arange(sub.num_points, dtype=torch.float32)
    opt = FusedAdam(model.optimizer_params(), chunk_elems=4096, rows={"semantic": (model.semantic_params(), 0.0025)})
    for i in range(3):  # moments: features_dc's and the logits' first column hold the same values
        m, v = opt.moment_views(6 * i + 3)
        m.copy_(torch.randn(m.shape, generator=torch.Generator().manual_seed(i)))
        v.copy_(m.abs())
        sm, sv = opt.row_moment_views("semantic", i)
        sm[:, 0], sv[:, 0] = m[:, 0, 0], v[:, 0, 0]
    before = [sub.num_points for sub in model.all_models.values()]
    model.step = 3400
    model.refinement_after(opt, 3400, generator=torch.Generator().manual_seed(0))
    after = [sub.num_points for sub in model.all_models.values()]
    assert before != after
    for i, sub in enumerate(model.all_models.values()):
        assert sub.semantic_logits.shape == (sub.num_points, 2) and isinstance(sub.semantic_logits, torch.nn.Parameter)
        assert torch.equal(sub.semantic_logits[:, 0], sub.gauss_params["features_dc"][:, 0, 0])
        m, v = opt.moment_views(6 * i + 3)
        sm, sv = opt.row_moment_views("semantic", i)
        assert torch.equal(sm[:, 0], m[:, 0, 0]) and torch.equal(sv[:, 0], v[:, 0, 0])
        assert opt.row_tensors()["semantic"][i] is sub.semantic_logits
