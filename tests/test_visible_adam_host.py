"""Host logic of the selective Adam step (gsplat's visible_adam) that needs no GPU: the sgn_adam_rows tables FusedAdam.step_table
builds (which flag byte each tensor's row 0 reads, its row width), the "seen" masks TrainStep keeps for accumulated row groups,
and the refusal under data parallelism."""
import types

import numpy as np
import pytest
import torch

from street_gaussians_ns_b200.optim import ADAM_DTYPE, ADAM_ROWS_DTYPE, FusedAdam

ROWS = [5, 3, 7]          # rows of the three sub-models
WIDTHS = [3, 3, 4, 3, 45, 1]
C = 4                     # semantic classes


def make_opt(extra=True, rows=True):
    g = torch.Generator().manual_seed(0)
    params = [[torch.randn(n, 3, generator=g), torch.randn(n, 3, generator=g), torch.randn(n, 4, generator=g),
               torch.randn(n, 1, 3, generator=g), torch.randn(n, 15, 3, generator=g), torch.randn(n, 1, generator=g)] for n in ROWS]
    ex = {"sky": (torch.randn(6, 2, 2, 3, generator=g), 0.005)} if extra else None
    rg = {"semantic": ([torch.randn(n, C, generator=g) for n in ROWS], 0.0025)} if rows else None
    return FusedAdam(params, chunk_elems=4096, extra=ex, rows=rg), params


def tensor_index(opt, tab):
    ptr = {t.data_ptr(): i for i, t in enumerate(opt._params)}
    return [ptr[int(p)] for p in tab["param"]]


def frame_row0(present):
    out, r = {}, 0
    for s in present:
        out[s] = r
        r += ROWS[s]
    return out


@pytest.mark.parametrize("full_layout", [False, True])
@pytest.mark.parametrize("present", [None, [0, 1, 2], [2, 0], [1], []])
@pytest.mark.parametrize("kinds", [None, [1, 4], [5]])
def test_flag_rows_of_the_six_tensors(present, full_layout, kinds):
    opt, _ = make_opt(extra=False, rows=False)
    ref, _ = make_opt(extra=False, rows=False)
    kw = {} if kinds is None else {"kinds": kinds}
    tab, rows = opt.step_table(present, full_layout=full_layout, visible=True, **kw)
    plain = ref.step_table(present, full_layout=full_layout, **kw)
    assert rows.dtype == ADAM_ROWS_DTYPE and tab.dtype == ADAM_DTYPE and len(rows) == len(tab)
    # the selective table is the dense one, field for field (pointers aside: two optimizers), and the step counts agree
    for f in ADAM_DTYPE.names:
        if f != "param":
            assert np.array_equal(tab[f], plain[f]), f
    assert np.array_equal(opt.steps, ref.steps)
    order = list(range(3)) if present is None else present
    r0 = frame_row0(order)
    want = [(s, k) for s in order for k in range(6) if kinds is None or k in kinds]
    assert tensor_index(opt, tab) == [6 * s + k for s, k in want]
    assert rows["flag_row0"].tolist() == [r0[s] for s, _ in want]
    assert rows["row_width"].tolist() == [WIDTHS[k] for _, k in want]


def test_extra_tensors_are_dense_and_row_groups_follow_their_sub_model():
    opt, params = make_opt()
    arena = torch.zeros(opt.moment_elems + 64)
    sky = opt.extra_tensors()["sky"]
    sem = opt.row_tensors()["semantic"]
    gsky = arena[opt.arena_elems:opt.arena_elems + sky.numel()]
    gsem = [None, arena[-64:-64 + ROWS[1] * C], arena[-40:-40 + ROWS[2] * C]]
    tab, rows = opt.step_table([2, 1], grad_arena=arena, extra_grads={"sky": gsky}, row_grads={"semantic": gsem}, visible=True)
    idx = tensor_index(opt, tab)
    r0 = frame_row0([2, 1])
    i_sky, i_sem = opt.extra_index["sky"], opt.row_index["semantic"]
    assert idx == [12 + k for k in range(6)] + [6 + k for k in range(6)] + [i_sky, i_sem + 1, i_sem + 2]
    assert rows["flag_row0"].tolist() == [r0[2]] * 6 + [r0[1]] * 6 + [-1, r0[1], r0[2]]
    assert rows["row_width"][-2:].tolist() == [C, C]
    # a row-group tensor of a sub-model that is not in the frame has no frame bytes: it needs its own
    gsem0 = [arena[-64:-64 + ROWS[0] * C], None, None]
    with pytest.raises(ValueError, match="row_flag_row0"):
        opt.step_table([2, 1], grad_arena=arena, row_grads={"semantic": gsem0}, visible=True)
    tab, rows = opt.step_table([2, 1], grad_arena=arena, row_grads={"semantic": gsem0}, visible=True,
                               row_flag_row0={"semantic": [100, 105, 108]})
    assert tensor_index(opt, tab)[-1] == i_sem and rows["flag_row0"][-1] == 100
    # the override replaces the frame's bytes for present sub-models too; nothing present: only the overridden tensors
    tab, rows = opt.step_table([], full_layout=True, grad_arena=arena, row_grads={"semantic": gsem}, visible=True,
                               row_flag_row0={"semantic": [100, 105, 108]})
    assert tensor_index(opt, tab) == [i_sem + 1, i_sem + 2] and rows["flag_row0"].tolist() == [105, 108]
    assert rows["row_width"].tolist() == [C, C]


def test_dense_call_is_unchanged_and_refuses_the_override():
    opt, _ = make_opt(extra=False, rows=False)
    tab = opt.step_table([0, 2])
    assert isinstance(tab, np.ndarray) and tab.dtype == ADAM_DTYPE
    with pytest.raises(AssertionError):
        opt.step_table([0, 2], row_flag_row0={"semantic": [0, 0, 0]})


# ---- TrainStep: the accumulated row groups' masks -------------------------------------------------------------------------
def make_step(accumulate=3):
    from street_gaussians_ns_b200.training import TrainStep
    from tests.test_refine import build_model
    model, _ = build_model()
    model.config.semantic_classes = C
    for sub in model.all_models.values():
        sub.__dict__["semantic_logits"] = torch.zeros(sub.num_points, C)
    opt = FusedAdam(model.optimizer_params(), chunk_elems=4096, rows={"semantic": (model.semantic_params(), 0.0025)})
    return model, opt, TrainStep(model, opt, refine_every=100, gradient_accumulation_steps={"semantic": accumulate}, visible_adam=True)


def test_seen_mask_layout_cycle_and_refinement():
    model, opt, st = make_step(accumulate=3)
    counts = [sub.num_points for sub in model.all_models.values()]
    stride = (sum(counts) + 15) // 16 * 16
    row0 = np.concatenate([[0], np.cumsum(counts)[:-1]])
    out = st._visible_flags(0, [0, 2], seen=False)  # nothing seen: the frame's bytes are zero
    buf = out["visible"]
    assert buf.dtype == torch.uint8 and buf.numel() == 2 * stride
    assert out["row_flag_row0"] == {"semantic": (stride + row0).tolist()}
    assert int(buf[:counts[0] + counts[2]].sum()) == 0
    # rows seen in the cycle (what sgn_visible_or writes) survive its later steps and are cleared where the next cycle starts
    buf[stride + 3] = 1
    buf[stride + row0[2] + 1] = 1
    buf[:4] = 1
    st._visible_flags(1, [1], seen=False)
    assert st._vis_buf is buf and int(buf[stride:].sum()) == 2 and int(buf[:counts[1]].sum()) == 0
    st._visible_flags(2, [], seen=False)
    assert int(buf[stride:].sum()) == 2
    st._visible_flags(3, [], seen=False)  # 3 % 3 == 0: a new cycle
    assert int(buf[stride:].sum()) == 0
    # a refinement that replaces sub-model 2's logits (and leaves the others) keeps only the others' masks
    buf[stride + 3] = 1
    buf[stride + row0[2] + 1] = 1

    def refine(o, step, **kw):
        sub = model.all_models["object_b"]
        sub.__dict__["semantic_logits"] = torch.zeros(sub.num_points, C)
        o.rebuild_pointers(model.optimizer_params(), rows={"semantic": model.semantic_params()})
    model.refinement_after = refine
    st._maybe_refine(100)
    assert st._vis_keep == {("semantic", 0), ("semantic", 1)}
    st._visible_flags(4, [], seen=False)
    assert st._vis_buf is not buf and st._vis_keep is None
    new = st._vis_buf
    assert int(new[stride + 3]) == 1 and int(new[stride + row0[2] + 1]) == 0 and int(new[stride:].sum()) == 1


def test_data_parallel_refuses_visible_adam_before_rendering(monkeypatch):
    from street_gaussians_ns_b200.model import _FullArenaSink
    from street_gaussians_ns_b200.training import TrainStep
    from tests.test_refine import build_model
    model, _ = build_model()
    opt = FusedAdam(model.optimizer_params(), chunk_elems=4096)
    step_fn = TrainStep(model, opt, refine_every=0, visible_adam=True)
    rendered = []
    monkeypatch.setattr(model, "get_outputs", lambda camera: rendered.append(camera))
    model._holder = types.SimpleNamespace(grad_arena=torch.zeros(8))
    model._grad_sink = _FullArenaSink()
    monkeypatch.setattr(step_fn, "world_size", lambda: 2)
    monkeypatch.setattr(step_fn, "_ensure_exchange", lambda: rendered.append("exchange"))
    with pytest.raises(NotImplementedError, match="visible_adam"):
        step_fn(700, camera=None, batch={}, all_cameras=[None, None])
    assert not rendered
