"""Selective Adam (gsplat's visible_adam) on the GPU.

* sgn_adam_step_visible, directed: row widths 1, 3, 4, 15, 45 and a semantic width, numel not a multiple of 4, parameters
  misaligned against 16 bytes (the scalar path), float4s that straddle a seen and an unseen row, all / no / random / run-like
  masks, dense and masked tensors in one launch.  A stepped element is bit-equal to oracle/step_ref64.adam_f32; every other
  element, the moment padding and the canaries around each parameter are bit-unchanged.  With every byte set the launch is
  bit-equal to sgn_adam_step.  Invalid arguments return SGN_ERR_INVALID.
* sgn_visible_or against a host OR.
* TrainStep(visible_adam=True) on a small street scene: rows with radius 0 keep their bits, the seen rows match a dense
  FusedAdam step on the same arena, an accumulated semantic cycle steps exactly the union of its frames' rows, a refinement
  inside the run keeps it working, and with the option off nothing changes."""
import ctypes as C

import numpy as np
import pytest
import torch

from street_gaussians_ns_b200 import _lib
from street_gaussians_ns_b200.optim import ADAM_ROWS_DTYPE, FusedAdam
from oracle import step_ref64 as ref
from tests.test_gpu_step_directed import AdamSet, adam_grads, adam_launch, adam_rows, bits

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
ERR_INVALID = -1
f32 = np.float32


def L():
    return _lib.load()


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


# ---- the kernel, directed ------------------------------------------------------------------------------------------------
# (rows, row width, masked): widths 1, 3, 4, 15, 45 and 10 (a semantic width); numels 21, 4099, 9000 ... not multiples of 4
TENSORS = [(4099, 1, True), (7, 3, True), (1500, 3, True), (1024, 4, True), (333, 15, True), (201, 45, True), (101, 10, True),
           (1000, 3, False), (5, 1, True), (0, 3, True), (9, 45, False), (2049, 45, True)]
FRONT = 13  # flag bytes in front of the first tensor's row 0


def flag_layout():
    row0, r = [], FRONT
    for n, w, masked in TENSORS:
        row0.append(r if masked else -1)
        r += n if masked else 0
    return row0, r + 17  # and bytes behind the last row


def make_mask(kind, rng, nbytes):
    if kind == "all":
        return np.ones(nbytes, np.uint8)
    if kind == "none":
        return np.zeros(nbytes, np.uint8)
    if kind == "random":
        return (rng.random(nbytes) < 0.5).astype(np.uint8) * rng.integers(1, 256, nbytes).astype(np.uint8)  # any non-zero byte
    # runs of seen and unseen rows, as a camera sees a street
    out, i, on = np.zeros(nbytes, np.uint8), 0, False
    while i < nbytes:
        k = int(rng.integers(1, 40))
        out[i:i + k] = on
        i += k
        on = not on
    return out


def rows_table(row0):
    rows = np.zeros(len(TENSORS), ADAM_ROWS_DTYPE)
    rows["flag_row0"] = row0
    rows["row_width"] = [w for _, w, _ in TENSORS]
    return rows


def visible_launch(tab, rows, nchunks, grads, m, v, vis):
    raw = np.concatenate([tab.view(np.uint8).reshape(-1), rows.view(np.uint8).reshape(-1)])
    dev = torch.from_numpy(raw.copy()).to(DEV)
    return L().sgn_adam_step_visible(_p(dev), C.c_void_p(dev.data_ptr() + tab.nbytes), len(tab), nchunks, C.c_void_p(grads),
                                     _p(m), _p(v), _p(vis), None)


def elem_mask(mask, r0, n, w):
    if r0 < 0:
        return np.ones(n * w, bool)
    return np.repeat(mask[r0:r0 + n] != 0, w)


@pytest.mark.parametrize("misaligned", [False, True])
@pytest.mark.parametrize("kinds", [("all", "none", "random"), ("random", "runs", "random"), ("runs", "all", "none")])
def test_visible_steps_match_replay_and_leave_the_rest(misaligned, kinds):
    numels = [n * w for n, w, _ in TENSORS]
    offs = [(1 + i % 3) if misaligned else 0 for i in range(len(numels))]
    s = AdamSet(numels, offs, seed=7)
    rng = np.random.default_rng(13)
    row0, nbytes = flag_layout()
    rows = rows_table(row0)
    lrs = [1.6e-4, 0.005, 0.001, 0.0025, 0.0025 / 20, 0.05] * 2
    for step, kind in enumerate(kinds, start=1):
        mask = make_mask(kind, rng, nbytes)
        # canary bytes in front of and behind the buffer the kernel is given: never read as a row
        vis_buf = torch.from_numpy(np.concatenate([np.full(16, 0xA5, np.uint8), mask, np.full(16, 0xA5, np.uint8)])).to(DEV)
        vis = vis_buf[16:16 + nbytes]
        grads = [adam_grads(rng, n, step) for n in numels]
        s.set_grads(grads, s.arena_off)
        tab, nch = adam_rows(numels, [step] * len(numels), lrs, s.arena_off, s.arena_off, s.params)
        assert visible_launch(tab, rows, nch, s.grad_base(), s.m, s.v, vis) == 0
        for i, ((n, w, _), gr) in enumerate(zip(TENSORS, grads)):
            o, k = int(s.arena_off[i]), numels[i]
            p1, m1, v1 = ref.adam_f32(s.p_host[i], gr, s.m_host[o:o + k], s.v_host[o:o + k], tab[i])
            e = elem_mask(mask, row0[i], n, w)
            s.p_host[i] = np.where(e, p1, s.p_host[i]).astype(f32)
            s.m_host[o:o + k] = np.where(e, m1, s.m_host[o:o + k])
            s.v_host[o:o + k] = np.where(e, v1, s.v_host[o:o + k])
        s.check(offs)  # parameters with their canaries, and both moment arenas (padding included)
        assert np.array_equal(vis_buf.cpu().numpy()[16:16 + nbytes], mask)


@pytest.mark.parametrize("misaligned", [False, True])
def test_all_rows_visible_equals_the_dense_step(misaligned):
    numels = [n * w for n, w, _ in TENSORS]
    offs = [(3 - i % 4) if misaligned else 0 for i in range(len(numels))]
    row0, nbytes = flag_layout()
    outs = []
    for selective in (False, True):
        s = AdamSet(numels, offs, seed=21)
        rng = np.random.default_rng(22)
        vis = torch.ones(nbytes, dtype=torch.uint8, device=DEV)
        for step in range(1, 4):
            grads = [adam_grads(rng, n, step) for n in numels]
            s.set_grads(grads, s.arena_off)
            tab, nch = adam_rows(numels, [step] * len(numels), [0.01] * len(numels), s.arena_off, s.arena_off, s.params)
            if selective:
                assert visible_launch(tab, rows_table(row0), nch, s.grad_base(), s.m, s.v, vis) == 0
            else:
                assert adam_launch(tab, nch, s.grad_base(), s.m, s.v) == 0
        torch.cuda.synchronize()
        outs.append(([bits(b.cpu().numpy().view(f32)) for b in s.p_bufs], bits(s.m.cpu().numpy()), bits(s.v.cpu().numpy())))
    (pa, ma, va), (pb, mb, vb) = outs
    assert all(np.array_equal(a, b) for a, b in zip(pa, pb)) and np.array_equal(ma, mb) and np.array_equal(va, vb)


def test_visible_argument_errors():
    s = AdamSet([8], [0], seed=1)
    tab, nch = adam_rows([8], [1], [0.01], [0], [0], s.params)
    rows = np.zeros(1, ADAM_ROWS_DTYPE)
    rows["flag_row0"], rows["row_width"] = 0, 2
    raw = np.concatenate([tab.view(np.uint8).reshape(-1), rows.view(np.uint8).reshape(-1), np.zeros(16, np.uint8)])
    dev = torch.from_numpy(raw).to(DEV)
    t, r = _p(dev), C.c_void_p(dev.data_ptr() + 64)
    vis = torch.ones(4, dtype=torch.uint8, device=DEV)
    g, m, v = C.c_void_p(s.grad_base()), _p(s.m), _p(s.v)
    f = L().sgn_adam_step_visible
    assert f(None, r, 1, nch, g, m, v, _p(vis), None) == ERR_INVALID
    assert f(t, None, 1, nch, g, m, v, _p(vis), None) == ERR_INVALID
    assert f(t, r, 1, nch, None, m, v, _p(vis), None) == ERR_INVALID
    assert f(t, r, 1, nch, g, None, v, _p(vis), None) == ERR_INVALID
    assert f(t, r, 1, nch, g, m, None, _p(vis), None) == ERR_INVALID
    assert f(t, r, 1, nch, g, m, v, None, None) == ERR_INVALID
    assert f(t, r, 0, nch, g, m, v, _p(vis), None) == ERR_INVALID
    assert f(t, r, 8193, nch, g, m, v, _p(vis), None) == ERR_INVALID
    assert b"8193" in L().sgn_last_error()
    assert f(t, r, 1, nch, C.c_void_p(s.grad_base() + 4), m, v, _p(vis), None) == ERR_INVALID
    assert f(t, r, 1, nch, g, C.c_void_p(s.m.data_ptr() + 8), v, _p(vis), None) == ERR_INVALID
    assert f(t, C.c_void_p(dev.data_ptr() + 68), 1, nch, g, m, v, _p(vis), None) == ERR_INVALID  # rows table misaligned
    assert f(t, r, 1, 0, g, m, v, _p(vis), None) == 0  # no chunks: nothing to do
    o = L().sgn_visible_or
    segs = torch.zeros(3, dtype=torch.int64, device=DEV)
    assert o(None, 1, 4, _p(vis), _p(vis), None) == ERR_INVALID
    assert o(_p(segs), 0, 4, _p(vis), _p(vis), None) == ERR_INVALID
    assert o(_p(segs), 1, 4, None, _p(vis), None) == ERR_INVALID
    assert o(C.c_void_p(segs.data_ptr() + 4), 1, 4, _p(vis), _p(vis), None) == ERR_INVALID


def test_visible_or_matches_host():
    rng = np.random.default_rng(3)
    counts = [0, 1000, 1, 37, 0, 5000, 12]
    present = [5, 1, 3, 6, 2, 0]
    row0 = np.concatenate([[0], np.cumsum(counts)[:-1]])
    base = 20000  # the mask sits behind the frame's bytes, as TrainStep lays them out
    n = sum(counts[s] for s in present)
    flags = (rng.random(n) < 0.3).astype(np.uint8)
    seen0 = (rng.random(sum(counts)) < 0.2).astype(np.uint8)
    buf = np.full(base + sum(counts) + 16, 0xEE, np.uint8)
    buf[:n] = flags
    buf[base:base + sum(counts)] = seen0
    want = buf.copy()
    f0 = np.concatenate([[0], np.cumsum([counts[s] for s in present])[:-1]])
    for s, a in zip(present, f0):
        want[base + row0[s]:base + row0[s] + counts[s]] |= flags[a:a + counts[s]]
    segs = np.stack([f0, base + row0[present], np.asarray([counts[s] for s in present])], 1).astype(np.int64)
    d = torch.from_numpy(buf).to(DEV)
    ds = torch.from_numpy(segs).to(DEV)
    assert L().sgn_visible_or(_p(ds), len(present), n, _p(d), _p(d), None) == 0
    assert np.array_equal(d.cpu().numpy(), want)


# ---- the training loop -----------------------------------------------------------------------------------------------------
def _scene(semantic=False):
    import street_gaussians_ns_b200.synthetic as syn
    from street_gaussians_ns_b200.model import ActorPose, SceneGraphConfig, SceneGraphRasterModel
    sc = syn.WaymoScene(scale=0.02, num_frames=20, n_actors=4)
    frame_list = list(range(sc.num_frames))

    def poses_at(t):
        f = int(t)
        return [ActorPose(str(a), rot, center, f, frame_list, frame_id=f) for a, rot, center in sc.boxes_at(f)]
    cfg = SceneGraphConfig(use_sky_sphere=False, ssim_lambda=0.0, refine_record=True, semantic_classes=3 if semantic else 0,
                           semantic_loss_mult=0.1 if semantic else 0.0)
    model = SceneGraphRasterModel(sc.background.to(DEV), {k: v.to(DEV) for k, v in sc.actors.items()}, cfg, poses_at=poses_at).to(DEV)
    model.train()
    g = torch.Generator().manual_seed(5)
    batch = {"image": (torch.rand(sc.height, sc.width, 3, generator=g) * 255).to(torch.uint8).to(DEV)}
    if semantic:
        batch["semantic"] = torch.randint(0, 3, (sc.height, sc.width, 1), generator=g).to(DEV)
    return sc, model, batch


class StepSpy:
    """Wraps FusedAdam.step: records, per call, everything the step read (arena, gradients, flags, radii) and the optimizer's
    state before it."""

    def __init__(self, model, opt, check=True):
        self.model, self.opt, self.real, self.calls, self.check = model, opt, opt.step, [], check
        opt.step = self

    def __call__(self, arena, **kw):
        opt = self.opt
        torch.cuda.synchronize()
        rec = dict(kw)
        rec["arena"] = arena.clone()
        if kw.get("row_grads"):
            rec["row_grads"] = {k: [None if g is None else g.clone() for g in gs] for k, gs in kw["row_grads"].items()}
        if kw.get("visible") is not None:
            rec["visible"] = kw["visible"].clone()
        h = self.model._holder
        rec["radii"] = None if h is None or h.radii is None else h.radii.clone()
        rec["before"] = ([t.detach().clone() for t in opt._params], opt.exp_avg.clone(), opt.exp_avg_sq.clone(), opt.steps.copy())
        self.real(arena, **kw)
        torch.cuda.synchronize()
        if self.check:  # against the state right after this step (a later step or refinement changes it)
            rec["stepped_rows"] = check_step(opt, rec)
        self.calls.append(rec)


def dense_twin(opt, rec):
    """A FusedAdam over copies of the state before ``rec``'s step, stepped densely with the same arena and gradients."""
    ps, m, v, steps = rec["before"]
    k = opt.num_segments
    rows = {name: ([ps[i0 + s].clone() for s in range(k)], opt.lrs["row:" + name]) for name, i0 in opt.row_index.items()}
    tw = FusedAdam([[ps[6 * s + j].clone() for j in range(6)] for s in range(k)], lrs=dict(opt.lrs), rows=rows or None)
    tw.exp_avg.copy_(m)
    tw.exp_avg_sq.copy_(v)
    tw.steps[:] = steps
    kw = {key: rec[key] for key in ("present", "full_layout", "kinds", "row_grads") if rec.get(key) is not None}
    tw.step(rec["arena"], **kw)
    torch.cuda.synchronize()
    return tw


def check_step(opt, rec):
    """After ``rec``'s step: every tensor row whose flag byte is set equals the dense twin, every other row -- and every tensor
    that was not stepped -- kept its bits (parameter and both moments)."""
    tw = dense_twin(opt, rec)
    ps0, m0, v0, steps0 = rec["before"]
    present = rec["present"]
    counts = [int(opt._params[6 * s].shape[0]) for s in range(opt.num_segments)]
    frame0 = dict(zip(present, np.concatenate([[0], np.cumsum([counts[s] for s in present])[:-1]]).astype(int)))
    flags = rec["visible"].cpu().numpy()
    n = sum(counts[s] for s in present)
    if rec["radii"] is not None and rec["radii"].shape[0] == n:
        assert np.array_equal(flags[:n] != 0, rec["radii"].cpu().numpy() > 0)
    stepped_rows = 0
    for i, t in enumerate(opt._params):
        a0, b0 = int(opt.offsets[i]), int(opt.offsets[i]) + t.numel()
        got = (t.detach(), opt.exp_avg[a0:b0].view(t.shape), opt.exp_avg_sq[a0:b0].view(t.shape))
        old = (ps0[i], m0[a0:b0].view(t.shape), v0[a0:b0].view(t.shape))
        if opt.steps[i] == steps0[i] or t.numel() == 0:
            assert all(torch.equal(x, y) for x, y in zip(got, old)), i
            continue
        s = int(opt._sub_of[i])
        name = next((nm for nm, i0 in opt.row_index.items() if i0 <= i < i0 + opt.num_segments), None)
        r0 = (rec.get("row_flag_row0") or {}).get(name, [None] * opt.num_segments)[s] if name else None
        r0 = frame0[s] if r0 is None else r0
        seen = torch.from_numpy(flags[r0:r0 + counts[s]] != 0).to(DEV).view(-1, *([1] * (t.dim() - 1)))
        stepped_rows += int(seen.sum())
        twin = (tw._params[i], tw.exp_avg[a0:b0].view(t.shape), tw.exp_avg_sq[a0:b0].view(t.shape))
        for x, y, z in zip(got, twin, old):
            want = torch.where(seen, y, z)
            assert torch.equal(x.view(torch.int32), want.contiguous().view(torch.int32)), (i, name)
    return stepped_rows


def test_train_steps_keep_unseen_rows_and_match_the_dense_step_on_seen_rows():
    from street_gaussians_ns_b200.training import TrainStep
    sc, model, batch = _scene()
    opt = FusedAdam(model.optimizer_params())
    fn = TrainStep(model, opt, refine_every=100000, visible_adam=True)
    spy = StepSpy(model, opt)
    for k, step in enumerate(range(599, 603)):
        fn(step, sc.cameras[3 * k + 1], batch)
    assert len(spy.calls) == 4
    for rec in spy.calls:
        assert rec["visible"] is not None and rec["radii"] is not None
        r = rec["radii"].cpu().numpy()
        assert 0 < (r > 0).sum() < r.size  # some rows seen, some not: the test means something
        assert rec["stepped_rows"] > 0


def test_refinement_inside_the_run():
    from street_gaussians_ns_b200.training import TrainStep
    sc, model, batch = _scene()
    opt = FusedAdam(model.optimizer_params())
    fn = TrainStep(model, opt, visible_adam=True)  # the reference's per-sub-model cadence: a refinement at 600
    spy = StepSpy(model, opt)
    n0 = [s.num_points for s in model.all_models.values()]
    for k, step in enumerate(range(599, 603)):
        fn(step, sc.cameras[k + 1], batch)
        if step == 600:
            assert [s.num_points for s in model.all_models.values()] != n0
    assert len(spy.calls) == 4 and all(rec["stepped_rows"] > 0 for rec in spy.calls)  # steps 601, 602: the new layout


def test_accumulated_semantic_cycle_steps_the_union_of_its_frames():
    from street_gaussians_ns_b200.training import TrainStep
    sc, model, batch = _scene(semantic=True)
    opt = FusedAdam(model.optimizer_params(), rows={"semantic": (model.semantic_params(), 0.0025)})
    fn = TrainStep(model, opt, refine_every=100000, gradient_accumulation_steps={"semantic": 3}, visible_adam=True)
    spy = StepSpy(model, opt)
    names = list(model.all_models._modules)
    union = {}
    for k, step in enumerate(range(3, 6)):  # one cycle: 3 % 3 == 0 starts it, 5 is its due step
        fn(step, sc.cameras[4 * k], batch)
        rec = spy.calls[-1]
        flags = rec["visible"].cpu().numpy()
        r = 0
        for s in rec["present"]:
            n = model.all_models[names[s]].num_points
            union[s] = union.get(s, np.zeros(n, bool)) | (flags[r:r + n] != 0)
            r += n
    rec = spy.calls[-1]
    assert rec.get("row_grads") and "semantic" in rec["row_flag_row0"]
    # the mask the step read is the union of the cycle's frames, per sub-model
    flags = rec["visible"].cpu().numpy()
    for s, r0 in enumerate(rec["row_flag_row0"]["semantic"]):
        n = model.all_models[names[s]].num_points
        want = union.get(s, np.zeros(n, bool))
        assert np.array_equal(flags[r0:r0 + n] != 0, want), names[s]
    assert any(u.any() and not u.all() for u in union.values())
    assert rec["stepped_rows"] > 0
    # the steps before the due step left the logits alone
    for rec in spy.calls[:-1]:
        assert not rec.get("row_grads")


def test_off_is_unchanged(monkeypatch):
    from street_gaussians_ns_b200 import raster
    from street_gaussians_ns_b200.training import TrainStep
    monkeypatch.setattr(raster, "DETERMINISTIC", True)
    outs = []
    for kw in ({}, {"visible_adam": False}):
        sc, model, batch = _scene()
        opt = FusedAdam(model.optimizer_params())
        fn = TrainStep(model, opt, refine_every=100000, **kw)
        spy = StepSpy(model, opt, check=False)
        for k, step in enumerate(range(599, 602)):
            fn(step, sc.cameras[2 * k], batch)
        torch.cuda.synchronize()
        assert all(rec.get("visible") is None and "row_flag_row0" not in rec for rec in spy.calls)
        outs.append(([t.detach().clone() for t in opt._params], opt.exp_avg.clone(), opt.exp_avg_sq.clone()))
    (pa, ma, va), (pb, mb, vb) = outs
    assert all(torch.equal(a, b) for a, b in zip(pa, pb)) and torch.equal(ma, mb) and torch.equal(va, vb)
