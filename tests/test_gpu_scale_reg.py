"""The scale regularisation (csrc/scale_reg.cu) through its C entry points, the render node and the model, on the GPU.

Bars: against the float64 oracle (oracle/scale_reg_ref64.py) the value within 1e-6 relative and every gradient element within
1e-6 relative (plus 1e-6 of g = 0.1 v / N where the exact gradient cancels to 0); against torch's fp32 autograd of nerfstudio's
expression on the same GPU -- the reference for rows whose fp32 ratio sits exactly on max_ratio, where fp32 and float64 take
different branches -- 1e-6 relative.  Model gradients within 1e-5 relative L2 of the torch path."""
import ctypes as C

import numpy as np
import pytest
import torch

import street_gaussians_ns_b200.synthetic as syn
from oracle.scale_reg_ref64 import scale_reg, scale_reg_grad
from street_gaussians_ns_b200 import _lib, raster
from street_gaussians_ns_b200.model import ActorPose, SceneGraphConfig, SceneGraphRasterModel, _FullArenaSink
from street_gaussians_ns_b200.optim import FusedAdam
from street_gaussians_ns_b200.scene import PARAM_NAMES
from street_gaussians_ns_b200.training import TrainStep
from tests.scale_reg_cases import cases

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


class Table:
    """A hand-built device segment table over fresh scales tensors (the only field the kernels read), with a gradient table
    whose scales slices are pre-filled with random values."""

    def __init__(self, rows: np.ndarray, counts, posed=(), seed=0, prefill=1e-3):
        rows = np.ascontiguousarray(rows, np.float32)
        assert sum(counts) == rows.shape[0]
        rng = np.random.default_rng(seed)
        self.counts = np.asarray(counts, np.int64)
        o = np.concatenate([[0], np.cumsum(self.counts)])
        self.scales = [torch.from_numpy(rows[o[i]:o[i + 1]].copy()).to(DEV) for i in range(len(counts))]
        self.prefill = [torch.from_numpy(rng.standard_normal((n, 3)).astype(np.float32) * np.float32(prefill)).to(DEV) for n in counts]
        self.grads = [p.clone() for p in self.prefill]
        chunks = (self.counts + 127) // 128
        host = np.zeros(len(counts), raster.SEG_DTYPE)
        host["count"], host["row0"] = self.counts, o[:-1]
        host["chunk0"] = np.concatenate([[0], np.cumsum(chunks)[:-1]])
        host["scales"] = [t.data_ptr() for t in self.scales]
        host["has_pose"][list(posed)] = 1
        host["R"] = np.eye(3, dtype=np.float32).reshape(-1)
        self.dev = torch.from_numpy(host.view(np.uint8).reshape(-1)).to(DEV)
        gt = np.zeros((len(counts), 6), np.uint64)
        gt[:, 1] = [t.data_ptr() for t in self.grads]
        self.gdev = torch.from_numpy(gt.view(np.uint8).reshape(-1)).to(DEV)
        self.nseg, self.N, self.num_chunks = len(counts), int(self.counts.sum()), int(chunks.sum())
        self.rows = rows


def fwd(tab: Table, max_ratio: float) -> torch.Tensor:
    L = _lib.load()
    out = torch.full((1,), -1.0, device=DEV)
    sb = L.sgn_scale_reg_scratch_bytes()
    scratch = torch.empty(sb, device=DEV, dtype=torch.uint8)
    _lib.check(L.sgn_scale_reg_fwd(_ptr(tab.dev), tab.nseg, tab.N, tab.num_chunks, max_ratio, _ptr(out), _ptr(scratch), sb, _stream()),
               "sgn_scale_reg_fwd")
    return out


def bwd(tab: Table, max_ratio: float, v: float) -> None:
    L = _lib.load()
    vt = torch.tensor([v], device=DEV, dtype=torch.float32)
    _lib.check(L.sgn_scale_reg_bwd(_ptr(tab.dev), _ptr(tab.gdev), tab.nseg, tab.N, tab.num_chunks, max_ratio, _ptr(vt), _stream()),
               "sgn_scale_reg_bwd")


def torch_fp32(rows: torch.Tensor, max_ratio: float, v: float):
    """nerfstudio's expression in fp32 on the GPU: (value, gradient, ratio per row)."""
    x = rows.clone().requires_grad_(True)
    s = torch.exp(x)
    r = s.amax(dim=-1) / s.amin(dim=-1)
    val = 0.1 * (torch.maximum(r, torch.tensor(max_ratio, device=DEV)) - max_ratio).mean()
    (val * v).backward()
    return val.detach(), x.grad, r.detach()


ALL = cases(dtype=np.float32)
MIXED = np.concatenate([ALL[k] for k in sorted(ALL)])


def _mixed(n, seed):
    rng = np.random.default_rng(seed)
    idx = rng.integers(0, MIXED.shape[0], n)
    return MIXED[idx] + rng.uniform(-0.5, 0.5, (n, 1)).astype(np.float32)  # a common shift keeps ratios and ties


def _on_device_ties(max_ratio, n, seed=0):
    """Rows [a, a, b] whose fp32 ratio on this GPU is exactly max_ratio (found with torch.exp on the device)."""
    rng = np.random.default_rng(seed)
    a = rng.uniform(-6, 1, 20000).astype(np.float32)
    b = (a + np.float32(np.log(max_ratio))).astype(np.float32)
    cand = np.stack([b, np.nextafter(b, np.float32(np.inf)), np.nextafter(b, np.float32(-np.inf))], 1)
    ea = torch.exp(torch.from_numpy(a).to(DEV))[:, None]
    ok = (torch.exp(torch.from_numpy(cand).to(DEV)) / ea == max_ratio).cpu().numpy()
    has = ok.any(1)
    pick = cand[np.arange(a.size), ok.argmax(1)][has][:n]
    a = a[has][:n]
    assert a.size == n
    return np.stack([a, a, pick], 1).astype(np.float32)


TABLES = {
    "one_row": ([1], ()),
    "127_1_129": ([127, 1, 129], (1, 2)),
    "empty_segments": ([0, 300, 0, 0, 5, 128], (2, 3, 4)),
    "33_segments": ([1000] + [int(x) for x in np.random.default_rng(33).integers(0, 700, 32)], tuple(range(1, 33))),
    "multi_chunk": ([128 * 40 + 17], ()),
}


def _rows_for(counts, seed, ties=0, max_ratio=10.0):
    n = int(sum(counts))
    rows = _mixed(n, seed)
    if ties:
        k = min(ties, n)
        rows[np.random.default_rng(seed + 1).choice(n, k, replace=False)] = _on_device_ties(max_ratio, k, seed)
    return rows


def check_directed(tab: Table, max_ratio: float, v: float = 0.7):
    val = fwd(tab, max_ratio)
    again = fwd(tab, max_ratio)
    torch.cuda.synchronize()
    assert torch.equal(val, again)
    want = scale_reg(tab.rows, max_ratio)
    # rows whose ratio is within a few fp32 ulps of max_ratio add terms that fp32 exp / division cannot resolve: their rounding
    # (a few ulps of the ratio each, as torch's fp32 has it too) is allowed on top of the relative bar
    s64 = np.exp(tab.rows.astype(np.float64))
    r64 = s64.max(1) / s64.min(1)
    near = np.where(r64 > max_ratio * (1 - 1e-5), 4 * 2.0 ** -23 * r64, 0.0)
    tol_val = 1e-6 * abs(want) + 0.1 * float(near.mean() if near.size else 0.0) + 1e-12
    assert abs(float(val) - want) <= tol_val, (float(val), want)
    bwd(tab, max_ratio, v)
    torch.cuda.synchronize()
    got = torch.cat(tab.grads).double().cpu().numpy()
    pre = torch.cat(tab.prefill).double().cpu().numpy()
    rows_t = torch.from_numpy(tab.rows).to(DEV)
    tv, tg, r32 = torch_fp32(rows_t, max_ratio, v)
    r32 = r32.cpu().numpy()
    below = r32 < np.float32(max_ratio)
    # rows without a gradient are not written: the pre-filled values come back exactly
    assert np.array_equal(torch.cat(tab.grads).cpu().numpy()[below], torch.cat(tab.prefill).cpu().numpy()[below])
    added = got - pre
    ulp = 2.0 * np.spacing(np.abs(got).astype(np.float32)).astype(np.float64)  # the rounding of the add into the pre-filled arena
    g_scale = 0.1 * abs(v) / max(tab.N, 1)
    # against float64 where fp32 and float64 take the same branch of max(r, max_ratio)
    same = ((r32 >= max_ratio) == (r64 >= max_ratio)) & (r32 != np.float32(max_ratio)) & (r64 != max_ratio)
    want_g = scale_reg_grad(tab.rows, max_ratio, v)
    err = np.abs(added - want_g)[same]
    tol = (1e-6 * np.abs(want_g) + 1e-6 * g_scale + ulp)[same]
    assert (err <= tol).all(), float((err - tol).max())
    # against torch's fp32 autograd on every row, ties on max_ratio included
    tg = tg.double().cpu().numpy()
    assert (np.abs(added - tg) <= 1e-6 * np.abs(tg) + 1e-6 * g_scale + ulp).all()
    assert abs(float(val) - float(tv)) <= 1e-6 * abs(float(tv)) + 1e-12
    return val


@pytest.mark.parametrize("name", list(TABLES))
@pytest.mark.parametrize("max_ratio", [10.0, 2.5])
def test_directed_tables(name, max_ratio):
    counts, posed = TABLES[name]
    rows = _rows_for(counts, seed=len(counts), ties=20, max_ratio=max_ratio)
    check_directed(Table(rows, counts, posed), max_ratio)


@pytest.mark.parametrize("case", sorted(ALL))
def test_each_case(case):
    rows = ALL[case]
    n = rows.shape[0]
    check_directed(Table(rows, [n // 3, 0, n - n // 3], posed=(2,)), 10.0, v=1.9)


def test_three_way_tie_at_max_ratio_one():
    rows = ALL["all_equal"]
    check_directed(Table(rows, [rows.shape[0]]), 1.0)


def test_fp32_ties_take_half():
    rows = _on_device_ties(10.0, 300)
    tab = Table(rows, [300])
    check_directed(tab, 10.0)
    # exactly half of what the same rows get with a threshold one fp32 step lower (zero pre-fill: the gradients themselves)
    half, full = Table(rows, [300], prefill=0.0), Table(rows, [300], prefill=0.0)
    bwd(half, 10.0, 1.0)
    bwd(full, float(np.nextafter(np.float32(10.0), np.float32(0.0))), 1.0)
    torch.cuda.synchronize()
    assert float(full.grads[0].abs().min()) > 0
    assert torch.equal(2.0 * half.grads[0], full.grads[0])


@pytest.mark.parametrize("n", [1, 129, 1 << 20, 3_000_001])
def test_row_counts(n):
    rows = _rows_for([n], seed=n, ties=50)
    counts = [n] if n < 1000 else [n // 2 - 3, 0, 77, n - n // 2 - 74]
    check_directed(Table(rows, counts, posed=tuple(range(1, len(counts)))), 10.0)


def test_zero_rows_is_nan_and_launches_nothing_backward():
    tab = Table(np.zeros((0, 3), np.float32), [])
    L = _lib.load()
    out = fwd(tab, 10.0)
    torch.cuda.synchronize()
    assert torch.isnan(out).all()
    n0 = L.sgn_launch_count()
    bwd(tab, 10.0, 1.0)
    assert L.sgn_launch_count() == n0


def test_errors_launch_nothing():
    L = _lib.load()
    tab = Table(_mixed(200, 1), [200])
    out = torch.empty(1, device=DEV)
    sb = L.sgn_scale_reg_scratch_bytes()
    scratch = torch.empty(sb, device=DEV, dtype=torch.uint8)
    v = torch.ones(1, device=DEV)
    n0 = L.sgn_launch_count()
    s = _stream()
    assert L.sgn_scale_reg_fwd(None, 1, 200, 2, 10.0, _ptr(out), _ptr(scratch), sb, s) == -1
    assert L.sgn_scale_reg_fwd(_ptr(tab.dev), 1, 200, 2, 10.0, None, _ptr(scratch), sb, s) == -1
    assert L.sgn_scale_reg_fwd(_ptr(tab.dev), 1, 200, 2, 10.0, _ptr(out), None, sb, s) == -1
    assert L.sgn_scale_reg_fwd(_ptr(tab.dev), 0, 200, 2, 10.0, _ptr(out), _ptr(scratch), sb, s) == -1
    assert L.sgn_scale_reg_fwd(_ptr(tab.dev), 1, -1, 2, 10.0, _ptr(out), _ptr(scratch), sb, s) == -1
    assert L.sgn_scale_reg_fwd(_ptr(tab.dev), 1, 200, 2, 10.0, _ptr(out), _ptr(scratch), sb - 1, s) == -3
    assert L.sgn_scale_reg_bwd(None, _ptr(tab.gdev), 1, 200, 2, 10.0, _ptr(v), s) == -1
    assert L.sgn_scale_reg_bwd(_ptr(tab.dev), None, 1, 200, 2, 10.0, _ptr(v), s) == -1
    assert L.sgn_scale_reg_bwd(_ptr(tab.dev), _ptr(tab.gdev), 1, 200, 2, 10.0, None, s) == -1
    assert L.sgn_scale_reg_bwd(_ptr(tab.dev), _ptr(tab.gdev), 0, 200, 2, 10.0, _ptr(v), s) == -1
    assert L.sgn_launch_count() == n0
    assert b"sgn_scale_reg_bwd" in L.sgn_last_error()
    torch.cuda.synchronize()
    assert torch.equal(torch.cat(tab.grads), torch.cat(tab.prefill))


# ---- model -----------------------------------------------------------------------------------------------------------

def _needles(model, every=7, by=3.0):
    """Stretch one axis of every ``every``-th row by e^by so that many rows are above max_gauss_ratio."""
    with torch.no_grad():
        for sub in model.all_models.values():
            sc = sub.gauss_params["scales"]
            sc[::every, 0] += by


def _small_model(seed=3, actors=True, **cfg):
    fr = syn.make_frame(n_background=20000, n_actors=3 if actors else 0, n_per_actor=1500, width=320, height=240, seed=seed,
                        actor_shift=np.array([1.0, 0.0, -1.0]))
    poses = [ActorPose(s.name.replace("object_", ""), s.rot, s.center, 21, list(range(85))) for s in fr.segments[1:]]
    # one more actor that is never in view: its rows must get no gradient
    extra = syn.make_actor(500, seed=99)
    actors_ = {s.name.replace("object_", ""): s.params.to(DEV) for s in fr.segments[1:]}
    actors_["hidden"] = extra.to(DEV)
    model = SceneGraphRasterModel(fr.segments[0].params.to(DEV), actors_, SceneGraphConfig(use_sky_sphere=False, **cfg),
                                  poses_at=lambda t: poses).to(DEV)
    model.train()
    _needles(model)
    gt = torch.rand(240, 320, 3, generator=torch.Generator().manual_seed(2)).to(DEV)
    return fr, model, gt


def _cfg4_model(**cfg):
    sc = syn.WaymoScene()
    frame_list = list(range(sc.num_frames))

    def poses_at(t):
        f = int(t)
        return [ActorPose(str(a), rot, center, f, frame_list, frame_id=f) for a, rot, center in sc.boxes_at(f)]
    model = SceneGraphRasterModel(sc.background.to(DEV), {k: v.to(DEV) for k, v in sc.actors.items()},
                                  SceneGraphConfig(use_sky_sphere=False, **cfg), poses_at=poses_at).to(DEV)
    model.train()
    _needles(model)
    gt = (torch.rand(sc.height, sc.width, 3, generator=torch.Generator().manual_seed(5)) * 255).to(torch.uint8).to(DEV)
    return sc, model, gt


def _grads(model):
    return {(n, k): (None if sub.gauss_params[k].grad is None else sub.gauss_params[k].grad.detach().clone())
            for n, sub in model.all_models.items() for k in PARAM_NAMES}


def _zero(model):
    for p in model.parameters():
        p.grad = None


def _run(model, camera, batch, step):
    _zero(model)
    model.step = step
    out = model.get_outputs(camera)
    losses = model.get_loss_dict(out, batch)
    sum(losses.values()).backward()
    torch.cuda.synchronize()
    return out, losses, _grads(model)


def rel_l2(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


def test_model_parity_cfg4(monkeypatch):
    monkeypatch.setattr(raster, "DETERMINISTIC", True)
    sc, model, gt = _cfg4_model(use_scale_regularization=True)
    cam = sc.cameras[5 * 40 + 1]
    batch = {"image": gt}
    out_on, losses_on, g_on = _run(model, cam, batch, 20)
    visible = list(model.visible_model_names)
    assert len(visible) > 1
    model.config.use_scale_regularization = False
    out_off, losses_off, g_off = _run(model, cam, batch, 20)
    assert "scale_reg" not in losses_off
    # the torch path's term over the visible rows
    model.config.use_scale_regularization, model.config.fused_loss = True, False
    reg_t = model._scale_reg_loss(fused=False)
    assert float(losses_on["scale_reg"].detach()) == pytest.approx(float(reg_t.detach()), rel=1e-6)
    assert float(losses_on["scale_reg"].detach()) > 0
    sc_t = torch.autograd.grad(reg_t, [model.all_models[n].gauss_params["scales"] for n in visible])
    for (n, k), g in g_on.items():
        if n not in visible:
            assert g is None and g_off[(n, k)] is None
        elif k == "scales":
            assert rel_l2(g, g_off[(n, k)] + sc_t[visible.index(n)]) < 1e-5, n
            assert not torch.equal(g, g_off[(n, k)])
        else:
            assert torch.equal(g, g_off[(n, k)]), (n, k)
    for k in out_off:
        assert torch.equal(out_on[k], out_off[k]), k
    # the full torch path through get_loss_dict gives the same value
    losses_t = model.get_loss_dict(out_off, batch)
    assert float(losses_t["scale_reg"].detach()) == pytest.approx(float(losses_on["scale_reg"].detach()), rel=1e-6)


def test_one_adam_step_lowers_the_ratio_of_rows_above():
    fr, model, gt = _small_model(use_scale_regularization=True)
    model.step = 20
    out = model.get_outputs(fr.camera)
    losses = model.get_loss_dict(out, {"image": gt})
    _zero(model)
    losses["scale_reg"].backward()
    before = {n: model.all_models[n].gauss_params["scales"].detach().clone() for n in model.visible_model_names}
    opt = FusedAdam(model.optimizer_params())
    present = model.present_submodels()
    opt.step(model._holder.grad_arena, present=present)
    torch.cuda.synchronize()
    n_above = 0
    for n, x0 in before.items():
        x1 = model.all_models[n].gauss_params["scales"].detach()
        s0, s1 = torch.exp(x0), torch.exp(x1)
        r0 = s0.amax(-1) / s0.amin(-1)
        r1 = s1.amax(-1) / s1.amin(-1)
        above = r0 > 10.0
        n_above += int(above.sum())
        assert (r1[above] < r0[above]).all(), n
        assert torch.equal(x1[r0 < 10.0], x0[r0 < 10.0]), n
    assert n_above > 100


def test_gating_and_off_path_bits(monkeypatch):
    monkeypatch.setattr(raster, "DETERMINISTIC", True)
    assert SceneGraphConfig().use_scale_regularization is False
    res = {}
    for on in (False, True):
        fr, model, gt = _small_model(use_scale_regularization=on)
        for step in (21, 20):
            out, losses, g = _run(model, fr.camera, {"image": gt}, step)
            res[(on, step)] = (out, losses, g)
    for step in (21, 20):
        out0, l0, g0 = res[(False, step)]
        out1, l1, g1 = res[(True, step)]
        assert "scale_reg" not in l0 and "scale_reg" in l1
        assert all(torch.equal(out0[k], out1[k]) for k in out0) and out0.keys() == out1.keys()
        assert all(torch.equal(l0[k], l1[k]) for k in l0)
        if step == 21:  # a zero without gradient, and every gradient the same bits
            assert float(l1["scale_reg"]) == 0.0 and not l1["scale_reg"].requires_grad
            assert all((a is None and b is None) or torch.equal(a, b) for a, b in zip(g0.values(), g1.values()))
        else:
            assert l1["scale_reg"].requires_grad and float(l1["scale_reg"]) > 0


def test_gradient_accumulation_gives_the_sum(monkeypatch):
    monkeypatch.setattr(raster, "DETERMINISTIC", True)
    fr, model, gt = _small_model(use_scale_regularization=True)
    _, _, g1 = _run(model, fr.camera, {"image": gt}, 20)
    out = model.get_outputs(fr.camera)  # .grad still set: the render's arena is added in
    sum(model.get_loss_dict(out, {"image": gt}).values()).backward()
    torch.cuda.synchronize()
    g2 = _grads(model)
    for key, a in g1.items():
        if a is None:
            assert g2[key] is None
        else:
            assert torch.equal(g2[key], a + a), key


def test_level0_forward_backward_matches_render(monkeypatch):
    monkeypatch.setattr(raster, "DETERMINISTIC", True)
    fr, model, gt = _small_model(use_scale_regularization=True)
    frame = model._frame(fr.camera)
    settings = model._settings(class_streams=True)
    w, a = (t.to(DEV) for t in syn.cotangents(240, 320))
    a = a[..., None].contiguous()
    params = [t for seg in frame.segments for t in seg.params.tensors()]
    for p in params:
        p.grad = None
    out, h = raster.render_frame(frame, settings, scale_reg=10.0)
    v = torch.tensor(0.37, device=DEV)
    torch.autograd.backward([out["rgb"], out["accumulation"], out["scale_reg"]], [w, a, v])
    res, h0 = raster.forward_backward(frame, settings, {"rgb": w, "accumulation": a, "scale_reg": v}, scale_reg=10.0)
    torch.cuda.synchronize()
    assert torch.equal(res["scale_reg"], out["scale_reg"].detach())
    assert torch.equal(h0.grad_arena, h.grad_arena)


@pytest.mark.parametrize("fused_loss", [True, False])
def test_nothing_in_view_steps_only_the_scales(fused_loss):
    """After a step in view (non-zero moments everywhere), a frame with nothing in view steps the scales of the frame's
    sub-models and nothing else: the other five tensors keep their values, moments and step counts, as torch.optim.Adam skips
    a parameter whose grad is None.  The same on the torch path, whose term never reaches the render."""
    fr, model, gt = _small_model(use_scale_regularization=True, fused_loss=fused_loss)
    c2w = np.array([[-1, 0, 0, 0], [0, 1, 0, 0], [0, 0, -1, 1e5]], np.float32)  # far away, looking away from the scene
    cam = syn.make_camera(320, 240, c2w=c2w, time=21.0)
    opt = FusedAdam(model.optimizer_params())
    step_fn = TrainStep(model, opt, refine_every=100000)
    step_fn(19, fr.camera, {"image": gt})
    visible = list(model.visible_model_names)
    subs = list(model.all_models)
    state = {}
    for n in visible:
        for j, k in enumerate(PARAM_NAMES):
            i = 6 * subs.index(n) + j
            m_, v_ = opt.moment_views(i)
            assert float(m_.abs().max()) > 0 or k == "features_rest"
            state[(n, k)] = (model.all_models[n].gauss_params[k].detach().clone(), m_.clone(), v_.clone(), int(opt.steps[i]))
    step_fn(20, cam, {"image": gt})
    torch.cuda.synchronize()
    assert model._holder.M == 0
    for n in visible:
        for j, k in enumerate(PARAM_NAMES):
            i = 6 * subs.index(n) + j
            x0, m0, v0, st0 = state[(n, k)]
            m_, v_ = opt.moment_views(i)
            x1 = model.all_models[n].gauss_params[k].detach()
            if k == "scales":
                assert not torch.equal(x1, x0) and int(opt.steps[i]) == st0 + 1, n
            else:
                assert torch.equal(x1, x0) and torch.equal(m_, m0) and torch.equal(v_, v0) and int(opt.steps[i]) == st0, (n, k)


def test_nothing_in_view_gradient_is_the_term():
    fr, model, gt = _small_model(use_scale_regularization=True)
    c2w = np.array([[-1, 0, 0, 0], [0, 1, 0, 0], [0, 0, -1, 1e5]], np.float32)
    cam = syn.make_camera(320, 240, c2w=c2w, time=21.0)
    model.step = 20
    out = model.get_outputs(cam)
    assert model._holder.M == 0 and float(out["rgb"].abs().sum()) == 0
    losses = model.get_loss_dict(out, {"image": gt})
    assert losses["scale_reg"].requires_grad
    _zero(model)
    losses["scale_reg"].backward()
    torch.cuda.synchronize()
    visible = list(model.visible_model_names)
    rows = torch.cat([model.all_models[n].gauss_params["scales"].detach() for n in visible]).cpu().numpy()
    want = scale_reg_grad(rows, 10.0)
    got = torch.cat([model.all_models[n].gauss_params["scales"].grad for n in visible]).double().cpu().numpy()
    assert np.abs(got - want).max() <= 1e-5 * np.abs(want).max()
    for n in visible:
        assert float(model.all_models[n].gauss_params["means"].grad.abs().max()) == 0.0


@pytest.mark.parametrize("full_arena", [False, True])
def test_train_step_torch_path_matches_fused(monkeypatch, full_arena):
    """One TrainStep at step 20 from the same state: the torch path's term (whose gradient reaches .grad before the render's
    backward runs) is in the arena the optimizer steps, as the fused path's is.  Each path's term is its arena minus the arena
    of the same path with the switch off."""
    monkeypatch.setattr(raster, "DETERMINISTIC", True)
    res = {}
    for fused in (True, False):
        for on in (True, False):
            fr, model, gt = _small_model(use_scale_regularization=on, fused_loss=fused, ssim_lambda=0.0,
                                         full_gradient_arena=full_arena)
            opt = FusedAdam(model.optimizer_params())
            stepped = []
            real = opt.step

            def spy(arena, *a, _real=real, _out=stepped, **k):
                _out.append(arena.clone())
                return _real(arena, *a, **k)
            opt.step = spy
            losses = TrainStep(model, opt, refine_every=100000)(20, fr.camera, {"image": gt})
            torch.cuda.synchronize()
            assert ("scale_reg" in losses) == on and len(stepped) == 1
            visible = list(model.visible_model_names)
            grads = {n: model.all_models[n].gauss_params["scales"].grad.detach().clone() for n in visible}
            scales = {n: model.all_models[n].gauss_params["scales"].detach().clone() for n in visible}
            res[(fused, on)] = (grads, scales, stepped[0], visible)
    (gf, sf, af, vis), (gfo, _, afo, _) = res[(True, True)], res[(True, False)]
    (gt_, st, at, _), (gto, _, ato, _) = res[(False, True)], res[(False, False)]
    assert af.shape == at.shape
    term_f, term_t = af - afo, at - ato
    assert float(term_f.abs().max()) > 0
    assert rel_l2(term_t, term_f) < 1e-5  # the arenas the optimizer read carry the same term
    for n in vis:
        assert rel_l2(gt_[n] - gto[n], gf[n] - gfo[n]) < 1e-5, n  # and .grad agrees with them
        d = (st[n] - sf[n]).abs()
        assert float((d > 1e-6).float().mean()) < 1e-4, n


def test_level0_refuses_ranged_exchange_with_the_term():
    fr, model, gt = _small_model(use_scale_regularization=True)
    frame = model._frame(fr.camera)
    with pytest.raises(AssertionError):
        raster.forward_backward(frame, model._settings(class_streams=True), {}, scale_reg=10.0, chunk_ranges=[(0, 1)])


def test_eval_does_not_render_the_term():
    fr, model, gt = _small_model(use_scale_regularization=True)
    model.step = 20
    out = model.get_outputs(fr.camera)
    train_val = float(model.get_loss_dict(out, {"image": gt})["scale_reg"].detach())
    model.eval()
    out = model.get_outputs_for_camera(fr.camera)
    assert model.__dict__.get("_scale_reg") is None
    with torch.no_grad():
        v = model.get_loss_dict(out, {"image": gt})["scale_reg"]
    assert not v.requires_grad and float(v) == train_val


def test_deterministic_steps_repeat_bit_for_bit(monkeypatch):
    monkeypatch.setattr(raster, "DETERMINISTIC", True)
    runs = []
    for _ in range(2):
        fr, model, gt = _small_model(use_scale_regularization=True)
        opt = FusedAdam(model.optimizer_params())
        step_fn = TrainStep(model, opt, refine_every=100000)
        for s in (20, 21, 30):
            losses = step_fn(s, fr.camera, {"image": gt})
            assert "scale_reg" in losses
        torch.cuda.synchronize()
        runs.append({n: p.detach().clone() for n, p in model.named_parameters()})
    a, b = runs
    assert a.keys() == b.keys()
    assert not [k for k in a if not torch.equal(a[k], b[k])]


def test_data_parallel_refuses_the_term(monkeypatch):
    fr, model, gt = _small_model(use_scale_regularization=True)
    opt = FusedAdam(model.optimizer_params())
    step_fn = TrainStep(model, opt, refine_every=100000)
    monkeypatch.setattr(step_fn, "world_size", lambda: 2)
    model.config.full_gradient_arena = True
    model._grad_sink = _FullArenaSink()
    called = []
    monkeypatch.setattr(model, "get_outputs", lambda camera: called.append(camera))
    with pytest.raises(NotImplementedError):
        step_fn(20, fr.camera, {"image": gt}, all_cameras=[fr.camera, fr.camera])
    assert not called
