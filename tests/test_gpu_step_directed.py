"""The step kernels after the render -- the loss epilogue, the densification statistics, the fused Adam and the gradient
exchange -- on hand-built inputs (tests/step_cases.py) against the host statements of oracle/step_ref64.py, through the C
entry points of libsgn_raster.so.

  * sgn_loss_fwd / sgn_loss_bwd: images from 1x1 to 1920x1280, float and uint8 ground truth, with and without a mask,
    views offset by 1..3 floats / bytes (the scalar loops), each term alone, grad_losses null and not, every output
    pointer null alone.  The L1 and sky cotangents equal the float32 replay bit for bit (ties give exactly 0); the entropy
    cotangent is within 4 U k (|log oa| + |log(1 - oa)|) of float64; each forward term is within step_ref64.loss_fwd_bound
    (first-order rounding of the summation tree, doubled) and bit-identical across two runs.
  * sgn_densify_stats: one, 33 and 1024 segments, empty segments, a first row0 > 0 with gaps, mixed ``first`` flags, two
    calls in a row.  Each segment's statistics sit inside a larger buffer filled with a canary pattern, with a margin in
    front of at least the first segment's row0 and behind of at least the rows up to the next segment: a write at a
    negative or too-large index lands in memory this test owns.  Every element is bit-equal to the replay and every
    canary is untouched.
  * sgn_adam_step / FusedAdam: tensors of 0 .. 8193 elements (empty ones first, in the middle and last), parameters at
    aligned and misaligned addresses (the scalar path), a gradient at a negative grad_offset, zero and tiny gradients,
    steps 1..5 with sub-models absent, 8192 tensors (8193 refused), tables cut by rows_in_range / rows_in_slices.  All
    bit-equal to the float32 replay (the kernel's sqrtf and division are IEEE, so the replay is exact).
  * sgn_allreduce_sym without multicast, emulated on one GPU: the ``world`` replicas are buffers on this device listed in
    the peer table, and ranks 0 .. world-1 are launched in order on one stream.  That order meets the kernel's contract:
    each rank reduces only its own part, and every other part is still unreduced when its owner runs.  Every live float4
    equals the rank-order fp32 sum times ``scale`` on every replica; skipped units, padding and the gaps between slices
    keep what was written (non-zero values, so a unit exchanged by mistake shows).  The multicast path
    (multimem.ld_reduce / st) needs an NVSwitch fabric and is checked by tools/test_collective.py on several GPUs.
  * Argument errors of the four entry points.

Observed on an H100 80GB HBM3 (700 W power limit): 289 tests in 28 s.  Nine one-token mutants each fail this file: the
densify kernel without its `i < 0` return and with `i > count` (2 tests each, the tables with a first row0 > 0), the
entropy clamp's open interval (111), `n3 % 2` in the forward (6) and the backward (4), the scalar Adam loop's `k < 3` (3),
and in rows_unseen / my_part `rem + 3 > w` (16), `ra + more` unclamped (20) and `len4 / world` (29).  test_gpu_model.py,
test_gpu_adam.py and test_reference_vectors.py catch none of the five of them that are safe to run there.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from street_gaussians_ns_b200 import _lib
from street_gaussians_ns_b200.optim import ADAM_DTYPE, FusedAdam
from oracle import step_ref64 as ref
from tests import step_cases as sc

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
ERR_INVALID, ERR_WORKSPACE = -1, -3
f32 = np.float32
CANARY = np.int32(0x7FBADBAD)  # a NaN payload no kernel writes


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def host(t):
    torch.cuda.synchronize()
    return t.cpu().numpy()


def bits(a):
    return np.ascontiguousarray(a, dtype=f32).view(np.int32)


def placed(arr: np.ndarray, off_elems: int):
    """A device copy of ``arr`` starting ``off_elems`` elements past a 16-byte boundary (the buffer keeps it alive)."""
    flat = np.ascontiguousarray(arr).reshape(-1)
    per16 = 16 // flat.itemsize
    buf = torch.zeros(flat.size + per16 + 16, dtype=torch.from_numpy(flat[:0]).dtype, device=DEV)
    v = buf[off_elems:off_elems + flat.size]
    assert (v.data_ptr() % 16) // flat.itemsize == off_elems
    v.copy_(torch.from_numpy(flat))
    return v


def L():
    return _lib.load()


# ---- loss epilogue ------------------------------------------------------------------------------------------------------
def loss_in(c: sc.LossCase, d: dict):
    li, keep = _lib.LossIn(), []
    o_rgb, o_gt, _ = c.off

    def put(name, arr, off=0):
        if arr is not None:
            t = placed(arr, off)
            keep.append(t)
            setattr(li, name, t.data_ptr())
    put("rgb", d["rgb"], o_rgb)
    if d["gt"] is not None:
        put("gt_u8" if d["gt"].dtype == np.uint8 else "gt_f32", d["gt"], c.u8_off if d["gt"].dtype == np.uint8 else o_gt)
    put("mask", d["mask"])
    put("accumulation", d["accumulation"])
    put("sky_mask", d["sky_mask"])
    put("object_acc", d["object_acc"])
    li.w_l1, li.w_sky, li.w_entropy = c.w
    return li, keep


def loss_fwd(c, li):
    sb = L().sgn_loss_scratch_bytes()
    scratch = torch.full((sb,), 0xFF, dtype=torch.uint8, device=DEV)
    out = torch.full((3,), float("nan"), device=DEV)
    _lib.check(L().sgn_loss_fwd(c.H, c.W, C.byref(li), _p(out), _p(scratch), sb, None), "sgn_loss_fwd")
    return host(out)


def loss_bwd(c, li, g, outs=("rgb", "acc", "obj")):
    P = c.P
    o_v = c.off[2]
    v_rgb = placed(np.full(3 * P, np.nan, f32), o_v) if "rgb" in outs else None
    v_acc = torch.full((P,), float("nan"), device=DEV) if "acc" in outs else None
    v_obj = torch.full((P,), float("nan"), device=DEV) if "obj" in outs else None
    gd = None if g is None else torch.tensor(g, dtype=torch.float32, device=DEV)
    _lib.check(L().sgn_loss_bwd(c.H, c.W, C.byref(li), _p(gd), _p(v_rgb), _p(v_acc), _p(v_obj), None), "sgn_loss_bwd")
    return [None if t is None else host(t) for t in (v_rgb, v_acc, v_obj)]


@pytest.mark.parametrize("case", sc.LOSS_CASES, ids=lambda c: c.name)
def test_loss_forward_within_bound_and_deterministic(case):
    d = sc.loss_inputs(case)
    li, keep = loss_in(case, d)
    a, b = loss_fwd(case, li), loss_fwd(case, li)
    assert np.array_equal(bits(a), bits(b))
    want = ref.loss_fwd64(case.P, **d, w=case.w)
    bound = ref.loss_fwd_bound(case.P, **d, w=case.w)
    err = np.abs(a.astype(np.float64) - want)
    assert np.all(err <= bound), (a, want, err, bound)
    for i, t in enumerate(("l1", "sky", "ent")):
        if t not in case.terms or case.w[i] == 0.0:
            assert a[i] == 0.0, t


def _check_bwd(case, d, got, g):
    gg = (1.0, 1.0, 1.0) if g is None else g
    v_rgb, v_acc, _ = ref.loss_bwd_f32(case.P, d["rgb"], d["gt"], d["mask"], d["sky_mask"], d["object_acc"], case.w, gg)
    if got[0] is not None:
        if v_rgb is None:
            v_rgb = np.full(3 * case.P, np.nan, f32)   # no rgb input: the output is not written
        assert np.array_equal(bits(got[0]), bits(v_rgb)), np.flatnonzero(bits(got[0]) != bits(v_rgb))[:10]
    if got[1] is not None:
        assert np.array_equal(bits(got[1]), bits(v_acc))
    if got[2] is not None:
        if d["object_acc"] is None:
            assert np.all(np.isnan(got[2]))
        else:
            want = ref.ent_bwd64(case.P, d["object_acc"], case.w[2], gg[2])
            bound = ref.ent_bwd_bound(case.P, d["object_acc"], case.w[2], gg[2])
            err = np.abs(got[2].astype(np.float64) - want)
            assert np.all(err <= bound), (np.max(err - bound), np.argmax(err - bound))
            x = d["object_acc"].reshape(-1)
            outside = (x < ref.CLAMP_LO) | (x > ref.CLAMP_HI)
            assert np.all(got[2][outside] == 0)


@pytest.mark.parametrize("case", sc.LOSS_CASES, ids=lambda c: c.name)
def test_loss_backward_matches_replay(case):
    d = sc.loss_inputs(case)
    li, keep = loss_in(case, d)
    for g in (None, (0.7, -1.3, 2.5)):
        _check_bwd(case, d, loss_bwd(case, li, g), g)
    if d["rgb"] is not None:   # ties: exactly zero
        tie = (ref.gt_f32(d["gt"]) == d["rgb"]).reshape(-1)
        got = loss_bwd(case, li, None, ("rgb",))[0]
        assert np.all(got[tie] == 0)


@pytest.mark.parametrize("case", [c for c in sc.LOSS_CASES if c.P <= 256 and c.terms == ("l1", "sky", "ent")][:8],
                         ids=lambda c: c.name)
def test_loss_backward_each_output_null_alone(case):
    d = sc.loss_inputs(case)
    li, keep = loss_in(case, d)
    for drop in ("rgb", "acc", "obj"):
        outs = tuple(x for x in ("rgb", "acc", "obj") if x != drop)
        _check_bwd(case, d, loss_bwd(case, li, (0.5, 2.0, -3.0), outs), (0.5, 2.0, -3.0))


def test_loss_argument_errors():
    c = sc.LossCase("e", 4, 4)
    d = sc.loss_inputs(c)
    li, keep = loss_in(c, d)
    sb = L().sgn_loss_scratch_bytes()
    assert sb == 3 * 1056 * 4
    scratch = torch.zeros(sb, dtype=torch.uint8, device=DEV)
    out = torch.zeros(3, device=DEV)
    assert L().sgn_loss_fwd(0, 4, C.byref(li), _p(out), _p(scratch), sb, None) == ERR_INVALID
    assert L().sgn_loss_fwd(4, -1, C.byref(li), _p(out), _p(scratch), sb, None) == ERR_INVALID
    assert L().sgn_loss_fwd(4, 4, None, _p(out), _p(scratch), sb, None) == ERR_INVALID
    assert L().sgn_loss_fwd(4, 4, C.byref(li), None, _p(scratch), sb, None) == ERR_INVALID
    assert L().sgn_loss_fwd(4, 4, C.byref(li), _p(out), None, sb, None) == ERR_INVALID
    assert L().sgn_loss_fwd(4, 4, C.byref(li), _p(out), _p(scratch), sb - 4, None) == ERR_WORKSPACE
    assert b"scratch" in L().sgn_last_error()
    both = _lib.LossIn.from_buffer_copy(li)
    both.gt_u8 = both.gt_f32
    assert L().sgn_loss_fwd(4, 4, C.byref(both), _p(out), _p(scratch), sb, None) == ERR_INVALID
    assert L().sgn_loss_bwd(4, 4, C.byref(both), None, None, None, None, None) == ERR_INVALID
    neither = _lib.LossIn.from_buffer_copy(li)
    neither.gt_f32 = None
    assert L().sgn_loss_fwd(4, 4, C.byref(neither), _p(out), _p(scratch), sb, None) == ERR_INVALID
    assert L().sgn_loss_bwd(0, 4, C.byref(li), None, None, None, None, None) == ERR_INVALID


# ---- densification statistics ----------------------------------------------------------------------------------------
MARGIN = 37  # canary floats around every window, beyond the margins the table's layout needs


def densify_layout(c: sc.DensifyCase):
    """Each segment's window [start, start + count) in one flat buffer per statistic, segments in REVERSE order (so that a
    segment's pointer plus its row offset never lands on another segment's data), with a margin in front of at least the
    first row0 and behind of at least the rows up to the next segment (or to N)."""
    starts, pos = [0] * len(c.segs), 0
    first_row0 = c.segs[0][0]
    for s in reversed(range(len(c.segs))):
        r0, n, _ = c.segs[s]
        nxt = c.segs[s + 1][0] if s + 1 < len(c.segs) else c.N
        pos += MARGIN + first_row0
        starts[s] = pos
        pos += n + max(nxt - r0 - n, 0) + 1 + MARGIN
    return starts, pos


def densify_table(c, starts, bufs, first_override=None):
    tab = (_lib.DensifySegment * len(c.segs))()
    for j, (r0, n, first) in enumerate(c.segs):
        tab[j].row0, tab[j].count = int(r0), int(n)
        tab[j].first = int(first) if first_override is None else first_override
        tab[j].xys_grad_norm, tab[j].vis_counts, tab[j].max_2Dsize = (b.data_ptr() + 4 * int(starts[j]) for b in bufs)
    return torch.frombuffer(bytearray(bytes(tab)), dtype=torch.uint8).to(DEV)


@pytest.mark.parametrize("case", sc.DENSIFY_CASES, ids=lambda c: c.name)
def test_densify_stats_match_replay_and_leave_canaries(case):
    starts, total = densify_layout(case)
    init = np.full(total, CANARY, np.int32)
    want = [init.copy() for _ in range(3)]
    for j, (r0, n, first) in enumerate(case.segs):  # the statistics earlier calls left (read by first = 0 segments)
        for k, a in enumerate(case.prior(n, j)):
            want[k][starts[j]:starts[j] + n] = bits(a)
    bufs = [torch.from_numpy(w.copy()).to(DEV) for w in want]
    for call in range(2):
        v, radii = case.inputs(call)
        vd, rd = torch.from_numpy(v).to(DEV), torch.from_numpy(radii).to(DEV)
        raw = densify_table(case, starts, bufs, None if call == 0 else 0)
        _lib.check(L().sgn_densify_stats(_p(raw), len(case.segs), case.N, _p(vd), _p(rd), case.H, case.W, None), "sgn_densify_stats")
        for j, (r0, n, first) in enumerate(case.segs):
            sl = slice(starts[j], starts[j] + n)
            prev = tuple(w[sl].view(f32) for w in want)
            got = ref.densify_f32(v[r0:r0 + n, :2], radii[r0:r0 + n], bool(first) and call == 0, prev, case.H, case.W)
            for k in range(3):
                want[k][sl] = bits(got[k])
        for k, name in enumerate(("xys_grad_norm", "vis_counts", "max_2Dsize")):
            g = host(bufs[k]).view(np.int32)
            bad = np.flatnonzero(g != want[k])
            assert bad.size == 0, (name, call, bad[:10], [(i, int(g[i]), int(want[k][i])) for i in bad[:3]])


def test_densify_argument_errors():
    t = torch.zeros(64, device=DEV)
    r = torch.zeros(4, dtype=torch.int32, device=DEV)
    raw = torch.zeros(64, dtype=torch.uint8, device=DEV)
    assert L().sgn_densify_stats(_p(raw), -1, 4, _p(t), _p(r), 8, 8, None) == ERR_INVALID
    assert L().sgn_densify_stats(_p(raw), 1, -1, _p(t), _p(r), 8, 8, None) == ERR_INVALID
    assert L().sgn_densify_stats(_p(raw), 1, 4, _p(t), _p(r), 0, 8, None) == ERR_INVALID
    assert L().sgn_densify_stats(None, 1, 4, _p(t), _p(r), 8, 8, None) == ERR_INVALID
    assert L().sgn_densify_stats(_p(raw), 1, 4, None, _p(r), 8, 8, None) == ERR_INVALID
    assert L().sgn_densify_stats(_p(raw), 1, 4, _p(t), None, 8, 8, None) == ERR_INVALID
    assert L().sgn_densify_stats(_p(raw), 1, 4, C.c_void_p(t.data_ptr() + 4), _p(r), 8, 8, None) == ERR_INVALID
    assert L().sgn_densify_stats(None, 0, 4, None, None, 8, 8, None) == 0   # nothing to do
    assert L().sgn_densify_stats(None, 3, 0, None, None, 8, 8, None) == 0


# ---- fused Adam -----------------------------------------------------------------------------------------------------------
CHUNK = 4096


def adam_rows(numels, steps, lrs, arena_offsets, grad_offsets, params):
    tab = np.zeros(len(numels), ADAM_DTYPE)
    tab["param"] = [p.data_ptr() for p in params]
    tab["arena_offset"], tab["grad_offset"], tab["numel"] = arena_offsets, grad_offsets, numels
    ch = [(n + CHUNK - 1) // CHUNK for n in numels]
    tab["chunk0"] = np.concatenate([[0], np.cumsum(ch)[:-1]])
    tab["beta1"], tab["beta2"], tab["eps"] = 0.9, 0.999, 1e-15
    tab["one_minus_beta1"], tab["one_minus_beta2"] = 1.0 - 0.9, 1.0 - 0.999
    st = np.asarray(steps, np.float64)
    tab["step_size"] = np.asarray(lrs) / (1.0 - 0.9 ** st)
    tab["sqrt_bc2"] = np.sqrt(1.0 - 0.999 ** st)
    return tab, int(sum(ch))


def adam_launch(tab, nchunks, grads, m, v):
    dev_tab = torch.from_numpy(tab.view(np.uint8).reshape(-1).copy()).to(DEV)
    return L().sgn_adam_step(_p(dev_tab), len(tab), nchunks, C.c_void_p(grads), _p(m), _p(v), None)


class AdamSet:
    """Parameters (each in its own canary-padded buffer, at a chosen float offset from 16-byte alignment), a gradient arena
    with room before its base for negative grad offsets, and the two moment arenas."""

    def __init__(self, numels, param_offs, seed, front=64):
        rng = np.random.default_rng(seed)
        self.numels = list(numels)
        self.pads = [4 * ((n + 3) // 4) for n in numels]
        self.arena_off = np.concatenate([[0], np.cumsum(self.pads)[:-1]]).astype(np.int64)
        A = int(sum(self.pads))
        self.front = front
        self.p_host = [rng.normal(size=n).astype(f32) for n in numels]
        self.p_bufs, self.params = [], []
        for n, o, ph in zip(numels, param_offs, self.p_host):
            buf = torch.from_numpy(np.full(n + 8, CANARY, np.int32)).to(DEV)
            view = buf[o:o + n].view(torch.float32)
            view.copy_(torch.from_numpy(ph))
            self.p_bufs.append(buf)
            self.params.append(view)
        self.m = torch.zeros(max(A, 4), device=DEV)
        self.v = torch.zeros(max(A, 4), device=DEV)
        self.g = torch.zeros(front + max(A, 4), device=DEV)
        self.m_host, self.v_host = np.zeros(max(A, 4), f32), np.zeros(max(A, 4), f32)

    def grad_base(self):
        return self.g.data_ptr() + 4 * self.front

    def set_grads(self, grads, grad_offsets):
        gh = np.zeros(self.g.numel(), f32)
        for gr, o in zip(grads, grad_offsets):
            gh[self.front + o:self.front + o + gr.size] = gr
        self.g.copy_(torch.from_numpy(gh))

    def replay(self, tab, grads, present):
        for i, gr in zip(present, grads):
            o, n = int(self.arena_off[i]), self.numels[i]
            row = tab[list(present).index(i)]
            self.p_host[i], self.m_host[o:o + n], self.v_host[o:o + n] = ref.adam_f32(
                self.p_host[i], gr, self.m_host[o:o + n], self.v_host[o:o + n], row)

    def check(self, param_offs):
        torch.cuda.synchronize()
        assert np.array_equal(bits(self.m.cpu().numpy()), bits(self.m_host))
        assert np.array_equal(bits(self.v.cpu().numpy()), bits(self.v_host))
        for i, (buf, o, n) in enumerate(zip(self.p_bufs, param_offs, self.numels)):
            b = buf.cpu().numpy()
            assert np.array_equal(b[o:o + n], bits(self.p_host[i])), i
            assert np.all(b[:o] == CANARY) and np.all(b[o + n:] == CANARY), i


def adam_grads(rng, n, step):
    g = rng.normal(size=n).astype(f32) * (10.0 ** rng.uniform(-3, 1, n)).astype(f32)
    g[rng.random(n) < 0.2] = 0.0                      # rows without a gradient: moments decay
    tiny = rng.random(n) < 0.05
    g[tiny] = (rng.choice([-1, 1], tiny.sum()) * 10.0 ** rng.uniform(-22, -14, tiny.sum())).astype(f32)  # around eps
    return g


NUMELS = [0, 1, 3, 4, 5, 0, 4095, 4096, 4097, 8193, 7, 0]


@pytest.mark.parametrize("misaligned", [False, True])
def test_adam_steps_match_replay(misaligned):
    offs = [(1 + i % 3) if misaligned else 0 for i in range(len(NUMELS))]
    s = AdamSet(NUMELS, offs, seed=4)
    rng = np.random.default_rng(11)
    steps = np.zeros(len(NUMELS), int)
    lrs = [1.6e-4, 0.005, 0.001, 0.0025, 0.0025 / 20, 0.05] * 2
    for step in range(5):
        present = [i for i in range(len(NUMELS)) if not (step in (1, 3) and i % 4 == 1)]  # some tensors absent in some steps
        steps[present] += 1
        # present tensors' gradients back to back from the arena's base, two of them in front of it (negative grad_offset):
        # the 5-element tensor at -12 (the float4 path) and the 3-element one at -39 (the scalar path)
        neg = {4: -12, 2: -39}
        goff, o = [], 0
        for i in present:
            if i in neg:
                goff.append(neg[i])
            else:
                goff.append(o)
                o += s.pads[i]
        grads = [adam_grads(rng, NUMELS[i], step) for i in present]
        s.set_grads(grads, goff)
        tab, nch = adam_rows([NUMELS[i] for i in present], steps[present], [lrs[i] for i in present],
                             s.arena_off[present], goff, [s.params[i] for i in present])
        assert adam_launch(tab, nch, s.grad_base(), s.m, s.v) == 0
        s.replay(tab, grads, present)
        s.check(offs)


def test_adam_misaligned_equals_aligned():
    outs = []
    for offs in ([0] * len(NUMELS), [3, 2, 1] * 4):
        s = AdamSet(NUMELS, offs, seed=9)
        rng = np.random.default_rng(12)
        for step in range(1, 4):
            grads = [adam_grads(rng, n, step) for n in NUMELS]
            s.set_grads(grads, s.arena_off)
            tab, nch = adam_rows(NUMELS, [step] * len(NUMELS), [0.01] * len(NUMELS), s.arena_off, s.arena_off, s.params)
            assert adam_launch(tab, nch, s.grad_base(), s.m, s.v) == 0
        torch.cuda.synchronize()
        outs.append(([bits(p.cpu().numpy()) for p in s.params], bits(s.m.cpu().numpy()), bits(s.v.cpu().numpy())))
    (pa, ma, va), (pb, mb, vb) = outs
    assert all(np.array_equal(a, b) for a, b in zip(pa, pb)) and np.array_equal(ma, mb) and np.array_equal(va, vb)


def test_adam_8192_tensors_and_8193_refused():
    n = 8192
    numels = [1 + (i % 5) for i in range(n)]
    s = AdamSet(numels, [i % 4 for i in range(n)], seed=2)
    rng = np.random.default_rng(3)
    grads = [adam_grads(rng, k, 1) for k in numels]
    s.set_grads(grads, s.arena_off)
    tab, nch = adam_rows(numels, [1] * n, [0.003] * n, s.arena_off, s.arena_off, s.params)
    assert adam_launch(tab, nch, s.grad_base(), s.m, s.v) == 0
    s.replay(tab, grads, list(range(n)))
    s.check([i % 4 for i in range(n)])
    big = np.concatenate([tab, tab[:1]])
    assert adam_launch(big, nch + 1, s.grad_base(), s.m, s.v) == ERR_INVALID
    assert b"8193" in L().sgn_last_error()


def test_adam_argument_errors():
    s = AdamSet([8], [0], seed=1)
    tab, nch = adam_rows([8], [1], [0.01], [0], [0], s.params)
    dev_tab = torch.from_numpy(tab.view(np.uint8).reshape(-1).copy()).to(DEV)
    g = C.c_void_p(s.grad_base())
    assert L().sgn_adam_step(None, 1, nch, g, _p(s.m), _p(s.v), None) == ERR_INVALID
    assert L().sgn_adam_step(_p(dev_tab), 1, nch, None, _p(s.m), _p(s.v), None) == ERR_INVALID
    assert L().sgn_adam_step(_p(dev_tab), 1, nch, g, None, _p(s.v), None) == ERR_INVALID
    assert L().sgn_adam_step(_p(dev_tab), 1, nch, g, _p(s.m), None, None) == ERR_INVALID
    assert L().sgn_adam_step(_p(dev_tab), 0, nch, g, _p(s.m), _p(s.v), None) == ERR_INVALID
    assert L().sgn_adam_step(_p(dev_tab), 1, nch, C.c_void_p(s.grad_base() + 4), _p(s.m), _p(s.v), None) == ERR_INVALID
    assert L().sgn_adam_step(_p(dev_tab), 1, nch, g, C.c_void_p(s.m.data_ptr() + 8), _p(s.v), None) == ERR_INVALID
    assert L().sgn_adam_step(_p(dev_tab), 1, 0, g, _p(s.m), _p(s.v), None) == 0   # no chunks: nothing to do
    s.check([0])


def test_fused_adam_refuses_another_chunk_size_on_cuda():
    p = [[torch.zeros(10, k, device=DEV) for k in (3, 3, 4, 3, 45, 1)]]
    with pytest.raises(ValueError, match="chunk"):
        FusedAdam(p, chunk_elems=8192)
    assert FusedAdam(p, chunk_elems=CHUNK)._chunk == CHUNK


def _fused_pair(seed):
    rng = np.random.default_rng(seed)
    shapes = [(2000, 3), (2000, 3), (2000, 4), (2000, 5, 3), (2000, 15, 3), (2000, 1),
              (1, 3), (1, 3), (1, 4), (1, 1, 3), (1, 15, 3), (1, 1),
              (1367, 3), (1367, 3), (1367, 4), (1367, 1, 3), (1367, 15, 3), (1367, 1)]
    host_p = [rng.normal(size=s).astype(f32) for s in shapes]
    mk = lambda: [[torch.from_numpy(host_p[6 * k + j].copy()).to(DEV) for j in range(6)] for k in range(3)]  # noqa: E731
    return mk(), mk()


@pytest.mark.parametrize("mode", ["ranges", "slices"])
def test_fused_adam_range_cut_equals_whole_table(mode):
    whole_p, cut_p = _fused_pair(21)
    whole, cut = FusedAdam(whole_p), FusedAdam(cut_p)
    A = whole.arena_elems
    rng = np.random.default_rng(22)
    for step in range(4):
        present = None if step != 2 else [0, 2]
        arena = torch.from_numpy(rng.normal(size=A).astype(f32)).to(DEV)
        whole.step(arena, present=present, full_layout=True)
        tab = cut.step_table(present, full_layout=True)
        # cuts inside a chunk, at chunk edges (multiples of 4096 floats from a tensor's start) and inside small tensors
        o4, o6, o12 = (int(cut.offsets[i]) for i in (4, 6, 12))
        edges = sorted({0, A} | {4, 4096, 4100, 6000, 6000 + 4096, 12000, 24000, 24004, 30000, o4 + 4096, o4 + 8196,
                                 o6 + 4, o12 + 4096, A - 4})
        ranges = [(a, b) for a, b in zip(edges[:-1], edges[1:]) if b > a]
        if mode == "ranges":
            for a, b in ranges:
                cut.launch(cut.rows_in_range(tab, a, b), arena)
        else:
            groups = [ranges[0::2], ranges[1::2]]
            for grp in groups:
                cut.launch(cut.rows_in_slices(tab, [(a, b - a) for a, b in grp]), arena)
        torch.cuda.synchronize()
        for ps_w, ps_c in zip(whole_p, cut_p):
            for a, b in zip(ps_w, ps_c):
                assert torch.equal(a.view(torch.int32), b.view(torch.int32))
        assert torch.equal(whole.exp_avg.view(torch.int32), cut.exp_avg.view(torch.int32))
        assert torch.equal(whole.exp_avg_sq.view(torch.int32), cut.exp_avg_sq.view(torch.int32))


# ---- gradient exchange ----------------------------------------------------------------------------------------------------
FLAGS_PAD = 64


def exchange_run(c: sc.ExchangeCase, world: int, scale: float, skip: bool):
    rng = np.random.default_rng(40 + c.seed * 10 + world)
    A = c.arena
    flag_off = 4 * (A + 16)                                   # flags behind each replica's arena, at flags_byte_offset
    R = c.union_rows
    nfloat = A + 16 + (R + FLAGS_PAD + 3) // 4 + 4
    reps_host = [(rng.normal(size=A) * 10.0 ** rng.uniform(-3, 3, A)).astype(f32) for _ in range(world)]
    for rh in reps_host:
        rh[rng.random(A) < 0.05] = 0.0
    bufs = []
    for rh in reps_host:
        b = torch.zeros(nfloat, device=DEV)
        b[:A] = torch.from_numpy(rh).to(DEV)
        bufs.append(b)
    peers = torch.tensor([b.data_ptr() for b in bufs], dtype=torch.int64, device=DEV)
    union = None
    if skip:
        flags = sc.rank_flags(c, world)
        # each rank's flags from radii > 0 (sgn_visible_flags), written behind its replica
        for r, b in enumerate(bufs):
            radii = torch.from_numpy(np.where(flags[r] != 0, rng.integers(1, 50, R), -rng.integers(0, 3, R)).astype(np.int32)).to(DEV)
            fl = b.view(torch.uint8)[flag_off:flag_off + R]
            _lib.check(L().sgn_visible_flags(_p(radii), R, _p(fl), None), "sgn_visible_flags")
        union = torch.full((R + FLAGS_PAD,), 7, dtype=torch.uint8, device=DEV)
        _lib.check(L().sgn_visible_union(_p(peers), flag_off, world, R, _p(union), None), "sgn_visible_union")
        u = host(union)
        assert np.array_equal(u[:R], flags.max(axis=0)) and np.all(u[R:] == 7)
    n = len(c.slices)
    offs = (C.c_int64 * n)(*[s.off for s in c.slices])
    lens = (C.c_int64 * n)(*[s.length for s in c.slices])
    widths = (C.c_int32 * n)(*[s.width for s in c.slices])
    row0 = (C.c_int64 * n)(*[s.row0 for s in c.slices])
    rows = (C.c_int64 * n)(*[s.nrows for s in c.slices])
    for rank in range(world):
        _lib.check(L().sgn_allreduce_sym(_p(bufs[rank]), None, _p(peers), rank, world, n, offs, lens, widths, row0, rows,
                                         _p(union), C.c_float(scale), c.max_ctas, None), "sgn_allreduce_sym")
    got = [host(b)[:A] for b in bufs]
    # expected: the original everywhere, the rank-order sum times scale on every live unit of every slice
    exp = [rh.copy() for rh in reps_host]
    u = host(union) if skip else None
    for s in c.slices:
        if s.length == 0:
            continue
        seg = slice(s.off, s.off + s.length)
        total = ref.exchange_f32([rh[seg] for rh in reps_host], scale)
        live = np.ones(s.length // 4, bool)
        if skip and s.width:
            live = ~ref.skipped_units(s.length // 4, s.width, s.nrows, u[s.row0:s.row0 + s.nrows])
        lf = np.repeat(live, 4)
        for e in exp:
            e[seg][lf] = total[lf]
    for r in range(world):
        bad = np.flatnonzero(bits(got[r]) != bits(exp[r]))
        assert bad.size == 0, (r, bad[:10])
    return exp


@pytest.mark.parametrize("case", sc.EXCHANGE_CASES, ids=lambda c: c.name)
@pytest.mark.parametrize("world", [1, 2, 3, 4, 8])
def test_exchange_matches_rank_order_sum(case, world):
    skip = case.union_rows > 0
    for scale in (1.0, 1.0 / world):
        exchange_run(case, world, scale, skip)
    if skip and case.pattern != "all":   # the case has units to skip (their non-zero values must survive)
        flags = sc.rank_flags(case, world).max(axis=0)
        assert any(ref.skipped_units(s.length // 4, s.width, s.nrows, flags[s.row0:s.row0 + s.nrows]).any()
                   for s in case.slices if s.width)


def test_exchange_argument_errors():
    buf = torch.zeros(1024, device=DEV)
    peers = torch.tensor([buf.data_ptr()], dtype=torch.int64, device=DEV)
    vis = torch.ones(64, dtype=torch.uint8, device=DEV)

    def call(nslices=1, offs=(0,), lens=(16,), widths=(0,), row0=(0,), rows=(0,), local=None, rank=0, world=1, union=None,
             peer=True):
        n = max(nslices, len(offs))
        mk = lambda t, v: (t * n)(*(list(v) * n)[:n])  # noqa: E731
        return L().sgn_allreduce_sym(_p(buf) if local is None else local, None, _p(peers) if peer else None, rank, world,
                                     nslices, mk(C.c_int64, offs), mk(C.c_int64, lens), mk(C.c_int32, widths),
                                     mk(C.c_int64, row0), mk(C.c_int64, rows), _p(union), C.c_float(1.0), 0, None)
    assert call(peer=False) == ERR_INVALID
    assert call(local=C.c_void_p(0)) == ERR_INVALID
    assert call(rank=1, world=1) == ERR_INVALID
    assert call(world=0) == ERR_INVALID
    assert call(nslices=49, offs=[16 * i for i in range(49)], lens=[16]) == ERR_INVALID
    assert call(nslices=-1) == ERR_INVALID
    assert call(local=C.c_void_p(buf.data_ptr() + 4)) == ERR_INVALID
    assert call(offs=(2,)) == ERR_INVALID and call(lens=(6,)) == ERR_INVALID
    assert call(widths=(4,), rows=(5,), union=vis) == ERR_INVALID              # 5 rows of 4 floats in 16 floats
    assert call(widths=(4097,), rows=(0,), union=vis) == ERR_INVALID
    # a row-skipping slice of 2^31 floats: refused before anything is launched (rows_unseen counts floats in 32 bits).
    # A second slice with a bad offset follows, so that a build without the check refuses the call too, on that slice.
    assert call(nslices=2, offs=(0, 2), lens=(1 << 31, 16), widths=(1, 0), rows=(1 << 31, 0), union=vis) == ERR_INVALID
    assert b"2^31" in L().sgn_last_error()
    assert call(nslices=2, offs=(0, 2), lens=((1 << 31) - 4, 16), widths=(1, 0), rows=(100, 0), union=vis) == ERR_INVALID
    assert b"16-byte" in L().sgn_last_error()
    # flags / union
    r = torch.ones(8, dtype=torch.int32, device=DEV)
    assert L().sgn_visible_flags(None, 8, _p(vis), None) == ERR_INVALID
    assert L().sgn_visible_flags(_p(r), -1, _p(vis), None) == ERR_INVALID
    assert L().sgn_visible_union(None, 0, 1, 8, _p(vis), None) == ERR_INVALID
    assert L().sgn_visible_union(_p(peers), 0, 0, 8, _p(vis), None) == ERR_INVALID
    torch.cuda.synchronize()
