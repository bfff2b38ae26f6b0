"""The float64 blend reference (oracle/blend_ref64.py) checked on the CPU: its forward against the C oracle on the lists
of the test_gpu_parity.py scenes, its backward against central differences of its own forward on tiny tiles, and the
hand-built cases (tests/blend_cases.py) against what each was built to exercise."""
import numpy as np
import pytest

import street_gaussians_ns_b200.synthetic as syn
from oracle import blend_ref64 as ref
from oracle import oracle_c
from tests import blend_cases as bc

PARITY_SCENES = {
    "small_actors": dict(n_background=20000, n_actors=6, n_per_actor=1500, width=320, height=240, seed=3,
                         actor_shift=np.array([1.0, 0.0, -1.0])),
    "ragged_edge": dict(n_background=8000, n_actors=2, n_per_actor=500, width=200, height=136, seed=9,
                        actor_shift=np.array([1.5, 0.0, 0.0])),
    "odd_many_actors": dict(n_background=12000, n_actors=9, n_per_actor=300, width=333, height=177, seed=21,
                            actor_shift=np.array([0.5, 0.0, -2.0]), c2w=syn.waymo_rig(4)[6]),
    "dense_small_image": dict(n_background=60000, n_actors=3, n_per_actor=4000, width=96, height=80, seed=5,
                              actor_shift=np.array([1.0, 0.0, 2.0]), fourier_dim=1),
}


@pytest.mark.parametrize("name", list(PARITY_SCENES))
def test_forward_matches_c_oracle(name):
    fr = syn.make_frame(**PARITY_SCENES[name])
    orc = oracle_c.Oracle(fr)
    fw = orc.forward()
    N = fw.N
    rec = np.zeros((N, 12), np.float32)
    rec[:, 0:2], rec[:, 2:5], rec[:, 5] = fw.xys, fw.conics, fw.opac
    rec[:, 6:9], rec[:, 9] = fw.rgbs, fw.depths
    ids = fw.sorted_ids.astype(np.int64)
    payload = (ids | (fw.cls[ids].astype(np.int64) << 31)).astype(np.uint32).view(np.int32)
    cls_ids, cls_bins = bc.partition(payload, fw.tile_bins)
    H, W = fr.camera.height, fr.camera.width
    inp = ref.Inputs(W, H, rec, payload, fw.tile_bins, cls_ids, cls_bins)
    r = ref.forward(inp, ref.Opts())
    ok = (fw.fragile == 0) & (r["margin"] >= 1e-4)
    assert ok.mean() > 0.95
    np.testing.assert_allclose(r["raw"][ok], fw.img[ok], rtol=1e-5, atol=2e-5)  # depth sums reach ~15
    np.testing.assert_allclose(r["final_T"][0][ok], fw.final_T[ok], rtol=0, atol=1e-5)
    # the C oracle leaves 0 where nothing was blended, the kernels' convention (and the reference's) is -1
    c_idx = lambda idx: np.where(idx < 0, 0, idx)
    np.testing.assert_array_equal(c_idx(r["final_idx"][0])[ok], fw.final_idx[ok])
    okc = ok & (fw.fragile_obj == 0) & (fw.fragile_bg == 0)
    np.testing.assert_allclose(r["final_T"][1][okc], fw.obj_T[okc], rtol=0, atol=1e-5)
    np.testing.assert_allclose(r["final_T"][2][okc], fw.bg_T[okc], rtol=0, atol=1e-5)
    # the class streams' last entries: the C oracle gives list positions, the reference sub-list positions
    for c, slot, fi in ((1, 1, fw.obj_idx), (0, 2, fw.bg_idx)):
        got = r["final_idx"][slot]
        if slot == 2:  # BG_SAME_AS_MAIN: the main stream's last entry
            got = np.where(got == ref.BG_SAME_AS_MAIN, r["final_idx"][0], got)
        pos = np.full(max(len(payload), 1), -1, np.int64)
        for t in range(fw.tile_bins.shape[0]):
            s0, s1 = fw.tile_bins[t]
            seg = np.arange(s0, s1)[(payload[s0:s1] < 0) == bool(c)]
            pos[cls_bins[c, t, 0]:cls_bins[c, t, 1]] = seg
        mapped = np.where(got >= 0, pos[np.maximum(got, 0)], -1)
        if slot == 2:
            mapped = np.where(r["final_idx"][slot] == ref.BG_SAME_AS_MAIN, r["final_idx"][0], mapped)
        np.testing.assert_array_equal(c_idx(mapped)[okc], fi[okc])


def _loss(case, rec, sky, cot):
    inp = case.inp
    fw = ref.forward(ref.Inputs(inp.width, inp.height, rec, inp.sorted_ids, inp.tile_bins, inp.cls_ids, inp.cls_bins, sky),
                     case.opts)
    return sum(float((np.asarray(cot[k], np.float64).reshape(fw[k].shape) * fw[k]).sum()) for k in cot)


@pytest.mark.parametrize("shape", [(16, 16, 1), (20, 18, 2), (9, 21, 3)])
def test_backward_matches_central_differences(shape):
    w, h, seed = shape
    case = bc.tiny(w, h, seed)
    cot = bc.cotangents(case, "rand", seed=seed)
    g, v_sky, _, _ = ref.backward(case.inp, case.opts, cot)
    rec = case.inp.records.astype(np.float64)
    sky = case.inp.sky.astype(np.float64)
    worst = 0.0
    for n in range(rec.shape[0]):
        for col in range(10):
            hstep = 1e-6 * max(1.0, abs(rec[n, col]))
            rp, rm = rec.copy(), rec.copy()
            rp[n, col] += hstep
            rm[n, col] -= hstep
            fd = (_loss(case, rp, sky, cot) - _loss(case, rm, sky, cot)) / (2 * hstep)
            scale = np.abs(g[:, col]).max() + 1e-12
            worst = max(worst, abs(fd - g[n, col]) / (abs(g[n, col]) + 1e-3 * scale))
    assert worst < 1e-4, worst
    for (i, j, c) in [(0, 0, 0), (h - 1, w - 1, 2), (h // 2, w // 3, 1)]:
        sp, sm = sky.copy(), sky.copy()
        sp[i, j, c] += 1e-6
        sm[i, j, c] -= 1e-6
        fd = (_loss(case, rec, sp, cot) - _loss(case, rec, sm, cot)) / 2e-6
        assert abs(fd - v_sky[i, j, c]) <= 1e-6 * max(1.0, abs(fd))


def test_cases_exercise_what_they_are_built_for():
    """Guards against a case silently losing the path it exists for (e.g. after a change of the builder)."""
    c = bc.get("lengths")
    lens = np.diff(c.inp.tile_bins, axis=1)[:, 0]
    assert lens.tolist() == bc.LENGTHS
    c = bc.get("termination")
    fi = c.fwd["final_idx"][0]
    # tiles 0-2: every pixel's main stream stops at entry 13, 7 and 31 of its tile (the last blended entry is the one before)
    for t, stop in ((0, 13), (1, 7), (2, 31)):
        assert np.all(fi[:, 16 * t:16 * t + 16] == c.inp.tile_bins[t, 0] + stop - 1)
    assert (c.fwd["accumulation"][:, 48:64] < 0.999).all()  # tile 3 never stops
    t4 = c.fwd["final_T"][0][:, 64:80]
    assert (t4 <= 1e-3).any() and (t4 > 0.1).any()  # tile 4: stopped and live pixels side by side
    c = bc.get("objects")
    assert c.fwd["tile_depth"][1].max() > 32  # the residual crosses a 32-entry batch
    assert c.fwd["tile_depth"][1][3] == 1     # exactly one object entry behind the exit point
    assert c.inp.cls_bins[0, 1, 1] == c.inp.cls_bins[0, 1, 0] and (c.fwd["final_idx"][2][:, 16:32] == -1).any()
    c = bc.get("split_default")
    lens = np.diff(c.inp.tile_bins, axis=1)[:, 0]
    assert [ref.strips_for(n, 768) for n in lens[:7]] == [1, 2, 2, 4, 4, 8, 8]
    c = bc.get("large")
    assert c.inp.tile_bins.shape[0] == 120 * 80 and np.diff(c.inp.tile_bins, axis=1).sum() > 5000
