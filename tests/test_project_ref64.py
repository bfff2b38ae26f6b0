"""The float64 projection reference (oracle/project_ref64.py) checked on the CPU: its forward against oracle_torch and the C
oracle on the test_gpu_parity.py scenes, its backward against central differences of its own forward on a tiny case with a
clamped, a posed and an sh_degree_to_use < sh_degree Gaussian, and the hand-built cases (tests/project_cases.py) against what
each was built to exercise."""
import numpy as np
import pytest
import torch

import street_gaussians_ns_b200.synthetic as syn
from oracle import oracle_c, oracle_torch
from oracle import project_ref64 as ref
from tests import project_cases as pc
from tests.test_blend_ref64 import PARITY_SCENES


@pytest.mark.parametrize("name", list(PARITY_SCENES))
def test_forward_matches_oracles(name):
    fr = syn.make_frame(**PARITY_SCENES[name])
    st = ref.Settings()
    fw = ref.forward(fr, st)
    _, cat = oracle_torch.compose(fr, torch.float64, requires_grad=False)
    ot = oracle_torch.project(cat, fr.camera, use_spec_exp=False)
    rgb, opac = oracle_torch.colours(cat, fr.camera, 3, 3)
    vis = fw["vis"]
    ok = fw["margin"] >= pc.MARGIN
    assert ok.mean() > 0.99
    np.testing.assert_array_equal(vis[ok], ot["visible"].numpy()[ok])
    np.testing.assert_array_equal(fw["radii"][ok], ot["radii"].numpy()[ok])
    np.testing.assert_array_equal(fw["num_tiles_hit"][ok], ot["num_tiles_hit"].numpy()[ok])
    rec = fw["records"]
    np.testing.assert_allclose(rec[vis, 0:2], ot["xys"].numpy()[vis], rtol=1e-12, atol=1e-9)
    np.testing.assert_allclose(rec[vis, 2:5], ot["conics"].numpy()[vis], rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(rec[vis, 9], ot["depths"].numpy()[vis], rtol=1e-12)
    np.testing.assert_allclose(rec[vis, 5], opac.numpy()[vis], rtol=1e-12)
    np.testing.assert_allclose(rec[vis, 6:9], rgb.numpy()[vis], rtol=1e-10, atol=1e-12)
    # the exact section of the C oracle (fp32, spec exp) takes the same integer decisions wherever the margins allow
    orc = oracle_c.Oracle(fr).project()
    np.testing.assert_array_equal(fw["radii"][ok], orc["radii"][ok])
    np.testing.assert_array_equal(fw["num_tiles_hit"][ok], orc["num_tiles_hit"][ok])
    bb = np.concatenate([fw["tmin"], fw["tmax"]], 1)
    np.testing.assert_array_equal(bb[ok & vis], orc["tile_bbox"][ok & vis])
    np.testing.assert_allclose(rec[vis, 0:2], orc["xys"][vis], rtol=1e-5, atol=1e-3)


def _tiny():
    b = pc._cam(48, 32, 77, ref.Settings(sh_degree=3, sh_degree_to_use=1))
    s0, s1 = b.segment(0), b.segment(1, pose=(0.4, (0.3, 0.1, -4.0)), F=3)
    b.add(s0, 0, 0, 4.0, (1.0, 0.6, 0.8), u=1.2 * b.limx, v=0.1, fixed=True)     # x clamped
    b.add(s0, 0, 0, 5.0, (1.5, 1.2, 1.0), u=-1.3 * b.limx, v=-1.2 * b.limy, fixed=True)  # both clamped
    b.add(s0, 20.0, 14.0, 3.0, (0.05, 0.02, 0.03))
    b.add(s1, 30.0, 10.0, 4.5, (0.08, 0.03, 0.05))
    b.add(s1, 0, 0, 6.0, (1.5, 0.9, 1.2), u=0.2, v=1.25 * b.limy, fixed=True)     # posed, y clamped
    return b.settle("tiny", notes={})


def test_backward_matches_central_differences():
    case = _tiny()
    fw = case.fwd
    assert fw["vis"].all() and (fw["clampx"] != 0).sum() >= 2 and (fw["clampy"] != 0).sum() >= 2
    v_all = pc.v_records(case, "all", seed=3)
    # the SH view direction is detached (as in the reference model), so the means are checked without the rgb cotangent
    v_geo = v_all.copy()
    v_geo[:, 6:9] = 0
    grads = {id(v_all): ref.backward(case.frame, case.st, v_all), id(v_geo): ref.backward(case.frame, case.st, v_geo)}
    worst = 0.0
    for si, seg in enumerate(case.frame.segments):
        for name in ("means", "scales", "quats", "features_dc", "features_rest", "opacities"):
            v = v_geo if name == "means" else v_all
            g = grads[id(v)]
            t = getattr(seg.params, name)
            base = t.clone()
            flat = t.view(-1)
            for j in range(flat.numel()):
                h = 1e-6 * max(1.0, abs(float(base.view(-1)[j])))
                vals = []
                for sgn in (1, -1):
                    p64 = base.double().clone().view(-1)
                    p64[j] += sgn * h
                    setattr(seg.params, name, p64.view(base.shape))
                    vals.append(float((ref.forward(case.frame, case.st)["rec"].detach().numpy() * v[:, :10]).sum()))
                setattr(seg.params, name, base)
                fd = (vals[0] - vals[1]) / (2 * h)
                an = g[si][name].reshape(-1)[j]
                worst = max(worst, abs(fd - an) / (abs(an) + 1e-6 * np.abs(g[si][name]).max() + 1e-9))
    assert worst < 1e-5, worst


def test_cases_exercise_what_they_are_built_for():
    c = pc.get("fov_clamp")
    fw = c.fwd
    v = fw["vis"]
    for arr in (fw["clampx"], fw["clampy"]):
        assert (v & (arr == 1)).sum() >= 3 and (v & (arr == -1)).sum() >= 3
    assert (v & (fw["clampx"] != 0) & (fw["clampy"] != 0)).sum() >= 3
    segrows = c.frame.segments[0].params.num_points
    assert (v[segrows:] & (fw["clampx"][segrows:] != 0)).any()  # posed rows clamped too
    c = pc.get("near_plane")
    assert (~c.fwd["unclipped"]).sum() >= 4 and c.fwd["vis"][0] and not c.fwd["vis"][1]
    big = 5  # the Gaussian 2 cm in front of the camera: AABB clamped on all four sides
    tiles = ((64 + 15) // 16, (48 + 15) // 16)
    assert tuple(c.fwd["tmin"][big]) == (0, 0) and tuple(c.fwd["tmax"][big]) == tiles and c.fwd["radii"][big] > 64
    c = pc.get("staged_mix")
    vis = c.fwd["vis"]
    assert vis[0:128:2].all() and not vis[1:128:2].any() and not vis[128:256].any()
    assert not vis[256:383].any() and vis[383]
    c = pc.get("layout")
    assert [s.params.num_points for s in c.frame.segments] == [1, 127, 0, 128, 129, 255, 0]
    assert len(pc.get("nseg1024").frame.segments) == 1024
    assert sorted({s.params.fourier_dim for s in pc.get("posed40").frame.segments}) == list(range(1, 9))
    for name in pc.CASES:
        if name.startswith("colour_d") and not name.startswith("colour_d0"):
            pre = pc.get(name).fwd["pre"][pc.get(name).fwd["vis"]]
            assert ((pre < 0).sum(0) > 0).all() and ((pre > 0).sum(0) > 0).all(), name
    c = pc.get("touch_bw2")
    area = (c.fwd["tmax"][:, 0] - c.fwd["tmin"][:, 0]) * (c.fwd["tmax"][:, 1] - c.fwd["tmin"][:, 1]) * c.fwd["vis"]
    assert (area > 1024).any() and ((area > 1) & (area <= 32)).any() and ((area > 32) & (area <= 1024)).any()
    assert len(c.notes["near_tau"]) >= 10
    assert all(n in pc.CASES for n in ("edges_333x177_bw2", "edges_333x177_bw3", "edges_333x177_bw7", "edges_333x177_bw8",
                                       "edges_333x177_bw16", "edges_1x1_bw16", "edges_17x3_bw16"))
