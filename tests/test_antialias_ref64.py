"""CPU checks of the antialiased mode's references: the float64 compensation (oracle/project_aa_ref64.py) against finite
differences and its closed form, and the C oracle in that mode (oracle/oracle_aa.py: the float32 projection and its
backward with the float64 compensation) against the float64 statement on the directed cases, with the bars of tests/test_gpu_project_directed.py (the
row's float32 noise: the float64 statement evaluated in float32), and for the geometry gradients at least
COND_K eps32 kappa of the row's scale (tests/antialias_cases.py comp_condition: the chain through cov2d)."""
import numpy as np
import pytest
import torch

from oracle import oracle_aa, oracle_c
from oracle import project_aa_ref64 as aa
from oracle import project_ref64 as ref
from street_gaussians_ns_b200 import raster
from tests import antialias_cases as ac
from tests import project_cases as pc

FWD_K, FWD_R, BWD_K, BWD_R = 8.0, 2e-6, 8.0, 5e-4


def test_compensation_closed_form_and_finite_differences():
    rng = np.random.default_rng(0)
    c00, c11 = rng.uniform(1e-3, 5.0, 200), rng.uniform(1e-3, 5.0, 200)
    c01 = rng.uniform(-0.9, 0.9, 200) * np.sqrt(c00 * c11)
    a, b, c = (torch.tensor(x, dtype=torch.float64, requires_grad=True) for x in (c00 + 0.3, c01, c11 + 0.3))
    comp = aa.compensation(a, b, c)
    want = np.sqrt((c00 * c11 - c01 ** 2) / ((c00 + 0.3) * (c11 + 0.3) - c01 ** 2))
    assert np.allclose(comp.detach().numpy(), want, rtol=1e-12)
    g = torch.autograd.grad(comp.sum(), (a, b, c))
    h = 1e-7
    for k, x in enumerate((a, b, c)):
        args = [t.detach().clone() for t in (a, b, c)]
        args[k] = args[k] + h
        up = aa.compensation(*args).numpy()
        args[k] = args[k] - 2 * h
        dn = aa.compensation(*args).numpy()
        assert np.allclose(g[k].numpy(), (up - dn) / (2 * h), rtol=1e-5, atol=1e-8)
    # the clamp: a rank-one covariance has comp 0 and a finite, zero gradient through it
    z = [torch.tensor([v], dtype=torch.float64, requires_grad=True) for v in (1.3, 1.0, 1.3)]
    cz = aa.compensation(*z)
    assert float(cz.detach()) == 0.0
    gz = torch.autograd.grad(cz.sum(), z)
    assert all(float(t) == 0.0 for t in gz)


def test_unknown_mode_raises():
    with pytest.raises(ValueError):
        raster.rasterize_mode_flag("mip")
    assert raster.rasterize_mode_flag("classic") == 0 and raster.rasterize_mode_flag("antialiased") == 1


@pytest.mark.parametrize("name", ["shapes", "posed40", "comp_edges"])
def test_c_oracle_antialiased_against_float64(name):
    case = ac.comp_edges() if name == "comp_edges" else pc.get(name)
    st = case.st
    orc = oracle_aa.AntialiasedOracle(case.frame, st.sh_degree, st.deg_use, st.block_width, st.clip_thresh)
    pr = orc.project()
    fw = aa.forward(case.frame, st)
    f32 = aa.forward(case.frame, st, torch.float32)
    vis = fw["vis"]
    kappa = ac.comp_condition(fw["records"])
    r64 = fw["records"][:, 5]
    noise = np.maximum(np.abs(f32["records"][:, 5] - r64), ac.EPS32 * kappa * np.abs(r64))
    bar = FWD_K * noise + FWD_R * np.maximum(np.abs(r64), 1e-3)
    assert np.all(np.abs(pr["opac"] - r64)[vis] <= bar[vis])
    assert np.all(pr["opac"][~vis] == 0)
    classic = oracle_c.Oracle(case.frame, st.sh_degree, st.deg_use, st.block_width, st.clip_thresh).project()
    assert np.all(pr["opac"][vis] <= classic["opac"][vis])
    # backward: the opacity cotangent alone, and every cotangent
    for kind in ("opacity", "all"):
        v = pc.v_records(case, kind)
        fwo = orc.forward(class_renders=False)
        got = orc.project_bwd(fwo, v[:, 0:2], v[:, 9], v[:, 2:5], v[:, 6:9], v[:, 5])
        want = aa.backward(case.frame, st, v)
        w32 = aa.backward(case.frame, st, v, torch.float32)
        row0 = 0
        for g, w, n32 in zip(got, want, w32):
            n = len(g["means"])
            kap = kappa[row0:row0 + n]
            row0 += n
            if not n:
                continue
            geo = np.max([np.abs(w[k].reshape(n, -1)).max(1) for k in ("means", "scales", "quats")], 0)
            for k in ("means", "scales", "quats", "opacities"):
                gv, wv, v32 = (x.astype(np.float64).reshape(n, -1) for x in (g[k], w[k], n32[k]))
                scale = geo if k != "opacities" else np.abs(wv).max(1)
                bar = np.maximum(BWD_K * np.abs(v32 - wv).max(1), BWD_R * scale)
                if k != "opacities":
                    bar = np.maximum(bar, ac.COND_K * ac.EPS32 * kap * scale)
                assert np.all(np.abs(gv - wv).max(1) <= bar), (name, kind, k)
