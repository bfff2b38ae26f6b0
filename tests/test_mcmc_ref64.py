"""CPU checks of the float64 MCMC statement (oracle/mcmc_ref64.py) against closed forms, quadrature, gsplat's own forms
written in torch, and autograd.  No GPU."""
import numpy as np
import pytest
import torch
from scipy import integrate

from oracle import mcmc_ref64 as R

OPACITIES = [1e-4, 0.005, 0.01, 0.1, 0.3, 0.5, 0.7, 0.9, 0.99, 0.999, 1 - 2.0 ** -23]


@pytest.mark.parametrize("N", list(range(1, 52)))
def test_closed_form_denominator_equals_double_sum(N):
    for o in OPACITIES:
        op = 1.0 - (1.0 - o) ** (1.0 / N)
        a, b = R.denom_closed(op, N), R.denom_double_sum(op, N)
        assert abs(a - b) <= 1e-9 * abs(b), (o, N, a, b)


@pytest.mark.parametrize("N", [1, 2, 3, 5, 10, 25, 51])
@pytest.mark.parametrize("o", [0.01, 0.3, 0.8, 0.99])
def test_opacity_identity(N, o):
    """N copies of opacity o' stack to o: 1 - (1 - o')^N = o."""
    _, _, op = R.relocation(o, np.ones(3), N - 1, 0.0)
    assert abs(1.0 - (1.0 - op) ** N - o) <= 1e-13


@pytest.mark.parametrize("N", [1, 2, 3, 7, 20, 51])
@pytest.mark.parametrize("o", [0.02, 0.5, 0.95])
def test_integral_identity(N, o):
    """N copies of (o', s_new) integrate, in 1D, to what the original Gaussian (o, s) integrates to."""
    s = 0.7
    _, s_new, op = R.relocation(o, np.array([s]), N - 1, 0.0)
    sn = float(s_new[0])
    lhs, _ = integrate.quad(lambda x: 1.0 - (1.0 - op * np.exp(-x * x / (2 * sn * sn))) ** N, -np.inf, np.inf, epsabs=1e-13, epsrel=1e-12)
    rhs = o * s * np.sqrt(2 * np.pi)
    assert abs(lhs - rhs) <= 1e-8 * rhs, (lhs, rhs)


def test_single_copy_leaves_the_row_unchanged():
    for o in OPACITIES[2:-1]:
        s = np.array([0.3, 1.0, 2.5])
        o_new, s_new, op = R.relocation(o, s, 0, 0.005)
        assert abs(op - o) <= 1e-15 and abs(o_new - o) <= 1e-15
        assert np.allclose(s_new, s, rtol=1e-15, atol=0)


def test_clamps():
    # a faint row drawn many times falls under min_opacity and is clamped there; a row at 1 is clamped below 1
    o_new, _, op = R.relocation(0.01, np.ones(3), 50, 0.005)
    assert op < 0.005 and o_new == float(np.float32(0.005))
    o_new, _, _ = R.relocation(1 - 2.0 ** -24, np.ones(3), 0, 0.005)
    assert o_new == R.EPS_CLAMP


def _rows(n, seed=0):
    g = np.random.default_rng(seed)
    rows = {"means": g.normal(size=(n, 3)), "scales": g.normal(-3, 0.5, (n, 3)), "quats": g.normal(size=(n, 4)),
            "features_dc": g.normal(size=(n, 2, 3)), "opacities": g.normal(0, 1.5, (n, 1)), "semantic_logits": g.normal(size=(n, 3)),
            "filter_3d": g.uniform(0, 0.01, n)}
    rows = {k: v.astype(np.float32) for k, v in rows.items()}
    moments = {k: (g.normal(size=rows[k].shape), g.uniform(0.1, 1, rows[k].shape)) for k in
               ("means", "scales", "quats", "features_dc", "opacities", "semantic_logits")}
    return rows, moments


def test_relocate_semantics():
    rows, moments = _rows(8)
    rows["opacities"][[2, 5], 0] = [-6.0, -8.0]  # dead: sigmoid <= 0.005
    assert list(R.dead_rows(rows["opacities"], 0.005)) == [2, 5]
    new, nm = R.relocate(rows, moments, [0, 0], 0.005)
    lo, ls = R.relocation_params(rows["opacities"][0, 0], rows["scales"][0], 2, 0.005)
    assert new["opacities"][0, 0] == lo and np.array_equal(new["scales"][0], ls)
    for k, t in new.items():
        for d in (2, 5):
            assert np.array_equal(t[d], t[0]), k                      # dead rows copy the updated source
        for r in (1, 3, 4, 6, 7):
            assert np.array_equal(t[r], rows[k][r].astype(np.float64)), k  # untouched rows
        if k not in ("opacities", "scales"):
            assert np.array_equal(t[0], rows[k][0].astype(np.float64))
    for k, (m, v) in nm.items():
        assert not m[0].any() and not v[0].any()                      # the source's moments are zeroed
        for r in (1, 2, 3, 4, 5, 6, 7):                               # the dead rows keep theirs, as gsplat's relocate
            assert np.array_equal(m[r], moments[k][0][r]) and np.array_equal(v[r], moments[k][1][r])


def test_relocate_without_dead_rows_changes_nothing():
    rows, moments = _rows(6, 1)
    rows["opacities"][:] = 0.0
    new, nm = R.relocate(rows, moments, [], 0.005)
    for k in rows:
        assert np.array_equal(new[k], rows[k].astype(np.float64))


def test_add_semantics():
    rows, moments = _rows(6, 2)
    new, nm = R.add(rows, moments, [3, 1, 3], 0.005)
    assert new["means"].shape[0] == 9
    for k, t in new.items():
        assert np.array_equal(t[6], t[3]) and np.array_equal(t[7], t[1]) and np.array_equal(t[8], t[3]), k
    lo3, ls3 = R.relocation_params(rows["opacities"][3, 0], rows["scales"][3], 2, 0.005)
    lo1, _ = R.relocation_params(rows["opacities"][1, 0], rows["scales"][1], 1, 0.005)
    assert new["opacities"][3, 0] == lo3 and new["opacities"][1, 0] == lo1 and np.array_equal(new["scales"][3], ls3)
    assert np.array_equal(new["opacities"][[0, 2, 4, 5]], rows["opacities"][[0, 2, 4, 5]].astype(np.float64))
    for k, (m, v) in nm.items():
        assert np.array_equal(m[:6], moments[k][0]) and np.array_equal(v[:6], moments[k][1])  # sources keep their moments
        assert not m[6:].any() and not v[6:].any()                                              # appended rows start at zero


def test_draws_from_uniforms_skip_zero_weights():
    w = np.array([0.0, 0.2, 0.0, 0.0, 0.5, 0.3, 0.0])
    u = np.array([0.0, 0.1, 0.2 / 1.0 - 1e-15, 0.2, 0.69, 0.7, 0.999999])
    d = R.draws_from_uniforms(w, u)
    assert list(d) == [1, 1, 1, 4, 4, 5, 5]
    assert all(w[r] > 0 for s in R.acceptable_draws(w, u) for r in s)


def test_noise_matches_gsplat_form():
    g = torch.Generator().manual_seed(0)
    n = 500
    scales = torch.randn(n, 3, generator=g) * 0.5 - 2
    quats = torch.randn(n, 4, generator=g) * 3  # not unit
    opac = torch.randn(n, 1, generator=g) * 4
    opac[:50] = -8.0  # faint rows: the gate is open
    eps = torch.randn(n, 3, generator=g)
    lr = 1.6e-4 * 5e5
    # gsplat's inject_noise_to_position, in float64 from the same float32 o and s (the gate's slope of 100 turns torch.sigmoid's
    # one-ulp differences from 1 / (1 + exp(-x)) into 1e-5 relative)
    o = torch.from_numpy(R.sigmoid32(opac.numpy())).double().flatten()
    gate = 1 / (1 + torch.exp(-100 * ((1 - o) - 0.995)))
    q = torch.nn.functional.normalize(quats.double(), dim=-1)
    w, x, y, z = q.unbind(-1)
    Rm = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
                      2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
                      2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1).reshape(n, 3, 3)
    M = Rm * torch.exp(scales).double()[:, None, :]
    covars = M @ M.transpose(-1, -2)
    want = torch.einsum("bij,bj->bi", covars, eps.double() * gate[:, None] * lr).numpy()
    got = R.noise_delta(scales.numpy(), quats.numpy(), opac.numpy(), eps.numpy(), lr)
    # per row, against the row's size: the components cancel, and torch.exp and numpy's exp differ by an ulp in float32
    assert (np.abs(got - want).max(1) <= 1e-6 * np.abs(want).max(1)).all()
    # the gate closes for opaque rows: at o = 0.5 it is exp(-49.5)
    assert np.abs(got[:50]).max() > 0 and np.abs(got[60:][o[60:].numpy() > 0.5]).max() < 1e-12 * np.abs(got[:50]).max()


def test_regularisers_match_torch_autograd():
    g = torch.Generator().manual_seed(1)
    opac = (torch.randn(300, 1, generator=g) * 3).double().requires_grad_(True)
    scales = (torch.randn(300, 3, generator=g) - 2).double().requires_grad_(True)
    lo = 0.01 * torch.sigmoid(opac).mean()
    ls = 0.02 * torch.exp(scales).mean()
    (lo + ls).backward()
    ro, rs = R.regularisers(opac.detach().float().numpy(), scales.detach().float().numpy(), 0.01, 0.02)
    assert abs(ro - lo.item()) <= 1e-7 * lo.item() and abs(rs - ls.item()) <= 1e-7 * ls.item()
    go, gs = R.regulariser_grads(opac.detach().float().numpy(), scales.detach().float().numpy(), 0.01, 0.02)
    assert np.allclose(go, opac.grad.numpy(), rtol=1e-6) and np.allclose(gs, scales.grad.numpy(), rtol=1e-6)


def test_settings_and_schedule():
    import street_gaussians_ns_b200.mcmc as M
    from street_gaussians_ns_b200.model import SceneGraphConfig
    s = M.MCMCSettings()
    assert (s.cap_max, s.noise_lr, s.min_opacity, s.refine_start, s.refine_stop, s.refine_every) == (1_000_000, 5e5, 0.005, 500, 25_000, 100)
    assert not M.due(s, 500) and M.due(s, 600) and not M.due(s, 650) and not M.due(s, 25_000) and M.due(s, 24_900)
    assert M.num_added(1000, s) == 50 and M.num_added(999_990, s) == 10 and M.num_added(2_000_000, s) == 0 and M.num_added(19, s) == 0
    c = SceneGraphConfig()
    assert c.strategy == "default" and c.object_mcmc.cap_max == 100_000 and c.mcmc_opacity_reg == c.mcmc_scale_reg == 0.01
