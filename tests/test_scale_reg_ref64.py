"""oracle/scale_reg_ref64.py against float64 torch autograd of nerfstudio's expression (CPU)."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.scale_reg_ref64 import scale_reg, scale_reg_grad, scale_reg_segments  # noqa: E402
from tests.scale_reg_cases import cases, exact_ratio_rows, segments  # noqa: E402


def torch_term(scales: torch.Tensor, max_ratio: float) -> torch.Tensor:
    """nerfstudio 1.0 SplatfactoModel.get_loss_dict's scale_reg, as written there."""
    scale_exp = torch.exp(scales)
    scale_reg = torch.maximum(scale_exp.amax(dim=-1) / scale_exp.amin(dim=-1), torch.tensor(max_ratio, dtype=scales.dtype)) - max_ratio
    return 0.1 * scale_reg.mean()


def torch_value_grad(rows: np.ndarray, max_ratio: float, v: float = 1.0):
    x = torch.tensor(rows, dtype=torch.float64, requires_grad=True)
    val = torch_term(x, max_ratio)
    (val * v).backward()
    return float(val.detach()), x.grad.numpy()


def atol(rows: np.ndarray, v: float = 1.0) -> float:
    """Where the exact gradient is 0 but autograd's is not: an element that is the max and the min gets g / mn - g r / mn with
    r = 1, which rounds to a few ulp of g = 0.1 v / N rather than to 0."""
    return 1e-13 * 0.1 * abs(v) / rows.shape[0]


ALL = cases()


@pytest.mark.parametrize("name", sorted(ALL))
@pytest.mark.parametrize("max_ratio", [10.0, 1.0, 2.5])
def test_value_and_grad_match_torch(name, max_ratio):
    rows = ALL[name] if max_ratio == 10.0 else cases(max_ratio)[name]
    val, grad = torch_value_grad(rows, max_ratio, v=0.7)
    assert scale_reg(rows, max_ratio) == pytest.approx(val, rel=1e-14, abs=1e-300)
    np.testing.assert_allclose(scale_reg_grad(rows, max_ratio, v=0.7), grad, rtol=1e-13, atol=atol(rows, 0.7))


def test_mixed_rows_match_torch():
    rows = np.concatenate([ALL[k] for k in sorted(ALL)])
    rows = rows[np.random.default_rng(3).permutation(rows.shape[0])]
    val, grad = torch_value_grad(rows, 10.0)
    assert scale_reg(rows, 10.0) == pytest.approx(val, rel=1e-14)
    np.testing.assert_allclose(scale_reg_grad(rows, 10.0), grad, rtol=1e-13, atol=1e-300)


def test_tie_at_max_ratio_takes_half():
    """torch.maximum hands half of the cotangent to the ratio when it equals max_ratio: pinned against torch itself."""
    rows = exact_ratio_rows(10.0, 8)
    s = np.exp(rows)
    assert (s.max(1) / s.min(1) == 10.0).all()
    _, grad = torch_value_grad(rows, 10.0)
    above = rows.copy()
    above[:, 2] = np.nextafter(above[:, 2], np.inf) + 1e-9  # the same rows strictly above the threshold
    _, grad_above = torch_value_grad(above, 10.0)
    np.testing.assert_allclose(grad, 0.5 * grad_above, rtol=1e-7)
    np.testing.assert_allclose(scale_reg_grad(rows, 10.0), grad, rtol=1e-13)


def test_rows_below_threshold_have_zero_gradient():
    for name in ("all_equal", "distinct_below", "just_below"):
        g = scale_reg_grad(ALL[name], 10.0)
        assert (g == 0).all(), name
    assert scale_reg(ALL["distinct_below"], 10.0) == 0.0


def test_three_way_tie_gets_both_shares():
    """max_ratio 1 puts rows of three equal scales at the tie: each element is the max and the min."""
    rows = ALL["all_equal"]
    val, grad = torch_value_grad(rows, 1.0)
    np.testing.assert_allclose(scale_reg_grad(rows, 1.0), grad, rtol=1e-13, atol=atol(rows))
    assert val == 0.0


@pytest.mark.parametrize("sizes", [(1,), (127, 1, 129), (300, 0, 5, 64, 128, 200), (1000, 3)])
def test_segments_of_uneven_size(sizes):
    rows = np.concatenate([ALL["random"], ALL["max_tie_2"], ALL["min_tie_2"], ALL["at_ratio"]])
    segs = segments(rows, sizes)
    val, grads = scale_reg_segments(segs, 10.0, v=1.3)
    tv, tg = torch_value_grad(rows, 10.0, v=1.3)
    assert val == pytest.approx(tv, rel=1e-14)
    np.testing.assert_allclose(np.concatenate(grads), tg, rtol=1e-13, atol=1e-300)
    assert [g.shape[0] for g in grads] == [s.shape[0] for s in segs]


def test_no_rows_is_nan():
    assert np.isnan(scale_reg(np.zeros((0, 3)), 10.0))
    assert np.isnan(float(torch_term(torch.zeros(0, 3, dtype=torch.float64), 10.0)))
    assert scale_reg_grad(np.zeros((0, 3)), 10.0).shape == (0, 3)


def test_model_torch_path_is_nerfstudio_expression():
    """SceneGraphRasterModel's fused_loss=False term over its visible sub-models (host logic, CPU tensors)."""
    from street_gaussians_ns_b200.model import SceneGraphConfig, SceneGraphRasterModel
    from street_gaussians_ns_b200.scene import GaussianSet

    def gs(n, seed):
        g = torch.Generator().manual_seed(seed)
        return GaussianSet(torch.randn(n, 3, generator=g), torch.randn(n, 3, generator=g) * 1.5 - 4, torch.randn(n, 4, generator=g),
                           torch.randn(n, 1, 3, generator=g), torch.randn(n, 15, 3, generator=g), torch.randn(n, 1, generator=g))
    m = SceneGraphRasterModel(gs(50, 0), {"a": gs(7, 1), "b": gs(9, 2)},
                              SceneGraphConfig(use_scale_regularization=True, fused_loss=False))
    m.visible_model_names = ["background", "object_b"]
    m.step = 20
    reg = m._scale_reg_loss(fused=False)
    rows = torch.cat([m.all_models["background"].gauss_params["scales"], m.all_models["object_b"].gauss_params["scales"]])
    assert float(reg.detach()) == pytest.approx(scale_reg(rows.detach().double().numpy(), 10.0), rel=1e-5)
    reg.backward()
    assert m.all_models["object_a"].gauss_params["scales"].grad is None
    g = scale_reg_grad(rows.detach().double().numpy(), 10.0)
    np.testing.assert_allclose(m.all_models["background"].gauss_params["scales"].grad.double().numpy(), g[:50], rtol=1e-4, atol=1e-12)
    m.step = 21
    z = m._scale_reg_loss(fused=False)
    assert float(z) == 0.0 and not z.requires_grad
    assert not SceneGraphConfig().use_scale_regularization and SceneGraphConfig().max_gauss_ratio == 10.0
