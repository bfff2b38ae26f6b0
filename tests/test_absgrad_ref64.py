"""CPU checks of the float64 absolute screen-space gradient (oracle/absgrad_ref64.py) and of the absgrad switches of the
refinement config and the model.

  * on tiny hand-built cases, each pixel's main-stream gradient per row from torch float64 autograd of a straight
    restatement of the forward, summed in absolute value, matches the oracle to 1e-12;
  * the signed sum of the same terms is blend_ref64.backward's v_records[:, 0:2] for main-stream cotangents;
  * an isotropic Gaussian centred on a pixel corner under a cotangent antisymmetric about it has v_xy = 0 and an
    absolute gradient far from 0 -- the case the absolute statistic exists for;
  * refine.make_config thresholds at densify_absgrad_thresh only with absgrad, and the MCMC strategy refuses absgrad.
"""
import numpy as np
import pytest
import torch

from oracle import absgrad_ref64 as aref
from oracle import blend_ref64 as ref
from tests import blend_cases as bc

MAIN_KINDS = [("rgb",), ("accumulation",), ("depth",), ("rgb", "accumulation", "depth")]


def _torch_losses(xy: torch.Tensor, case, cot):
    """[P] per-pixel <cotangent, main-stream output> as a float64 torch function of the rows' means; every skip / stop
    decision is taken on detached values (the cases keep them 1e-3 from their thresholds)."""
    inp, opts = case.inp, case.opts
    rec = torch.from_numpy(np.asarray(inp.records, np.float64))
    H, W = inp.height, inp.width
    ids = np.asarray(inp.sorted_ids, np.int64) & ref.ID_MASK
    tb = np.asarray(inp.tile_bins, np.int64)
    raw = torch.zeros(H * W, 4, dtype=torch.float64)
    Tfin = torch.ones(H * W, dtype=torch.float64)
    for t in range(inp.tiles):
        rows = ids[tb[t, 0]:tb[t, 1]]
        if len(rows) == 0:
            continue
        tx, ty = t % inp.tiles_x, t // inp.tiles_x
        r, c = np.divmod(np.arange(16 * 16), 16)
        i, j = ty * 16 + r, tx * 16 + c
        ok = (i < H) & (j < W)
        i, j = i[ok], j[ok]
        px = torch.from_numpy(j + 0.5)[:, None]
        py = torch.from_numpy(i + 0.5)[:, None]
        R = rec[rows]
        dx = xy[rows, 0][None, :] - px
        dy = xy[rows, 1][None, :] - py
        sigma = 0.5 * R[:, 2] * dx * dx + R[:, 3] * dx * dy + 0.5 * R[:, 4] * dy * dy
        rawa = R[:, 5] * torch.exp(-sigma)
        valid = (sigma.detach() >= 0) & (rawa.detach() >= ref.ALPHA_MIN)
        alpha = torch.where(valid, torch.clamp(rawa, max=opts.clamp_fwd), torch.zeros_like(rawa))
        # stop BEFORE an entry whose new transmittance would be <= 1e-4
        Tc = torch.cumprod(1.0 - alpha.detach(), 1)
        stop = valid & (Tc <= ref.T_STOP)
        L = len(rows)
        ks = torch.where(stop.any(1), stop.int().argmax(1), torch.full((len(i),), L))
        blended = valid & (torch.arange(L)[None, :] < ks[:, None])
        a = torch.where(blended, alpha, torch.zeros_like(alpha))
        T = torch.cumprod(1.0 - a, 1)
        Tprev = torch.cat([torch.ones_like(T[:, :1]), T[:, :-1]], 1)
        w = a * Tprev
        pid = torch.from_numpy(i * W + j)
        raw = raw.index_put((pid,), w @ R[:, 6:10])
        Tfin = Tfin.index_put((pid,), T[:, -1])
    acc = 1.0 - Tfin
    loss = torch.zeros(H * W, dtype=torch.float64)
    if "rgb" in cot:
        cl = torch.clamp(raw[:, :3], max=1.0)
        fin = cl
        if opts.has_sky:
            sky = torch.from_numpy(np.asarray(inp.sky, np.float64).reshape(-1, 3))
            fin = cl * acc[:, None] + sky * (1.0 - acc[:, None])
        if opts.eval_clamp:
            fin = torch.clamp(fin, 0.0, 1.0)
        loss = loss + (fin * torch.from_numpy(np.asarray(cot["rgb"], np.float64).reshape(-1, 3))).sum(1)
    if "accumulation" in cot:
        loss = loss + acc * torch.from_numpy(np.asarray(cot["accumulation"], np.float64).reshape(-1))
    if "depth" in cot:
        ok = acc.detach() > 1e-3
        dep = torch.where(ok, raw[:, 3] / torch.where(ok, acc, torch.ones_like(acc)), torch.full_like(acc, 10.0))
        loss = loss + dep * torch.from_numpy(np.asarray(cot["depth"], np.float64).reshape(-1))
    return loss


def _autograd_absgrad(case, cot):
    xy = torch.from_numpy(np.asarray(case.inp.records, np.float64)[:, 0:2].copy())
    J = torch.autograd.functional.jacobian(lambda v: _torch_losses(v, case, cot), xy)  # [P, N, 2]
    return J.abs().sum(0).numpy(), J.sum(0).numpy()


@pytest.mark.parametrize("sky", [False, True])
@pytest.mark.parametrize("kinds", MAIN_KINDS, ids=["+".join(k) for k in MAIN_KINDS])
def test_oracle_matches_autograd(kinds, sky):
    case = bc.tiny(20, 18, 501 + int(sky), sky=sky, n=4)
    full = bc.cotangents(case, "rand")
    cot = {k: full[k] for k in kinds}
    want_abs, want_signed = _autograd_absgrad(case, cot)
    got, bound, signed = aref.absgrad(case.inp, case.opts, cot)
    scale = max(np.abs(want_abs).max(), 1e-300)
    assert np.abs(got - want_abs).max() <= 1e-12 * scale
    assert np.abs(signed - want_signed).max() <= 1e-12 * scale
    assert np.all(bound >= got * (1 - 1e-12))
    assert got.max() > 0


@pytest.mark.parametrize("name", ["lengths", "lengths_sky_eval", "objects", "raw_mode", "shape_15x33"])
def test_signed_sum_is_v_xy(name):
    case = bc.get(name)
    full = bc.cotangents(case, "rand")
    cot = {k: full[k] for k in ("rgb", "accumulation", "depth")}
    got, bound, signed = aref.absgrad(case.inp, case.opts, cot)
    v = ref.backward(case.inp, case.opts, cot)[0][:, 0:2]
    scale = max(np.abs(got).max(), 1e-300)
    assert np.abs(signed - v).max() <= 1e-12 * scale
    assert np.all(got >= np.abs(signed) - 1e-12 * scale)


def cancellation_case():
    """One isotropic Gaussian (sigma 3 px) centred on the pixel corner (8, 8) of one tile, and an accumulation cotangent
    sign(x - 8) sign(y - 8): every pixel's term has a mirror image of opposite sign in x and in y."""
    b = bc.Builder(16, 16, 7)
    g = b.gauss(8.0, 8.0, 3.0, o=0.8, rgb=(0.5, 0.5, 0.5), depth=2.0)
    b.lists[0] = [g]
    inp = b.inputs()
    x = np.arange(16) + 0.5
    cot = {"accumulation": (np.sign(x[:, None] - 8.0) * np.sign(x[None, :] - 8.0)).astype(np.float32)}
    return inp, ref.Opts(), cot


def test_cancellation_case():
    inp, opts, cot = cancellation_case()
    got, _, signed = aref.absgrad(inp, opts, cot)
    v = ref.backward(inp, opts, cot)[0][:, 0:2]
    assert np.abs(v).max() <= 1e-12 and np.abs(signed).max() <= 1e-12
    assert got.min() > 0.5, got  # |v_xy| = 0, the absolute statistic is of order one


def test_make_config_threshold():
    from street_gaussians_ns_b200 import refine
    s = refine.RefineSettings()
    assert s.densify_absgrad_thresh == pytest.approx(0.0008)
    off = refine.make_config(s, 1000, (64, 48), True)
    on = refine.make_config(s, 1000, (64, 48), True, absgrad=True)
    assert off.densify_grad_thresh == pytest.approx(s.densify_grad_thresh)
    assert on.densify_grad_thresh == pytest.approx(s.densify_absgrad_thresh)
    assert on.max_size == off.max_size  # the normalisation * 0.5 * max(H, W) is the same


def test_mcmc_refuses_absgrad():
    from street_gaussians_ns_b200 import model as mdl
    from street_gaussians_ns_b200.synthetic import make_background
    bg = make_background(64, seed=1)
    with pytest.raises(ValueError, match="absgrad"):
        mdl.SceneGraphRasterModel(bg, {}, mdl.SceneGraphConfig(strategy="mcmc", absgrad=True))
    mdl.SceneGraphRasterModel(bg, {}, mdl.SceneGraphConfig(absgrad=True))  # the default strategy takes it
