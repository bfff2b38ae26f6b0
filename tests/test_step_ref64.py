"""Pins oracle/step_ref64.py on the CPU: the loss statements against the torch expressions of ``get_loss_dict`` in
float64 (values and autograd cotangents) and against the reference's own loss values in tests/golden/reference_vectors.npz;
the densification replay against after_train's torch expressions and the golden statistics; Adam against
torch.optim.Adam; the exchange's parts and skipped units against a brute-force enumeration, float by float."""
import os

import numpy as np
import pytest
import torch

from oracle import step_ref64 as ref
from tests import step_cases as sc

f32 = np.float32
GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "reference_vectors.npz"))


def torch_losses64(rgb, gt, mask, acc, sky, oa, w):
    """get_loss_dict's torch expressions (model.py, fused_loss=False) in float64, with autograd."""
    gt_img = torch.from_numpy(ref.gt_float(gt)) if gt is not None else None
    out, leaves = [], []
    if rgb is not None:
        r = torch.from_numpy(rgb.astype(np.float64)).requires_grad_(True)
        leaves.append(r)
        g, rr = gt_img, r
        if mask is not None:
            m = torch.from_numpy(mask.astype(np.float64))
            g, rr = g * m, r * m
        out.append(float(f32(w[0])) * torch.abs(g - rr).mean())
    if acc is not None:
        a = torch.from_numpy(acc.astype(np.float64)).requires_grad_(True)
        leaves.append(a)
        out.append(float(f32(w[1])) * (torch.from_numpy(sky != 0) * a).mean())
    if oa is not None:
        o = torch.from_numpy(oa.astype(np.float64)).requires_grad_(True)
        leaves.append(o)
        c = torch.clamp(o, min=float(ref.CLAMP_LO), max=float(ref.CLAMP_HI))
        out.append(float(f32(w[2])) * -(c * torch.log(c) + (1.0 - c) * torch.log(1.0 - c)).mean())
    return out, leaves


def test_clamp_bounds_are_torchs():
    assert ref.CLAMP_HI == f32(1 - 1e-5) and ref.CLAMP_LO == f32(1e-5)
    # torch clamps a float32 tensor at the fp32 bounds, and passes the gradient at them (closed interval)
    x = torch.tensor([ref.CLAMP_LO, ref.CLAMP_HI, np.nextafter(ref.CLAMP_LO, f32(0)), np.nextafter(ref.CLAMP_HI, f32(1))],
                     requires_grad=True)
    torch.clamp(x, min=1e-5, max=1 - 1e-5).sum().backward()
    assert x.grad.tolist() == [1.0, 1.0, 0.0, 0.0]


@pytest.mark.parametrize("case", [c for c in sc.LOSS_CASES if c.P <= 100_000], ids=lambda c: c.name)
def test_loss_statement_matches_torch_float64(case):
    d = sc.loss_inputs(case)
    got = ref.loss_fwd64(case.P, **d, w=case.w)
    terms, leaves = torch_losses64(d["rgb"], d["gt"], d["mask"], d["accumulation"], d["sky_mask"], d["object_acc"], case.w)
    want = {t: float(v.detach()) for t, v in zip([t for t in ("l1", "sky", "ent") if t in case.terms], terms)}
    for i, t in enumerate(("l1", "sky", "ent")):
        np.testing.assert_allclose(got[i], want.get(t, 0.0), rtol=1e-13, atol=1e-300, err_msg=t)
    g = (0.7, -1.3, 2.5)
    sum(gi * tv for gi, tv in zip([g[i] for i, t in enumerate(("l1", "sky", "ent")) if t in case.terms], terms)).backward()
    v64 = ref.loss_bwd64(case.P, d["rgb"], d["gt"], d["mask"], d["sky_mask"], d["object_acc"], case.w, g)
    present = [v for v in v64 if v is not None]
    assert len(present) == len(leaves)
    for v, leaf in zip(present, leaves):
        np.testing.assert_allclose(v, leaf.grad.numpy().reshape(-1), rtol=1e-11, atol=1e-18)
    # the float32 replay: L1 / sky cotangents are k-scaled signs (exact up to k's rounding), entropy within its bound
    v32 = ref.loss_bwd_f32(case.P, d["rgb"], d["gt"], d["mask"], d["sky_mask"], d["object_acc"], case.w, g)
    if d["rgb"] is not None:
        # away from ties: a u8 ground truth is u8 / 255 in float64 but fp32(u8) / 255.f in the kernel
        gf, r = ref.gt_float(d["gt"]).reshape(-1), d["rgb"].astype(np.float64).reshape(-1)
        far = np.abs(gf - r) > 4 * ref.U * (np.abs(gf) + np.abs(r))
        np.testing.assert_allclose(v32[0][far], v64[0][far], rtol=4 * ref.U, atol=0)
    if d["object_acc"] is not None:
        assert np.all(np.abs(v32[2].astype(np.float64) - v64[2]) <= ref.ent_bwd_bound(case.P, d["object_acc"], case.w[2], g[2])
                      + abs(v64[2]) * 4 * ref.U)


def test_loss_ties_have_a_zero_cotangent():
    c = next(x for x in sc.LOSS_CASES if x.name.startswith("16x16") and x.mask == "frac")
    d = sc.loss_inputs(c)
    v = ref.loss_bwd_f32(c.P, d["rgb"], d["gt"], d["mask"], d["sky_mask"], d["object_acc"], c.w)[0]
    tie = (ref.gt_f32(d["gt"]) == d["rgb"]).reshape(-1)
    assert tie.sum() > 20 and np.all(v[tie] == 0) and np.all(v[~tie & (np.repeat(d["mask"].reshape(-1), 3) != 0)] != 0)


@pytest.mark.parametrize("tag", ["plain", "masked"])
def test_loss_statement_matches_the_reference_values(tag):
    w = GOLD["loss_weights"]   # ssim_lambda, sky mult, entropy mult, stop_split_at
    sem = GOLD["loss_semantic"]
    mask = GOLD["loss_mask"] if tag == "masked" else None
    P = sem.size
    got = ref.loss_fwd64(P, GOLD["loss_rgb"], GOLD["loss_gt"], mask, GOLD["loss_accumulation"], (sem == 2).astype(np.uint8),
                         GOLD["loss_object_acc"], w=(1 - w[0], w[1], w[2]))
    np.testing.assert_allclose(got, GOLD[f"loss_{tag}"], rtol=1e-6, atol=0)


def test_loss_bound_is_the_stated_one():
    """The forward bound of the 1920x1280 case: a summation depth of 52 additions for L1 (28 per thread, 3 inside a float4
    unit, 8 + 5 + 8 in the trees) and 34 for the per-pixel terms."""
    assert ref.sum_depth(3 * 1920 * 1280) == 28 + 3 + 8 + 5 + 8
    assert ref.sum_depth(1920 * 1280) == 10 + 3 + 8 + 5 + 8
    c = next(x for x in sc.LOSS_CASES if x.name == "1280x1920_plain")
    d = sc.loss_inputs(c)
    b = ref.loss_fwd_bound(c.P, **d, w=c.w) / ref.loss_fwd64(c.P, **d, w=c.w)
    assert np.all(b < 1e-4) and np.all(b > 1e-6), b


def test_densify_replay_matches_after_train_expressions():
    for call in range(2):
        n = GOLD["stats_radii_0"].shape[0]
        H, W = (int(x) for x in GOLD["stats_size"])
        prev = None if call == 0 else tuple(GOLD[f"stats_{k}_0"] for k in ("xys_grad_norm", "vis_counts", "max_2Dsize"))
        got = ref.densify_f32(GOLD[f"stats_xys_grad_{call}"], GOLD[f"stats_radii_{call}"], call == 0, prev, H, W)
        for k, g in zip(("xys_grad_norm", "vis_counts", "max_2Dsize"), got):
            np.testing.assert_allclose(g, GOLD[f"stats_{k}_{call}"], rtol=2e-6, atol=0, err_msg=k)
        assert n == got[0].shape[0]
    # torch's statements (sgn_splatfacto.py:513-541) on a directed case, second call
    c = sc.DENSIFY_CASES[0]
    v, r = c.inputs(1)
    prev = c.prior(c.N, 0)
    got = ref.densify_f32(v[:, :2], r, False, prev, c.H, c.W)
    vis = torch.from_numpy(r > 0)
    grads = torch.from_numpy(v[:, :2]).norm(dim=-1)
    g0, c0, m0 = (torch.from_numpy(x.copy()) for x in prev)
    c0[vis] += 1
    g0[vis] = grads[vis] + g0[vis]
    m0[vis] = torch.maximum(m0[vis], torch.from_numpy(r).float()[vis] / float(max(c.H, c.W)))
    np.testing.assert_array_equal(got[1], c0.numpy())
    np.testing.assert_allclose(got[0], g0.numpy(), rtol=2e-7, atol=0)
    np.testing.assert_allclose(got[2], m0.numpy(), rtol=2e-7, atol=0)


def _adam_row(lr, step, betas=(0.9, 0.999), eps=1e-15):
    from street_gaussians_ns_b200.optim import ADAM_DTYPE
    row = np.zeros(1, ADAM_DTYPE)[0]
    b1, b2 = betas
    row["beta1"], row["beta2"], row["eps"] = b1, b2, eps
    row["one_minus_beta1"], row["one_minus_beta2"] = 1.0 - b1, 1.0 - b2
    row["step_size"], row["sqrt_bc2"] = lr / (1.0 - b1 ** step), np.sqrt(1.0 - b2 ** step)
    return row


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_adam_statement_matches_torch_adam(dtype):
    """adam64 equals torch.optim.Adam in float64.  adam_f32 agrees with it in float32 to 2e-6 of each array's largest
    magnitude: torch's CPU kernels fuse the lerp into an fma (m + w1 (g - m) cancels when m is small against g, so m may
    differ by many ulps of itself) and form step_size * m / denom in another order; the kernel rounds each operation as
    adam_f32 states, which the GPU tests hold it to bit for bit."""
    rng = np.random.default_rng(3)
    n = 4097
    p0 = rng.normal(size=n).astype(f32)
    p = torch.from_numpy(p0.astype(np.float64 if dtype == torch.float64 else f32)).requires_grad_(True)
    opt = torch.optim.Adam([p], lr=0.005, eps=1e-15, foreach=False)
    mine, m, v = p0.copy(), np.zeros(n, f32), np.zeros(n, f32)
    m64, v64, p64 = np.zeros(n), np.zeros(n), p0.astype(np.float64)
    for step in range(1, 6):
        g = rng.normal(size=n).astype(f32) * (rng.random(n) > 0.3)
        g[:8] = [1e-15, -1e-15, 1e-20, 0, 1e-30, 3e-16, -2e-38, 1e-44]
        p.grad = torch.from_numpy(g.astype(np.float64) if dtype == torch.float64 else g.copy())
        opt.step()
        if dtype == torch.float64:
            p64, m64, v64 = ref.adam64(p64, g, m64, v64, 0.005, step)
        else:
            mine, m, v = ref.adam_f32(mine, g, m, v, _adam_row(0.005, step))
    st = opt.state[p]
    if dtype == torch.float64:
        np.testing.assert_allclose(p64, p.detach().numpy(), rtol=1e-14, atol=0)
        np.testing.assert_allclose(v64, st["exp_avg_sq"].numpy(), rtol=1e-14, atol=0)
    else:
        for a, b in ((mine, p.detach().numpy()), (m, st["exp_avg"].numpy()), (v, st["exp_avg_sq"].numpy())):
            np.testing.assert_allclose(a, b, rtol=0, atol=2e-6 * float(np.abs(b).max()))
            assert np.mean(a == b) > 0.5


def test_exchange_parts_cover_every_unit_once():
    for world in (1, 2, 3, 4, 8):
        for len4 in list(range(0, 40)) + [1000, 1001, 4096 * 3 + 7]:
            parts = [ref.my_part(len4, r, world) for r in range(world)]
            owner = -np.ones(len4, int)
            for r, (b, e) in enumerate(parts):
                assert 0 <= b <= e <= len4 and e - b <= -(-len4 // world)
                assert np.all(owner[b:e] == -1)
                owner[b:e] = r
            assert np.all(owner >= 0) and np.all(np.diff(owner) >= 0)   # every unit once, parts in rank order


def _skipped_brute(length, width, nrows, vis_rows):
    skip = []
    for i in range(length // 4):
        seen = False
        for fl in range(4 * i, 4 * i + 4):
            r = fl // width
            if r < nrows and vis_rows[r]:
                seen = True
        skip.append(not seen)
    return np.array(skip, bool)


@pytest.mark.parametrize("case", [c for c in sc.EXCHANGE_CASES if c.union_rows], ids=lambda c: c.name)
def test_exchange_skipped_units_match_enumeration(case):
    for world in case.worlds:
        union = sc.rank_flags(case, world).max(axis=0)
        for sl in case.slices:
            vis = union[sl.row0:sl.row0 + sl.nrows]
            got = ref.skipped_units(sl.length // 4, sl.width, sl.nrows, vis)
            np.testing.assert_array_equal(got, _skipped_brute(sl.length, sl.width, sl.nrows, vis), err_msg=f"w={sl.width}")
            if case.pattern == "none":
                assert got.all()
            if case.pattern == "all":
                assert got.sum() == sl.length // 4 - (-(-sl.width * sl.nrows // 4)) and not got[0]


def test_cases_drive_what_they_are_named_for():
    shapes = {(c.H, c.W) for c in sc.LOSS_CASES}
    assert {(1, 1), (7, 1), (2, 1), (6, 3), (1280, 1920)} <= shapes
    assert any(c.P * 3 % 2 == 1 for c in sc.LOSS_CASES) and any(c.P * 3 % 4 == 2 for c in sc.LOSS_CASES)
    assert {c.u8_off for c in sc.LOSS_CASES} == {0, 1, 2, 3} and {o for c in sc.LOSS_CASES for o in c.off} == {0, 1, 2, 3}
    for c in sc.DENSIFY_CASES:
        ends = [r0 + n for r0, n, _ in c.segs]
        assert all(a <= b for a, b in zip(ends[:-1], [r0 for r0, _, _ in c.segs[1:]])) and ends[-1] <= c.N
    assert any(c.segs[0][0] > 0 for c in sc.DENSIFY_CASES)
    assert {len(c.segs) for c in sc.DENSIFY_CASES} >= {1, 33, 1024}
    assert any(c.H > c.W for c in sc.DENSIFY_CASES) and any(c.W > c.H for c in sc.DENSIFY_CASES)
    widths = {sl.width for c in sc.EXCHANGE_CASES for sl in c.slices}
    assert {1, 2, 3, 4, 5, 6, 9, 45} <= widths
    assert max(len(c.slices) for c in sc.EXCHANGE_CASES) == 48
    for c in sc.EXCHANGE_CASES:
        for sl in c.slices:
            assert sl.off % 4 == 0 and sl.length % 4 == 0 and sl.nrows * sl.width <= sl.length
            assert sl.off + sl.length <= c.arena and (not sl.width or sl.row0 + sl.nrows < c.union_rows)
