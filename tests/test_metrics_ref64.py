"""CPU checks of the per-step metrics: the float64 oracle (oracle/metrics_ref64.py) on closed-form cases and against the
reference's torch expressions in float64, and the argument validation of sgn_metrics through ctypes (no launch, no GPU)."""
import ctypes
import math

import numpy as np
import pytest
import torch

from oracle import metrics_ref64 as ref


def test_constant_offset_gives_the_closed_form_psnr():
    rng = np.random.default_rng(1)
    gt = (rng.integers(0, 48, (7, 9, 3)) / 64.0).astype(np.float32)
    c = 2.0 ** -4  # exact in fp32 together with gt: every difference is exactly c
    rgb = (gt + np.float32(c)).astype(np.float32)
    assert ref.psnr(rgb, gt) == pytest.approx(-20.0 * math.log10(c), abs=1e-12)
    # a constant fractional mask m scales the difference: 10 log10(1 / (m c)^2)
    m = np.full((7, 9, 1), 0.5, np.float32)
    assert ref.psnr(rgb, gt, m) == pytest.approx(-20.0 * math.log10(0.5 * c), abs=1e-12)


def test_equal_images_and_all_zero_mask_give_inf():
    rgb = np.random.default_rng(2).random((5, 4, 3)).astype(np.float32)
    assert ref.psnr(rgb, rgb.copy()) == math.inf
    other = np.random.default_rng(3).random((5, 4, 3)).astype(np.float32)
    assert ref.psnr(rgb, other, np.zeros((5, 4, 1), np.float32)) == math.inf


def test_uint8_gt_is_read_as_float_over_255():
    u8 = np.random.default_rng(4).integers(0, 256, (6, 5, 3)).astype(np.uint8)
    rgb = np.random.default_rng(5).random((6, 5, 3)).astype(np.float32)
    f = (torch.from_numpy(u8).float() / 255.0).numpy()
    assert ref.psnr(rgb, u8) == ref.psnr(rgb, f)
    assert ref.psnr(f, u8) == math.inf


def test_zero_log_scale_and_zero_logit():
    s = [np.zeros((10, 3), np.float32), np.zeros((3, 3), np.float32)]
    o = [np.zeros((10, 1), np.float32), np.zeros((3, 1), np.float32)]
    assert ref.param_means(s, o) == (1.0, 0.0, 0.5)


def test_empty_means_are_nan_and_overflow_is_inf():
    e = ref.param_means([np.zeros((0, 3), np.float32)], [np.zeros((0, 1), np.float32)])
    assert all(math.isnan(v) for v in e)
    assert math.isnan(ref.radii_mean(np.zeros(0, np.int32)))
    big = ref.param_means([np.full((2, 3), 100.0, np.float32)], [np.array([[100.0], [-100.0]], np.float32)])
    assert big[0] == math.inf and big[1] == 100.0 and big[2] == pytest.approx(0.5, abs=1e-15)
    # torch gives the same inf for the overflowing fp32 exp
    assert torch.exp(torch.full((2, 3), 100.0)).mean().item() == math.inf


def test_oracle_matches_the_reference_expressions_in_float64():
    """get_metrics_dict's torch statements (sgn_splatfacto.py:1031-1037) evaluated in float64 on the concatenation."""
    rng = np.random.default_rng(6)
    scales = [rng.normal(-3, 1, (n, 3)).astype(np.float32) for n in (300, 0, 129)]
    opac = [rng.normal(0, 3, (n, 1)).astype(np.float32) for n in (300, 0, 129)]
    radii = rng.integers(0, 40, 429).astype(np.int32)
    rgb = rng.random((12, 17, 3)).astype(np.float32)
    gt = rng.random((12, 17, 3)).astype(np.float32)
    mask = rng.random((12, 17, 1)).astype(np.float32)
    got = ref.metrics(rgb, gt, mask, scales, opac, radii)
    S = torch.from_numpy(np.concatenate(scales)).double()
    O = torch.from_numpy(np.concatenate(opac)).double()
    g, r, m = (torch.from_numpy(a) for a in (gt, rgb, mask))
    d = (g * m - r * m).double()
    want = [10 * math.log10(1 / float((d ** 2).mean())), float(torch.exp(S).mean()), float(S.mean()),
            float(torch.sigmoid(O).mean()), float(torch.from_numpy(radii).double().mean())]
    np.testing.assert_allclose(got[1:], want[1:], rtol=1e-12, atol=0)
    assert abs(got[0] - want[0]) <= 1e-6  # the squares are fp32 in the oracle (as in the kernel): 2^-24 relative each


@pytest.fixture(scope="module")
def lib():
    import street_gaussians_ns_b200.build as b
    from street_gaussians_ns_b200 import _lib
    b.build()
    return _lib.load(), _lib


def test_argument_validation_without_gpu(lib):
    L, mod = lib
    p = ctypes.c_void_p(256)
    sb = L.sgn_metrics_scratch_bytes()
    assert sb > 0
    li = mod.LossIn()
    li.rgb, li.gt_u8 = 256, 256
    launches = L.sgn_launch_count()

    def call(info=li, table=p, nseg=1, radii=p, out=p, scratch=p, nbytes=sb, H=8, W=8):
        return L.sgn_metrics(H, W, ctypes.byref(info) if info is not None else None, table, nseg, 128, 1, radii, out, scratch,
                             nbytes, None)

    assert call(table=None, nseg=2) == -1 and b"null segment table" in L.sgn_last_error()
    both = mod.LossIn()
    both.rgb, both.gt_u8, both.gt_f32 = 256, 256, 256
    assert call(info=both) == -1 and b"exactly one" in L.sgn_last_error()
    nogt = mod.LossIn()
    nogt.rgb = 256
    assert call(info=nogt) == -1 and b"exactly one" in L.sgn_last_error()
    assert call(nbytes=sb - 1) == -3 and b"scratch too small" in L.sgn_last_error()
    assert call(out=None) == -1 and call(scratch=None) == -1
    assert call(H=0) == -1 and b"empty image" in L.sgn_last_error()
    assert call(nseg=-1) == -1
    assert L.sgn_launch_count() == launches  # nothing was launched
