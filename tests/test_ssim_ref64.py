"""CPU checks of the SSIM loss term: the float64 oracle (oracle/ssim_ref64.py) against torch float64 autograd of model.ssim
and against central differences; the window taps against torch's fp32 window (and the kernel's copy of them); and the
argument validation of sgn_ssim_fwd / sgn_ssim_bwd through ctypes (no launch, no GPU)."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from oracle import ssim_ref64 as ref
from street_gaussians_ns_b200.model import _gauss_window, ssim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _images(H, W, seed, mask_kind=None):
    rng = np.random.default_rng(seed)
    gt = rng.random((H, W, 3))
    rgb = np.clip(0.6 * gt + 0.4 * rng.random((H, W, 3)), 0, 1)
    mask = None
    if mask_kind == "binary":
        mask = (rng.random((H, W, 1)) > 0.3).astype(np.float64)
    elif mask_kind == "fractional":
        mask = rng.random((H, W, 1))
    return rgb, gt, mask


def _torch_loss64(rgb, gt, mask, weight, taps=None):
    y = torch.tensor(rgb, dtype=torch.float64, requires_grad=True)
    x = torch.tensor(gt, dtype=torch.float64)
    xm, ym = x, y
    if mask is not None:
        m = torch.tensor(mask, dtype=torch.float64)
        xm, ym = x * m, y * m
    loss = weight * (1 - ssim(xm.permute(2, 0, 1)[None], ym.permute(2, 0, 1)[None]))
    loss.backward()
    return float(loss.detach()), y.grad.numpy()


@pytest.mark.parametrize("H,W,mask_kind", [(11, 11, None), (12, 13, "binary"), (20, 23, None), (24, 17, "fractional")])
def test_oracle_matches_torch_float64_autograd(H, W, mask_kind):
    rgb, gt, mask = _images(H, W, H * 100 + W, mask_kind)
    weight = 0.2
    lt, gt_grad = _torch_loss64(rgb, gt, mask, weight)
    lo, go, _ = ref.ssim_loss(rgb, gt, mask, weight=weight, taps=ref.window())  # torch's window in float64
    assert abs(lo - lt) <= 1e-12 * abs(lt)
    assert np.linalg.norm(go - gt_grad) <= 1e-12 * np.linalg.norm(gt_grad)
    assert np.abs(go - gt_grad).max() <= 1e-12 * np.abs(gt_grad).max()


@pytest.mark.parametrize("mask_kind", [None, "fractional"])
def test_oracle_gradient_against_central_differences(mask_kind):
    H, W = 13, 14
    rgb, gt, mask = _images(H, W, 7, mask_kind)
    weight, g = 0.7, 1.3
    _, grad, _ = ref.ssim_loss(rgb, gt, mask, weight=weight, grad=g)
    h = 1e-6
    fd = np.zeros_like(rgb)
    for idx in np.ndindex(*rgb.shape):
        p, m = rgb.copy(), rgb.copy()
        p[idx] += h
        m[idx] -= h
        fd[idx] = g * (ref.ssim_loss(p, gt, mask, weight=weight)[0] - ref.ssim_loss(m, gt, mask, weight=weight)[0]) / (2 * h)
    assert np.abs(fd - grad).max() <= 1e-7 * np.abs(grad).max()
    # the value is linear in the weight, the gradient in weight and incoming gradient
    l1, g1, _ = ref.ssim_loss(rgb, gt, mask)
    assert ref.ssim_loss(rgb, gt, mask, weight=weight)[0] == pytest.approx(weight * l1, rel=1e-14)
    assert np.allclose(grad, weight * g * g1, rtol=1e-13, atol=0)


def test_identical_images_give_zero_loss_and_gradient():
    rgb, _, _ = _images(15, 16, 3)
    loss, grad, maps = ref.ssim_loss(rgb, rgb)
    assert abs(loss) < 1e-14 and np.abs(grad).max() < 1e-15
    assert np.allclose(maps["S"], 1.0, rtol=0, atol=1e-14)


def test_window_taps_are_torch_float32():
    w = _gauss_window(11, 1.5, "cpu", torch.float32).numpy()
    assert w.dtype == np.float32 and np.array_equal(w, ref.TAPS_F32)
    # the kernels' copy of the taps (csrc/ssim.cu kTaps, hex float literals)
    src = open(os.path.join(ROOT, "street-gaussians-ns_b200", "csrc", "ssim.cu")).read()
    body = re.search(r"kTaps\[11\]\s*=\s*\{(.*?)\}", src, flags=re.S).group(1)
    lits = [float.fromhex(s.strip().rstrip("f")) for s in body.split(",")]
    assert np.array_equal(np.array(lits, dtype=np.float32), ref.TAPS_F32)
    assert np.abs(ref.window() - w).max() < 1e-8


@pytest.fixture(scope="module")
def lib():
    import street_gaussians_ns_b200.build as b
    from street_gaussians_ns_b200 import _lib
    b.build()
    return _lib.load(), _lib


def test_workspace_bytes(lib):
    L, _ = lib
    assert L.sgn_ssim_workspace_bytes(10, 40) == 0 and L.sgn_ssim_workspace_bytes(40, 10) == 0
    for H, W in ((11, 11), (37, 53), (1280, 1920)):
        maps = 36 * (H - 10) * (W - 10)
        blocks = -(-(W - 10) // 32) * -(-(H - 10) // 16)
        assert L.sgn_ssim_workspace_bytes(H, W) == maps + -(-12 * blocks // 256) * 256


def test_argument_validation_without_gpu(lib):
    L, mod = lib
    p = ctypes.c_void_p(256)
    li = mod.LossIn()
    li.rgb, li.gt_u8 = 256, 256
    launches = L.sgn_launch_count()
    big = 1 << 40

    def fwd(H, W, info, nbytes=big):
        return L.sgn_ssim_fwd(H, W, ctypes.byref(info), 0.2, p, p, nbytes, None)

    for H, W in ((10, 40), (40, 10), (5, 5)):
        assert fwd(H, W, li) == -1 and b"11 x 11" in L.sgn_last_error()
        assert L.sgn_ssim_bwd(H, W, ctypes.byref(li), 0.2, None, p, p, None) == -1
        assert b"11 x 11" in L.sgn_last_error()
    both = mod.LossIn()
    both.rgb, both.gt_u8, both.gt_f32 = 256, 256, 256
    assert fwd(32, 32, both) == -1 and b"exactly one" in L.sgn_last_error()
    assert L.sgn_ssim_bwd(32, 32, ctypes.byref(both), 0.2, None, p, p, None) == -1
    nogt = mod.LossIn()
    nogt.rgb = 256
    assert fwd(32, 32, nogt) == -1
    norgb = mod.LossIn()
    norgb.gt_u8 = 256
    assert fwd(32, 32, norgb) == -1 and b"rgb" in L.sgn_last_error()
    need = L.sgn_ssim_workspace_bytes(32, 32)
    assert fwd(32, 32, li, need - 1) == -3 and b"workspace" in L.sgn_last_error()
    assert L.sgn_launch_count() == launches  # nothing was launched
