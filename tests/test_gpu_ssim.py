"""The SSIM loss term on the GPU (csrc/ssim.cu through loss.fused_ssim_loss and model.get_loss_dict) against the float64
oracle (oracle/ssim_ref64.py).  The accuracy bars are set by torch fp32 model.ssim's own errors on the same case on the
same GPU: e_t (value), r_t (gradient relative L2), m_t (gradient max-abs over max|ref|):

    value     |d| <= max(2 e_t, 2e-6), and <= 1e-4
    gradient  rel L2 <= max(2 r_t, 2e-5), and <= 5e-4;  max-abs <= max(2 m_t, 5e-5) * max|ref|

When SGN_SSIM_REPORT_DIR is set, the observed errors of every case are written there as JSON lines."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import ssim_ref64 as ref
from street_gaussians_ns_b200 import _lib
from street_gaussians_ns_b200.loss import fused_ssim_loss
from street_gaussians_ns_b200.model import ssim

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
WEIGHT, GRAD = 0.2, 1.7  # the reference's ssim_lambda; an incoming gradient != 1
SIZES = [(11, 11), (11, 40), (40, 11), (12, 13), (37, 53), (129, 257), (240, 320), (1280, 1920)]
CONTENTS = ["random", "smooth", "near_constant", "saturated", "equal"]
MASKS = [None, "binary", "fractional"]


def make_case(H, W, content, mask_kind, seed=0):
    """(gt uint8 [H,W,3], rgb float32 [H,W,3], mask float32 [H,W,1] or None) as numpy arrays."""
    rng = np.random.default_rng([H, W, CONTENTS.index(content), MASKS.index(mask_kind), seed])
    if content == "random":
        gt = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        rgb = rng.random((H, W, 3), dtype=np.float32)
    elif content == "smooth":
        yy, xx = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
        base = 0.5 + 0.4 * np.sin(xx / 9.0 + np.arange(3)[:, None, None] * 0.7).transpose(1, 2, 0) * np.cos(yy / 13.0)[..., None]
        gt = np.clip(np.rint(255 * (base + 0.02 * rng.standard_normal((H, W, 3)))), 0, 255).astype(np.uint8)
        rgb = np.clip(base + 0.05 * rng.standard_normal((H, W, 3)), 0, 1).astype(np.float32)
    elif content == "near_constant":  # E[y^2] - mu_y^2 cancels
        gt = (128 + rng.integers(-1, 2, (H, W, 3))).astype(np.uint8)
        rgb = (0.5 + 1e-3 * rng.standard_normal((H, W, 3))).astype(np.float32)
    elif content == "saturated":  # 0 / 1 blocks, different in gt and rgb
        gt = (255 * (rng.random((H // 4 + 1, W // 4 + 1, 3)) > 0.5)).astype(np.uint8).repeat(4, 0).repeat(4, 1)[:H, :W]
        rgb = (rng.random((H // 3 + 1, W // 3 + 1, 3)) > 0.5).astype(np.float32).repeat(3, 0).repeat(3, 1)[:H, :W].copy()
    else:  # equal: x == y
        gt = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        rgb = gt.astype(np.float32) / np.float32(255)
    mask = None
    if mask_kind == "binary":
        mask = (rng.random((H, W, 1)) > 0.3).astype(np.float32)
    elif mask_kind == "fractional":
        mask = rng.random((H, W, 1), dtype=np.float32)
    return np.ascontiguousarray(gt), np.ascontiguousarray(rgb), mask


def gt_float(gt_u8):
    return gt_u8.astype(np.float32) / np.float32(255)  # the kernels' u8 / 255.0f (IEEE division)


def run_fused(rgb, gt, mask, weight=WEIGHT, grad=GRAD):
    y = torch.from_numpy(rgb).to(DEV).requires_grad_(True)
    m = None if mask is None else torch.from_numpy(mask).to(DEV)
    loss = fused_ssim_loss(y, torch.from_numpy(gt).to(DEV), mask=m, weight=weight)
    (loss * grad).backward()
    return loss.detach(), y.grad


def run_torch(rgb, gt_f, mask, weight=WEIGHT, grad=GRAD):
    y = torch.from_numpy(rgb).to(DEV).requires_grad_(True)
    x = torch.from_numpy(gt_f).to(DEV)
    ym = y
    if mask is not None:
        m = torch.from_numpy(mask).to(DEV)
        x, ym = x * m, y * m
    loss = weight * (1 - ssim(x.permute(2, 0, 1)[None], ym.permute(2, 0, 1)[None]))
    (loss * grad).backward()
    return float(loss.detach()), y.grad.cpu().numpy().astype(np.float64)


def errors(loss, v, l_ref, v_ref):
    d = v - v_ref
    return (abs(loss - l_ref), float(np.linalg.norm(d) / max(np.linalg.norm(v_ref), 1e-300)),
            float(np.abs(d).max() / max(np.abs(v_ref).max(), 1e-300)))


def report(**kw):
    d = os.environ.get("SGN_SSIM_REPORT_DIR")
    if d:
        os.makedirs(d, exist_ok=True)
        with open(os.path.join(d, "ssim_errors.jsonl"), "a") as f:
            f.write(json.dumps(kw) + "\n")


def check_case(H, W, content, mask_kind):
    gt, rgb, mask = make_case(H, W, content, mask_kind)
    gf = gt_float(gt)
    l_ref, v_ref, _ = ref.ssim_loss(rgb, gf, mask, weight=WEIGHT, grad=GRAD)
    l_u8, v_u8 = run_fused(rgb, gt, mask)
    l_f32, v_f32 = run_fused(rgb, gf, mask)
    l_again, v_again = run_fused(rgb, gt, mask)
    # uint8 and float gt read the same values; two runs are bit-identical (fixed-order sums, a gather backward)
    assert torch.equal(l_u8, l_f32) and torch.equal(v_u8, v_f32)
    assert torch.equal(l_u8, l_again) and torch.equal(v_u8, v_again)
    l_t, v_t = run_torch(rgb, gf, mask)
    loss, v = float(l_u8), v_u8.cpu().numpy().astype(np.float64)
    e_f, r_f, m_f = errors(loss, v, l_ref, v_ref)
    e_t, r_t, m_t = errors(l_t, v_t, l_ref, v_ref)
    report(H=H, W=W, content=content, mask=mask_kind, e=e_f, e_t=e_t, r=r_f, r_t=r_t, m=m_f, m_t=m_t,
           vmax=float(np.abs(v).max()), vmax_t=float(np.abs(v_t).max()))
    assert e_f <= max(2 * e_t, 2e-6) and e_f <= 1e-4, (e_f, e_t)
    if content == "equal":
        # the exact gradient is 0: what is left is rounding, far below the 1/count scale of a gradient element
        k = WEIGHT * GRAD / (3 * (H - 10) * (W - 10))
        assert np.abs(v).max() <= max(2 * np.abs(v_t).max(), 1e-3 * k), (np.abs(v).max(), np.abs(v_t).max(), k)
        return
    assert r_f <= max(2 * r_t, 2e-5) and r_f <= 5e-4, (r_f, r_t)
    assert m_f <= max(2 * m_t, 5e-5), (m_f, m_t)


@pytest.mark.parametrize("H,W", SIZES)
def test_sizes(H, W):
    check_case(H, W, "random", None)


@pytest.mark.parametrize("mask_kind", MASKS)
@pytest.mark.parametrize("content", CONTENTS)
@pytest.mark.parametrize("H,W", [(37, 53), (129, 257)])
def test_contents_and_masks(H, W, content, mask_kind):
    check_case(H, W, content, mask_kind)


@pytest.mark.parametrize("content,mask_kind", [("smooth", "fractional"), ("saturated", "binary")])
def test_full_size(content, mask_kind):
    check_case(1280, 1920, content, mask_kind)


def test_weight_and_incoming_gradient_scale_linearly():
    gt, rgb, mask = make_case(129, 257, "smooth", "fractional")
    l1, v1 = run_fused(rgb, gt, mask, weight=1.0, grad=1.0)
    l2, v2 = run_fused(rgb, gt, mask, weight=0.35, grad=-2.5)
    assert float(l2) == pytest.approx(0.35 * float(l1), rel=1e-6)
    assert torch.allclose(v2, -2.5 * 0.35 * v1, rtol=1e-5, atol=1e-12)
    l0 = fused_ssim_loss(torch.from_numpy(rgb).to(DEV).requires_grad_(True), torch.from_numpy(gt).to(DEV), weight=0.0)
    assert float(l0) == 0.0 and not l0.requires_grad


@pytest.mark.parametrize("H,W", [(10, 40), (40, 10), (10, 10)])
def test_small_image_raises(H, W):
    rgb = torch.rand(H, W, 3, device=DEV, requires_grad=True)
    gt = torch.zeros(H, W, 3, device=DEV, dtype=torch.uint8)
    with pytest.raises(_lib.SgnError, match="11 x 11"):
        fused_ssim_loss(rgb, gt, weight=0.2)


def test_no_host_synchronisation():
    gt, rgb, mask = make_case(240, 320, "random", "binary")
    y = torch.from_numpy(rgb).to(DEV).requires_grad_(True)
    g, m = torch.from_numpy(gt).to(DEV), torch.from_numpy(mask).to(DEV)
    fused_ssim_loss(y, g, mask=m, weight=WEIGHT).backward()  # first call: module load, allocator
    torch.cuda.synchronize()
    y.grad = None
    torch.cuda.set_sync_debug_mode("error")
    try:
        loss = fused_ssim_loss(y, g, mask=m, weight=WEIGHT)
        loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert y.grad is not None and torch.isfinite(y.grad).all()


# ---- model.get_loss_dict ----------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def model_setup():
    import street_gaussians_ns_b200.synthetic as syn
    from street_gaussians_ns_b200.model import ActorPose, SceneGraphConfig, SceneGraphRasterModel
    fr = syn.make_frame(n_background=20000, n_actors=4, n_per_actor=1500, width=320, height=240, seed=3,
                        actor_shift=np.array([1.0, 0.0, -1.0]))
    bg = fr.segments[0].params.to(DEV)
    actors = {s.name.replace("object_", ""): s.params.to(DEV) for s in fr.segments[1:]}
    poses = [ActorPose(s.name.replace("object_", ""), s.rot, s.center, 21, list(range(85))) for s in fr.segments[1:]]
    model = SceneGraphRasterModel(bg, actors, SceneGraphConfig(use_sky_sphere=False, ssim_lambda=0.2),
                                  poses_at=lambda t: poses).to(DEV)
    model.train()
    model.step = 30000
    H, W = fr.camera.height, fr.camera.width
    g = torch.Generator().manual_seed(4)
    image = (torch.rand(H, W, 3, generator=g) * 255).to(torch.uint8).to(DEV)
    mask = (torch.rand(H, W, 1, generator=g) > 0.1).float().to(DEV)
    return fr, model, image, mask


def test_get_loss_dict_simloss_and_rgb_cotangent(model_setup):
    fr, model, image, mask = model_setup
    with torch.no_grad():
        rgb0 = model.get_outputs(fr.camera)["rgb"].detach().clone()
    gt_np = image.cpu().numpy()
    rgb_np, mask_np = rgb0.cpu().numpy(), mask.cpu().numpy()
    l_ref, v_ref, _ = ref.ssim_loss(rgb_np, gt_float(gt_np), mask_np, weight=0.2)
    res = {}
    try:
        for fused in (False, True):
            model.config.fused_loss = fused
            rgb = rgb0.clone().requires_grad_(True)
            losses = model.get_loss_dict({"rgb": rgb, "accumulation": torch.ones_like(rgb[..., :1]),
                                          "object_acc": torch.zeros_like(rgb[..., :1])}, {"image": image, "mask": mask})
            losses["simloss"].backward()
            res[fused] = (set(losses), float(losses["simloss"].detach()), rgb.grad.cpu().numpy().astype(np.float64))
    finally:
        model.config.fused_loss = True
    assert res[True][0] == res[False][0]
    e_t, r_t, m_t = errors(res[False][1], res[False][2], l_ref, v_ref)
    e_f, r_f, m_f = errors(res[True][1], res[True][2], l_ref, v_ref)
    report(case="get_loss_dict", e=e_f, e_t=e_t, r=r_f, r_t=r_t, m=m_f, m_t=m_t)
    assert e_f <= max(2 * e_t, 2e-6) and e_f <= 1e-4, (e_f, e_t)
    assert r_f <= max(2 * r_t, 2e-5) and r_f <= 5e-4, (r_f, r_t)
    assert m_f <= max(2 * m_t, 5e-5), (m_f, m_t)


def test_full_model_backward_deterministic(model_setup, monkeypatch):
    from street_gaussians_ns_b200 import raster
    from street_gaussians_ns_b200.scene import PARAM_NAMES
    fr, model, image, mask = model_setup
    monkeypatch.setattr(raster, "DETERMINISTIC", True)
    grads = {}
    try:
        for fused in (False, True):
            model.config.fused_loss = fused
            for p in model.parameters():
                p.grad = None
            out = model.get_outputs(fr.camera)
            losses = model.get_loss_dict(out, {"image": image, "mask": mask})
            assert float(losses["simloss"]) > 0
            sum(losses.values()).backward()
            grads[fused] = {(name, k): model.all_models[name].gauss_params[k].grad.detach().clone()
                            for name in model.visible_model_names for k in PARAM_NAMES}
    finally:
        model.config.fused_loss = True
    assert grads[True].keys() == grads[False].keys()
    worst = 0.0
    for key, a in grads[False].items():
        b = grads[True][key]
        rel = float(torch.linalg.vector_norm((b - a).double()) / max(float(torch.linalg.vector_norm(a.double())), 1e-30))
        worst = max(worst, rel)
        assert rel <= 1e-4, (key, rel)
    report(case="full_model_backward", worst_rel_l2=worst)
