"""The objects-only accumulation rendered inside the main blend traversal, forward and backward.

Scenes that force each path of the fused kernels: actors behind a dense background (the objects-only streams outlive the
main ones, so the traversal continues on the object sub-list), actors in front (the objects-only streams end inside the
main traversal), and a tiny image under a very dense background (tiles long enough to be split into 8 strips, forward
and backward).  Each is compared with the C oracle at the bars of test_gpu_parity.py, and the object slot of the saved
state (final_T, final_idx) with the separate objects-only pass that preceded the fusion, bit for bit
(tests/golden/fused_object_slot.npz, written by tests/golden/make_golden_fused_object_slot.py)."""
import os

import numpy as np
import pytest
import torch

import street_gaussians_ns_b200.synthetic as syn
from street_gaussians_ns_b200 import raster
from street_gaussians_ns_b200.scene import Frame, Segment
from oracle import oracle_c

pytestmark = pytest.mark.gpu

RGB_TOL = 1e-4
GRAD_TOL = 1e-3
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fused_object_slot.npz")

SCENES = {
    "actors_behind": dict(n_background=250000, n_actors=8, n_per_actor=3000, width=64, height=48, seed=11,
                          actor_shift=np.array([0.0, 0.0, -60.0])),
    "actors_in_front": dict(n_background=60000, n_actors=4, n_per_actor=3000, width=128, height=96, seed=12,
                            actor_shift=np.array([0.0, 0.0, 4.0])),
    "eight_strips": dict(n_background=300000, n_actors=3, n_per_actor=6000, width=64, height=48, seed=5,
                         actor_shift=np.array([1.0, 0.0, 2.0])),
}


def rel_l2(a, b):
    a = np.asarray(a, np.float64).reshape(-1)
    b = np.asarray(b, np.float64).reshape(-1)
    d = np.linalg.norm(b)
    return np.linalg.norm(a - b) / d if d > 0 else np.linalg.norm(a)


def to_cuda(frame: Frame, requires_grad=False) -> Frame:
    segs = []
    for s in frame.segments:
        p = s.params.to("cuda")
        if requires_grad:
            p.requires_grad_(True)
        segs.append(Segment(p, s.cls, s.rot, s.center, s.idft, s.name))
    return Frame(frame.camera, segs)


def forward_state(frame: Frame, settings: raster.RenderSettings):
    """The blend forward's outputs and saved per-pixel state, stage by stage (as raster.forward_backward runs them)."""
    params = [seg.params.tensors() for seg in frame.segments]
    device = params[0][0].device
    cs = raster.camera_struct(frame.camera, settings)
    bo = raster.blend_opts(settings, False)
    table = raster.SegmentTable(frame, params, device)
    proj = raster.project_fwd(table, cs, device)
    records, radii, _, _ = proj
    M, sorted_ids, tile_bins = raster.bin_and_sort(cs, records, radii, proj=proj)
    cls_ids, cls_bins = raster.class_lists(cs, M, sorted_ids, tile_bins)
    out = raster.blend_fwd(cs, bo, records, sorted_ids, tile_bins, None, cls_ids, cls_bins)
    torch.cuda.synchronize()
    return out, tile_bins


@pytest.fixture(scope="module", params=list(SCENES))
def scene(request):
    fr = syn.make_frame(**SCENES[request.param])
    orc = oracle_c.Oracle(fr)
    return request.param, fr, orc, orc.forward()


def test_forward_parity_and_object_slot_bits(scene):
    name, fr, orc, fw = scene
    frc = to_cuda(fr)
    out, tile_bins = forward_state(frc, raster.RenderSettings())
    ok = fw.fragile == 0
    alpha = 1 - fw.final_T
    assert np.abs(out["accumulation"].cpu().numpy()[..., 0] - alpha)[ok].max() <= RGB_TOL
    assert np.abs(out["object_acc"].cpu().numpy()[..., 0] - (1 - fw.obj_T))[fw.fragile_obj == 0].max() <= RGB_TOL
    assert np.abs(out["background_acc"].cpu().numpy()[..., 0] - (1 - fw.bg_T))[fw.fragile_bg == 0].max() <= RGB_TOL
    gold = np.load(GOLDEN)
    np.testing.assert_array_equal(out["final_T"][1].cpu().numpy(), gold[name + "_T"])
    np.testing.assert_array_equal(out["final_idx"][1].cpu().numpy(), gold[name + "_idx"])
    td = out["tile_depth"].cpu().numpy()
    lens = (tile_bins[:, 1] - tile_bins[:, 0]).cpu().numpy()
    if name == "actors_behind":  # the objects-only streams ran past the main traversal
        assert td[1].max() > 0
    if name == "eight_strips":  # forward: lists above 4 x 1024 entries; backward: depth above 4 x 384
        assert lens.max() > 4 * 1024 and (td[0] + td[1]).max() > 4 * 384


def test_backward_parity(scene):
    name, fr, orc, fw = scene
    frc = to_cuda(fr, requires_grad=True)
    out, holder = raster.render_frame(frc, raster.RenderSettings())
    H, W = fr.camera.height, fr.camera.width
    g = torch.Generator().manual_seed(7)
    ok = torch.from_numpy(((fw.fragile == 0) & (fw.fragile_obj == 0) & (fw.fragile_bg == 0)).astype(np.float32))
    w_rgb = torch.rand(H, W, 3, generator=g) * ok[..., None]
    w_a = torch.rand(H, W, generator=g) * ok
    w_o = torch.rand(H, W, generator=g) * ok
    w_b = torch.zeros(H, W)
    loss = ((out["rgb"] * w_rgb.cuda()).sum() + (out["accumulation"][..., 0] * w_a.cuda()).sum()
            + (out["object_acc"][..., 0] * w_o.cuda()).sum())
    loss.backward()
    torch.cuda.synchronize()
    img = torch.from_numpy(fw.img).requires_grad_(True)
    alpha = torch.from_numpy(1 - fw.final_T).requires_grad_(True)
    rgb_ref, a_ref, _ = oracle_c.post_ops(img, alpha, None, True)
    ((rgb_ref * w_rgb).sum() + (a_ref[..., 0] * w_a).sum()).backward()
    _, rastergrads = orc.backward(fw, img.grad.numpy(), alpha.grad.numpy(), w_o.numpy(), w_b.numpy())
    v = holder.v_records.cpu().numpy()
    assert rel_l2(v[:, 0:2], rastergrads["v_xy"]) <= GRAD_TOL
    assert rel_l2(v[:, 2:5], rastergrads["v_conic"]) <= GRAD_TOL
    assert rel_l2(v[:, 5], rastergrads["v_opac"]) <= GRAD_TOL
    assert rel_l2(v[:, 6:9], rastergrads["v_rgb"]) <= GRAD_TOL


def test_object_gradient_alone_and_deterministic_mode():
    """Only object_acc carries a cotangent: the whole gradient comes from the folded objects-only terms and the object
    residual.  Deterministic mode is bit-identical from run to run and agrees with the float-atomic path."""
    fr = syn.make_frame(**SCENES["actors_behind"])
    H, W = fr.camera.height, fr.camera.width
    _, v = syn.cotangents(H, W)
    cots = {"object_acc": v.cuda()}  # [H, W], as the accumulation cotangents of test_gpu_parity.py
    frc = to_cuda(fr)
    runs = []
    for _ in range(2):
        _, h = raster.forward_backward(frc, raster.RenderSettings(deterministic=True), cots)
        runs.append(h.v_records.clone())
    assert torch.equal(runs[0], runs[1])
    _, h = raster.forward_backward(frc, raster.RenderSettings(deterministic=False), cots)
    assert rel_l2(runs[0].cpu().numpy(), h.v_records.cpu().numpy()) < 1e-5
    orc = oracle_c.Oracle(fr)
    fw = orc.forward()
    w_o = (v.numpy() * (fw.fragile_obj == 0)).astype(np.float32)
    _, h = raster.forward_backward(frc, raster.RenderSettings(), {"object_acc": torch.from_numpy(w_o).cuda()})
    _, rastergrads = orc.backward(fw, np.zeros_like(fw.img), np.zeros_like(fw.final_T), w_o, np.zeros_like(w_o))
    vr = h.v_records.cpu().numpy()
    assert np.abs(vr[:, 0:2]).max() > 0
    assert rel_l2(vr[:, 0:2], rastergrads["v_xy"]) <= GRAD_TOL
    assert rel_l2(vr[:, 2:5], rastergrads["v_conic"]) <= GRAD_TOL
    assert rel_l2(vr[:, 5], rastergrads["v_opac"]) <= GRAD_TOL
