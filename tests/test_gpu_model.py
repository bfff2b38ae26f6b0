"""Level-2 surface (SceneGraphRasterModel.get_outputs / get_loss_dict, the reference's nerfstudio Model methods on
the hot path, street_gaussians_ns/sgn_splatfacto_scene_graph.py:305-391) against the autograd path of
raster.render_frame on the same frame: outputs identical, parameter gradients delivered through the gradient sink
equal to the per-leaf autograd gradients, and torch's accumulate-unless-zeroed semantics."""
import numpy as np
import pytest
import torch

import street_gaussians_ns_b200.synthetic as syn
from street_gaussians_ns_b200 import raster
from street_gaussians_ns_b200.model import ActorPose, SceneGraphConfig, SceneGraphRasterModel
from street_gaussians_ns_b200.scene import PARAM_NAMES, Frame, Segment

pytestmark = pytest.mark.gpu


def rel_l2(a, b):
    return float(np.linalg.norm((a - b).ravel()) / max(np.linalg.norm(b.ravel()), 1e-30))


@pytest.fixture(scope="module")
def setup():
    fr = syn.make_frame(n_background=20000, n_actors=4, n_per_actor=1500, width=320, height=240, seed=3,
                        actor_shift=np.array([1.0, 0.0, -1.0]))
    dev = torch.device("cuda", 0)
    bg = fr.segments[0].params.to(dev)
    actors = {s.name.replace("object_", ""): s.params.to(dev) for s in fr.segments[1:]}
    poses = [ActorPose(s.name.replace("object_", ""), s.rot, s.center, 21, list(range(85))) for s in fr.segments[1:]]
    model = SceneGraphRasterModel(bg, actors, SceneGraphConfig(use_sky_sphere=False, ssim_lambda=0.0),
                                  poses_at=lambda t: poses).to(dev)
    model.train()
    model.step = 30000
    gt = torch.rand(fr.camera.height, fr.camera.width, 3, generator=torch.Generator().manual_seed(2)).to(dev)
    return fr, model, gt


def _loss(model, out, gt):
    return sum(model.get_loss_dict(out, {"image": gt}).values())


def _model_grads(model):
    # PARAM_NAMES order (a ParameterDict built from a plain dict iterates its keys SORTED)
    return torch.cat([model.all_models[name].gauss_params[k].grad.reshape(-1) for name in model.visible_model_names
                      for k in PARAM_NAMES])


def test_model_matches_render_frame_autograd(setup):
    fr, model, gt = setup
    for p in model.parameters():
        p.grad = None
    out = model.get_outputs(fr.camera)
    loss = _loss(model, out, gt)
    loss.backward()
    got = _model_grads(model).clone()
    # the same frame through the per-leaf autograd path
    frame = model._frame(fr.camera)
    frc = Frame(fr.camera, [Segment(type(s.params)(*[t.detach().clone().requires_grad_(True) for t in s.params.tensors()]),
                                    s.cls, s.rot, s.center, s.idft, s.name) for s in frame.segments])
    out2, h2 = raster.render_frame(frc, model._settings(class_streams=True))
    for k in ("rgb", "accumulation", "depth", "object_acc", "background_acc"):
        assert torch.equal(out[k].detach(), out2[k].detach()), k
    loss2 = _loss(model, out2, gt)
    loss2.backward()
    ref = torch.cat([t.grad.reshape(-1) for seg in frc.segments for t in seg.params.tensors()])
    assert float(loss) == pytest.approx(float(loss2), rel=1e-6)
    assert rel_l2(got.cpu().numpy(), ref.cpu().numpy()) < 1e-5
    # side effects the densification reads (sgn_splatfacto.py:513-541)
    assert model.xys.grad is not None and model.xys.grad.shape == model.xys.shape
    sub = model.all_models[model.visible_model_names[1]]
    assert sub.xys.grad.shape[0] == sub.num_points and sub.radii.shape[0] == sub.num_points
    assert model._holder.grad_arena.numel() >= got.numel()


def test_gradients_accumulate_unless_zeroed(setup):
    fr, model, gt = setup
    for p in model.parameters():
        p.grad = None
    _loss(model, model.get_outputs(fr.camera), gt).backward()
    g1 = _model_grads(model).clone()
    _loss(model, model.get_outputs(fr.camera), gt).backward()  # no zero_grad: torch semantics = sum
    g2 = _model_grads(model).clone()
    assert rel_l2(g2.cpu().numpy(), 2 * g1.cpu().numpy()) < 1e-4
    for p in model.parameters():
        p.grad = None
    _loss(model, model.get_outputs(fr.camera), gt).backward()
    assert rel_l2(_model_grads(model).cpu().numpy(), g1.cpu().numpy()) < 1e-5


def test_eval_outputs_and_no_grad(setup):
    fr, model, gt = setup
    model.eval()
    try:
        with torch.no_grad():
            out = model.get_outputs(fr.camera)
        for k in ("rgb", "accumulation", "depth", "object_acc", "background_acc", "background_rgb", "object_rgb"):
            assert k in out and torch.isfinite(out[k]).all(), k
        assert float(out["rgb"].min()) >= 0.0 and float(out["rgb"].max()) <= 1.0  # eval clamp (sgn_splatfacto.py:974-975)
        assert not out["rgb"].requires_grad
    finally:
        model.train()


@pytest.mark.parametrize("u8", [False, True])
def test_fused_loss_epilogue_matches_torch(setup, u8):
    """loss.py (SURVEY.md 8f rank 2) against the reference's torch expressions (sgn_splatfacto.py:1079-1093,
    scene graph :386-389): loss values and the cotangents that reach rgb / accumulation / object_acc."""
    fr, model, gt = setup
    H, W = fr.camera.height, fr.camera.width
    g = torch.Generator().manual_seed(11)
    dev = gt.device
    rgb0 = torch.rand(H, W, 3, generator=g).to(dev)
    acc0 = torch.rand(H, W, 1, generator=g).to(dev)
    obj0 = torch.rand(H, W, 1, generator=g).to(dev)
    obj0[:4] = 0.0          # clamp region: no gradient
    obj0[4:8] = 1.0
    semantic = (torch.rand(H, W, 1, generator=g) > 0.7).to(dev).long() * 2
    mask = (torch.rand(H, W, 1, generator=g) > 0.2).float().to(dev)
    image = (torch.rand(H, W, 3, generator=g) * 255).to(torch.uint8).to(dev) if u8 else gt
    res = {}
    for fused in (False, True):
        model.config.fused_loss = fused
        for with_mask in (False, True):
            rgb, acc, obj = (t.clone().requires_grad_(True) for t in (rgb0, acc0, obj0))
            batch = {"image": image, "semantic": semantic}
            if with_mask:
                batch["mask"] = mask
            losses = model.get_loss_dict({"rgb": rgb, "accumulation": acc, "object_acc": obj}, batch)
            assert set(losses) == {"Ll1", "simloss", "sky_accumulation", "object_acc_entropy_loss"}
            assert float(losses["simloss"]) == 0.0  # ssim_lambda == 0: the key the reference always emits, as an exact zero
            (2.0 * losses["Ll1"] + 0.5 * losses["sky_accumulation"] + 3.0 * losses["object_acc_entropy_loss"]).backward()
            res[(fused, with_mask)] = ({k: float(v) for k, v in losses.items()}, rgb.grad, acc.grad, obj.grad)
    model.config.fused_loss = True
    for with_mask in (False, True):
        (l0, *g0), (l1, *g1) = res[(False, with_mask)], res[(True, with_mask)]
        for k in l0:
            assert l1[k] == pytest.approx(l0[k], rel=2e-6), k
        for a, b in zip(g0, g1):
            assert torch.allclose(a, b, rtol=1e-5, atol=1e-12)


def test_after_train_statistics_match_reference_expressions(setup):
    """sgn_densify_stats (SURVEY.md 8f rank 3) against the torch statements of every sub-model's after_train
    (sgn_splatfacto.py:513-541), over two steps (creation, then accumulation on visible rows)."""
    fr, model, gt = setup
    model.step = 100  # < stop_split_at: statistics are still collected
    try:
        for sub in model.all_models.values():
            sub.xys_grad_norm = sub.vis_counts = sub.max_2Dsize = None
        ref = {}
        for it in range(2):
            for p in model.parameters():
                p.grad = None
            _loss(model, model.get_outputs(fr.camera), gt).backward()
            model.after_train(model.step)
            for name in model.visible_model_names:
                sub = model.all_models[name]
                vis = (sub.radii > 0).flatten()
                grads = sub.xys.grad.detach().norm(dim=-1)
                if name not in ref:
                    r = dict(g=grads.clone(), c=torch.ones_like(grads), m=torch.zeros_like(sub.radii, dtype=torch.float32))
                    ref[name] = r
                else:
                    r = ref[name]
                    r["c"][vis] = r["c"][vis] + 1
                    r["g"][vis] = grads[vis] + r["g"][vis]
                r["m"][vis] = torch.maximum(r["m"][vis], sub.radii.detach()[vis] / float(max(model.last_size)))
        for name, r in ref.items():
            sub = model.all_models[name]
            assert torch.equal(sub.vis_counts, r["c"]), name
            assert torch.allclose(sub.max_2Dsize, r["m"], rtol=2e-6, atol=0), name   # radii * (1/max) vs torch's own rounding
            assert torch.allclose(sub.xys_grad_norm, r["g"], rtol=2e-6, atol=1e-12), name
        bgm = model.all_models["background"]
        assert float(bgm.vis_counts.max()) == 2.0 and float(bgm.vis_counts.min()) == 1.0 and float(bgm.xys_grad_norm.sum()) > 0
        model.step = model.config.stop_split_at  # statistics frozen after refinement stops (:516-518)
        before = model.all_models["background"].vis_counts.clone()
        model.after_train(model.step)
        assert torch.equal(model.all_models["background"].vis_counts, before)
    finally:
        model.step = 30000


def test_after_train_past_the_background_stop_split_at(setup):
    """object_refine.stop_split_at > refine.stop_split_at, at a step between the two: after_train collects the actors'
    statistics only, so the segment table starts at the first actor's row (row0 > 0).  The actors' statistics follow the
    torch statements of after_train (sgn_splatfacto.py:513-541) and the background's are left as they were."""
    fr, model, gt = setup
    c = model.config
    saved = (c.refine.stop_split_at, c.object_refine.stop_split_at)
    c.refine.stop_split_at, c.object_refine.stop_split_at = 100, 200
    model.step = 150
    try:
        for sub in model.all_models.values():
            sub.xys_grad_norm = sub.vis_counts = sub.max_2Dsize = None
        bgm = model.all_models["background"]
        n_bg = bgm.num_points
        fill = [torch.full((n_bg,), v, device=gt.device) for v in (0.25, 3.0, 0.125)]
        bgm.xys_grad_norm, bgm.vis_counts, bgm.max_2Dsize = (t.clone() for t in fill)
        ref = {}
        for it in range(2):
            for p in model.parameters():
                p.grad = None
            _loss(model, model.get_outputs(fr.camera), gt).backward()
            model.after_train(model.step)
            for name in model.visible_model_names:
                if name == "background":
                    continue
                sub = model.all_models[name]
                vis = (sub.radii > 0).flatten()
                grads = sub.xys.grad.detach().norm(dim=-1)
                if name not in ref:
                    ref[name] = r = dict(g=grads.clone(), c=torch.ones_like(grads), m=torch.zeros_like(sub.radii, dtype=torch.float32))
                else:
                    r = ref[name]
                    r["c"][vis] = r["c"][vis] + 1
                    r["g"][vis] = grads[vis] + r["g"][vis]
                r["m"][vis] = torch.maximum(r["m"][vis], sub.radii.detach()[vis] / float(max(model.last_size)))
        assert len(ref) == 4 and model._slices[1][1].start == n_bg
        for name, r in ref.items():
            sub = model.all_models[name]
            assert torch.equal(sub.vis_counts, r["c"]), name
            assert torch.allclose(sub.max_2Dsize, r["m"], rtol=2e-6, atol=0), name
            assert torch.allclose(sub.xys_grad_norm, r["g"], rtol=2e-6, atol=1e-12), name
        for got, want in zip((bgm.xys_grad_norm, bgm.vis_counts, bgm.max_2Dsize), fill):
            assert torch.equal(got, want)
    finally:
        c.refine.stop_split_at, c.object_refine.stop_split_at = saved
        model.step = 30000


def test_device_resident_frame_table_and_pose_content_key():
    """SURVEY 8f rank 4: prepare_frames() builds every timestamp's segment rows once (one upload); get_outputs then indexes
    the resident table.  Same images as the per-frame host build; a box moved IN PLACE at a fixed timestamp (what the
    reference's bbox_optimizer.apply_to_bbox does every step) is noticed by content and re-staged."""
    dev = torch.device("cuda", 0)
    sc = syn.WaymoScene(scale=0.04, num_frames=12, actor_range=20.0)
    cfg = SceneGraphConfig(use_sky_sphere=False, ssim_lambda=0.0)
    boxes = {f: [ActorPose(str(a), rot.copy(), center.copy(), f, list(range(sc.num_frames))) for a, rot, center in sc.boxes_at(f)]
             for f in range(sc.num_frames)}

    def build():
        m = SceneGraphRasterModel(sc.background.to(dev), {k: v.to(dev) for k, v in sc.actors.items()}, cfg,
                                  poses_at=lambda t: boxes[int(t)]).to(dev)
        m.train()
        m.step = 5000
        return m

    plain, resident = build(), build()
    nbytes = resident.prepare_frames([float(f) for f in range(sc.num_frames)])
    assert nbytes == sum((1 + len(boxes[f])) * 168 for f in range(sc.num_frames))
    for ci in (0, 7, 23, 58):
        cam = sc.cameras[ci]
        a, b = plain.get_outputs(cam), resident.get_outputs(cam)
        assert resident._holder is not None and plain.visible_model_names == resident.visible_model_names
        for k in ("rgb", "accumulation", "depth", "object_acc", "background_acc"):
            assert torch.equal(a[k], b[k]), (ci, k)
    # the resident rows were used as they are (no rebuild): the Frame handed to the rasterizer carries the prebuilt block
    fr = resident._frame(sc.cameras[7])
    assert fr._prebuilt is not None and fr._prebuilt.dev.data_ptr() >= resident.__dict__["_frame_table_blob"].data_ptr()
    # move one box in place: identity unchanged, content changed -> the image must change and match a fresh model's
    cam = sc.cameras[5]  # frame 1, the forward-looking rig camera: the nearest boxes are in view
    before = resident.get_outputs(cam)["rgb"].clone()
    for pose in boxes[int(cam.time)]:
        pose.center[0] += 0.75
    after = resident.get_outputs(cam)["rgb"]
    assert not torch.equal(before, after)
    assert torch.equal(after, build().get_outputs(cam)["rgb"])


def test_model_without_the_count_read_back_matches_the_exact_path(setup):
    """SceneGraphConfig.async_binning: get_outputs without the per-frame host read-back of the intersection count -- same images,
    same gradients; an empty view gets the reference's early-out depth (0, not the 10 of an empty pixel) on the device."""
    fr, model, gt = setup
    for p in model.parameters():
        p.grad = None
    ref = model.get_outputs(fr.camera)
    _loss(model, ref, gt).backward()
    g_ref = _model_grads(model).clone()
    raster._ASYNC_STATE.clear()
    model.config.async_binning = True
    try:
        for it in range(3):  # the first frame learns the count, the next ones run without the read-back
            for p in model.parameters():
                p.grad = None
            out = model.get_outputs(fr.camera)
            _loss(model, out, gt).backward()
        assert isinstance(model._holder.M, raster.LazyCount)
        for k in ("rgb", "accumulation", "depth", "object_acc", "background_acc"):
            assert torch.equal(out[k].detach(), ref[k].detach()), k
        assert rel_l2(_model_grads(model).cpu().numpy(), g_ref.cpu().numpy()) < 1e-5
        # nothing in view: look away from the scene
        import street_gaussians_ns_b200.synthetic as syn2
        away = syn2.make_camera(fr.camera.width, fr.camera.height, c2w=np.array([[-1.0, 0, 0, 0], [0, 1.0, 0, 0], [0, 0, -1.0, 500.0]]),
                                time=fr.camera.time)
        empty = model.get_outputs(away)
        assert isinstance(model._holder.M, raster.LazyCount) and int(model._holder.M) == 0
        assert float(empty["depth"].abs().max()) == 0.0 and float(empty["accumulation"].abs().max()) == 0.0
    finally:
        model.config.async_binning = None
