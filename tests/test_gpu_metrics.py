"""The per-step metrics kernel (csrc/metrics.cu through loss.fused_metrics) and the model surface built on it
(get_metrics_dict, get_image_metrics_and_images, TrainStep(metrics=True)) on the GPU.

Bars: against the float64 oracle (oracle/metrics_ref64.py) each mean within 1e-6 relative, psnr within 1e-5 dB, the radii mean
equal to the oracle's value rounded once to fp32, inf / NaN exactly where the oracle has them; against torch's fp32 statement
of the reference's expressions on the same GPU, 1e-5 relative and 1e-4 dB."""
import ctypes
import math
import types

import numpy as np
import pytest
import torch

from oracle import metrics_ref64 as ref
from oracle import ssim_ref64
from street_gaussians_ns_b200 import _lib, raster
from street_gaussians_ns_b200.loss import METRIC_NAMES, fused_metrics

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
SIZES = [(1, 1), (11, 11), (37, 53), (1280, 1920)]
MASKS = [None, "binary", "fractional"]


def make_image(H, W, u8, mask_kind, seed=0):
    rng = np.random.default_rng([H, W, int(u8), MASKS.index(mask_kind), seed])
    gt = rng.integers(0, 256, (H, W, 3), dtype=np.uint8) if u8 else rng.random((H, W, 3), dtype=np.float32)
    rgb = rng.random((H, W, 3), dtype=np.float32)
    mask = None
    if mask_kind == "binary":
        mask = (rng.random((H, W, 1)) > 0.3).astype(np.float32)
    elif mask_kind == "fractional":
        mask = rng.random((H, W, 1), dtype=np.float32)
    return gt, rgb, mask


def dev(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def check_against_oracle(got, want):
    got = got.cpu().numpy().astype(np.float64)
    for i, name in enumerate(METRIC_NAMES):
        g, w = got[i], want[i]
        if math.isnan(w) or math.isinf(w):
            assert (math.isnan(g) and math.isnan(w)) or g == w, (name, g, w)
        elif name == "psnr":
            assert abs(g - w) <= 1e-5, (name, g, w)
        elif name == "radii_mean":
            assert g == float(np.float32(w)), (name, g, w)
        else:
            assert abs(g - w) <= 1e-6 * abs(w), (name, g, w)


@pytest.mark.parametrize("H,W", SIZES)
@pytest.mark.parametrize("u8", [True, False])
@pytest.mark.parametrize("mask_kind", MASKS)
def test_psnr_against_the_oracle(H, W, u8, mask_kind):
    gt, rgb, mask = make_image(H, W, u8, mask_kind)
    got = fused_metrics(dev(rgb), dev(gt), dev(mask))
    torch.cuda.synchronize()
    want = ref.metrics(rgb, gt, mask)
    check_against_oracle(got, want)
    assert all(math.isnan(v) for v in got[1:].tolist())  # no table, no radii


@pytest.mark.parametrize("u8,mask_kind", [(True, None), (False, None), (False, "fractional"), (True, "binary")])
def test_equal_images_give_inf(u8, mask_kind):
    gt, _, mask = make_image(37, 53, u8, mask_kind, seed=1)
    rgb = ref.gt_float(gt)
    got = fused_metrics(dev(rgb), dev(gt), dev(mask))
    assert got[0].item() == math.inf and ref.psnr(rgb, gt, mask) == math.inf


def make_table(counts, seed=0, scale_rows=None, logit_rows=None, zero_radii=False):
    """A device segment table over fresh scales / opacities tensors (the fields sgn_metrics reads); returns (table-like
    object, radii, host copies).  ``scale_rows`` / ``logit_rows``: {(segment, row): value} overrides."""
    rng = np.random.default_rng([seed, len(counts)])
    scales = [rng.normal(-3.0, 1.0, (n, 3)).astype(np.float32) for n in counts]
    opac = [rng.normal(0.0, 3.0, (n, 1)).astype(np.float32) for n in counts]
    for (s, r), v in (scale_rows or {}).items():
        scales[s][r] = v
    for (s, r), v in (logit_rows or {}).items():
        opac[s][r] = v
    ts, to = [dev(a) for a in scales], [dev(a) for a in opac]
    counts = np.asarray(counts, np.int64)
    chunks = (counts + 127) // 128
    host = np.zeros(len(counts), raster.SEG_DTYPE)
    host["count"] = counts
    host["row0"] = np.concatenate([[0], np.cumsum(counts)[:-1]])
    host["chunk0"] = np.concatenate([[0], np.cumsum(chunks)[:-1]])
    host["scales"] = [t.data_ptr() for t in ts]
    host["opacities"] = [t.data_ptr() for t in to]
    N = int(counts.sum())
    radii = np.zeros(N, np.int32) if zero_radii else rng.integers(0, 60, N).astype(np.int32)
    tab = types.SimpleNamespace(dev=torch.from_numpy(host.view(np.uint8).reshape(-1)).to(DEV), nseg=len(counts), N=N,
                                num_chunks=int(chunks.sum()), keep=(ts, to))
    return tab, dev(radii), (scales, opac, radii)


def _counts33():
    head = [5000, 0, 127, 128, 129, 1, 256, 257, 0, 383, 384, 385, 2000]
    rng = np.random.default_rng(33)
    return head + [int(x) if x % 5 else 0 for x in rng.integers(0, 700, 33 - len(head))]


TABLES = {
    "one_129": dict(counts=[129]),
    "two_127_128": dict(counts=[127, 128]),
    "leading_empty": dict(counts=[0, 200]),
    "33_segments": dict(counts=_counts33()),
    "zero_radii": dict(counts=[300, 129], zero_radii=True),
    "exp_overflow": dict(counts=[130, 5], scale_rows={(0, 7): 100.0}),
    "logits_pm100": dict(counts=[128, 3], logit_rows={(0, 0): 100.0, (0, 1): -100.0, (1, 2): -100.0}),
    "multi_chunk": dict(counts=[128 * 40 + 17]),
}


@pytest.mark.parametrize("name", list(TABLES))
def test_parameter_terms_against_the_oracle(name):
    tab, radii, (scales, opac, r) = make_table(seed=3, **TABLES[name])
    got = fused_metrics(table=tab, radii=radii)
    torch.cuda.synchronize()
    want = ref.metrics(scales=scales, opacities=opac, radii=r)
    check_against_oracle(got, want)
    assert math.isnan(got[0].item())
    if name == "exp_overflow":
        assert got[1].item() == math.inf
    if name == "zero_radii":
        assert got[4].item() == 0.0


def test_zero_rows_give_nan():
    tab, radii, _ = make_table([0])
    got = fused_metrics(table=tab, radii=radii)
    assert all(math.isnan(v) for v in got.tolist())


def test_image_and_table_together_and_bit_identical_runs():
    gt, rgb, mask = make_image(1280, 1920, True, "fractional", seed=5)
    tab, radii, (scales, opac, r) = make_table(_counts33(), seed=5)
    a = fused_metrics(dev(rgb), dev(gt), dev(mask), table=tab, radii=radii)
    b = fused_metrics(dev(rgb), dev(gt), dev(mask), table=tab, radii=radii)
    torch.cuda.synchronize()
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    check_against_oracle(a, ref.metrics(rgb, gt, mask, scales, opac, r))


def test_error_returns_launch_nothing():
    L = _lib.load()
    gt, rgb, _ = make_image(11, 11, True, None)
    g, x = dev(gt), dev(rgb)
    tab, radii, _ = make_table([129])
    out = torch.empty(5, device=DEV)
    sb = L.sgn_metrics_scratch_bytes()
    scratch = torch.empty(sb, device=DEV, dtype=torch.uint8)
    li = _lib.LossIn()
    li.rgb, li.gt_u8 = x.data_ptr(), g.data_ptr()
    both = _lib.LossIn()
    both.rgb, both.gt_u8, both.gt_f32 = x.data_ptr(), g.data_ptr(), x.data_ptr()
    neither = _lib.LossIn()
    neither.rgb = x.data_ptr()
    p = raster._ptr

    def call(info=li, table=tab.dev, nseg=1, nbytes=sb):
        return L.sgn_metrics(11, 11, ctypes.byref(info), p(table), nseg, tab.N, tab.num_chunks, p(radii), p(out), p(scratch), nbytes,
                             raster._stream())

    torch.cuda.synchronize()
    launches = L.sgn_launch_count()
    assert call(table=None) == -1 and b"null segment table" in L.sgn_last_error()
    assert call(info=both) == -1 and b"exactly one" in L.sgn_last_error()
    assert call(info=neither) == -1 and b"exactly one" in L.sgn_last_error()
    assert call(nbytes=sb - 1) == -3 and b"scratch too small" in L.sgn_last_error()
    assert L.sgn_launch_count() == launches
    assert call() == 0 and L.sgn_launch_count() == launches + 2
    with pytest.raises(_lib.SgnError):
        fused_metrics(x, None)


# ---- model level ------------------------------------------------------------------------------------------------------
def torch_statement(model, rgb, gt):
    """The reference's get_metrics_dict expressions (sgn_splatfacto.py:1031-1037) in fp32 over torch.cat of the visible
    sub-models, on the GPU."""
    subs = [model.all_models[n] for n in model.visible_model_names]
    scales = torch.cat([s.gauss_params["scales"].detach() for s in subs])
    opac = torch.cat([s.gauss_params["opacities"].detach() for s in subs])
    g = gt.float() / 255.0 if gt.dtype == torch.uint8 else gt
    mse = torch.mean((rgb.detach() - g) ** 2)
    return {"psnr": float(10 * torch.log10(1 / mse)), "gaussian_count": sum(s.num_points for s in subs),
            "scale_mean": float(torch.exp(scales).mean()), "log_scale_mean": float(scales.mean()),
            "sigmoid_opacity": float(torch.sigmoid(opac).mean()), "self.radii": float(model.radii.float().mean())}, (subs, g)


@pytest.fixture(scope="module")
def cfg4():
    """The config-4 scene of tools/train_cfg4.py: 5 cameras x 85 frames, 2 M Gaussians in 33 sub-models, 1920 x 1280."""
    import street_gaussians_ns_b200.synthetic as syn
    from street_gaussians_ns_b200.model import ActorPose, SceneGraphConfig, SceneGraphRasterModel
    sc = syn.WaymoScene(actor_range=45.0)
    frame_list = list(range(sc.num_frames))

    def poses_at(t):
        f = int(t)
        return [ActorPose(str(a), rot, center, f, frame_list) for a, rot, center in sc.boxes_at(f)]

    cfg = SceneGraphConfig(use_sky_sphere=False, async_binning=False)
    model = SceneGraphRasterModel(sc.background.to(DEV), {k: v.to(DEV) for k, v in sc.actors.items()}, cfg, poses_at=poses_at).to(DEV)
    model.train()
    model.step = 600
    gt = (torch.rand(sc.height, sc.width, 3, generator=torch.Generator().manual_seed(5)) * 255).to(torch.uint8).to(DEV)
    with torch.no_grad():  # the capacity of the list buffers, learnt with the read-back on (as tools/train_cfg4.py does)
        for cam in sc.cameras[::7]:
            model.get_outputs(cam)
            raster.async_learn(DEV, int(model._holder.M))
    return sc, model, gt


def test_get_metrics_dict_on_config4_against_torch_and_oracle_without_sync(cfg4):
    sc, model, gt = cfg4
    model.config.async_binning = True
    try:
        for cam in (sc.cameras[212], sc.cameras[3]):
            out = model.get_outputs(cam)
            torch.cuda.synchronize()
            torch.cuda.set_sync_debug_mode("error")
            try:
                d = model.get_metrics_dict(out, {"image": gt})
            finally:
                torch.cuda.set_sync_debug_mode(0)
            assert list(d) == ["psnr", "gaussian_count", "scale_mean", "log_scale_mean", "sigmoid_opacity", "self.radii"]
            assert isinstance(d["gaussian_count"], int)
            for k, v in d.items():
                if k != "gaussian_count":
                    assert isinstance(v, torch.Tensor) and v.dim() == 0 and v.is_cuda, k
            want, (subs, g) = torch_statement(model, out["rgb"], gt)
            assert d["gaussian_count"] == want["gaussian_count"] == model.radii.shape[0]
            assert len(subs) > 1  # actors in view
            assert abs(float(d["psnr"]) - want["psnr"]) <= 1e-4
            for k in ("scale_mean", "log_scale_mean", "sigmoid_opacity", "self.radii"):
                assert abs(float(d[k]) - want[k]) <= 1e-5 * abs(want[k]), (k, float(d[k]), want[k])
            o = ref.metrics(out["rgb"].detach().cpu().numpy(), gt.cpu().numpy(), None,
                            [s.gauss_params["scales"].detach().cpu().numpy() for s in subs],
                            [s.gauss_params["opacities"].detach().cpu().numpy() for s in subs], model.radii.cpu().numpy())
            got = torch.stack([d[k] for k in ("psnr", "scale_mean", "log_scale_mean", "sigmoid_opacity", "self.radii")])
            check_against_oracle(got, o)
            # the torch fallback of the model itself gives the same numbers
            model.config.fused_loss = False
            try:
                fb = model.get_metrics_dict(out, {"image": gt})
            finally:
                model.config.fused_loss = True
            assert fb["gaussian_count"] == d["gaussian_count"]
            for k in ("scale_mean", "log_scale_mean", "sigmoid_opacity", "self.radii"):
                assert abs(float(fb[k]) - float(d[k])) <= 1e-5 * abs(float(d[k])), k
            assert abs(float(fb["psnr"]) - float(d["psnr"])) <= 1e-4
    finally:
        model.config.async_binning = False


def small_model():
    import street_gaussians_ns_b200.synthetic as syn
    from street_gaussians_ns_b200.model import ActorPose, SceneGraphConfig, SceneGraphRasterModel
    fr = syn.make_frame(n_background=20000, n_actors=3, n_per_actor=1500, width=320, height=240, seed=3,
                        actor_shift=np.array([1.0, 0.0, -1.0]))
    bg = fr.segments[0].params.to(DEV)
    actors = {s.name.replace("object_", ""): s.params.to(DEV) for s in fr.segments[1:]}
    poses = [ActorPose(s.name.replace("object_", ""), s.rot, s.center, 21, list(range(85))) for s in fr.segments[1:]]
    model = SceneGraphRasterModel(bg, actors, SceneGraphConfig(use_sky_sphere=False), poses_at=lambda t: poses).to(DEV)
    return fr, model


@pytest.mark.parametrize("mask_kind", [None, "binary", "fractional"])
def test_get_image_metrics_and_images(mask_kind):
    fr, model = small_model()
    model.eval()
    calls = []

    def lpips(a, b):
        calls.append((a.clone(), b.clone()))
        return torch.tensor(0.125, device=DEV)

    model.lpips = lpips
    out = model.get_outputs_for_camera(fr.camera)
    H, W = fr.camera.height, fr.camera.width
    gt_np, _, mask_np = make_image(H, W, True, mask_kind, seed=9)
    batch = {"image": dev(gt_np)}
    if mask_np is not None:
        batch["mask"] = dev(mask_np)
    before = {k: v.clone() for k, v in out.items()}, {k: v.clone() for k, v in batch.items()}
    metrics, images = model.get_image_metrics_and_images(out, batch)
    assert list(metrics) == ["psnr", "ssim", "lpips"] and all(isinstance(v, float) for v in metrics.values())
    rgb = out["rgb"].cpu().numpy()
    assert abs(metrics["psnr"] - ref.psnr(rgb, gt_np, mask_np)) <= 1e-5
    loss, _, _ = ssim_ref64.ssim_loss(rgb, ref.gt_float(gt_np), mask_np, weight=1.0)
    assert abs(metrics["ssim"] - (1.0 - loss)) <= 1e-5
    assert metrics["lpips"] == 0.125 and len(calls) == 1
    g = batch["image"].float() / 255.0
    m = batch["mask"] if mask_np is not None else torch.ones(H, W, 1, device=DEV)
    assert torch.equal(calls[0][0], (g * m).permute(2, 0, 1)[None]) and torch.equal(calls[0][1], (out["rgb"] * m).permute(2, 0, 1)[None])
    assert list(images) == ["img", "accumulation", "depth"]
    assert torch.equal(images["img"], torch.cat([g, out["rgb"]], dim=1))
    for k, v in before[0].items():
        assert torch.equal(out[k], v), k
    for k, v in before[1].items():
        assert torch.equal(batch[k], v), k
    model.lpips = None
    metrics, _ = model.get_image_metrics_and_images(out, batch)
    assert "lpips" not in metrics


def _train(metrics, steps):
    from street_gaussians_ns_b200.optim import FusedAdam
    from street_gaussians_ns_b200.training import TrainStep
    fr, model = small_model()
    model.train()
    opt = FusedAdam(model.optimizer_params())
    step_fn = TrainStep(model, opt, refine_every=0, metrics=metrics)
    gt = (torch.rand(240, 320, 3, generator=torch.Generator().manual_seed(2)) * 0.5 + 0.25).to(DEV)
    losses = []
    for step in steps:
        losses.append({k: v.detach().clone() for k, v in step_fn(step, fr.camera, {"image": gt}).items()})
    torch.cuda.synchronize()
    state = {f"{n}.{k}": p.detach().clone() for n, sub in model.all_models.items() for k, p in sub.gauss_params.items()}
    return losses, state, step_fn


def test_train_step_with_metrics_is_bit_identical(monkeypatch):
    monkeypatch.setattr(raster, "DETERMINISTIC", True)
    steps = [600, 601, 602]
    la, sa, fa = _train(False, steps)
    lb, sb, fb = _train(True, steps)
    assert fa.metrics is None
    assert list(fb.metrics) == ["psnr", "gaussian_count", "scale_mean", "log_scale_mean", "sigmoid_opacity", "self.radii"]
    assert math.isfinite(float(fb.metrics["psnr"]))
    for a, b in zip(la, lb):
        assert a.keys() == b.keys() and all(torch.equal(a[k], b[k]) for k in a)
    assert sa.keys() == sb.keys() and all(torch.equal(sa[k], sb[k]) for k in sa)
