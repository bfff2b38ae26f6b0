"""The model's metrics against the reference's own code.

tests/golden/reference_metrics.npz holds what the reference's ``get_metrics_dict`` and ``get_image_metrics_and_images`` return
after its own ``get_outputs`` (tests/golden/make_golden_reference_metrics.py).  On the CPU, ``SceneGraphRasterModel`` takes
its torch statement of the same expressions; fed the reference's rendered image and radii, it must give the same keys in the
same order (``"self.radii"`` included, no refine counters), the same means over the same rows (only the visible sub-models:
an actor with zero rows or without a box at the timestamp does not count), and in eval the psnr / ssim of the masked images
with ``img`` built before the mask."""
import math
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_reference_metrics as mg  # noqa: E402

from street_gaussians_ns_b200.model import ActorPose, SceneGraphConfig, SceneGraphRasterModel  # noqa: E402
from street_gaussians_ns_b200.scene import GaussianSet  # noqa: E402

GOLD = np.load(mg.OUT)


def cpu_model(kind, training=True):
    fr = mg.frame_of(kind)
    actors = {s.name[len("object_"):]: s.params for s in fr.segments[1:]}
    poses = [ActorPose(s.name[len("object_"):], s.rot, s.center, int(fr.camera.time), list(range(85))) for s in fr.segments[1:]]
    if kind in ("zero", "nobox"):
        actors["extra"] = GaussianSet(**mg.extra_params(kind, fr.segments[1].params))
        if kind == "zero":
            poses.append(ActorPose("extra", fr.segments[1].rot, fr.segments[1].center, int(fr.camera.time), list(range(85))))
    model = SceneGraphRasterModel(fr.segments[0].params, actors, SceneGraphConfig(use_sky_sphere=False), poses_at=lambda t: poses)
    model.train(training)
    model.step = 30000
    model._frame(fr.camera)  # the visible sub-models of the timestamp, as get_outputs selects them
    return fr, model


@pytest.mark.parametrize("kind", mg.SCENES)
def test_get_metrics_dict_torch_statement_matches_the_reference(kind):
    fr, model = cpu_model(kind)
    assert list(model.visible_model_names) == list(GOLD[f"{kind}_visible"])
    model.__dict__["radii"] = torch.from_numpy(GOLD[f"{kind}_radii"])
    out = {"rgb": torch.from_numpy(GOLD[f"{kind}_rgb"])}
    d = model.get_metrics_dict(out, {"image": torch.from_numpy(GOLD[f"{kind}_gt"])})
    assert list(d) == list(GOLD[f"{kind}_keys"])  # reference's order; no refine counters
    want = dict(zip(GOLD[f"{kind}_keys"], GOLD[f"{kind}_values"]))
    assert isinstance(d["gaussian_count"], int) and d["gaussian_count"] == int(want["gaussian_count"])
    for k in ("psnr", "scale_mean", "log_scale_mean", "sigmoid_opacity", "self.radii"):
        assert float(d[k]) == pytest.approx(want[k], rel=1e-6, abs=0), k


def test_excluded_sub_models_do_not_change_the_metrics():
    """An actor with zero rows, or one without a box at the timestamp, leaves every value as in the scene without it."""
    for kind in ("zero", "nobox"):
        np.testing.assert_array_equal(GOLD[f"{kind}_values"], GOLD["act_values"])
        assert list(GOLD[f"{kind}_visible"]) == list(GOLD["act_visible"])
    assert "object_extra" not in list(GOLD["nobox_visible"])


@pytest.mark.parametrize("masked", [False, True])
def test_get_image_metrics_and_images_torch_statement_matches_the_reference(masked):
    p = "eval_mask" if masked else "eval"
    _, model = cpu_model("act", training=False)
    calls = []

    def lpips(a, b):
        calls.append((a.clone(), b.clone()))
        return torch.tensor(0.25)

    model.lpips = lpips
    rgb = torch.from_numpy(GOLD[f"{p}_rgb"])
    H, W = rgb.shape[:2]
    outputs = {"rgb": rgb.clone(), "accumulation": torch.zeros(H, W, 1), "depth": torch.ones(H, W, 1)}
    batch = {"image": torch.from_numpy(GOLD[f"{p}_image"])}
    if masked:
        batch["mask"] = torch.from_numpy(GOLD[f"{p}_mask"])
    image_before = batch["image"].clone()
    metrics, images = model.get_image_metrics_and_images(outputs, batch)
    assert list(metrics) == list(GOLD[f"{p}_keys"]) == ["psnr", "ssim", "lpips"]
    assert all(isinstance(v, float) for v in metrics.values())
    want = dict(zip(GOLD[f"{p}_keys"], GOLD[f"{p}_values"]))
    assert metrics["psnr"] == pytest.approx(want["psnr"], rel=1e-6)
    assert metrics["ssim"] == pytest.approx(want["ssim"], rel=1e-5, abs=1e-7)
    assert metrics["lpips"] == 0.25 and len(calls) == 1
    # the lpips callable gets the masked [1,3,H,W] gt and rgb, in that order
    g = image_before.float() / 255.0
    m = batch["mask"] if masked else torch.ones(H, W, 1)
    torch.testing.assert_close(calls[0][0], (g * m).permute(2, 0, 1)[None], rtol=0, atol=0)
    torch.testing.assert_close(calls[0][1], (rgb * m).permute(2, 0, 1)[None], rtol=0, atol=0)
    # img is cat([gt, rgb], dim=1) built before masking; accumulation / depth come as the model's maps
    assert list(images) == list(GOLD[f"{p}_image_keys"])
    np.testing.assert_array_equal(images["img"].numpy(), GOLD[f"{p}_img"])
    # unlike the reference, nothing is multiplied by the mask in place
    assert torch.equal(outputs["rgb"], rgb) and torch.equal(batch["image"], image_before)


def test_psnr_of_equal_images_is_inf_on_the_torch_path():
    _, model = cpu_model("act", training=False)
    rgb = torch.rand(16, 16, 3)
    metrics, _ = model.get_image_metrics_and_images({"rgb": rgb, "accumulation": rgb[..., :1], "depth": rgb[..., :1]},
                                                    {"image": rgb.clone()})
    assert metrics["psnr"] == math.inf and "lpips" not in metrics


def test_get_outputs_for_camera_rejects_a_crop_box():
    fr, model = cpu_model("act", training=False)
    with pytest.raises(ValueError):
        model.get_outputs_for_camera(fr.camera, obb_box=object())
