"""Generates tests/golden/reference_metrics.npz: what THE REFERENCE'S OWN ``get_metrics_dict`` (sgn_splatfacto.py:1015-1040, as
the scene graph inherits it) and ``get_image_metrics_and_images`` (:1109-1187) return after its own ``get_outputs``, on the CPU
(tests/golden/reference_glue.py explains how the reference's model code runs here).

What is not the reference's code here:
  * ``m.psnr``: torchmetrics ``PeakSignalNoiseRatio(data_range=1.0)`` on one pair, restated (10 log10(1 / mse));
  * ``m.ssim``: this library's torch restatement of pytorch_msssim's SSIM (``street_gaussians_ns_b200.model.ssim``);
  * ``m.lpips``: a stand-in that records its arguments and returns 0.25;
  * nerfstudio's colour maps are the identity (the images are not pinned, only their keys).

Scenes (64 x 48, 1200 background + 2 actors x 200 Gaussians, training at step 30000):
  act      the two actors have boxes at the timestamp;
  zero     plus an actor with a box and ZERO rows (skipped by get_outputs, scene graph :337-338);
  nobox    plus an actor with rows and NO box at the timestamp;
  noact    the scene without actors.
Per scene ``k``: ``{k}_keys`` (the dict's keys in order), ``{k}_values`` (float64, same order), ``{k}_rgb`` (outputs["rgb"]),
``{k}_radii`` (self.radii), ``{k}_gt`` (the image), ``{k}_visible`` (visible_model_names).
Eval (scene ``act`` in eval mode, the image as uint8, with and without a mask): ``eval{_mask}_keys`` / ``_values`` of the
metrics dict, ``eval{_mask}_image_keys``, ``eval{_mask}_img`` and the image / mask / rgb inputs.

    SGN_REFERENCE_ROOT=<checkout of street-gaussians-ns> python tests/golden/make_golden_reference_metrics.py
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import reference_glue as rg  # noqa: E402  (puts the repo root on sys.path)
import make_golden_reference_glue as mg  # noqa: E402
import reference_loader as rl  # noqa: E402

OUT = os.path.join(HERE, "reference_metrics.npz")
SEED, FOURIER = 31, 5
SCENES = ("act", "zero", "nobox", "noact")
EXTRA_ROWS = 150  # rows of the actor that has no box at the timestamp


def frame_of(kind):
    return mg.no_actors_scene() if kind == "noact" else mg.live_scene(SEED, FOURIER)


def extra_params(kind, like):
    """The additional sub-model of scenes ``zero`` / ``nobox``: zero rows, or EXTRA_ROWS seeded rows shaped like ``like``."""
    n = 0 if kind == "zero" else EXTRA_ROWS
    g = torch.Generator().manual_seed(77)
    out = {}
    for k in rg.PARAMS:
        t = getattr(like, k)
        out[k] = (torch.randn((n,) + tuple(t.shape[1:]), generator=g) * 0.5 + (-2.0 if k == "scales" else 0.0)).float()
    return out


def gt_image(H, W):
    return torch.rand(H, W, 3, generator=torch.Generator().manual_seed(8))


def eval_mask(H, W):
    return (torch.rand(H, W, 1, generator=torch.Generator().manual_seed(9)) > 0.3).float()


def _psnr(preds, target):
    return 10.0 * torch.log10(1.0 / torch.mean((preds - target) ** 2))


class _SSIM(torch.nn.Module):
    def forward(self, x, y):
        from street_gaussians_ns_b200.model import ssim
        return ssim(x, y)


def reference_model(kind, training):
    base, _ = rl.load()
    fr = frame_of(kind)
    m, cam = rg.build_reference_model(fr, training=training)
    m.refine_record_dict = {}  # populate_modules (sgn_splatfacto.py:314)
    m.psnr, m.ssim = _psnr, _SSIM()
    if kind in ("zero", "nobox"):
        params = extra_params(kind, fr.segments[1].params)
        sub_cfg = base.SplatfactoModelConfig(use_sky_sphere=False, fourier_features_dim=FOURIER)
        sub = rl.bare_model(base, params, sub_cfg, step=30000, idx=len(m.all_models))
        sub.xys = sub.depths = sub.radii = sub.conics = sub.num_tiles_hit = sub.last_size = None
        m.all_models["object_extra"] = sub
        if kind == "zero":  # a box at the timestamp, but no rows
            a = m.object_annos.annos[0]
            m.object_annos.annos.append(types.SimpleNamespace(trackId="extra", frame=a.frame, center=a.center, rot=a.rot))
            m.object_annos.objects_frames["extra"] = list(range(85))
    base.colormaps.apply_colormap = lambda x, **k: x
    base.colormaps.apply_depth_colormap = lambda x, **k: x
    return fr, m, cam


def build():
    d = {}
    for kind in SCENES:
        fr, m, cam = reference_model(kind, training=True)
        H, W = fr.camera.height, fr.camera.width
        out = m.get_outputs(cam)
        batch = {"image": gt_image(H, W)}
        md = m.get_metrics_dict(out, batch)
        d[f"{kind}_keys"] = np.array(list(md))
        d[f"{kind}_values"] = np.array([float(v) for v in md.values()], np.float64)
        d[f"{kind}_rgb"] = out["rgb"].detach().numpy()
        d[f"{kind}_radii"] = m.radii.numpy()
        d[f"{kind}_gt"] = batch["image"].numpy()
        d[f"{kind}_visible"] = np.array(m.visible_model_names)
    for masked in (False, True):
        fr, m, cam = reference_model("act", training=False)
        H, W = fr.camera.height, fr.camera.width
        calls = []

        def lpips(a, b):
            calls.append((tuple(a.shape), tuple(b.shape)))
            return torch.tensor(0.25)

        m.lpips = lpips
        with torch.no_grad():
            out = m.get_outputs(cam)
        image = (gt_image(H, W) * 255).to(torch.uint8)
        batch = {"image": image}
        if masked:
            batch["mask"] = eval_mask(H, W)
        rgb_in = out["rgb"].clone()
        metrics, images = m.get_image_metrics_and_images(out, batch)
        assert calls == [((1, 3, H, W), (1, 3, H, W))]
        p = "eval_mask" if masked else "eval"
        d[f"{p}_keys"] = np.array(list(metrics))
        d[f"{p}_values"] = np.array([float(v) for v in metrics.values()], np.float64)
        d[f"{p}_image_keys"] = np.array(list(images))
        d[f"{p}_img"] = images["img"].numpy()
        d[f"{p}_rgb"] = rgb_in.numpy()
        d[f"{p}_image"] = image.numpy()
        if masked:
            d[f"{p}_mask"] = batch["mask"].numpy()
    return d


if __name__ == "__main__":
    d = build()
    np.savez_compressed(OUT, **d)
    print(OUT, os.path.getsize(OUT) // 1024, "KiB")
    for k in SCENES + ("eval", "eval_mask"):
        print(k, list(d[f"{k}_keys"]), d[f"{k}_values"])
